"""CPU: the bars, inputs and coverage of tests/test_reg_matrix_gpu.py, and the regulariser C-ABI's refusals.

For every case of the GPU module the oracle runs once in float32 and once in float64 on the same float32 inputs and
cotangents; the float32 run's worst error (fraction of each array's largest float64 magnitude, as the GPU module measures the
kernels) is what float32 arithmetic costs at that case.  Each bar stays a fixed headroom above it.  The chunked oracle matches
oracle.dbw_path.regularisers; every case's inputs keep the function's decisions clear of float32 rounding; and the case table
follows the kernels' CTA and chunk sizes as csrc/dbw_reg.cu defines them."""
import ctypes
import functools
import os
import re
import types

import pytest
import torch

from oracle import dbw_path as D
from tests import test_reg_matrix_gpu as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# a bar is at least HEADROOM x the float32 oracle's deviation; a bar above 2e-6 is at most BAR_FACTOR * 4 x it (CPUs differ
# in their float32 rounding by a factor of two or so)
HEADROOM = 4


def _acc(out, name, e):
    out[name] = max(out.get(name, 0.), e)


@functools.lru_cache(maxsize=None)
def float32_deviations():
    out = {}
    for case in M.CASES:
        x = M.reg_inputs(case['name'])
        v64, g64 = M.oracle(case, x, torch.float64)
        v32, g32 = M.oracle(case, x, torch.float32)
        for n in v64:
            _acc(out, f'val.{n}', M.rel_err(v32[n], v64[n]))
        for k in g64:
            _acc(out, f'g.{k}', M.rel_err(g32[k], g64[k]))
    return out


def test_every_bar_is_measured_and_every_loose_bar_explained():
    assert set(float32_deviations()) == set(M.BARS)
    assert {k for k, v in M.BARS.items() if v > 2e-6} <= set(M.BAR_NOTES)


@pytest.mark.parametrize('name', sorted(M.BARS))
def test_bar_sits_a_fixed_multiple_above_float32_rounding(name):
    dev, bar = float32_deviations()[name], M.BARS[name]
    assert HEADROOM * dev <= bar, f'{name}: float32 oracle deviates by {dev:.3g} of max; bar {bar:.3g} leaves less than {HEADROOM}x'
    assert bar <= 2e-6 or bar <= 4 * M.BAR_FACTOR * dev, f'{name}: bar {bar:.3g} is loose for a float32 deviation of {dev:.3g}'


@pytest.mark.parametrize('name', [c['name'] for c in M.CASES if c['terms'] == 7 and c['coarse']
                                  and c['n_blocks'] ** 2 * c['n_points'] <= 500_000])
def test_chunked_oracle_matches_dbw_path(name, monkeypatch):
    """the module's oracle, in chunks of 3 blocks, against D.regularisers (the opacities as sigmoid(alpha_logit) * keep)"""
    monkeypatch.setattr(M, 'CHUNK_PAIRS', 3 * M.BY_NAME[name]['n_points'])
    case, x = M.BY_NAME[name], M.reg_inputs(name)
    vals, grads = M.oracle(case, x, torch.float64)
    a = x['alpha_full'].double()
    keep = a > 0
    p = {k: x[k].double().clone().requires_grad_(True) for k in ('texture_bkg', 'texture_ground', 'textures', 'S', 'R_6d', 'T', 'sq_eps')}
    p['alpha_logit'] = torch.where(keep, torch.logit(a), torch.zeros_like(a)).requires_grad_(True)
    tpl = types.SimpleNamespace(n_blocks=case['n_blocks'], ratio=M.RATIO, scale_min=M.SCALE_MIN)
    ref = D.regularisers(tpl, p, coarse=True, keep=keep, tv_type=case['norm'], unit_samples=x['unit_samples'].double(),
                         weights=case['w'])
    cot = M.cotangents(case)
    sum(cot[n] * ref[n] for n in ref).backward()
    for n in ref:
        assert abs(vals[n].item() - ref[n].item()) <= 1e-12 * max(abs(ref[n].item()), 1e-30), n
    for k in p:
        want = p[k].grad
        got = grads['alpha_full'] * a * (1 - a) * keep if k == 'alpha_logit' else grads[k]
        assert (got - want).abs().max().item() <= 1e-12 * max(want.abs().max().item(), 1e-30), k


def _tv_stacks(x):
    return ((x['texture_bkg'], False), (x['texture_ground'], False), (x['textures'], True))


@pytest.mark.parametrize('name', [c['name'] for c in M.CASES])
def test_inputs_are_decisive(name):
    """no point's overlap excess within OCC_MARGIN of 0, no block-frame coordinate within CLAMP_MARGIN of +-5, no texel pair's
    squared difference within L2_MARGIN (relative) of l2's 1e-6 clamp, no channel difference nonzero but below L1_MARGIN,
    every opacity 0 or far above the parsimony root's 1e-6 clamp"""
    case, x = M.BY_NAME[name], M.reg_inputs(name)
    if case['terms'] & M.OV:
        exc, gap = M.overlap_decisions(x)
        assert exc.abs().min().item() >= M.OCC_MARGIN
        assert gap.min().item() >= M.CLAMP_MARGIN
    if case['terms'] & M.TV:
        for logits, wrap in _tv_stacks(x):
            for d in M.tv_pairs(M.sigmoid_maps(logits.double()), wrap):
                assert ((d == 0) | (d.abs() >= M.L1_MARGIN)).all()
                assert ((d.pow(2).sum(-1) / 1e-6 - 1).abs() >= M.L2_MARGIN).all()
    a = x['alpha_full']
    assert ((a == 0) | (a >= 0.5)).all()


def _constants():
    src = open(os.path.join(ROOT, 'differentiable-blocksworld_b200', 'csrc', 'dbw_reg.cu')).read()
    return {n: int(re.search(rf'constexpr int {n} = (\d+);', src).group(1)) for n in ('REG_OV_CHUNK', 'REG_THREADS', 'REG_TV_TEXELS')}


def test_case_table_covers_the_kernels_seams():
    """block counts around the overlap CTAs' shared-memory chunk, point counts around their CTA size, TV segment boundaries
    (background | ground | blocks) inside a forward CTA, inside one forward thread's strided texels and inside a backward CTA,
    plateau maps under l1 and l2, a case with an environment smaller than the blocks' maps, sides 2 and 3"""
    c = _constants()
    chunk, threads, texels = c['REG_OV_CHUNK'], c['REG_THREADS'], c['REG_TV_TEXELS']
    ov = [case for case in M.CASES if case['terms'] & M.OV]
    assert {chunk - 1, chunk, chunk + 1, 2 * chunk + 1} <= {case['n_blocks'] for case in ov}
    assert {1, threads - 1, threads, threads + 1} <= {case['n_points'] for case in ov}
    assert {'none', 'some', 'all'} <= {case['kill'] for case in ov}
    tv = [case for case in M.CASES if case['terms'] & M.TV]
    fwd = threads * texels
    bounds = [b for case in tv for b in (case['env'] ** 2, 2 * case['env'] ** 2)]

    def straddles(b):                    # some thread's texel i lies before the boundary and its texel i + 1 at or after it
        base = b // fwd * fwd
        return any(base + t + i * threads < b <= base + t + (i + 1) * threads for t in range(threads) for i in range(texels - 1))

    assert any(b % fwd for b in bounds), 'no TV segment boundary inside a forward CTA'
    assert any(straddles(b) for b in bounds), "no TV segment boundary inside a forward thread's strided texels"
    assert any(b % threads for b in bounds), 'no TV segment boundary inside a backward CTA'
    assert {'l1', 'l2'} <= {case['norm'] for case in tv if case['maps'] == 'plateau'}
    assert {'l1', 'l2', 'l2sq'} <= {case['norm'] for case in tv if not case['coarse']}
    assert any(case['env'] < case['txt'] for case in tv)
    assert {2, 3} <= {case['txt'] for case in tv} and {2, 3} <= {case['env'] for case in tv}
    assert {case['terms'] for case in M.CASES} == set(range(1, 8))
    assert all(case['terms'] == M.TV for case in M.CASES if not case['coarse'])       # losses.regularisers' fine phase


# ---------------------------------------------------------------------------------------------------------- refusals
_FAKE = {k: 0x1000 * (i + 1) for i, k in enumerate(M.LEAVES + ('unit_samples',))}      # never dereferenced: nothing launches


def _valid(**kw):
    return M.reg_struct(dict(M.BY_NAME['PTO'], **kw), _FAKE)


def _refused(rc, what):
    from dbw_b200 import _lib
    return rc != 0 and what.encode() in _lib.lib().dbw_last_error()


def _ws(r):
    from dbw_b200 import _lib
    n = ctypes.c_size_t(0)
    return _lib.lib().dbw_regularisers_workspace_bytes(ctypes.byref(r) if r is not None else None, ctypes.byref(n)), n.value


def test_make_plan_refuses_what_it_cannot_run():
    """every argument check of the plan, through the workspace query (no kernel is launched); what a term that is off would
    read may be missing"""
    assert _ws(_valid())[0] == 0
    assert _refused(_ws(None)[0], 'null argument')
    bad = [
        (dict(terms=8 | 7), {}, 'unknown bits'),
        (dict(n_blocks=0), {}, 'n_blocks < 1'),
        (dict(terms=M.PAR), dict(alpha_full=None), 'null alpha_full'),
        (dict(terms=M.OV), dict(alpha_full=None), 'null alpha_full'),
        (dict(env=1), {}, 'env_size and txt_size'),
        (dict(txt=1), {}, 'env_size and txt_size'),
        (dict(n_points=0), {}, 'n_points < 1'),
    ] + [((), {k: None}, 'null texture') for k in ('texture_bkg', 'texture_ground', 'textures')] \
      + [((), {k: None}, 'null block parameter') for k in ('S', 'R_6d', 'T', 'sq_eps', 'unit_samples')]
    for kw, ptrs, what in bad:
        r = M.reg_struct(dict(M.BY_NAME['PTO'], **dict(kw)), dict(_FAKE, **ptrs))
        assert _refused(_ws(r)[0], what), (kw, ptrs, what)
    for norm in (-1, 3):
        r = _valid()
        r.tv_norm = norm
        assert _refused(_ws(r)[0], 'bad tv_norm'), norm
    # a term that is off reads none of its inputs
    off = [(dict(terms=M.PAR | M.OV, env=0, txt=0), ('texture_bkg', 'texture_ground', 'textures')),
           (dict(terms=M.PAR | M.TV, n_points=0), ('S', 'R_6d', 'T', 'sq_eps', 'unit_samples')),
           (dict(terms=M.TV), ('S', 'R_6d', 'T', 'sq_eps', 'unit_samples', 'alpha_full'))]
    for kw, absent in off:
        r = M.reg_struct(dict(M.BY_NAME['PTO'], **kw), {k: v for k, v in _FAKE.items() if k not in absent})
        assert _ws(r)[0] == 0, kw


def test_entries_refuse_a_missing_output_or_a_workspace_one_byte_short():
    """forward: a NULL output of a term that is on, a NULL workspace, the reported size minus one byte; backward: a NULL
    upstream gradient of a term that is on, the same workspace checks.  All refused before any launch."""
    from dbw_b200 import _lib
    L = _lib.lib()
    r = _valid()
    rc, n = _ws(r)
    assert rc == 0 and n > 0
    ws, out = ctypes.c_void_p(0x9000), [ctypes.c_void_p(0xA000 + 4 * i) for i in range(3)]
    grads = [ctypes.c_void_p(0xB000 + 0x100 * i) for i in range(8)]
    for i in range(3):
        o = list(out)
        o[i] = None
        assert _refused(L.dbw_regularisers_forward(ctypes.byref(r), *o, ws, n, None), 'null output of a term that is on'), i
        assert _refused(L.dbw_regularisers_backward(ctypes.byref(r), *o, *grads, ws, n, None), 'null upstream gradient'), i
    assert _refused(L.dbw_regularisers_forward(ctypes.byref(r), *out, None, n, None), 'workspace too small')
    assert _refused(L.dbw_regularisers_forward(ctypes.byref(r), *out, ws, n - 1, None), 'workspace too small')
    assert _refused(L.dbw_regularisers_backward(ctypes.byref(r), *out, *grads, None, n, None), 'workspace too small')
    assert _refused(L.dbw_regularisers_backward(ctypes.byref(r), *out, *grads, ws, n - 1, None), 'workspace too small')
