"""CPU: the bars of tests/test_scene_matrix_gpu.py against the float64 oracle's own float32 evaluation.

For every case of the GPU module the oracle runs once in float32 and once in float64 on the same float32 inputs and cotangents;
the float32 run's worst error (fraction of each array's largest float64 magnitude, as the GPU module measures the kernels) is
what float32 arithmetic costs at that case.  Each bar stays a fixed headroom above it: a kernel may round differently from the
CPU, not by an order of magnitude more."""
import functools

import pytest
import torch

from tests import test_scene_matrix_gpu as M

# a bar is at least HEADROOM x the float32 oracle's deviation; a bar above 2e-6 is at most BAR_FACTOR * 4 x it (CPUs differ
# in their float32 rounding by a factor of two or so)
HEADROOM = 4


def _acc(out, name, e):
    out[name] = max(out.get(name, 0.), e)


@functools.lru_cache(maxsize=None)
def float32_deviations():
    out = {}
    for case in M.GEOM_CASES:
        for seed in (0, 1):                                        # the seam test's inputs, then the C-ABI test's
            x = M.geom_inputs(case, seed)
            wb, wg = M.geom_cotangents(x, seed)
            b64, g64, grads64 = M.oracle_geometry_grads(x, torch.float64, wb, wg)
            b32, g32, grads32 = M.oracle_geometry_grads(x, torch.float32, wb, wg)
            _acc(out, 'geom.verts', max(M.rel_err(b32, b64), M.rel_err(g32, g64)))
            for n, a, b in zip(M.GEOM_LEAVES, grads32, grads64):
                _acc(out, M.geom_bar(n, case), M.rel_err(a, b))
    for case in M.OPACITY_CASES:
        lg, noise, _ = M.opacity_inputs(case)
        N, thr = case[0], case[2]
        ga, gk = torch.randn(N, generator=M._gen(2), dtype=torch.float64), torch.randn(N, generator=M._gen(3), dtype=torch.float64)
        runs = {dt: M.oracle_opacity(lg, noise, thr, dt) for dt in (torch.float32, torch.float64)}
        for i in (1, 2):
            _acc(out, 'opacity.alpha', M.rel_err(runs[torch.float32][i], runs[torch.float64][i]))
        for wa, wk in ((ga, gk), (ga, None), (None, gk)):
            g = {dt: torch.autograd.grad(sum((r[i] * w.to(dt)).sum() for i, w in ((1, wa), (2, wk)) if w is not None), r[0],
                                         retain_graph=True)[0] for dt, r in runs.items()}
            _acc(out, 'opacity.g_logit', M.rel_err(g[torch.float32], g[torch.float64]))
    tex_launches = M.TEX_CASES + [[(M.CELLS4, 2, 64, 8, 0, 0, 5.), (M.CELLS4, 5, 40, 8, 0, 0, 5.)]]
    for case in tex_launches:
        for k, job in enumerate(case):
            x, w = M.tex_inputs(case, k), M.tex_cotangent(job, k)
            o64, g64 = M.oracle_texture_grads(job, x, w, torch.float64)
            o32, g32 = M.oracle_texture_grads(job, x, w, torch.float32)
            _acc(out, 'tex.out', M.rel_err(o32, o64))
            _acc(out, 'tex.grad', M.rel_err(g32, g64))
    for phase in M.CHAIN_PHASES:
        ws = M.chain_cotangents(phase, M.chain_shapes(phase))
        o64, keep64, g64 = M.chain_oracle(phase, torch.float64, ws)
        o32, keep32, g32 = M.chain_oracle(phase, torch.float32, ws)
        for k in M.CHAIN_OUTPUTS:
            if o64[k] is not None:
                _acc(out, f'chain.{k}', M.rel_err(o32[k], o64[k]))
        for k in M.CHAIN_LEAVES:
            if g64[k] is not None:
                _acc(out, f'chain.{k}', M.rel_err(g32[k], g64[k]))
    return out


def test_every_bar_is_measured_and_every_loose_bar_explained():
    assert set(float32_deviations()) == set(M.BARS)
    assert {k for k, v in M.BARS.items() if v > 2e-6} <= set(M.BAR_NOTES)


@pytest.mark.parametrize('name', sorted(M.BARS))
def test_bar_sits_a_fixed_multiple_above_float32_rounding(name):
    dev, bar = float32_deviations()[name], M.BARS[name]
    assert HEADROOM * dev <= bar, f'{name}: float32 oracle deviates by {dev:.3g} of max; bar {bar:.3g} leaves less than {HEADROOM}x'
    assert bar <= 2e-6 or bar <= 4 * M.BAR_FACTOR * dev, f'{name}: bar {bar:.3g} is loose for a float32 deviation of {dev:.3g}'


def test_keep_decisions_do_not_depend_on_precision():
    """the opacity and model-chain cases keep their logits clear of logit(threshold): float32 and float64 keep the same blocks"""
    for case in M.OPACITY_CASES:
        lg, noise, _ = M.opacity_inputs(case)
        assert torch.equal(torch.sigmoid(lg) > case[2], torch.sigmoid(lg.double()) > case[2]) or case[2] < 0
    for phase in M.CHAIN_PHASES:
        _, thr = M.chain_phase_settings(phase)[2:4]
        lg = M.chain_params(phase)['alpha_logit']
        assert ((torch.sigmoid(lg.double()) - thr).abs() > 1e-3).all()
