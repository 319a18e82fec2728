"""GPU: the coarse phase's blocks loss pass in its own kernel (blocks_loss_kernel, the BLOCKS instantiation of the forward
body) against the generic raster_forward_kernel<128, true> (dbw_debug_generic_blocks_loss(1)), on the same inputs.  The loss and the
environment's gradient image are bit-identical; the leaf gradients agree to the rounding of the atomics' order (1e-6 of
each array's largest magnitude, or 4x the spread of two generic runs).  The generic kernel itself is pinned to the
two-kernel path by test_fused_blocks_grad_gpu.py and to the float64 oracle by test_epilogue_matrix_gpu.py."""
import ctypes
from copy import deepcopy

import pytest
import torch

from oracle import dbw_path as D
from tests.test_fused_blocks_grad_gpu import KEYS, NAMES, _Spy
from tests.test_raster_matrix_gpu import BANDS, _close_to_cuda, _pack_maps

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _scene(dev, Kf, alpha, n_blocks=4, H=40, W=56, B=2, dist=2.75, seed=13):
    """test_fused_blocks_grad_gpu's scene (environment + blocks over cell maps) with a block count and a camera distance"""
    from dbw_b200 import Renderer
    from dbw_b200.fused_loss import ScenePass
    from dbw_b200.scene_ops import cell_map_table
    tpl = D.SceneTemplate(n_blocks=n_blocks, txt_size=16)
    p = D.init_params(n_blocks, 16, seed=seed)
    R, T, K = D.ring_cameras(B, dist=dist, jitter=0.3, seed=seed)
    env = tpl.build_env(p)
    blocks, blk_alpha = tpl.build_blocks(p)

    def renderer(**kw):
        r = Renderer((H, W), z_clip=0.001, cameras={'name': 'perspective'}, **kw).to(dev)
        r.update_cameras(device=dev, K=K[None].to(dev))
        return r

    em, et = _pack_maps(env['maps'], True)
    g = torch.Generator().manual_seed(seed)
    cells = torch.rand(n_blocks * 4 * 4, 4, generator=g)
    cells[:, 3] = 0
    i32 = lambda t: t.to(dev).to(torch.int32)
    env_pass = ScenePass(i32(env['faces']), env['faces_verts_uvs'].to(dev), i32(env['face_map']), et,
                         renderer(faces_per_pixel=1, sigma=0), n_static_faces=tpl.bkg_faces.shape[0])
    group = {None: 1, 'face': 1, 'block': tpl.BNF, 'view_block': tpl.BNF}[alpha]
    blk_pass = ScenePass(i32(blocks['faces']), blocks['faces_verts_uvs'].to(dev), i32(blocks['face_map']),
                         cell_map_table(n_blocks, 16, 4, 1, 1), renderer(faces_per_pixel=Kf, sigma=1e-4, detach_bary=True),
                         alpha_group=group)
    a = blk_alpha.detach() * torch.linspace(0.6, 1.2, len(blk_alpha))
    ba = {None: None, 'face': a.repeat_interleave(tpl.BNF), 'block': a, 'view_block': a.repeat(B)}[alpha]
    leaf = lambda t: t.to(dev).requires_grad_(True)
    x = dict(ev=leaf(env['verts'].detach()), em=leaf(em), bv=leaf(blocks['verts'].detach()), bm=leaf(cells.reshape(-1)),
             ba=None if ba is None else leaf(ba), R=R.to(dev), T=T.to(dev),
             imgs=torch.rand(B, 3, H, W, generator=g).to(dev), fmap=i32(blocks['face_map']))
    return x, env_pass, blk_pass


class _GEnvSpy(_Spy):
    """also runs every dbw_render_forward_loss_grad call once more into a private g_env with the kernel `generic` selects,
    and keeps that copy: (generic, g_env) per call"""

    def __init__(self, L):
        super().__init__(L)
        self.g_env = []

    def __getattr__(self, name):
        fn = getattr(self.L, name)
        if name != 'dbw_render_forward_loss_grad':
            return super().__getattr__(name)

        def call(*args):
            self.calls.append((name, args))
            ep = args[12]._obj
            cfg = args[0]._obj
            mine = type(ep).from_buffer_copy(ep)
            g = torch.zeros(cfg.n_views, 4, cfg.height, cfg.width, device='cuda')       # the alpha plane may stay unwritten
            part = torch.zeros(ep.n_partials, device='cuda')
            mine.g_env, mine.loss_partials = g.data_ptr(), part.data_ptr()
            rc = fn(*args[:12], ctypes.byref(mine), *args[13:])
            if rc == 0:
                self.g_env.append(g)
            return rc if rc != 0 else fn(*args)
        return call


@pytest.fixture
def genv_spy(monkeypatch):
    from dbw_b200 import _lib, fused_loss
    s = _GEnvSpy(_lib.lib())
    monkeypatch.setattr(fused_loss._lib, 'lib', lambda: s)
    yield s


def _set_generic(on):
    from dbw_b200 import _lib
    _lib.lib().dbw_debug_generic_blocks_loss(1 if on else 0)


def _run(x, env_pass, blk_pass, generic, view_rows=None):
    """(loss, leaf gradients in KEYS order, launches of blocks_loss_kernel)"""
    from dbw_b200 import _lib
    from dbw_b200.fused_loss import scene_mse
    L = _lib.lib()
    _set_generic(generic)
    L.dbw_timing_reset()
    L.dbw_timing_enable(1)
    try:
        loss = scene_mse(x['ev'], x['em'], x['bv'], x['bm'], x['ba'], x['R'], x['T'], x['imgs'], env_pass, blk_pass,
                         x['fmap'], view_rows=view_rows)
        leaves = [x[k] for k in KEYS if x[k] is not None and x[k].requires_grad]
        g = torch.autograd.grad(loss, leaves)
        torch.cuda.synchronize()
        launches = _lib.kernel_time_ms(2)[1]
    finally:
        L.dbw_timing_enable(0)
        L.dbw_timing_reset()
        _set_generic(False)
    return loss.detach(), list(g), launches


def _ab(x, env_pass, blk_pass, spy, expect_dedicated=True, view_rows=None, nonzero=True):
    spy.g_env.clear()
    l_g, g_g, n_g = _run(x, env_pass, blk_pass, True, view_rows)
    _, g_g2, _ = _run(x, env_pass, blk_pass, True, view_rows)
    ge_generic = list(spy.g_env)
    spy.g_env.clear()
    l_n, g_n, n_n = _run(x, env_pass, blk_pass, False, view_rows)
    ge_new = list(spy.g_env)
    assert n_g == 0
    assert (n_n > 0) == expect_dedicated, n_n
    assert torch.equal(l_n, l_g), (l_n.item(), l_g.item())
    assert ge_new and len(ge_new) * 2 == len(ge_generic)
    for a, b in zip(ge_new, ge_generic):
        assert torch.equal(a, b)
    names = NAMES[:4] + (('alpha',) if x['ba'] is not None else ())
    for a, b, b2, name in zip(g_n, g_g, g_g2, names):
        assert b.abs().max() > 0 or not nonzero, name
        _close_to_cuda(a, b, b2, name, floor=1e-6)
    return l_n


@pytest.mark.parametrize('alpha', [None, 'face', 'block', 'view_block'])
@pytest.mark.parametrize('Kf', [10, 25])
def test_dedicated_kernel_matches_generic(Kf, alpha, genv_spy):
    x, env_pass, blk_pass = _scene(_dev(), Kf, alpha)
    _ab(x, env_pass, blk_pass, genv_spy)


def test_many_opacity_entries_fall_back_to_generic(genv_spy):
    """per-face opacities of 8 blocks: 640 entries per view, more than the shared-memory table holds -> generic kernel"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'face', n_blocks=8)
    _ab(x, env_pass, blk_pass, genv_spy, expect_dedicated=False)


@pytest.mark.parametrize('Kf', [10, 25])
def test_z_clipped_views(Kf, genv_spy):
    """cameras among the blocks: faces straddle the near plane, the views have z-clipped slots (sorted offer order)"""
    x, env_pass, blk_pass = _scene(_dev(), Kf, 'view_block', n_blocks=8, dist=0.45, seed=5)
    _ab(x, env_pass, blk_pass, genv_spy)


@pytest.mark.parametrize('Kf', [10, 25])
def test_chunked_path(Kf, genv_spy):
    """8 blocks in a 16 x 16 image: a tile lists far more than 64 faces, the list is refilled (chunked path)"""
    x, env_pass, blk_pass = _scene(_dev(), Kf, 'view_block', n_blocks=8, H=16, W=16)
    _ab(x, env_pass, blk_pass, genv_spy)


def test_row_bands(genv_spy):
    dev = _dev()
    x, env_pass, blk_pass = _scene(dev, 10, 'view_block', H=72, W=40)
    for rows in BANDS:          # an empty and a one-row band among them
        _ab(x, env_pass, blk_pass, genv_spy, view_rows=torch.tensor(rows, dtype=torch.int32, device=dev), nonzero=False)


def test_graph_replay():
    """forward + backward captured in a CUDA graph with each kernel: replays give the eager loss bit for bit"""
    from dbw_b200.fused_loss import scene_mse
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    leaves = [x[k] for k in KEYS if x[k] is not None]

    def step():
        loss = scene_mse(x['ev'], x['em'], x['bv'], x['bm'], x['ba'], x['R'], x['T'], x['imgs'], env_pass, blk_pass, x['fmap'])
        return loss.detach(), torch.autograd.grad(loss, leaves)

    out = {}
    for generic in (True, False):
        _set_generic(generic)
        try:
            l_eager, g_eager = step()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    step()
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                l_static, g_static = step()
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(l_static, l_eager)
            out[generic] = (l_static.clone(), [g.clone() for g in g_static], [g.clone() for g in g_eager])
        finally:
            _set_generic(False)
    assert torch.equal(out[True][0], out[False][0])
    for a, b, b2, name in zip(out[False][1], out[True][1], out[True][2], NAMES):
        _close_to_cuda(a, b, b2, name, floor=1e-6)


def test_dedicated_kernel_runs_at_the_bench_shape():
    """an eager training step of bench.py's dtu model runs blocks_loss_kernel for its blocks pass, and the generic kernel
    once dbw_debug_generic_blocks_loss(1) asks for it"""
    import bench
    from dbw_b200 import _lib
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.parallel import ViewParallel
    w = bench.WORKLOADS['dtu']
    dev = _dev()
    torch.manual_seed(bench.SEED)
    model = DifferentiableBlocksWorld((w['height'], w['width']), **deepcopy(bench.model_cfg(w))).to(dev)
    model.train()
    vp = ViewParallel(model, seed=bench.SEED)
    inp = {k: v.to(dev) for k, v in bench.synthetic_inputs(w).items()}
    L = _lib.lib()
    counts = []
    for generic in (False, True):
        _set_generic(generic)
        L.dbw_timing_reset()
        L.dbw_timing_enable(1)
        try:
            vp.forward_backward(inp)
            torch.cuda.synchronize()
            counts.append((_lib.kernel_time_ms(2, w['faces_per_pixel'])[1], _lib.kernel_time_ms(0, w['faces_per_pixel'])[1]))
        finally:
            L.dbw_timing_enable(0)
            L.dbw_timing_reset()
            _set_generic(False)
    (d0, f0), (d1, f1) = counts
    assert d0 == f0 > 0, counts
    assert d1 == 0 and f1 > 0, counts
