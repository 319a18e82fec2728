"""GPU: the environment pass without what its backward never reads.  A hard single-layer pass without opacities keeps no
fragment colours, and the blocks loss epilogue leaves the alpha plane of g_env unwritten (env_alpha_unread).  With every
buffer the step allocates uninitialised filled with NaN, the gradients must still be finite.  They must equal the
computation that keeps both, forced on by dbw_debug_keep_unread_outputs: the loss bit for bit, the gradients to 4x the
spread of two runs of that computation (atomics add in varying order).  The cases are the fused scene of
test_fused_blocks_grad_gpu, row bands with an empty band among them, pose gradients, a CUDA-graph replay, and the bench's
model at a reduced image size."""
import ctypes
from copy import deepcopy

import pytest
import torch

from tests.test_fused_blocks_grad_gpu import NAMES, _compare, _dev, _scene, _step
from tests.test_raster_matrix_gpu import BANDS

pytestmark = pytest.mark.gpu


class _NaNTorch:
    """the torch module as fused_loss sees it, with torch.empty returning NaN (float) or 0xff bytes (workspaces: NaN floats)"""

    def __init__(self):
        self.n_empty = 0

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *shape, dtype=None, device=None):
        self.n_empty += 1
        t = torch.empty(*shape, dtype=dtype, device=device)
        return t.fill_(255) if t.dtype == torch.uint8 else t.fill_(float('nan'))


@pytest.fixture
def poison(monkeypatch):
    from dbw_b200 import fused_loss
    p = _NaNTorch()
    monkeypatch.setattr(fused_loss, 'torch', p)
    yield p


class _KeepUnread:
    """dbw_debug_keep_unread_outputs(1) for the duration: colours kept, g_env's alpha plane written"""

    def __enter__(self):
        from dbw_b200 import _lib
        _lib.lib().dbw_debug_keep_unread_outputs(1)

    def __exit__(self, *exc):
        from dbw_b200 import _lib
        _lib.lib().dbw_debug_keep_unread_outputs(0)


def _finite(gs):
    for g in gs:
        assert torch.isfinite(g).all()


def _old_and_new(run):
    """run() twice with the unread outputs kept, once without: (loss, grads) of each"""
    with _KeepUnread():
        old, old2 = run(), run()
    new = run()
    for r in (old, old2, new):
        _finite(r[1])
    return old, old2, new


def test_poisoned_buffers_match_the_path_that_keeps_them(poison):
    from dbw_b200 import _lib
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    (l_old, g_old), (_, g_old2), (l_new, g_new) = _old_and_new(lambda: _step(x, env_pass, blk_pass, True))
    assert poison.n_empty > 0
    assert torch.equal(l_new, l_old), (l_new.item(), l_old.item())
    _compare(g_new, g_old, g_old2, NAMES)
    # the environment pass really ran without colours: its settings declare no opacities
    cfg = env_pass.settings(x['ev'], x['em'], 2, None)[0]
    assert cfg.save_fragment_state == 2 and cfg.faces_per_pixel == 1 and cfg.sigma == 0
    sizes = []
    for keep in (1, 0):
        _lib.lib().dbw_debug_keep_unread_outputs(keep)
        fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(_lib.lib().dbw_workspace_bytes(ctypes.byref(cfg), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
        sizes.append(fwd.value)
    assert sizes[0] > sizes[1]


@pytest.mark.parametrize('fused', [False, True])
def test_two_kernel_blocks_path(fused, poison):
    """with the blocks pass differentiated by raster_backward_kernel too (g_env then comes from dbw_render_forward_loss)"""
    x, env_pass, blk_pass = _scene(_dev(), 3, None)
    (l_old, g_old), (_, g_old2), (l_new, g_new) = _old_and_new(lambda: _step(x, env_pass, blk_pass, fused))
    assert torch.equal(l_new, l_old)
    _compare(g_new, g_old, g_old2, NAMES[:4])


def test_row_bands(poison):
    """a partition of the rows (an empty band and a one-row band among them): rows outside a call's band are never written
    and never read"""
    dev = _dev()
    x, env_pass, blk_pass = _scene(dev, 10, 'view_block', H=72, W=40)

    def banded():
        tot, g_sum = None, None
        for rows in BANDS:
            l, g = _step(x, env_pass, blk_pass, True, view_rows=torch.tensor(rows, dtype=torch.int32, device=dev))
            tot = l if tot is None else tot + l
            g_sum = g if g_sum is None else [a + b for a, b in zip(g_sum, g)]
        return tot, g_sum
    (l_old, g_old), (_, g_old2), (l_new, g_new) = _old_and_new(banded)
    assert torch.equal(l_new, l_old)
    _compare(g_new, g_old, g_old2, NAMES, floor=1e-4)


def test_pose_gradients(poison):
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    x['R'].requires_grad_(True)
    x['T'].requires_grad_(True)
    (l_old, g_old), (_, g_old2), (l_new, g_new) = _old_and_new(lambda: _step(x, env_pass, blk_pass, True, extra=('R', 'T')))
    assert torch.equal(l_new, l_old)
    _compare(g_new, g_old, g_old2, NAMES + ('R', 'T'))


def test_graph_replay(poison):
    """forward + backward captured in a CUDA graph (the NaN fills are captured with it): a replay gives the eager results of
    the path that keeps the unread outputs"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    with _KeepUnread():
        l_eager, g_eager = _step(x, env_pass, blk_pass, True)
        _, g_eager2 = _step(x, env_pass, blk_pass, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _step(x, env_pass, blk_pass, True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        l_static, g_static = _step(x, env_pass, blk_pass, True)
    graph.replay()
    torch.cuda.synchronize()
    _finite(g_static)
    assert torch.equal(l_static, l_eager)
    _compare(g_static, g_eager, g_eager2, NAMES)


def test_bench_model(poison):
    """the bench's scene (its model configuration: 10 blocks, 256^2 textures, decoupled env + blocks, K = 10) at 6 views of
    96 x 128: loss and every parameter gradient"""
    import bench
    from dbw_b200.dbw import DifferentiableBlocksWorld
    dev = _dev()
    w = dict(bench.WORKLOADS['dtu'], n_views=6, height=96, width=128)
    torch.manual_seed(bench.SEED)
    model = DifferentiableBlocksWorld((w['height'], w['width']), **deepcopy(bench.model_cfg(w))).to(dev)
    model.train()
    inp = {k: v.to(dev) for k, v in bench.synthetic_inputs(w).items()}
    params = [p for p in model.parameters() if p.requires_grad]
    # the step's opacity noise, drawn once: every run renders the same scene
    model.opacity_noise_buffer = torch.randn(model.alpha_logit.shape, generator=torch.Generator().manual_seed(1)).to(dev)
    assert model._fused_loss_ok(inp['imgs'])

    def run():
        total = model(inp, None)['total']
        gs = torch.autograd.grad(total, params, allow_unused=True)
        return total.detach(), [g if g is not None else torch.zeros_like(p) for g, p in zip(gs, params)]
    (l_old, g_old), (_, g_old2), (l_new, g_new) = _old_and_new(run)
    assert torch.equal(l_new, l_old)
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    keep = [i for i, g in enumerate(g_old) if g.abs().max() > 0]
    assert len(keep) >= 5, names
    _compare([g_new[i] for i in keep], [g_old[i] for i in keep], [g_old2[i] for i in keep], [names[i] for i in keep])
