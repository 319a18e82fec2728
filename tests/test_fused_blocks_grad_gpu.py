"""GPU: the blocks pass differentiated inside its loss-epilogue forward kernel (fused_loss.FUSE_BLOCKS_BACKWARD:
dbw_render_forward_loss_grad + dbw_render_backward_deferred) against the two-kernel path it replaces (fragment records in
the workspace, then raster_backward_kernel).  The loss is bit-identical; the gradients agree to the rounding of the atomics'
order (4x the spread of two identical two-kernel runs, at least 1e-5 of the largest magnitude).  The two-kernel path itself
is pinned to the float64 oracle by test_raster_matrix_gpu.py."""
import ctypes

import pytest
import torch

from oracle import dbw_path as D
from tests.test_raster_matrix_gpu import BANDS, _close_to_cuda, _pack_maps

pytestmark = pytest.mark.gpu

NAMES = ('env verts', 'env maps', 'blocks verts', 'blocks cells', 'alpha')
KEYS = ('ev', 'em', 'bv', 'bm', 'ba')


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


class _Spy:
    """stands in for the loaded library: records (entry, args) of every call fused_loss makes"""

    def __init__(self, L):
        self.L, self.calls = L, []

    def __getattr__(self, name):
        fn = getattr(self.L, name)

        def call(*args):
            self.calls.append((name, args))
            return fn(*args)
        return call

    def names(self):
        return [n for n, _ in self.calls]


@pytest.fixture
def spy(monkeypatch):
    from dbw_b200 import _lib, fused_loss
    s = _Spy(_lib.lib())
    monkeypatch.setattr(fused_loss._lib, 'lib', lambda: s)
    yield s


def _scene(dev, Kf, alpha, H=40, W=56, B=2, seed=13):
    """environment (float4 atlas) + blocks over float4 CELL maps (4x decimated, circular padding 1 + 1) as the coarse phase of
    a training step renders them: (inputs, env pass, blocks pass)"""
    from dbw_b200 import Renderer
    from dbw_b200.fused_loss import ScenePass
    from dbw_b200.scene_ops import cell_map_table
    tpl = D.SceneTemplate(n_blocks=4, txt_size=16)
    p = D.init_params(4, 16, seed=seed)
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=seed)
    env = tpl.build_env(p)
    blocks, blk_alpha = tpl.build_blocks(p)
    assert blocks['maps'][0].shape == (16, 18, 3)

    def renderer(**kw):
        r = Renderer((H, W), z_clip=0.001, cameras={'name': 'perspective'}, **kw).to(dev)
        r.update_cameras(device=dev, K=K[None].to(dev))
        return r

    em, et = _pack_maps(env['maps'], True)
    g = torch.Generator().manual_seed(seed)
    cells = torch.rand(4 * 4 * 4, 4, generator=g)
    cells[:, 3] = 0
    i32 = lambda t: t.to(dev).to(torch.int32)
    env_pass = ScenePass(i32(env['faces']), env['faces_verts_uvs'].to(dev), i32(env['face_map']), et,
                         renderer(faces_per_pixel=1, sigma=0), n_static_faces=tpl.bkg_faces.shape[0])
    group = {None: 1, 'face': 1, 'block': tpl.BNF, 'view_block': tpl.BNF}[alpha]
    blk_pass = ScenePass(i32(blocks['faces']), blocks['faces_verts_uvs'].to(dev), i32(blocks['face_map']),
                         cell_map_table(4, 16, 4, 1, 1), renderer(faces_per_pixel=Kf, sigma=1e-4, detach_bary=True),
                         alpha_group=group)
    a = blk_alpha.detach() * torch.linspace(0.6, 1.2, len(blk_alpha))
    ba = {None: None, 'face': a.repeat_interleave(tpl.BNF), 'block': a, 'view_block': a.repeat(B)}[alpha]
    leaf = lambda t: t.to(dev).requires_grad_(True)
    x = dict(ev=leaf(env['verts'].detach()), em=leaf(em), bv=leaf(blocks['verts'].detach()), bm=leaf(cells.reshape(-1)),
             ba=None if ba is None else leaf(ba), R=R.to(dev), T=T.to(dev),
             imgs=torch.rand(B, 3, H, W, generator=g).to(dev), fmap=i32(blocks['face_map']))
    return x, env_pass, blk_pass


def _loss(x, env_pass, blk_pass, view_rows=None):
    from dbw_b200.fused_loss import scene_mse
    return scene_mse(x['ev'], x['em'], x['bv'], x['bm'], x['ba'], x['R'], x['T'], x['imgs'], env_pass, blk_pass, x['fmap'],
                     view_rows=view_rows)


def _step(x, env_pass, blk_pass, fused, view_rows=None, scale=1.0, extra=()):
    """(loss, gradients of the leaves that require grad, in KEYS order then `extra`) with the fused path on or off"""
    from dbw_b200 import fused_loss
    old, fused_loss.FUSE_BLOCKS_BACKWARD = fused_loss.FUSE_BLOCKS_BACKWARD, fused
    try:
        loss = _loss(x, env_pass, blk_pass, view_rows)
        leaves = [x[k] for k in KEYS + tuple(extra) if x[k] is not None and x[k].requires_grad]
        g = torch.autograd.grad(loss * scale, leaves)
    finally:
        fused_loss.FUSE_BLOCKS_BACKWARD = old
    return loss.detach(), list(g)


def _compare(got, ref, ref2, names, floor=1e-5):
    assert len(got) == len(ref) == len(names)
    for a, b, b2, name in zip(got, ref, ref2, names):
        assert b.abs().max() > 0, name
        _close_to_cuda(a, b, b2, name, floor=floor)


@pytest.mark.parametrize('alpha', [None, 'face', 'view_block'])
@pytest.mark.parametrize('Kf', [1, 3, 10, 25])
def test_fused_matches_two_kernel_path(Kf, alpha, spy):
    x, env_pass, blk_pass = _scene(_dev(), Kf, alpha)
    l2, g2 = _step(x, env_pass, blk_pass, False)
    _, g2b = _step(x, env_pass, blk_pass, False)
    assert 'dbw_render_forward_loss_grad' not in spy.names()
    spy.calls.clear()
    l1, g1 = _step(x, env_pass, blk_pass, True)
    names = spy.names()
    assert 'dbw_render_forward_loss_grad' in names and 'dbw_render_backward_deferred' in names
    assert 'dbw_render_forward_loss' not in names                  # the blocks pass wrote no d loss / d RGBA image
    assert torch.equal(l1, l2), (l1.item(), l2.item())
    _compare(g1, g2, g2b, NAMES[:4] + (('alpha',) if alpha else ()))


def test_fused_forward_writes_no_fragment_records(spy):
    """the fused forward runs with save_fragment_state = 0: its workspace is smaller by the two 16 B records per (pixel,
    layer) and the count per pixel"""
    from dbw_b200 import _lib
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    _step(x, env_pass, blk_pass, True)
    (args,) = [a for n, a in spy.calls if n == 'dbw_render_forward_loss_grad']
    cfg = args[0]._obj
    assert cfg.save_fragment_state == 0
    on = _lib.DbwRenderSettings.from_buffer_copy(cfg)
    on.save_fragment_state = 1
    sizes = []
    for c in (cfg, on):
        fwd, bwd = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(_lib.lib().dbw_workspace_bytes(ctypes.byref(c), ctypes.byref(fwd), ctypes.byref(bwd)), 'dbw_workspace_bytes')
        sizes.append(fwd.value)
    npx = cfg.n_views * cfg.height * cfg.width
    assert args[11] == sizes[0]                                   # the workspace the call was given
    assert sizes[1] - sizes[0] >= npx * cfg.faces_per_pixel * 32 + npx


@pytest.mark.parametrize('Kf', [3, 10])
def test_fused_row_bands(Kf):
    """row bands (an empty band and a one-row band among them): the fused gradients of a partition of the rows sum to the
    two-kernel gradient of the whole image"""
    dev = _dev()
    x, env_pass, blk_pass = _scene(dev, Kf, 'view_block', H=72, W=40)
    l_full, g_full = _step(x, env_pass, blk_pass, False)
    _, g_full2 = _step(x, env_pass, blk_pass, False)
    tot, g_sum = 0.0, None
    for rows in BANDS:
        l, g = _step(x, env_pass, blk_pass, True, view_rows=torch.tensor(rows, dtype=torch.int32, device=dev))
        tot += l.item()
        g_sum = g if g_sum is None else [a + b for a, b in zip(g_sum, g)]
    assert abs(tot - l_full.item()) <= 1e-6 * abs(l_full.item())
    _compare(g_sum, g_full, g_full2, NAMES, floor=1e-4)


def test_fused_upstream_scale():
    """the deferred fold multiplies by the upstream gradient of the loss (here loss x 0.37)"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    _, g2 = _step(x, env_pass, blk_pass, False, scale=0.37)
    _, g2b = _step(x, env_pass, blk_pass, False, scale=0.37)
    _, g1 = _step(x, env_pass, blk_pass, True, scale=0.37)
    _, g_unit = _step(x, env_pass, blk_pass, True)
    _compare(g1, g2, g2b, NAMES)
    assert (g1[2] - 0.37 * g_unit[2]).norm() <= 1e-5 * g1[2].norm()


def test_fused_partial_gradients(spy):
    """every subset of {blocks verts, blocks cells, alpha} requiring grad gets the gradients of the all-gradients call"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    _, g_all = _step(x, env_pass, blk_pass, True)
    _, g_all2 = _step(x, env_pass, blk_pass, False)
    full = dict(zip(KEYS, g_all))
    full2 = dict(zip(KEYS, g_all2))
    blk = ('bv', 'bm', 'ba')
    for mask in range(1, 7):
        want = [k for i, k in enumerate(blk) if mask >> i & 1]
        for k in blk:
            x[k].requires_grad_(k in want)
        spy.calls.clear()
        _, g = _step(x, env_pass, blk_pass, True)
        assert 'dbw_render_forward_loss_grad' in spy.names(), want
        got = dict(zip([k for k in KEYS if x[k].requires_grad], g))
        for k in want:
            _close_to_cuda(got[k], full[k], full2[k], f'{want}: {k}')
    for k in blk:
        x[k].requires_grad_(True)


def test_fused_pose_gradients():
    """g_R and g_T through the deferred fold's camera_grad_kernel equal the two-kernel path's"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    x['R'].requires_grad_(True)
    x['T'].requires_grad_(True)
    _, g2 = _step(x, env_pass, blk_pass, False, extra=('R', 'T'))
    _, g2b = _step(x, env_pass, blk_pass, False, extra=('R', 'T'))
    _, g1 = _step(x, env_pass, blk_pass, True, extra=('R', 'T'))
    _compare(g1, g2, g2b, NAMES + ('R', 'T'))


def test_fused_pose_gradients_alone(spy):
    """only the poses require grad: the fused forward still computes the vertex-path scratch the camera gradient needs"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    for k in KEYS:
        if x[k] is not None:
            x[k].requires_grad_(False)
    x['R'].requires_grad_(True)
    x['T'].requires_grad_(True)
    _, g2 = _step(x, env_pass, blk_pass, False, extra=('R', 'T'))
    _, g2b = _step(x, env_pass, blk_pass, False, extra=('R', 'T'))
    spy.calls.clear()
    _, g1 = _step(x, env_pass, blk_pass, True, extra=('R', 'T'))
    assert 'dbw_render_forward_loss_grad' in spy.names()
    _compare(g1, g2, g2b, ('R', 'T'))


def test_no_grad_runs_no_fused_differentiation(spy):
    from dbw_b200 import fused_loss
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
    assert fused_loss.FUSE_BLOCKS_BACKWARD
    l_grad, _ = _step(x, env_pass, blk_pass, True)
    spy.calls.clear()
    with torch.no_grad():
        l = _loss(x, env_pass, blk_pass)
    names = spy.names()
    assert 'dbw_render_forward_loss' in names and 'dbw_render_forward_loss_grad' not in names
    assert torch.equal(l, l_grad)


def test_fused_graph_replay_equals_eager():
    """forward + backward of the fused path captured in a CUDA graph: a replay gives the eager results"""
    x, env_pass, blk_pass = _scene(_dev(), 10, 'view_block')
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
    assert torch.equal(l_static, l_eager)
    _compare(g_static, g_eager, g_eager2, NAMES)
