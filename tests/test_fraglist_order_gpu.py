"""GPU: the fragments a pixel keeps where both halves of a z-clipped quad reach it, against the float64 oracle, exactly.

Of the two halves of a quad split by the near plane a pixel keeps the one nearer to it, and the rule acts on the list as it
stands, so the kept fragments depend on the order the faces are offered in (tests/test_fraglist_order_host.py).  The oracle
offers them in the clipped mesh's face order; raster_forward_kernel sorts its tile list into that order (fast path) or scans
and compacts in it (chunked path, coarse bins).  The parity tests of test_raster_matrix_gpu.py exclude every pixel whose
kept ids differ from the oracle's; here the excluded pixels are sorted by their margins instead:

- a NEAR-TIE is a pixel where some candidate face's inside test, halo test (|dist - blur|), depth order against another
  candidate, or the quad rule (| |d_A| - |d_B| |) is decided by less than an fp32 bound (_Margins), so float32 and float64
  may legitimately decide it differently;
- everything else is a REAL DISAGREEMENT, and there must be none.

At the DECISIVE pixels -- both halves of a quad are candidates and every margin is well above the bound -- the kept ids must
equal the oracle's exactly, and the image and gradients there are compared with no exclusion at all.  Two runs must be bit
identical (ids, distances, image)."""
import functools

import numpy as np
import pytest
import torch

from oracle import dbw_path as D
from oracle import pt3d
from tests.helpers import decision_mask, intrinsics, slots_to_clipped_idx
from tests.test_raster_matrix_gpu import IMG_TOL, _cams, _composite_loss, _dev, _dev_scene, _leaf, _oracle, _pack_maps, _pairs, _parity

pytestmark = pytest.mark.gpu

SIZE = (200, 264)                   # 4 x 5 coarse bins of 64 px
KS = [1, 2, 3, 10, 25]              # 1-3: raster_forward_kernel<256, *>, 10 and 25: <128, *>
SIGMAS = [1e-4, 5e-6]
# fp32 bounds of the margins: relative to the depth, to the squared halo radius, and to the face's coordinate scale
# (edge functions and squared distances are formed from NDC coordinates rounded to ~6e-8 of their magnitude)
REL_Z = 2e-5
REL_D = 2e-5
ABS_E = 1e-5


# ------------------------------------------------------------------------------------------------ float64 candidate margins
class _Margins:
    """per pixel of (B, H, W), from every (pixel, clipped face) candidate of the float64 oracle's rasterizer (raster_oracle.c):
    quad = both halves of some quad are candidates; near = some decision at the pixel is within the fp32 bounds above"""

    def __init__(self, fv, mesh_first, mesh_nfaces, neighbor, H, W, blur, persp):
        B = len(mesh_first)
        self.quad = np.zeros((B, H, W), bool)
        self.near = np.zeros((B, H, W), bool)
        fv = fv.detach().double().numpy()
        nb = neighbor.numpy() if neighbor is not None else np.full(len(fv), -1)
        xs = np.array([float(pt3d_ndc(W - 1 - x, W, H)) for x in range(W)])
        ys = np.array([float(pt3d_ndc(H - 1 - y, H, W)) for y in range(H)])
        sb = np.sqrt(blur)
        for n in range(B):
            cand = []                                      # (pixel, face, pz, |dist|)
            f0, f1 = int(mesh_first[n]), int(mesh_first[n] + mesh_nfaces[n])
            for f in range(f0, f1):
                (x0, y0, z0), (x1, y1, z1), (x2, y2, z2) = fv[f]
                if min(z0, z1, z2) < 1e-8:
                    continue
                area = (x2 - x0) * (y1 - y0) - (y2 - y0) * (x1 - x0)
                if abs(area) <= 1e-8:
                    continue
                cx = np.nonzero((xs >= min(x0, x1, x2) - sb) & (xs <= max(x0, x1, x2) + sb))[0]
                cy = np.nonzero((ys >= min(y0, y1, y2) - sb) & (ys <= max(y0, y1, y2) + sb))[0]
                if not len(cx) or not len(cy):
                    continue
                px, py = np.meshgrid(xs[cx], ys[cy])
                e = [(px - xa) * (yb - ya) - (py - ya) * (xb - xa)
                     for (xa, ya), (xb, yb) in (((x1, y1), (x2, y2)), ((x2, y2), (x0, y0)), ((x0, y0), (x1, y1)))]
                a = area + 1e-8
                w = [ei / a for ei in e]
                if persp:
                    t = [w[0] * z1 * z2, z0 * w[1] * z2, z0 * z1 * w[2]]
                    s = np.maximum(t[0] + t[1] + t[2], 1e-8)
                    w = [ti / s for ti in t]
                inside = (w[0] > 0) & (w[1] > 0) & (w[2] > 0)
                wc = [np.maximum(wi, 0) for wi in w]
                s = np.maximum(wc[0] + wc[1] + wc[2], 1e-5)
                pz = (wc[0] * z0 + wc[1] * z1 + wc[2] * z2) / s
                dist = np.minimum(np.minimum(_seg(px, py, x0, y0, x1, y1), _seg(px, py, x0, y0, x2, y2)), _seg(px, py, x1, y1, x2, y2))
                ok = (inside | (dist < blur)) & (pz >= 0)
                scale = max(1.0, np.abs(fv[f, :, :2]).max())
                # the inside test can only flip within ABS_E * scale of the triangle's boundary, the halo test near dist = blur
                near = (dist < (ABS_E * scale) ** 2) | (~inside & (np.abs(dist - blur) < REL_D * blur))
                pix = (cy[:, None] * W + cx[None, :])
                self.near[n].reshape(-1)[pix[near]] = True
                cand.append(np.stack([pix[ok].astype(np.float64), np.full(ok.sum(), f, np.float64), pz[ok], dist[ok]], 1))
            if not cand:
                continue
            c = np.concatenate(cand)
            pix, face, pz, dist = c[:, 0].astype(np.int64), c[:, 1].astype(np.int64), c[:, 2], c[:, 3]
            # depth order: the smallest gap between any two candidates of a pixel
            o = np.lexsort((pz, pix))
            same = pix[o][1:] == pix[o][:-1]
            gap = np.abs(pz[o][1:] - pz[o][:-1]) < REL_Z * np.maximum(pz[o][1:], 1e-3)
            self.near[n].reshape(-1)[pix[o][1:][same & gap]] = True
            # the quad rule: both halves candidates at a pixel, and how clearly it is decided
            Fc = len(fv)
            key = pix * Fc + face
            order = np.argsort(key)
            has_nb = nb[face] >= 0
            nkey = pix * Fc + np.where(has_nb, nb[face], 0)
            pos = np.searchsorted(key[order], nkey)
            pos = np.minimum(pos, len(key) - 1)
            both = has_nb & (key[order][pos] == nkey)
            self.quad[n].reshape(-1)[pix[both]] = True
            other = dist[order][pos]
            self.near[n].reshape(-1)[pix[both & (np.abs(dist - other) < REL_D * np.maximum(dist, blur))]] = True


def pt3d_ndc(i, S1, S2):
    rng = 2.0 * S1 / S2 if S1 > S2 else 2.0
    return -rng / 2 + (rng * i + rng / 2) / S1


def _seg(px, py, xa, ya, xb, yb):
    bx, by = xb - xa, yb - ya
    l2 = bx * bx + by * by
    if l2 <= 1e-8:
        return (px - xb) ** 2 + (py - yb) ** 2
    t = np.clip((bx * (px - xa) + by * (py - ya)) / l2, 0, 1)
    return (xa + t * bx - px) ** 2 + (ya + t * by - py) ** 2


def _clipped(ndc, faces, z_clip, persp):
    B, _, _ = ndc.shape
    Fn = faces.shape[0]
    fv = ndc.detach()[:, faces].reshape(B * Fn, 3, 3)
    c = pt3d.clip_faces(fv, torch.arange(B) * Fn, torch.full((B,), Fn), z_clip, persp)
    return c


def _check_decisions(tag, ids, frags, n_faces, margins):
    """kept ids: equal to the oracle's at every decisive pixel; every differing pixel is a near-tie.  Returns the number of
    decisive pixels."""
    got = slots_to_clipped_idx(ids, frags, n_faces)
    same = (got == frags.clipped_idx).all(-1).numpy()
    decisive = margins.quad & ~margins.near
    real = ~same & ~margins.near
    print(f'\n{tag}: pixels decided by the quad rule {int(margins.quad.sum())}, decisive {int(decisive.sum())}, '
          f'differing ids {int((~same).sum())} (near-ties {int((~same & margins.near).sum())}, real disagreements {int(real.sum())})')
    assert not (decisive & ~same).any(), f'{tag}: {int((decisive & ~same).sum())} decisive pixels keep other faces than the oracle'
    assert not real.any(), f'{tag}: {int(real.sum())} pixels disagree with the oracle by more than fp32 rounding'
    return int(decisive.sum())


def _img_tol(tag, ref, ref32, frags, frags32):
    """image tolerance with the float32 oracle as the model of fp32 rounding (DESIGN.md §4): twice its deviation from the
    float64 oracle where both keep the same faces, at least the matrix tests' 1e-4.  The halves of a quad clipped at the near
    plane interpolate vertices far outside the screen, and sigma = 5e-6 amplifies the rounding of distances by 1 / sigma."""
    same = (frags32.clipped_idx == frags.clipped_idx).all(-1)[:, None]
    dev32 = ((ref32.detach().double() - ref.detach()).abs() * same).max().item()
    print(f'\n{tag}: float32 oracle image deviation {dev32:.3e}')
    return max(IMG_TOL, 2 * dev32)


def _twice_identical(run):
    a, b = run(), run()
    for x, y, name in zip(a, b, ('image', 'ids', 'dists')):
        assert torch.equal(x.detach(), y.detach()), f'two runs differ in their {name}'
    return a


# ------------------------------------------------------------------------------------------------ scenes
def _world_scene():
    """the camera inside the geometry (test_z_clipped_scene_with_and_without_perspective_correction): environment and
    blocks straddle the near plane"""
    tpl = D.SceneTemplate(n_blocks=3, txt_size=32)
    p = D.init_params(3, 32, seed=3, dtype=torch.float64)
    R, T, K = _cams(3, seed=3, dist=0.45)
    K = K.clone(); K[0, 0] = K[1, 1] = 1.2
    return _leaf(D.join_scenes([tpl.build_env(p), tpl.build_blocks(p)[0]])), R, T, K


def _ndc_scene(n_faces=3000, B=2, seed=7):
    """NDC input: many overlapping triangles crowded into the centre of the image (tiles list more faces than the list capacity:
    the chunked path), their view depths spread across the near plane so that a quarter of them are split into quads, and
    faces lying in depth between the two halves of a quad along its halo"""
    g = torch.Generator().manual_seed(seed)
    c = (torch.rand(B, n_faces, 1, 2, generator=g, dtype=torch.float64) - 0.5) * 0.8
    xy = c + (torch.rand(B, n_faces, 3, 2, generator=g, dtype=torch.float64) - 0.5) * 0.8
    z = 0.1 + 1.9 * torch.rand(B, n_faces, 3, 1, generator=g, dtype=torch.float64)
    ndc = torch.cat([xy, z], -1).reshape(B, 3 * n_faces, 3)
    faces = torch.arange(3 * n_faces).reshape(n_faces, 3)
    maps = [torch.rand(16, 16, 3, generator=g, dtype=torch.float64).requires_grad_(True) for _ in range(4)]
    scene = {'verts': ndc[0], 'faces': faces, 'faces_verts_uvs': torch.rand(n_faces, 3, 2, generator=g, dtype=torch.float64),
             'face_map': torch.randint(0, 4, (n_faces,), generator=g), 'maps': maps}
    return scene, ndc.requires_grad_(True)


NDC_Z_CLIP, WORLD_Z_CLIP = 0.3, 0.05


@functools.lru_cache(maxsize=None)
def _margins(kind, sigma):
    """_Margins of a scene (the same for every K), computed once"""
    if kind == 'world':
        scene, R, T, K = _world_scene()
        ndc, z_clip = pt3d.world_to_ndc(scene['verts'].detach(), R, T, K), WORLD_Z_CLIP
    else:
        scene, ndc = _ndc_scene()
        z_clip = NDC_Z_CLIP
    c = _clipped(ndc, scene['faces'], z_clip, True)
    return _Margins(c.face_verts, c.mesh_first, c.mesh_nfaces, c.neighbor, *SIZE, D.blur_radius_from_sigma(sigma), True)


def _faces_covering_a_tile(fv, H, W):
    """faces of (F, 3, 3) NDC triangles that cover at least one pixel centre of the 16 x 16 pixel tile at the image centre"""
    x0, y0 = (W // 2) // 16 * 16, (H // 2) // 16 * 16
    xs = torch.tensor([pt3d_ndc(W - 1 - x, W, H) for x in range(x0, x0 + 16)], dtype=torch.float64)
    ys = torch.tensor([pt3d_ndc(H - 1 - y, H, W) for y in range(y0, y0 + 16)], dtype=torch.float64)
    px, py = (t.reshape(-1) for t in torch.meshgrid(xs, ys, indexing='ij'))
    v = fv.detach().double()[:, :, None, :2]                          # (F, 3, 1, 2)
    e = [(px - v[:, a, :, 0]) * (v[:, b, :, 1] - v[:, a, :, 1]) - (py - v[:, a, :, 1]) * (v[:, b, :, 0] - v[:, a, :, 0])
         for a, b in ((1, 2), (2, 0), (0, 1))]
    inside = ((e[0] > 0) & (e[1] > 0) & (e[2] > 0)) | ((e[0] < 0) & (e[1] < 0) & (e[2] < 0))
    return int(inside.any(1).sum())


def _cuda_render(d, R, T, K, sigma, Kf, z_clip, verts=None, ndc=False):
    from dbw_b200 import render_scene
    dev = d['maps'].device
    return render_scene(d['verts'] if verts is None else verts, d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'],
                        None if R is None else R.float().to(dev), None if T is None else T.float().to(dev), intrinsics(K),
                        SIZE, sigma, Kf, z_clip=z_clip, verts_are_ndc=ndc, return_ids=True, return_dists=True)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('sigma', SIGMAS)
@pytest.mark.parametrize('Kf', KS)
def test_world_scene_straddling_the_near_plane(Kf, sigma):
    dev = _dev()
    scene, R, T, K = _world_scene()
    z_clip = WORLD_Z_CLIP
    ref, frags = _oracle(scene, R, T, K, SIZE, sigma, Kf, z_clip=z_clip)
    assert frags.unclipped_to_clipped is not None
    margins = _margins('world', sigma)
    s32 = dict(scene, verts=scene['verts'].detach().float(), maps=[m.detach().float() for m in scene['maps']],
               faces_verts_uvs=scene['faces_verts_uvs'].float())
    ref32, frags32 = _oracle(s32, R.float(), T.float(), K.float(), SIZE, sigma, Kf, z_clip=z_clip)
    d = _dev_scene(scene, dev)
    out, ids, _ = _twice_identical(lambda: _cuda_render(d, R, T, K, sigma, Kf, z_clip))
    tag = f'world K={Kf} sigma={sigma}'
    _check_decisions(tag, ids, frags, scene['faces'].shape[0], margins)
    _parity(tag, scene, ref, frags, out, ids, _pairs(scene, d), seed=40 + Kf, max_ambiguous=1e-2,
            img_tol=_img_tol(tag, ref, ref32, frags, frags32))


@pytest.mark.parametrize('sigma', SIGMAS)
@pytest.mark.parametrize('Kf', KS)
def test_ndc_scene_with_faces_between_the_halves(Kf, sigma):
    dev = _dev()
    scene, ndc = _ndc_scene()
    z_clip = NDC_Z_CLIP
    _, _, K = _cams(2, seed=7)
    ref, frags = _oracle(scene, None, None, K, SIZE, sigma, Kf, z_clip=z_clip, ndc=ndc)
    c = _clipped(ndc, scene['faces'], z_clip, True)
    assert int((c.neighbor >= 0).sum()) > 200
    # the chunked path: the 16 x 16 pixel tile at the image centre lists more faces than either list capacity (64 at
    # <128, *>, 256 at <256, *>): faces that cover one of its pixels certainly reach it
    margins = _margins('ndc', sigma)
    assert _faces_covering_a_tile(c.face_verts[: int(c.mesh_nfaces[0])], *SIZE) > 256
    d = _dev_scene(scene, dev, want=('maps',))
    leaf = ndc.detach().float().to(dev).requires_grad_(True)
    out, ids, _ = _twice_identical(lambda: _cuda_render(d, None, None, K, sigma, Kf, z_clip, verts=leaf, ndc=True))
    tag = f'ndc K={Kf} sigma={sigma}'
    n = _check_decisions(tag, ids, frags, scene['faces'].shape[0], margins)
    assert n > 0, 'no pixel is decided by the quad rule'
    pairs = [('ndc', [ndc], leaf, lambda g: [g])] + _pairs(scene, d, verts=False)
    s32 = dict(scene, maps=[m.detach().float() for m in scene['maps']], faces_verts_uvs=scene['faces_verts_uvs'].float())
    ref32, frags32 = _oracle(s32, None, None, K, SIZE, sigma, Kf, z_clip=z_clip, ndc=ndc.detach().float())
    # a crowded scene: up to a quarter of the pixels hold a near-tie (every one of them checked above), those are excluded
    _parity(tag, scene, ref, frags, out, ids, pairs, seed=50 + Kf, max_ambiguous=0.4, img_tol=_img_tol(tag, ref, ref32, frags, frags32))


@pytest.mark.parametrize('Kf', [1, 3, 10, 25])
def test_loss_epilogue_straddling_the_near_plane(Kf):
    """dbw_render_forward_loss_grad (raster_forward_kernel<*, true>, the blocks pass of fused_loss.scene_mse) with the cameras
    inside the blocks: loss and gradients equal those of the plain render + composite path, and two runs agree to the order of
    the float atomics the gradients are summed with"""
    from dbw_b200 import Renderer
    from dbw_b200.fused_loss import ScenePass
    from tests.test_raster_matrix_gpu import _scene_mse
    dev = _dev()
    H, W = SIZE
    tpl = D.SceneTemplate(n_blocks=4, txt_size=16)
    p = D.init_params(4, 16, seed=13)
    R, T, K = D.ring_cameras(2, jitter=0.3, seed=13, dist=0.45)
    env = tpl.build_env(p)
    blocks, alpha = tpl.build_blocks(p)
    ndc = pt3d.world_to_ndc(blocks['verts'].detach().double(), R.double(), T.double(), K.double())
    fvz = ndc[:, blocks['faces'], 2]
    assert (((fvz < 0.05).sum(-1) == 1)).any(), 'no block face straddles the near plane'

    def renderer(**kw):
        r = Renderer((H, W), z_clip=0.05, cameras={'name': 'perspective'}, **kw).to(dev)
        r.update_cameras(device=dev, K=K[None].to(dev))
        return r

    def arrays(sc):
        maps, table = _pack_maps(sc['maps'], True)
        return sc['verts'].detach().to(dev).requires_grad_(True), maps.to(dev).requires_grad_(True), table

    ev, em, et = arrays(env)
    bv, bm, bt = arrays(blocks)
    i32 = lambda t: t.to(dev).to(torch.int32)
    env_pass = ScenePass(i32(env['faces']), env['faces_verts_uvs'].to(dev), i32(env['face_map']), et,
                         renderer(faces_per_pixel=1, sigma=0), n_static_faces=tpl.bkg_faces.shape[0])
    blk_pass = ScenePass(i32(blocks['faces']), blocks['faces_verts_uvs'].to(dev), i32(blocks['face_map']), bt,
                         renderer(faces_per_pixel=Kf, sigma=1e-4, detach_bary=True), alpha_group=tpl.BNF)
    ba = (alpha.detach() * torch.linspace(0.6, 1.2, len(alpha))).repeat(2).to(dev).requires_grad_(True)
    imgs = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(13)).to(dev)
    x = dict(ev=ev, em=em, bv=bv, bm=bm, ba=ba, R=R.to(dev), T=T.to(dev), imgs=imgs, fmap=i32(blocks['face_map']))
    la, ga = _scene_mse(x, env_pass, blk_pass)
    la2, ga2 = _scene_mse(x, env_pass, blk_pass)
    assert abs(la.item() - la2.item()) <= 1e-7 * abs(la.item())
    for a, b, name in zip(ga, ga2, ('env verts', 'env maps', 'blocks verts', 'blocks maps', 'alpha')):
        assert (a - b).norm() <= 1e-5 * b.norm(), f'{name}: two runs differ by {((a - b).norm() / b.norm()).item():.3e}'
    lb, gb = _composite_loss(x, env_pass, blk_pass)
    assert abs(la.item() - lb.item()) <= 1e-6 * abs(lb.item())
    for a, b, name in zip(ga, gb, ('env verts', 'env maps', 'blocks verts', 'blocks maps', 'alpha')):
        assert a is not None and b is not None and b.abs().max() > 0, name
        assert (a - b).norm() <= 1e-4 * b.norm(), (name, (a - b).norm().item(), b.norm().item())


@pytest.mark.parametrize('case', ['z-clipped persp', 'baseline K=10', 'baseline K=3'])
def test_existing_scenes_have_no_real_disagreement(case):
    """the margin-aware mask over the scenes of the existing parity tests: every pixel whose kept ids differ from the oracle's
    is a near-tie"""
    dev = _dev()
    if case == 'z-clipped persp':
        tpl = D.SceneTemplate(n_blocks=3, txt_size=32)
        p = D.init_params(3, 32, seed=3, dtype=torch.float64)
        R, T, K = _cams(3, seed=3, dist=0.45)
        K = K.clone(); K[0, 0] = K[1, 1] = 1.2
        scene = _leaf(D.join_scenes([tpl.build_env(p), tpl.build_blocks(p)[0]]))
        size, Kf, z_clip = (48, 48), 8, 0.05
    else:
        tpl = D.SceneTemplate(n_blocks=7, txt_size=16)
        p = D.init_params(7, 16, seed=3, dtype=torch.float64)
        scene = _leaf(tpl.build_blocks(p)[0])
        R, T, K = _cams(2, seed=3)
        size, Kf, z_clip = (48, 64), int(case.split('=')[1]), 0.001
    ref, frags = _oracle(scene, R, T, K, size, 1e-4, Kf, z_clip=z_clip)
    ndc = pt3d.world_to_ndc(scene['verts'].detach(), R, T, K)
    c = _clipped(ndc, scene['faces'], z_clip, True)
    margins = _Margins(c.face_verts, c.mesh_first, c.mesh_nfaces, c.neighbor, *size, D.blur_radius_from_sigma(1e-4), True)
    d = _dev_scene(scene, dev)
    from dbw_b200 import render_scene
    _, ids = render_scene(d['verts'], d['faces'], d['fvu'], d['fmap'], d['maps'], d['table'], R.float().to(dev), T.float().to(dev),
                          intrinsics(K), size, 1e-4, Kf, z_clip=z_clip, return_ids=True)
    _check_decisions(case, ids, frags, scene['faces'].shape[0], margins)
    amb = 1 - decision_mask(ids, frags, scene['faces'].shape[0]).mean().item()
    print(f'{case}: ambiguous pixels {amb * 100:.3f}%')
