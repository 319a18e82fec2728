"""Phong shading on the GPU: vertex normals (dbw_vertex_normals) against float64 and across calls; the Phong-shaded hard
render (dbw_render_forward_phong) against the float64 restatement of PyTorch3D's phong_shading (oracle/phong.py) for every
light type, with and without specular, z-clipped faces, opacities and per-view intrinsics; the resolving variant against
avg_pool2d of the 4x render, bit for bit; the eye_light views; and the refusals (soft phong, backward, gouraud)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dbw_path as D
from oracle import phong as P
from oracle import pt3d
from tests.helpers import scene_to_device, intrinsics, decision_mask

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


# ------------------------------------------------------------------ vertex normals
def _normal_meshes():
    from tests.test_phong_host import _meshes
    out = _meshes()
    tpl = D.SceneTemplate(n_blocks=4, txt_size=32)
    blocks, _ = tpl.build_blocks(D.init_params(4, 32, seed=3))
    out['blocks'] = (blocks['verts'], blocks['faces'])
    return out


@pytest.mark.parametrize('name', ['icosphere', 'cube', 'degenerate', 'noisy_icosphere', 'blocks'])
def test_vertex_normals_match_float64_and_repeat_bit_for_bit(name):
    from dbw_b200.renderer import vertex_face_list, vertex_normals
    from tests.test_phong_host import vertex_face_list as vf_ref
    dev = _dev()
    verts, faces = _normal_meshes()[name]
    v, f = verts.float().to(dev), faces.to(dev).to(torch.int32)
    vf = vertex_face_list(f, len(v))
    end, lst = vf_ref(faces.numpy(), len(v))
    assert np.array_equal(vf[0].cpu().numpy(), end) and np.array_equal(vf[1].cpu().numpy(), lst)
    n1, n2 = vertex_normals(v, f, vf), vertex_normals(v, f)
    assert torch.equal(n1, n2)
    ref = P.vertex_normals(verts.double(), faces.long())
    assert (n1.cpu().double() - ref).abs().max().item() < 1e-6


# ------------------------------------------------------------------ hard phong renders against the oracle
def _small():
    from tests.golden.make_golden import small_case
    tpl, p, R, T, K, _ = small_case()
    blocks, alpha = tpl.build_blocks(p)
    return {k: (v.detach() if torch.is_tensor(v) else v) for k, v in blocks.items()}, R, T, K, alpha.detach().repeat_interleave(tpl.BNF)


def _cube():
    from tests.golden.make_golden import cube_case
    tex, Rm, Tm, R, T, K = cube_case()
    return D.cube_scene(tex, scale=0.45, R=Rm, T=Tm), R, T, K, None


def _per_view_K(K, B):
    Kb = K.reshape(-1, 4, 4)[:1].repeat(B, 1, 1).clone()
    Kb[:, 0, 0] *= torch.linspace(0.8, 1.2, B)
    Kb[:, 1, 1] *= torch.linspace(1.1, 0.9, B)
    Kb[:, 0, 2] = torch.linspace(-0.05, 0.05, B)
    return Kb


def _scene64(scene):
    out = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in scene.items()}
    out['maps'] = [m.double() for m in scene['maps']]
    return out


def _oracle_frags(scene, R, T, K, size, z_clip):
    """the oracle's hard fragments, view by view when K holds one camera per view"""
    Ks = K.reshape(-1, 4, 4)
    if len(Ks) == 1:
        return D.render(_scene64(scene), R.double(), T.double(), Ks[0].double(), size, sigma=0, faces_per_pixel=1, z_clip=z_clip,
                        return_fragments=True)[1]
    fr = [_oracle_frags(scene, R[b:b + 1], T[b:b + 1], Ks[b], size, z_clip) for b in range(len(R))]
    Fn = scene['faces'].shape[0]
    # per-view fragments carry view-local ids: shift them to the batch-packed ids of one call over all views
    from types import SimpleNamespace
    cat = lambda k: torch.cat([getattr(f, k) for f in fr])
    p2f = torch.cat([torch.where(f.pix_to_face >= 0, f.pix_to_face + b * Fn, f.pix_to_face) for b, f in enumerate(fr)])
    return SimpleNamespace(pix_to_face=p2f, zbuf=cat('zbuf'), bary_coords=cat('bary_coords'), dists=cat('dists'),
                           clipped_idx=None, unclipped_to_clipped=None, parts=fr)


def _same_mask(ids, frags, Fn):
    if getattr(frags, 'parts', None) is not None:
        return torch.cat([decision_mask(ids[b:b + 1], f, Fn) for b, f in enumerate(frags.parts)])
    return decision_mask(ids, frags, Fn)


LIGHTS = {
    'ambient': {'name': 'ambient', 'ambient_color': [[0.9, 0.8, 0.7]]},
    'directional': {'name': 'directional'},                                        # PyTorch3D defaults: specular 0.2
    'directional-nospec': {'name': 'directional', 'direction': [[1, 0.25, -1]], 'ambient_color': [[0.7] * 3],
                           'diffuse_color': [[0.4] * 3], 'specular_color': [[0.] * 3]},
    'directional-spec': {'name': 'directional', 'direction': [[-0.3, 0.5, -1]], 'specular_color': [[0.6, 0.5, 0.4]]},
    'point': {'name': 'point', 'location': [[0.4, 1.5, -2.0]], 'specular_color': [[0.5] * 3]},
}

CASES = [  # (scene, light, z_clip, camera distance, faces_alpha, per-view K, size)
    ('small', 'directional', 0.001, None, False, False, (40, 48)),
    ('small', 'directional-nospec', 0.001, None, True, False, (40, 48)),
    ('small', 'point', 0.001, None, True, True, (33, 45)),
    ('small', 'ambient', 0.001, None, False, False, (40, 48)),
    ('small', 'directional-spec', 0.05, 0.6, False, False, (36, 36)),          # camera inside the scene: z-clipped faces
    ('cube', 'directional-spec', 0.001, None, False, False, (64, 64)),
    ('cube', 'point', 0.001, None, False, True, (48, 56)),
    ('cube', 'directional', 0.7, 1.0, False, False, (40, 40)),                 # the near plane cuts the cube
]


def _case(kind, dist):
    scene, R, T, K, fa = _small() if kind == 'small' else _cube()
    if dist is not None:
        R, T, K = D.ring_cameras(len(R), dist=dist, jitter=0.3, seed=5)
        K = K.clone(); K[0, 0] = K[1, 1] = 1.2
    return scene, R, T, K, fa


@pytest.mark.parametrize('case', CASES, ids=[f'{c[0]}-{c[1]}-z{c[2]}{"-alpha" if c[4] else ""}{"-K" if c[5] else ""}' for c in CASES])
@torch.no_grad()
def test_hard_phong_render_matches_float64_oracle(case):
    from dbw_b200 import render_scene
    from dbw_b200.renderer import render_scene_phong, phong_shading
    kind, light, z_clip, dist, with_alpha, per_view, size = case
    dev = _dev()
    scene, R, T, K, fa = _case(kind, dist)
    if with_alpha:
        fa = torch.linspace(0.2, 1.0, scene['faces'].shape[0])
    else:
        fa = None
    Kx = _per_view_K(K, len(R)) if per_view else K
    ref = P.render_phong(_scene64(scene), R.double(), T.double(), Kx.double(), size, lights=LIGHTS[light], z_clip=z_clip,
                         faces_alpha=fa.double() if fa is not None else None, background=(1., 1., 1.))
    sc = scene_to_device(scene, dev)
    intr = Kx.to(dev) if per_view else intrinsics(K)
    out = render_scene_phong(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                             intr, size, phong_shading(LIGHTS[light]), 1, z_clip=z_clip, background=(1., 1., 1.),
                             faces_alpha=fa.to(dev) if fa is not None else None)
    _, ids = render_scene(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                          intr, size, 0.0, 1, z_clip, return_ids=True)
    same = _same_mask(ids, _oracle_frags(scene, R, T, Kx, size, z_clip), scene['faces'].shape[0])
    assert same.mean() > 0.97
    assert ref[:, 3].mean() > 0.05                                               # the scene is in view
    err = ((out.cpu().double() - ref).abs() * same).max().item()
    assert err <= TOL, err
    if light != 'ambient' and fa is None:                                        # the lighting is not a constant factor
        raw = render_scene(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                           intr, size, 0.0, 1, z_clip, background=(1., 1., 1.))
        ratio = out[:, :3] / raw[:, :3].clamp(min=1e-3)
        inside = raw[:, 3:].expand(-1, 3, -1, -1) > 0.99
        assert ratio[inside].std() > 1e-2


@pytest.mark.parametrize('light', ['directional', 'point', 'ambient'])
@torch.no_grad()
def test_resolving_phong_equals_avg_pool_of_the_4x_phong_render(light):
    from dbw_b200.renderer import render_scene_phong, phong_shading
    dev = _dev()
    scene, R, T, K, _ = _small()
    sc = scene_to_device(scene, dev)
    size = (30, 38)
    sh = phong_shading(LIGHTS[light])
    for intr in (intrinsics(K), _per_view_K(K, len(R)).to(dev)):
        args = (sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev), intr)
        fa = torch.linspace(0.3, 1.0, scene['faces'].shape[0], device=dev)
        for alpha in (None, fa):
            big = render_scene_phong(*args, (4 * size[0], 4 * size[1]), sh, 1, z_clip=0.001, background=(0.2, 0.3, 0.4), faces_alpha=alpha)
            ref = F.avg_pool2d(big, 4)
            rgba, rgb8 = render_scene_phong(*args, size, sh, 4, z_clip=0.001, background=(0.2, 0.3, 0.4), faces_alpha=alpha,
                                            frames_u8=True)
            assert torch.equal(rgba, ref), f'{(rgba != ref).float().mean().item() * 100:.4f}% of the values differ'
            to_u8 = lambda x: (x * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8)
            assert torch.equal(rgb8, to_u8(rgba[:, :3]))
            bkg = torch.rand(len(R), 3, *size, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
            out, out8 = render_scene_phong(*args, size, sh, 4, z_clip=0.001, background=(0.2, 0.3, 0.4), faces_alpha=alpha, bkg=bkg,
                                           frames_u8=True)
            rec, a = ref.split([3, 1], dim=1)
            comp = rec * a + (1 - a) * bkg
            assert torch.equal(out[:, :3], comp) and torch.equal(out[:, 3:], a) and torch.equal(out8, to_u8(comp))


# ------------------------------------------------------------------ Renderer and views
def _meshes(dev, requires_grad=False):
    from dbw_b200 import Meshes, TexturesUV, join_meshes_as_scene
    tpl = D.SceneTemplate(n_blocks=3, txt_size=32)
    blocks, _ = tpl.build_blocks(D.init_params(3, 32, seed=3))
    nb = 3
    txt = TexturesUV(torch.stack(blocks['maps']).to(dev), tpl.block_faces_uvs[None].expand(nb, -1, -1).to(dev),
                     tpl.block_verts_uvs[None].expand(nb, -1, -1).to(dev))
    verts = blocks['verts'].reshape(nb, -1, 3).detach().to(dev).requires_grad_(requires_grad)
    return join_meshes_as_scene(Meshes(verts, tpl.block_faces[None].expand(nb, -1, -1).to(dev), txt))


def _oracle_scene(renderer, mesh):
    verts, faces, fvu, fmap, maps, table = renderer._scene(mesh)
    return {'verts': verts.detach().cpu(), 'faces': faces.cpu().long(), 'faces_verts_uvs': fvu.cpu(), 'face_map': fmap.cpu().long(),
            'maps': [maps[o:o + h * w * 3].reshape(h, w, 3).cpu() for o, h, w in table]}


def _viz_check(frames, scene, R, T, K, size, lights, z_clip, background, clamp):
    """frames (B,3,H,W) against the oracle's supersampled phong frames, on the pixels whose 16 samples the product and the
    oracle rasterize alike"""
    from dbw_b200 import render_scene
    dev = _dev()
    H, W = size
    ref = P.render_phong_viz(_scene64(scene), R.double(), T.double(), K.double(), size, lights=lights, z_clip=z_clip,
                             background=background)[:, :3]
    if clamp:
        ref = ref.clamp(0, 1)
    sc = scene_to_device(scene, dev)
    _, ids = render_scene(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                          intrinsics(K), (4 * H, 4 * W), 0.0, 1, z_clip, return_ids=True)
    frags = _oracle_frags(scene, R, T, K, (4 * H, 4 * W), z_clip)
    same = F.avg_pool2d(decision_mask(ids, frags, scene['faces'].shape[0]), 4) == 1
    assert same.float().mean() > 0.97
    err = ((frames.double() - ref).abs() * same).max().item()
    assert err <= TOL, err
    return ref, same


@torch.no_grad()
def test_eye_light_views_match_the_oracle(monkeypatch, tmp_path):
    from dbw_b200 import Renderer
    from dbw_b200 import views as V
    dev = _dev()
    mesh = _meshes(dev)
    K = D.ring_cameras(2, jitter=0.3, seed=3)[2]
    # K among the constructor's kwargs: the eye_light renderer of render_views is rebuilt from them, as in the reference
    # (renderer.py:343-351), so a K set later by update_cameras would not carry over
    rend = Renderer((30, 42), faces_per_pixel=10, z_clip=0.001, cameras={'name': 'perspective', 'K': K[None].to(dev)},
                    background_color=(1, 1, 1)).to(dev)
    scene = _oracle_scene(rend, mesh)
    n, elev, dist = 7, 30, 2.732
    R = V.look_at_view_transform(dist=1, elev=elev, azim=torch.linspace(-180, 180, n))[0]
    T = torch.tensor([[0., 0., dist]]).expand(n, -1)
    rot = V.render_rotated_views(mesh, n_views=n, elev=elev, dist=dist, renderer=rend, eye_light=True)
    ref, same = _viz_check(rot, scene, R, T, K, (30, 42), V.EYE_LIGHT_ROTATED, 0.001, (1., 1., 1.), clamp=True)
    # the lit frames differ from the unlit ones
    assert (rot - V.render_rotated_views(mesh, n_views=n, elev=elev, dist=dist, renderer=rend)).abs().max() > 0.05
    # the video's frames: the uint8 conversion of the same frames, made in the kernel
    written = []

    class _Capture:
        def __init__(self, *a, **k):
            pass

        def write(self, f):
            written.append(f.cpu())

        def __enter__(self):
            return self

        def __exit__(self, *exc):
            pass
    monkeypatch.setattr(V, 'VideoWriter', _Capture)
    V.save_mesh_as_video(mesh, tmp_path / 'rot.mp4', n_views=n, elev=elev, dist=dist, renderer=rend, eye_light=True)
    u8 = torch.cat(written)
    assert torch.equal(u8, (rot * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8))
    # trajectory views with their own light set
    Rt, Tt = V.get_circle_traj(dist=2.5, N_views=5)
    traj = V.render_views(mesh, Rt, Tt, renderer=rend, eye_light=True)
    _viz_check(traj, scene, Rt, Tt, K, (30, 42), V.EYE_LIGHT_VIEWS, 0.001, (1., 1., 1.), clamp=False)


@torch.no_grad()
def test_phong_renderer_forward_paths_agree():
    from dbw_b200 import Renderer
    dev = _dev()
    mesh = _meshes(dev)
    R, T, K = D.ring_cameras(3, jitter=0.3, seed=4)
    R, T = R.to(dev), T.to(dev)
    kw = dict(z_clip=0.001, cameras={'name': 'perspective', 'K': K[None].to(dev)}, shading_type='phong', lights={'name': 'point'})
    rend = Renderer((26, 34), sigma=0, faces_per_pixel=1, **kw).to(dev)
    viz = rend(mesh, R, T, viz_purpose=True)
    assert torch.equal(viz, rend.render_viz(mesh, R, T))
    big = Renderer((104, 136), sigma=0, faces_per_pixel=1, **kw).to(dev)
    assert torch.equal(viz, F.avg_pool2d(big(mesh, R, T), 4))
    scene = _oracle_scene(rend, mesh)
    ref = P.render_phong(_scene64(scene), R.cpu().double(), T.cpu().double(), K.double(), (26, 34), lights={'name': 'point'},
                         z_clip=0.001)
    hard = rend(mesh, R, T).cpu().double()
    assert ((hard - ref).abs() > TOL).float().mean() < 0.02                       # the rest: pixels rasterized differently


def test_phong_refusals():
    from dbw_b200 import Renderer
    dev = _dev()
    mesh = _meshes(dev, requires_grad=True)
    R, T, K = D.ring_cameras(2, jitter=0.3, seed=4)
    R, T = R.to(dev), T.to(dev)
    base = dict(z_clip=0.001, cameras={'name': 'perspective', 'K': K[None].to(dev)}, lights={'name': 'directional'})
    soft = Renderer((24, 24), shading_type='phong', **base).to(dev)                # sigma 1e-4, 25 faces per pixel
    with pytest.raises(NotImplementedError, match='soft phong'):
        soft(mesh, R, T)
    hard = Renderer((24, 24), shading_type='phong', sigma=0, faces_per_pixel=1, **base).to(dev)
    out = hard(mesh, R, T)
    assert out.requires_grad
    with pytest.raises(NotImplementedError, match='no backward'):
        out.sum().backward()
    gouraud = Renderer((24, 24), shading_type='gouraud', sigma=0, faces_per_pixel=1, **base).to(dev)
    for call in (lambda: gouraud(mesh, R, T), lambda: gouraud(mesh, R, T, viz_purpose=True), lambda: gouraud.render_viz(mesh, R, T)):
        with pytest.raises(NotImplementedError, match='gouraud'):
            call()
