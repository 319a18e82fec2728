"""The resolving hard render (dbw_render_forward_viz, Renderer.render_viz) and the view renders built on it (dbw_b200/views.py)
on the GPU: bit identity with today's viz_purpose path avg_pool2d(render at 4H x 4W, 4), agreement with the float64
oracle's supersampled render, the uint8 frames, chunking, and the videos qualitative_eval writes."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dbw_path as D
from tests.helpers import scene_to_device, intrinsics, decision_mask

pytestmark = pytest.mark.gpu


def _dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _scene(kind, n_views, seed=3, dist=2.75):
    tpl = D.SceneTemplate(n_blocks=4, txt_size=32)
    p = D.init_params(4, 32, seed=seed)
    R, T, K = D.ring_cameras(n_views, jitter=0.3, seed=seed, dist=dist)
    blocks, _ = tpl.build_blocks(p)
    scene = D.join_scenes([tpl.build_env(p), blocks]) if kind == 'env' else blocks
    return scene, R, T, K


def _per_view_K(K, B):
    Kb = K[None].repeat(B, 1, 1).clone()
    Kb[:, 0, 0] *= torch.linspace(0.8, 1.2, B)
    Kb[:, 1, 1] *= torch.linspace(1.1, 0.9, B)
    Kb[:, 0, 2] = torch.linspace(-0.05, 0.05, B)
    return Kb


def _today(sc, R, T, intr, size, shade, bg, z_clip):
    """the viz_purpose path of Renderer.forward: hard render at 4x, avg_pool2d"""
    from dbw_b200 import render_scene
    H, W = size
    out = render_scene(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R, T, intr,
                       (4 * H, 4 * W), 0.0, 1, z_clip, background=bg, face_shade=shade)
    return F.avg_pool2d(out, kernel_size=4, stride=4)


CASES = [  # (scene, views, frame size, lit, per-view K, background, z_clip, camera distance)
    ('env', 2, (40, 52), False, False, (0., 0., 0.), 0.001, 2.75),
    ('env', 3, (36, 20), False, False, (1., 1., 1.), 0.05, 0.45),          # z-clipped faces everywhere
    ('blocks', 2, (33, 47), True, False, (1., 1., 1.), 0.001, 2.75),       # renderer_light: flat shading, white
    ('env', 4, (24, 40), False, True, (0., 0., 0.), 0.001, 2.75),          # per-view intrinsics
    ('blocks', 1, (17, 29), True, True, (0., 0., 0.), 0.001, 2.75),
    ('env', 37, (20, 28), False, False, (1., 1., 1.), 0.001, 2.75),
]


@pytest.mark.parametrize('case', CASES, ids=[f'{c[0]}-B{c[1]}-{c[2][0]}x{c[2][1]}{"-lit" if c[3] else ""}{"-K" if c[4] else ""}'
                                             for c in CASES])
@torch.no_grad()
def test_resolving_kernel_equals_avg_pool_of_the_4x_render(case):
    from dbw_b200.renderer import render_scene_viz
    kind, B, size, lit, per_view, bg, z_clip, dist = case
    dev = _dev()
    scene, R, T, K = _scene(kind, B, dist=dist)
    if dist < 1:
        K = K.clone(); K[0, 0] = K[1, 1] = 1.2
    sc = scene_to_device(scene, dev)
    R, T = R.to(dev), T.to(dev)
    intr = _per_view_K(K, B).to(dev) if per_view else intrinsics(K)
    shade = D.flat_shade_multiplier(scene['verts'], scene['faces'], R.cpu()).float().to(dev) if lit else None
    ref = _today(sc, R, T, intr, size, shade, bg, z_clip)
    args = (sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R, T, intr, size)
    rgba, rgb8 = render_scene_viz(*args, z_clip=z_clip, background=bg, face_shade=shade, frames_u8=True)
    assert torch.equal(rgba, ref), f'{(rgba != ref).float().mean().item() * 100:.4f}% of the values differ'
    assert ref[:, 3].mean() > 0.02                                                 # the scene is in view
    to_u8 = lambda x: (x * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8)
    assert torch.equal(rgb8, to_u8(rgba[:, :3]))
    # background composite: one shared background and one per view
    g = torch.Generator(device=dev).manual_seed(1)
    for n_bkg in (1, B):
        bkg = torch.rand(n_bkg, 3, *size, device=dev, generator=g)
        out, out8 = render_scene_viz(*args, z_clip=z_clip, background=bg, face_shade=shade, bkg=bkg, frames_u8=True)
        rec, alpha = ref.split([3, 1], dim=1)
        comp = rec * alpha + (1 - alpha) * bkg
        assert torch.equal(out[:, :3], comp) and torch.equal(out[:, 3:], alpha)
        assert torch.equal(out8, to_u8(comp))


def _viz_oracle(scene, R, T, K, size, z_clip):
    """the float64 supersampled hard render: the oracle's hard render at 4H x 4W and its 4 x 4 box filter, with the
    fragments of the sample grid"""
    H, W = size
    sc64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in scene.items()}
    sc64['maps'] = [m.double() for m in scene['maps']]
    out, frags = D.render(sc64, R.double(), T.double(), K.double(), (4 * H, 4 * W), sigma=0, faces_per_pixel=1, z_clip=z_clip,
                          return_fragments=True)
    return F.avg_pool2d(out, 4), frags


@torch.no_grad()
def test_resolving_kernel_matches_float64_supersampled_oracle():
    from dbw_b200 import render_scene
    from dbw_b200.renderer import render_scene_viz
    dev = _dev()
    size = (28, 36)
    scene, R, T, K = _scene('env', 2)
    ref, frags = _viz_oracle(scene, R, T, K, size, 0.001)
    sc = scene_to_device(scene, dev)
    out = render_scene_viz(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                           intrinsics(K), size, z_clip=0.001).cpu().double()
    _, ids = render_scene(sc['verts'], sc['faces'], sc['faces_uvs'], sc['face_map'], sc['maps'], sc['table'], R.to(dev), T.to(dev),
                          intrinsics(K), (4 * size[0], 4 * size[1]), 0.0, 1, 0.001, return_ids=True)
    same = F.avg_pool2d(decision_mask(ids, frags, scene['faces'].shape[0]), 4) == 1      # all 16 samples decided alike
    assert same.float().mean() > 0.97
    err = ((out - ref).abs() * same).max().item()
    assert err <= 1e-4, err


# ------------------------------------------------------------------ Renderer / views
def _meshes(dev, lit=False):
    from dbw_b200 import Renderer, Meshes, TexturesUV, join_meshes_as_scene
    tpl = D.SceneTemplate(n_blocks=3, txt_size=32)
    p = D.init_params(3, 32, seed=3)
    blocks, _ = tpl.build_blocks(p)
    nb = 3
    txt = TexturesUV(torch.stack(blocks['maps']).to(dev), tpl.block_faces_uvs[None].expand(nb, -1, -1).to(dev),
                     tpl.block_verts_uvs[None].expand(nb, -1, -1).to(dev))
    mesh = join_meshes_as_scene(Meshes(blocks['verts'].reshape(nb, -1, 3).to(dev), tpl.block_faces[None].expand(nb, -1, -1).to(dev), txt))
    kw = dict(faces_per_pixel=10, z_clip=0.001, cameras={'name': 'perspective'})
    if lit:
        kw.update(sigma=0, faces_per_pixel=1, shading_type='flat', background_color=(1, 1, 1),
                  lights={'name': 'directional', 'direction': [[1, 0.25, -1]], 'ambient_color': [[0.7] * 3],
                          'diffuse_color': [[0.4] * 3], 'specular_color': [[0.] * 3]})
    R, T, K = D.ring_cameras(2, jitter=0.3, seed=3)
    rend = Renderer((30, 42), **kw).to(dev)
    rend.update_cameras(device=dev, K=K[None].to(dev))
    return rend, mesh, K


@pytest.mark.parametrize('lit', [False, True])
@torch.no_grad()
def test_render_viz_equals_forward_viz_purpose(lit):
    dev = _dev()
    rend, mesh, K = _meshes(dev, lit)
    R, T = D.ring_cameras(5, jitter=0.3, seed=4)[:2]
    R, T = R.to(dev), T.to(dev)
    assert torch.equal(rend.render_viz(mesh, R, T), rend(mesh, R, T, viz_purpose=True))
    Kb = _per_view_K(K, 5).to(dev)
    assert torch.equal(rend.render_viz(mesh, R, T, K=Kb), rend(mesh, R, T, viz_purpose=True, K=Kb))


@torch.no_grad()
def test_view_renders_do_not_depend_on_the_chunk_size():
    from dbw_b200 import views as V
    dev = _dev()
    rend, mesh, K = _meshes(dev)
    per_frame = rend.viz_bytes(mesh, 1)
    R, T = V.get_circle_traj(dist=2.5, N_views=23)
    bkg = torch.rand(3, 30, 42, generator=torch.Generator().manual_seed(5))
    for kw in ({}, {'bkg': bkg}, {'with_alpha': True}, {'with_edges': True, 'bkg': bkg}):
        outs = [V.render_views(mesh, R, T, renderer=rend, chunk_bytes=c * per_frame, **kw) for c in (1, 7, 23)]
        assert outs[0].shape[0] == 23 and all(torch.equal(outs[0], o) for o in outs[1:]), kw
    rot = [V.render_rotated_views(mesh, n_views=17, renderer=rend, bkg=bkg, chunk_bytes=c * per_frame) for c in (1, 7, 17)]
    assert rot[0].shape == (17, 3, 30, 42) and all(torch.equal(rot[0], o) for o in rot[1:])
    # with_edges: the chunk's render_viz, then draw_edges on it
    res = rend.render_viz(mesh, R[:7].to(dev), T[:7].to(dev))
    edged = rend.draw_edges(res[:, :3], mesh, R=R[:7].to(dev), T=T[:7].to(dev))
    assert torch.equal(V.render_views(mesh, R[:7], T[:7], renderer=rend, with_edges=True), edged.cpu())
    assert torch.equal(V.render_views(mesh, R[:7], T[:7], renderer=rend), res[:, :3].cpu())
    # the streamed video frames are the uint8 conversion of render_views' frames (no edges, no clamp: the kernel's own)
    frames = torch.cat(list(V._view_frames(mesh, R, T, rend, bkg.to(dev), u8=True, chunk_bytes=7 * per_frame)))
    ref = V.render_views(mesh, R, T, renderer=rend, bkg=bkg)
    assert torch.equal(frames.cpu(), (ref * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8))


def _read_mp4(path):
    import cv2
    cap = cv2.VideoCapture(str(path))
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f[..., ::-1])
    return np.stack(frames)


# mp4v (MPEG-4 part 2) is lossy: the first decoded frame of a trajectory is held to this PSNR against the uint8 frame
VIDEO_PSNR_MIN = 30.0


def test_qualitative_eval_writes_the_reference_videos(tmp_path):
    from copy import deepcopy
    from dbw_b200 import views as V
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from tests.test_model_gpu import CFG, _inputs
    dev = _dev()
    torch.manual_seed(5)
    model = DifferentiableBlocksWorld((48, 64), **deepcopy(CFG)).to(dev)
    model.set_cur_epoch(2000)
    with torch.no_grad():
        model.alpha_logit.copy_(torch.tensor([2., -2., 1., 3., -1.]))
    inp, *_ = _inputs(dev, B=3)

    class _Set:
        pc_gt = torch.rand(5000, 3, generator=torch.Generator().manual_seed(0))

    class _Loader(list):
        dataset = _Set()
        batch_size = 2

    loader = _Loader([({k: v[:2].cpu() for k, v in inp.items()}, {}), ({k: v[2:].cpu() for k, v in inp.items()}, {})])
    NV = 9
    assert model.qualitative_eval(loader, dev, path=tmp_path, NV=NV) == 3
    names = {f.name for f in tmp_path.iterdir()}
    videos = {'rotated_mesh.mp4'} | {f'{i}_rec_traj{s}.mp4' for i in range(3) for s in ('', '_syn')}
    assert videos <= names and 'gt.ply' in names
    from dbw_b200.dtu_eval import read_ply
    gt = read_ply(tmp_path / 'gt.ply')
    assert len(gt) == 3000
    for v in videos:
        fr = _read_mp4(tmp_path / v)
        assert fr.shape == (NV, 48, 64, 3), (v, fr.shape)
    # the first frame of view 0's trajectory against the render it encodes
    meshes = model.build_scene(filter_transparent=True)
    R_traj = V.get_circle_traj(N_views=NV)[0].to(dev)
    with torch.no_grad():
        _, u8 = model.renderer.render_viz(meshes, inp['R'][:1] @ R_traj[:1], inp['T'][:1], frames_u8=True)
    dec = _read_mp4(tmp_path / '0_rec_traj.mp4')[0].astype(np.float64)
    mse = ((dec - u8[0].cpu().numpy().astype(np.float64)) ** 2).mean()
    psnr = 10 * np.log10(255 ** 2 / max(mse, 1e-12))
    print(f'0_rec_traj.mp4 frame 0: PSNR {psnr:.2f} dB against the uint8 render')
    assert psnr > VIDEO_PSNR_MIN, psnr
