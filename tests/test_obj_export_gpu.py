"""GPU: the textured OBJ export (dbw_b200.export, csrc/dbw_export.cu).  The atlas kernel against a torch composition of the
same layout, bit for bit, on the model's own scenes; its block rectangles against the texels the fused renderer samples; a
round trip through the written files, rendered; and qualitative_eval's outputs.  The writer's format and the packer are
tested on the CPU (tests/test_obj_export_host.py).

DBW_OBJ_EXPORT_REPORT=<file> appends the round trip's measured render differences to <file>."""
import copy
import os
from copy import deepcopy

import numpy as np
import pytest
import torch

from oracle import dbw_path as D
from tests._obj_export_ref import compose_atlas, read_textured

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
CFG = {
    'mesh': {'n_blocks': 5, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 32},
    'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
    'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                   'decouple_rendering': True, 'opacity_noise': False},
    'loss': {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1},
}
IMG = (96, 128)


def _model(txt_size=32, n_blocks=5, upscale=1, alpha=(2., -2., 1., 3., -1.), seed=5, train=False, epoch=2000):
    """a model with random texture logits (a wide spread, so maps reach 0 and 1) and the given opacity logits"""
    from dbw_b200.dbw import DifferentiableBlocksWorld
    torch.manual_seed(seed)
    cfg = deepcopy(CFG)
    cfg['mesh'].update(n_blocks=n_blocks, txt_size=txt_size, txt_bkg_upscale=upscale)
    model = DifferentiableBlocksWorld(IMG, **cfg).to(DEV)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for t in (model.texture_bkg, model.texture_ground, model.textures):
            t.copy_(torch.randn(t.shape, generator=g) * 4)
        model.alpha_logit.copy_(torch.tensor(list(alpha)[:n_blocks]))
    model.set_cur_epoch(epoch)
    model.train(train)
    return model


def _cameras(B=4, seed=7):
    R, T, K = D.ring_cameras(B, jitter=0.3, seed=seed)
    return {'imgs': torch.zeros(B, 3, *IMG, device=DEV), 'R': R.float().to(DEV), 'T': T.float().to(DEV),
            'K': K.float()[None].expand(B, -1, -1).contiguous().to(DEV)}


def _torch_atlas(maps, layout):
    return compose_atlas([(m.detach().cpu() * 255.0).numpy().astype(np.uint8) for m in maps], layout)


def _kernel_atlas(scene):
    from dbw_b200 import export
    maps = export.scene_maps(scene.textures)
    atlas, layout = export.texture_atlas(maps)
    return atlas.cpu().numpy(), layout, maps


SCENES = {
    'eval_ts32': dict(),
    'eval_ts256': dict(txt_size=256),
    'bkg_upscale_2': dict(upscale=2),
    'no_kept_blocks': dict(alpha=(-3., -2., -4., -1., -5.)),
    'train_decimated': dict(train=True, epoch=10),
}


@pytest.mark.parametrize('name', list(SCENES))
def test_atlas_equals_torch_composition(name):
    model = _model(**SCENES[name])
    with torch.no_grad():
        scene = model.build_scene(filter_transparent=True)
    got, layout, maps = _kernel_atlas(scene)
    assert len(maps) - 2 == (0 if name == 'no_kept_blocks' else 3)
    if name == 'bkg_upscale_2':
        assert maps[0].shape[0] == maps[1].shape[0] == 2 * maps[2].shape[0]
    if name == 'train_decimated':                                 # decimate_txt live: 8 x 8 cells of equal texels
        assert torch.equal(maps[1][:8, :8], maps[1][:1, :1].expand(8, 8, 3))
        assert not torch.equal(maps[1][:8, :9], maps[1][:1, :1].expand(8, 9, 3))
    assert got.shape == (layout.height, layout.width, 3)
    assert np.array_equal(got, _torch_atlas(maps, layout))


def test_atlas_is_deterministic_and_covers_every_texel():
    """two calls give the same bytes, and an atlas buffer prefilled with garbage comes back equal to the composition"""
    from dbw_b200 import export
    model = _model()
    with torch.no_grad():
        scene = model.build_scene(filter_transparent=True)
    maps = export.scene_maps(scene.textures)
    a1, layout = export.texture_atlas(maps)
    torch.cuda.empty_cache()
    junk = torch.full((a1.numel() * 4,), 0xA5, dtype=torch.uint8, device=DEV)     # the allocator may hand this back
    del junk
    a2, _ = export.texture_atlas(maps)
    assert torch.equal(a1, a2)
    assert np.array_equal(a2.cpu().numpy(), _torch_atlas(maps, layout))


def test_block_rectangles_are_the_texels_the_renderer_samples():
    """eval mode: each kept block's rectangle == trunc(255 x) of the fused renderer's float4 atlas (scene_atlases) wherever
    that atlas and the scene's torch-sigmoid maps hold the same float; where the two sigmoids differ in the last bits the
    levels differ by at most one"""
    from dbw_b200.scene_ops import scene_atlases
    model = _model(txt_size=64)
    with torch.no_grad():
        scene = model.build_scene(filter_transparent=True)
        _, blk = scene_atlases(model.texture_bkg, model.texture_ground, model.textures, model.txt_padding)
    keep = (torch.sigmoid(model.alpha_logit) > 0.5).cpu()
    blk = blk[keep.to(DEV)][..., :3].contiguous()
    got, layout, maps = _kernel_atlas(scene)
    assert len(maps) - 2 == blk.shape[0] == 3
    n_same, n_diff = 0, 0
    for k in range(blk.shape[0]):
        x0, y0 = layout.origins[k + 2]
        h, w = blk.shape[1:3]
        rect = got[y0:y0 + h, x0:x0 + w]
        want = (blk[k].cpu() * 255.0).numpy().astype(np.uint8)
        same = (blk[k] == maps[k + 2]).cpu().numpy()
        assert np.array_equal(rect[same], want[same])
        assert np.abs(rect[~same].astype(int) - want[~same].astype(int)).max(initial=0) <= 1
        n_same, n_diff = n_same + same.sum(), n_diff + (~same).sum()
    print(f'block texels: {n_same} equal floats, {n_diff} differing in the last bits')


def _scene_meshes(scene, maps_u8_float):
    """the scene's geometry and UVs with its maps replaced"""
    from dbw_b200 import Meshes
    txt = copy.copy(scene.textures)
    txt.map_groups = maps_u8_float
    verts, faces = scene.get_mesh_verts_faces(0)
    return Meshes(verts[None], faces[None], txt)


@pytest.mark.parametrize('name', ['eval_ts32', 'eval_ts256', 'bkg_upscale_2'])
def test_round_trip_through_the_files_renders_the_same(name, tmp_path):
    """export, read the three files back, and render the in-memory geometry (a) with the file's vt, face-vt indices and
    atlas / 255 as one map and (b) with the scene's own UVs and maps quantised to trunc(255 x) / 255: the two agree within
    what the %f-rounded vt allow, 0.5e-6 (max(Wa, Ha) - 1) texels of displacement, plus 8 float32 ulps of a UV below 1
    (2^-21) for the renderer's interpolation of UVs across that many texels; texel values are in [0, 1], so a displacement
    of d texels changes a sample by at most d"""
    from dbw_b200 import Meshes, TexturesUV, export
    model = _model(**SCENES[name])
    with torch.no_grad():
        scene = model.build_scene(filter_transparent=True)
    export.save_mesh_as_obj(scene, tmp_path / 'scene.obj')
    (head, v, vt, fv, ft), kd, png = read_textured(tmp_path / 'scene.obj')
    assert head == ['', 'mtllib scene.mtl', 'usemtl mesh', ''] and kd == 'scene.png'
    verts, faces = scene.get_mesh_verts_faces(0)
    assert np.abs(v - verts.double().cpu().numpy()).max() <= 5e-7 + 1e-12
    assert np.array_equal(fv, faces.cpu().numpy())
    assert len(vt) == 3 * len(fv) and np.array_equal(ft, np.arange(3 * len(fv)).reshape(-1, 3))
    atlas = torch.from_numpy(png.copy()).to(DEV)
    Ha, Wa = png.shape[:2]
    mesh_a = Meshes(verts[None], faces[None],
                    TexturesUV((atlas.float() / 255)[None], torch.from_numpy(ft)[None].to(DEV),
                               torch.from_numpy(vt).float()[None].to(DEV)))
    mesh_b = _scene_meshes(scene, [(g * 255.0).to(torch.uint8).float() / 255 for g in scene.textures.map_groups])
    inp = _cameras()
    model._install_cameras(inp)
    K = model._view_K(inp)
    with torch.no_grad():
        a = model.renderer.render_viz(mesh_a.extend(4), inp['R'], inp['T'], K=K)
        b = model.renderer.render_viz(mesh_b.extend(4), inp['R'], inp['T'], K=K)
    d = (a - b).abs()
    bound = (0.5e-6 + 2.0 ** -21) * (max(Wa, Ha) - 1)
    line = f'{name}: atlas {Ha}x{Wa}, max |a - b| = {d.max().item():.3e}, mean = {d.mean().item():.3e}, bound {bound:.3e}'
    print(line)
    if os.environ.get('DBW_OBJ_EXPORT_REPORT'):
        with open(os.environ['DBW_OBJ_EXPORT_REPORT'], 'a') as fh:
            fh.write(line + '\n')
    assert (a[:, 3] > 0).float().mean() > 0.5                     # the views see the scene
    assert d.max().item() <= bound, line


def test_qualitative_eval_writes_textured_meshes(tmp_path):
    from dbw_b200 import export, geometry
    model = _model()
    inp = _cameras(B=2)
    loader = [({k: v.cpu() for k, v in inp.items()}, {})]
    model.qualitative_eval(loader, DEV, path=tmp_path, NV=2, n_inputs=1)
    for stem in ('mesh', 'mesh_full'):
        for ext in ('obj', 'mtl', 'png'):
            assert (tmp_path / f'{stem}.{ext}').exists(), (stem, ext)
        (head, v, vt, fv, ft), kd, png = read_textured(tmp_path / f'{stem}.obj')
        assert head[1] == f'mtllib {stem}.mtl' and kd == f'{stem}.png'
    with torch.no_grad():
        reduced = model.build_scene(filter_transparent=True, w_bkg=False, reduce_ground=True)
    verts, faces = geometry.load_obj(str(tmp_path / 'mesh.obj'))
    rv, rf = reduced.get_mesh_verts_faces(0)
    assert torch.equal(faces, rf.cpu()) and len(faces) == 128 + 3 * 80
    # the geometry-only file of the same scene has the same `v` records: load_obj reads the same floats
    export.save_mesh_as_obj(type(reduced)(rv[None], rf[None]), tmp_path / 'plain.obj')
    pv, pf = geometry.load_obj(str(tmp_path / 'plain.obj'))
    assert torch.equal(verts, pv) and torch.equal(faces, pf)
    assert (verts - rv.cpu()).abs().max().item() <= 5e-7 + 1e-7


def test_evaluate_mesh_reads_the_textured_file(tmp_path):
    """dtu_eval.evaluate_mesh(path) scores the textured file exactly as the geometry-only file of the same mesh"""
    from scipy.io import savemat
    from dbw_b200 import Meshes, TexturesUV, export
    from dbw_b200.dtu_eval import evaluate_mesh, write_ply
    here = os.path.dirname(os.path.abspath(__file__))
    gold = dict(np.load(os.path.join(here, 'golden', 'dtu_eval.npz')))
    root = tmp_path / 'DTU'
    (root / 'ObsMask').mkdir(parents=True)
    (root / 'Points' / 'stl').mkdir(parents=True)
    savemat(root / 'ObsMask' / 'ObsMask7_10.mat', {'ObsMask': gold['obs_mask'], 'BB': gold['bb'], 'Res': gold['res']})
    savemat(root / 'ObsMask' / 'Plane7.mat', {'P': gold['plane']})
    write_ply(root / 'Points' / 'stl' / 'stl007_total.ply', gold['stl'])
    verts = torch.from_numpy(gold['verts']).float().to(DEV)
    faces = torch.from_numpy(gold['faces']).long().to(DEV)
    F = faces.shape[0]
    g = torch.Generator().manual_seed(3)
    txt = TexturesUV(torch.rand(1, 8, 8, 3, generator=g).to(DEV), torch.arange(3 * F, device=DEV).reshape(1, F, 3),
                     torch.rand(1, 3 * F, 2, generator=g).to(DEV))
    export.save_mesh_as_obj(Meshes(verts[None], faces[None], txt), tmp_path / 'textured.obj')
    export.save_mesh_as_obj(Meshes(verts[None], faces[None]), tmp_path / 'plain.obj')
    assert (tmp_path / 'textured.png').exists() and not (tmp_path / 'plain.png').exists()
    run = tmp_path / 'run'
    run.mkdir()
    s_tex = evaluate_mesh(str(tmp_path / 'textured.obj'), 7, str(root), str(run), suffix='_tex', save_viz=False, seed=0)
    s_plain = evaluate_mesh(str(tmp_path / 'plain.obj'), 7, str(root), str(run), suffix='_plain', save_viz=False, seed=0)
    assert s_tex == s_plain and all(np.isfinite(list(s_tex.values())))
    assert abs(s_tex['avg'] - float(gold['scores'][2])) < 0.05 * float(gold['scores'][2])
