"""What a Phong-shaded turntable costs on the GPU: the 240 frames of save_mesh_as_video(eye_light=True) -- the scene model's
blocks (10 blocks, the bench.py scene) turning around +y, elevation 30, distance 2.732 -- two ways, alternating in one process:

  flat    today's lit visualisation: renderer_light (flat shading, src/model/dbw.py:139-143) through the resolving kernel
  phong   the eye_light renderer (views.EYE_LIGHT_ROTATED, Phong shading) through the Phong-shaded resolving kernel, vertex
          normals included

Both write the uint8 frames in the kernel, in chunks sized by views.CHUNK_BYTES.  Two shapes: 400x400 (DTU) and 576x768
(BlendedMVS).  Per shape and arm: frames/s (CUDA-synchronised wall clock, median of --repeat).  --check asserts that the phong
frames equal avg_pool2d of the Phong-shaded render at 4H x 4W bit for bit (float and uint8, all 240 frames), and that the
first frame, rendered at a quarter of each side, is within 1e-4 of the float64 oracle (oracle/phong.py) wherever both
rasterize the 16 samples of a pixel alike.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_phong.py [--repeat 5] [--check]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from copy import deepcopy

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'dtu': (400, 400), 'bmvs': (576, 768)}
N_FRAMES = 240
CFG = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
       'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
       'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                      'decouple_rendering': True, 'opacity_noise': False},
       'loss': {'rgb_weight': 1}}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


@torch.no_grad()
def video_arm(renderer, mesh, R, T, frames, keep=None):
    """frames (N,H,W,3) uint8 receives the video; keep: a list that collects the float frames (--check)"""
    from dbw_b200 import views as V
    for a, b in V._chunks(renderer, mesh, len(R), None):
        rgba, u8 = renderer.render_viz(mesh, R[a:b], T[a:b], frames_u8=True)
        frames[a:b] = u8
        if keep is not None:
            keep.append(rgba)


def timed(fn, *args):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def turntable(n, dev, elev=30, dist=2.732):
    from dbw_b200 import views as V
    R = V.look_at_view_transform(dist=1, elev=elev, azim=torch.linspace(-180, 180, n), device=dev)[0]
    return R, torch.tensor([[0., 0., dist]], device=dev).expand(n, -1)


@torch.no_grad()
def check_against_oracle(model, mesh, R, T, K, size):
    """first frame at `size` against the float64 oracle, on the pixels whose 16 samples both rasterize alike"""
    from dbw_b200 import Renderer, render_scene
    from dbw_b200 import views as V
    from oracle import dbw_path as D
    from oracle import phong as P
    from tests.helpers import decision_mask
    rend = V._eye_light(Renderer(size, **model.renderer.init_kwargs), size, V.EYE_LIGHT_ROTATED).to(R.device)
    rend.update_cameras(device=R.device, K=K[None].to(R.device))
    out = rend.render_viz(mesh, R[:1], T[:1]).cpu().double()
    verts, faces, fvu, fmap, maps, table = rend._scene(mesh)
    scene = {'verts': verts.cpu().double(), 'faces': faces.cpu().long(), 'faces_verts_uvs': fvu.cpu().double(),
             'face_map': fmap.cpu().long(), 'maps': [maps[o:o + h * w * 3].reshape(h, w, 3).cpu().double() for o, h, w in table]}
    big = (4 * size[0], 4 * size[1])
    R1, T1 = R[:1].cpu().double(), T[:1].cpu().double()
    ref = F.avg_pool2d(P.render_phong(scene, R1, T1, K.double(), big, lights=V.EYE_LIGHT_ROTATED, z_clip=rend.z_clip), 4)
    frags = D.render(scene, R1, T1, K.double(), big, sigma=0, faces_per_pixel=1, z_clip=rend.z_clip, return_fragments=True)[1]
    intr = tuple(float(K.reshape(4, 4)[i, j]) for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    _, ids = render_scene(verts, faces, fvu, fmap, maps, table, R[:1], T[:1], intr, big, 0.0, 1, rend.z_clip, return_ids=True)
    same = F.avg_pool2d(decision_mask(ids, frags, faces.shape[0]), 4) == 1
    err = ((out - ref).abs() * same).max().item()
    assert same.float().mean() > 0.97 and err <= 1e-4, (same.float().mean().item(), err)
    return err


def measure(shape, repeat, check):
    from dbw_b200 import Renderer
    from dbw_b200 import views as V
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.renderer import render_scene_phong
    from dbw_b200.synthetic import ring_cameras
    dev = torch.device('cuda')
    H, W = SHAPES[shape]
    torch.manual_seed(1)
    model = DifferentiableBlocksWorld((H, W), **deepcopy(CFG)).to(dev).eval()
    K = ring_cameras(1)[2]
    for r in (model.renderer, model.renderer_light):
        r.update_cameras(device=dev, K=K[None].to(dev))
    mesh = model.build_blocks(filter_transparent=True)
    R, T = turntable(N_FRAMES, dev)
    phong = V._eye_light(Renderer((H, W), **model.renderer.init_kwargs), (H, W), V.EYE_LIGHT_ROTATED).to(dev)
    phong.update_cameras(device=dev, K=K[None].to(dev))
    arms = {'flat': model.renderer_light, 'phong': phong}
    frames = {a: torch.empty(N_FRAMES, H, W, 3, dtype=torch.uint8, device=dev) for a in arms}
    res = {a: [] for a in arms}
    for a, r in arms.items():                        # warm-up of every shape either arm launches
        video_arm(r, mesh, R, T, frames[a])
    for _ in range(repeat):
        for a, r in arms.items():
            res[a].append(timed(video_arm, r, mesh, R, T, frames[a]))
    out = {a: {'frames_per_s': round(N_FRAMES / statistics.median(s), 1), 'median_s': round(statistics.median(s), 4)}
           for a, s in res.items()}
    out['phong_over_flat_time'] = round(statistics.median(res['phong']) / statistics.median(res['flat']), 3)
    if check:
        kept = []
        video_arm(phong, mesh, R, T, frames['phong'], kept)
        verts, faces, fvu, fmap, maps, table = phong._scene(mesh)
        from dbw_b200.renderer import phong_shading
        for a in range(0, N_FRAMES, 10):
            big = render_scene_phong(verts, faces, fvu, fmap, maps, table, R[a:a + 10], T[a:a + 10], phong.cameras.intrinsics(),
                                     (4 * H, 4 * W), phong_shading(phong.light_kwargs), 1, phong.z_clip,
                                     background=phong.background_color)
            pooled = F.avg_pool2d(big, 4)
            assert torch.equal(torch.cat(kept)[a:a + 10], pooled), 'resolved phong frames differ from avg_pool2d of the 4x render'
            assert torch.equal(frames['phong'][a:a + 10], (pooled[:, :3] * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8))
        out['bit_identical_to_pooled_4x'] = True
        out['oracle_max_err_quarter_size'] = check_against_oracle(model, mesh, R, T, K, (H // 4, W // 4))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=5)
    ap.add_argument('--check', action='store_true', help='check the phong frames against the 4x render and the float64 oracle')
    ap.add_argument('--shapes', default=','.join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_phong.py needs a CUDA device')
    name, power = card()
    out = {'gpu': name, 'power_limit_w': power, 'frames': N_FRAMES}
    for shape in args.shapes.split(','):
        out[f'{shape}_{SHAPES[shape][0]}x{SHAPES[shape][1]}'] = measure(shape, args.repeat, args.check)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
