"""What the textured OBJ export (`export.save_mesh_as_obj`, as `qualitative_eval` calls it for mesh_full.obj) costs on the GPU,
for the bench scene (10 blocks, TS 256) and the stress shape (50 blocks, TS 256), every block kept.  Per scene, the median
over --repeat of:

  atlas    export.texture_atlas: the job table, its copy to the device and the atlas kernel (CUDA events, device time), and
           the host wall time of the call up to a synchronise
  d2h      the one device-to-host copy of the uint8 atlas
  png      PIL's PNG encode and write of the atlas
  text     the per-corner UV remap and the .obj / .mtl text write
  total    save_mesh_as_obj end to end

--check asserts that the kernel's atlas equals a torch composition of the same layout bit for bit (each map
(map.cpu() * 255.0).numpy().astype(uint8), gutters as edge copies, the rest 0).  Files go to a temporary directory.  Prints
one JSON line with the card's name and power limit.

    python scripts/bench_export.py [--repeat 5] [--check]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from copy import deepcopy

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CFG = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
       'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
       'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                      'decouple_rendering': True, 'opacity_noise': False},
       'loss': {'rgb_weight': 1}}
SCENES = {'dtu_10': 10, 'stress_50': 50}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def scene_of(n_blocks, dev):
    from dbw_b200.dbw import DifferentiableBlocksWorld
    torch.manual_seed(0)
    cfg = deepcopy(CFG)
    cfg['mesh']['n_blocks'] = n_blocks
    model = DifferentiableBlocksWorld((400, 400), **cfg).to(dev)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for t in (model.texture_bkg, model.texture_ground, model.textures):
            t.copy_(torch.randn(t.shape, generator=g) * 3)
        model.alpha_logit.fill_(3.0)
    model.set_cur_epoch(2000)
    model.eval()
    with torch.no_grad():
        return model.build_scene(filter_transparent=True)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def one(scene, tmp):
    from dbw_b200 import export
    verts, faces = scene.get_mesh_verts_faces(0)
    maps = export.scene_maps(scene.textures)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    atlas, layout = export.texture_atlas(maps)
    e1.record()
    torch.cuda.synchronize()
    t = {'atlas_wall': (time.perf_counter() - t0) * 1e3, 'atlas_device': e0.elapsed_time(e1)}
    host, t['d2h'] = wall(lambda: atlas.cpu().numpy())
    _, t['png'] = wall(lambda: export.write_png(os.path.join(tmp, 'a.png'), host))

    def text():
        fvu, fmap = scene.textures.scene_arrays()
        sizes = [(int(m.shape[0]), int(m.shape[1])) for m in maps]
        uvs = export.remap_uvs(fvu.cpu().numpy(), fmap.cpu().numpy(), sizes, layout)
        F = int(faces.shape[0])
        with open(os.path.join(tmp, 'a.obj'), 'w') as fh:
            fh.write('\nmtllib a.mtl\nusemtl mesh\n\n')
            fh.write(export.obj_records(verts, faces, None, uvs.reshape(-1, 2), np.arange(3 * F).reshape(F, 3)))
        with open(os.path.join(tmp, 'a.mtl'), 'w') as fh:
            fh.write('newmtl mesh\nmap_Kd a.png\n')
    _, t['text'] = wall(text)
    _, t['total'] = wall(lambda: export.save_mesh_as_obj(scene, os.path.join(tmp, 'mesh_full.obj')))
    return t, atlas, layout, maps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=5)
    ap.add_argument('--check', action='store_true')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    name, power = card()
    result = {'bench': 'obj_export', 'card': name, 'power_limit_w': power, 'repeat': args.repeat, 'scenes': {}}
    with tempfile.TemporaryDirectory() as tmp:
        for sname, n_blocks in SCENES.items():
            scene = scene_of(n_blocks, dev)
            one(scene, tmp)                                                  # warm-up: library load, allocator, PIL
            runs = [one(scene, tmp) for _ in range(args.repeat)]
            _, atlas, layout, maps = runs[-1]
            med = {k: round(statistics.median(r[0][k] for r in runs), 3) for k in runs[0][0]}
            entry = {'maps': len(maps), 'atlas_hw': [layout.height, layout.width],
                     'texels_m': round(layout.height * layout.width / 1e6, 3), 'faces': int(scene.get_mesh_verts_faces(0)[1].shape[0]),
                     'ms': med, 'obj_bytes': os.path.getsize(os.path.join(tmp, 'mesh_full.obj')),
                     'png_bytes': os.path.getsize(os.path.join(tmp, 'mesh_full.png'))}
            if args.check:
                from tests._obj_export_ref import compose_atlas
                want = compose_atlas([(m.cpu() * 255.0).numpy().astype(np.uint8) for m in maps], layout)
                got = atlas.cpu().numpy()
                entry['check_bit_equal'] = bool(np.array_equal(got, want))
                assert entry['check_bit_equal'], sname
            result['scenes'][sname] = entry
    print(json.dumps(result))


if __name__ == '__main__':
    main()
