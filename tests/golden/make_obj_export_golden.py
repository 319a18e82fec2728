"""Generates tests/golden/obj_export.npz: the files the reference's OWN `save_obj` / `_save` (src/utils/mesh.py:306-486) of a
checkout of monniert/differentiable-blocksworld named by DBW_REFERENCE writes, extracted with `ast` by tests/_refextract.py
and run with a trivial PathManager, `_open_file` = open, pathlib.Path, PIL.Image and warnings.  For each case it freezes
the inputs, the .obj text, the .mtl text (textured cases) and the array of the written PNG.  The cases cover textured and
untextured meshes, decimal_places None and 3, negative, large and tiny coordinates, one face, and a texture map holding
values on and next to the k/255 boundaries.

    DBW_REFERENCE=/path/to/differentiable-blocksworld python tests/golden/make_obj_export_golden.py
"""
import os
import sys
import tempfile
import typing
import warnings
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from _refextract import extract, have_reference  # noqa: E402

OUT = os.path.join(HERE, 'obj_export.npz')

# name: (n_verts, n_faces, coordinate scale, textured, decimal_places, seed)
CASES = {
    'textured': (9, 7, 1.0, True, None, 1),
    'textured_dp3': (9, 7, 1.0, True, 3, 1),
    'plain': (6, 4, 1.0, False, None, 2),
    'plain_dp3': (6, 4, 1.0, False, 3, 2),
    'wide': (12, 10, 1e5, True, None, 3),
    'wide_dp3': (12, 10, 1e5, True, 3, 3),
    'tiny': (5, 3, 1e-6, True, None, 4),
    'one_face': (3, 1, 10.0, True, None, 5),
}


def inputs(name):
    """(verts (V,3) f32, faces (F,3) i64, verts_uvs (Vt,2) f32, faces_uvs (F,3) i64, texture_map (H,W,3) f32) of a case"""
    V, F, scale, _, _, seed = CASES[name]
    g = np.random.default_rng(seed)
    verts = ((g.random((V, 3)) * 2 - 1) * scale).astype(np.float32)
    verts[0] = [-scale, 0.0, -0.0]                                  # exact zeros of both signs
    faces = np.stack([g.permutation(V)[:3] for _ in range(F)]).astype(np.int64)
    Vt = V + 2
    verts_uvs = g.random((Vt, 2)).astype(np.float32)
    verts_uvs[0], verts_uvs[1] = [0.0, 1.0], [1.0, 0.0]
    faces_uvs = g.integers(0, Vt, (F, 3)).astype(np.int64)
    H, W = 5 + seed % 3, 7
    k = g.integers(0, 256, (H, W, 3)).astype(np.float32)
    tex = (k / np.float32(255.0)).astype(np.float32)                # on the boundaries (rounded to float32)
    nudge = g.integers(-1, 2, (H, W, 3))                            # and their float32 neighbours
    tex = np.where(nudge < 0, np.nextafter(tex, np.float32(0)), np.where(nudge > 0, np.nextafter(tex, np.float32(1)), tex))
    tex = np.clip(tex, 0, 1).astype(np.float32)
    tex[0, 0] = [0.0, 1.0, 0.5]
    return verts, faces, verts_uvs, faces_uvs, tex


class _PathManager:
    pass


def main():
    if not have_reference():
        print('DBW_REFERENCE is not a reference checkout: tests/golden/obj_export.npz left untouched')
        return
    from PIL import Image
    ns = extract('src/utils/mesh.py', {'save_obj', '_save'},
                 extra_ns={'Optional': typing.Optional, 'PathManager': _PathManager, 'Path': Path, 'Image': Image,
                           'warnings': warnings, '_open_file': lambda f, path_manager, mode: open(f, mode)})
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (_, _, _, textured, dp, _) in CASES.items():
            verts, faces, verts_uvs, faces_uvs, tex = inputs(name)
            obj = os.path.join(tmp, f'{name}.obj')
            kw = dict(verts_uvs=torch.from_numpy(verts_uvs), faces_uvs=torch.from_numpy(faces_uvs),
                      texture_map=torch.from_numpy(tex)) if textured else {}
            ns['save_obj'](obj, torch.from_numpy(verts), torch.from_numpy(faces), decimal_places=dp, **kw)
            for key, arr in zip(('verts', 'faces', 'verts_uvs', 'faces_uvs', 'texture_map'), (verts, faces, verts_uvs, faces_uvs, tex)):
                out[f'{name}/{key}'] = arr
            out[f'{name}/obj'] = np.frombuffer(open(obj, 'rb').read(), np.uint8)
            if textured:
                out[f'{name}/mtl'] = np.frombuffer(open(obj[:-4] + '.mtl', 'rb').read(), np.uint8)
                out[f'{name}/png'] = np.asarray(Image.open(obj[:-4] + '.png'))
    np.savez_compressed(OUT, **out)
    print(f'wrote {OUT}: {len(CASES)} cases')


if __name__ == '__main__':
    main()
