"""Plain numpy statements the OBJ-export tests compare against (tests/test_obj_export_host.py, tests/test_obj_export_gpu.py):
the atlas composed map by map, a float64 bilinear sampler with the renderer's texture addressing, and a small reader of the
exported .obj / .mtl / .png files.  Test infrastructure only: the package has no OBJ reader for textured files."""
import numpy as np


def compose_atlas(maps_u8, layout):
    """(Ha, Wa, C) atlas of already quantised (h, w, C) maps: each map at its layout origin, its 1-texel gutter a copy of
    its edge texels (np.pad mode='edge'), every other texel 0"""
    C = maps_u8[0].shape[2]
    atlas = np.zeros((layout.height, layout.width, C), maps_u8[0].dtype)
    for m, (x0, y0) in zip(maps_u8, layout.origins):
        h, w = m.shape[:2]
        atlas[y0 - 1:y0 + h + 1, x0 - 1:x0 + w + 1] = np.pad(m, ((1, 1), (1, 1), (0, 0)), mode='edge')
    return atlas


def sample_bilinear(tex, uv):
    """(N, C) float64 samples of an (h, w, C) map at (N, 2) UVs as the renderer reads it (csrc/dbw_math.cuh tex_tap:
    align_corners=True on the map flipped along H, border clamp): column u (w - 1), stored row (1 - v) (h - 1)"""
    tex = np.asarray(tex, np.float64)
    h, w = tex.shape[:2]
    x = np.clip(np.asarray(uv[:, 0], np.float64), 0, 1) * (w - 1)
    y = (1 - np.clip(np.asarray(uv[:, 1], np.float64), 0, 1)) * (h - 1)
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    return ((1 - fx) * (1 - fy) * tex[y0, x0] + fx * (1 - fy) * tex[y0, x1]
            + (1 - fx) * fy * tex[y1, x0] + fx * fy * tex[y1, x1])


def read_obj(path):
    """(header lines before the first record, v (V,3) float64, vt (Vt,2) float64, face vertex indices (F,3), face vt indices
    (F,3) or None), 0-based"""
    head, v, vt, fv, ft = [], [], [], [], []
    with open(path) as fh:
        for line in fh:
            tok = line.split()
            if tok and tok[0] == 'v':
                v.append([float(t) for t in tok[1:]])
            elif tok and tok[0] == 'vt':
                vt.append([float(t) for t in tok[1:]])
            elif tok and tok[0] == 'f':
                idx = [t.split('/') for t in tok[1:]]
                fv.append([int(i[0]) - 1 for i in idx])
                if len(idx[0]) > 1:
                    ft.append([int(i[1]) - 1 for i in idx])
            elif not v:
                head.append(line.rstrip('\n'))
    return (head, np.array(v, np.float64).reshape(-1, 3), np.array(vt, np.float64).reshape(-1, 2),
            np.array(fv, np.int64).reshape(-1, 3), np.array(ft, np.int64).reshape(-1, 3) if ft else None)


def read_textured(obj_path):
    """the export's three files: (read_obj(...), the .mtl's map_Kd file name, the PNG as an (H, W, 3) uint8 array)"""
    from pathlib import Path
    from PIL import Image
    obj = read_obj(obj_path)
    mtllib = [l.split()[1] for l in obj[0] if l.startswith('mtllib')]
    mtl_path = Path(obj_path).parent / mtllib[0]
    kd = [l.split()[1] for l in mtl_path.read_text().splitlines() if l.startswith('map_Kd')]
    png = np.asarray(Image.open(mtl_path.parent / kd[0]).convert('RGB'))
    return obj, kd[0], png
