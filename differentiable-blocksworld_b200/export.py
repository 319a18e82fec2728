"""Wavefront OBJ export of a reconstructed scene: the reference's `save_mesh_as_obj` (src/utils/mesh.py:286-297), which
`qualitative_eval` calls for `mesh_full.obj` and `mesh.obj`.  A textured scene is written as the reference's `save_obj`
writes it (src/utils/mesh.py:306-486), byte for byte for the same arrays:

- `{stem}.obj`: the header "\\nmtllib {stem}.mtl\\nusemtl mesh\\n\\n", `v` lines, `vt` lines (both "%f", or "%.{d}f" with
  `decimal_places`), then `f a/at b/bt c/ct` lines, 1-based, with no newline after the last face;
- `{stem}.mtl`: "newmtl mesh\\nmap_Kd {stem}.png\\n";
- `{stem}.png`: the texture as (texture_map * 255.0).astype(np.uint8), a float32 product then truncation.

A mesh without TexturesUV is written as geometry only (`f a b c`).

The scene's maps (TexturesUV.map_groups: background, ground, kept blocks) become one atlas whose layout is this module's own,
not PyTorch3D's `pack_rectangles` (see `atlas_layout`).  The atlas is composed and quantised on the device by the library's
kernel (csrc/dbw_export.cu, one launch) and read back with one copy; maps on the CPU raise, there is no CPU fallback."""
import ctypes
import math
import warnings
from collections import namedtuple
from pathlib import Path

import numpy as np
import torch

from . import _lib
from ._lib import DbwError, DbwAtlasJob, check
from .structures import TexturesUV

AtlasLayout = namedtuple('AtlasLayout', 'height width origins cells')
AtlasLayout.__doc__ = """atlas (height, width); per map the atlas (column, row) of its texel (0, 0) and the (width, height) of
its cell, which starts one texel up and left of that origin"""


def atlas_layout(sizes):
    """The shelf-packed atlas of maps of sizes [(h, w)], in their order.  Each map is a (h + 2) x (w + 2) rectangle: the map
    and a 1-texel gutter that replicates its edge texels, so a UV that rounds a hair past a map's edge still samples that
    map's colour, as padding_mode='border' does.  The atlas width is max(widest rectangle, ceil(sqrt(total rectangle area)));
    rectangles are placed left to right and a new shelf starts when the next one does not fit; the height is the sum of the
    shelf heights.  Each rectangle's cell runs to the next rectangle of its shelf (to the atlas's right edge for the last one)
    and down to the shelf's bottom, so the cells tile the atlas; texels outside the rectangles are 0."""
    if not sizes:
        raise ValueError('atlas_layout: no map')
    rects = [(int(w) + 2, int(h) + 2) for h, w in sizes]
    if min(min(r) for r in rects) < 3:
        raise ValueError(f'atlas_layout: empty map in {sizes}')
    area = sum(rw * rh for rw, rh in rects)
    side = math.isqrt(area)
    width = max(max(rw for rw, _ in rects), side + (side * side < area))
    shelves, x, y, shelf_h = [[]], 0, 0, 0
    origins = []
    for rw, rh in rects:
        if x + rw > width:
            y, x, shelf_h = y + shelf_h, 0, 0
            shelves.append([])
        origins.append((x + 1, y + 1))
        shelves[-1].append(len(origins) - 1)
        x += rw
        shelf_h = max(shelf_h, rh)
    height = y + shelf_h
    cells = [None] * len(rects)
    for shelf in shelves:
        sy = origins[shelf[0]][1] - 1
        sh = max(rects[k][1] for k in shelf)
        for n, k in enumerate(shelf):
            right = origins[shelf[n + 1]][0] - 1 if n + 1 < len(shelf) else width
            cells[k] = (right - (origins[k][0] - 1), sy + sh - (origins[k][1] - 1))
    return AtlasLayout(height, width, origins, cells)


def remap_uvs(faces_verts_uvs, face_map, sizes, layout):
    """(F, 3, 2) float64 atlas UVs of per-face-corner map UVs: the point a map's sampler reads (align_corners=True on the map
    flipped along H, border clamp; csrc/dbw_math.cuh tex_tap) is the point the atlas's sampler reads.  With (x0, y0) the
    map's origin in the atlas and u, v clamped to [0, 1]:
        u' = (x0 + u (w - 1)) / (Wa - 1),    v' = 1 - (y0 + (1 - v) (h - 1)) / (Ha - 1)"""
    uv = np.clip(np.asarray(faces_verts_uvs, dtype=np.float64), 0.0, 1.0)
    fm = np.asarray(face_map, dtype=np.int64)
    hw = np.asarray(sizes, dtype=np.float64)[fm]
    org = np.asarray(layout.origins, dtype=np.float64)[fm]
    out = np.empty_like(uv)
    out[..., 0] = (org[:, None, 0] + uv[..., 0] * (hw[:, None, 1] - 1.0)) / (layout.width - 1.0)
    out[..., 1] = 1.0 - (org[:, None, 1] + (1.0 - uv[..., 1]) * (hw[:, None, 0] - 1.0)) / (layout.height - 1.0)
    return out


def texture_atlas(maps):
    """((Ha, Wa, 3) uint8 device atlas, AtlasLayout) of a list of (h, w, 3) float32 CUDA maps, in one launch: each map at its
    atlas_layout place, texels quantised as (uint8)(x * 255.0f), gutters replicating the edge texels, the rest 0"""
    if not maps:
        raise ValueError('texture_atlas: no map')
    dev = maps[0].device
    for m in maps:
        if not m.is_cuda or m.device != dev:
            raise DbwError('texture_atlas: expected CUDA maps on one device (there is no CPU fallback)')
        if m.dtype != torch.float32 or m.dim() != 3 or m.shape[2] != 3:
            raise DbwError(f'texture_atlas: expected float32 (h, w, 3) maps, got {m.dtype} {tuple(m.shape)}')
    maps = [m.detach().contiguous() for m in maps]
    sizes = [(int(m.shape[0]), int(m.shape[1])) for m in maps]
    layout = atlas_layout(sizes)
    jobs = (DbwAtlasJob * len(maps))(*[DbwAtlasJob(m.data_ptr(), h, w, x0, y0, cw, ch)
                                       for m, (h, w), (x0, y0), (cw, ch) in zip(maps, sizes, layout.origins, layout.cells)])
    L = _lib.lib()
    atlas = torch.empty(layout.height, layout.width, 3, dtype=torch.uint8, device=dev)
    ws = torch.empty(L.dbw_texture_atlas_workspace_bytes(len(maps)), dtype=torch.uint8, device=dev)
    check(L.dbw_texture_atlas_u8(jobs, len(maps), layout.height, layout.width, ctypes.c_void_p(atlas.data_ptr()),
                                 ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                 ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), 'dbw_texture_atlas_u8')
    return atlas, layout


def scene_maps(textures):
    """the scene's maps in TexturesUV order (map_groups: background, ground, kept blocks), as (h, w, 3) views"""
    return [g[i] for g in textures.map_groups for i in range(g.shape[0])]


def save_mesh_as_obj(mesh, filename, decimal_places=None):
    """Write the first (only) mesh of a joined scene `mesh` as `filename` (.obj), plus, when it carries TexturesUV,
    `{stem}.mtl` and `{stem}.png` beside it, in the reference's format (module docstring).  The texture is the scene's
    atlas (atlas_layout); one `vt` is written per face corner, remapped into the atlas (remap_uvs)."""
    assert len(mesh) == 1
    verts, faces = mesh.get_mesh_verts_faces(0)
    txt = mesh.textures
    if not isinstance(txt, TexturesUV) or txt.n_maps() == 0:
        write_obj(filename, verts, faces, decimal_places)
        return
    maps = scene_maps(txt)
    atlas, layout = texture_atlas(maps)
    fvu, fmap = txt.scene_arrays()
    F = int(faces.shape[0])
    if fvu.shape[0] != F:
        raise ValueError(f'save_mesh_as_obj: the texture has {fvu.shape[0]} faces, the mesh {F}')
    sizes = [(int(m.shape[0]), int(m.shape[1])) for m in maps]
    uvs = remap_uvs(fvu.detach().cpu().numpy(), fmap.cpu().numpy(), sizes, layout)
    write_obj(filename, verts, faces, decimal_places, verts_uvs=uvs.reshape(-1, 2),
              faces_uvs=np.arange(3 * F, dtype=np.int64).reshape(F, 3), texture=atlas.cpu().numpy())


def _rows(a):
    return a.detach().cpu().tolist() if torch.is_tensor(a) else np.asarray(a).tolist()


def obj_records(verts, faces, decimal_places=None, verts_uvs=None, faces_uvs=None):
    """the .obj records after the header, as save_obj's `_save` writes them (src/utils/mesh.py:405-486): `v`, then `vt` and
    `f a/at ..` faces when verts_uvs and faces_uvs are given, else `f a b c` faces; no newline after the last face"""
    v, f = _rows(verts), _rows(faces)
    if not (len(v) or len(f)):
        warnings.warn("Empty 'verts' and 'faces' arguments provided")
        return ''
    fmt = '%f' if decimal_places is None else '%.' + '%df' % decimal_places
    parts = [''.join(f'v {fmt} {fmt} {fmt}\n' % tuple(r) for r in v)]
    if len(f) and (max(map(max, f)) >= len(v) or min(map(min, f)) < 0):
        warnings.warn('Faces have invalid indices')
    if verts_uvs is not None and faces_uvs is not None:
        parts.append(''.join(f'vt {fmt} {fmt}\n' % tuple(r) for r in _rows(verts_uvs)))
        parts.append('\n'.join('f %d/%d %d/%d %d/%d' % (a + 1, ta + 1, b + 1, tb + 1, c + 1, tc + 1)
                               for (a, b, c), (ta, tb, tc) in zip(f, _rows(faces_uvs))))
    else:
        parts.append('\n'.join('f %d %d %d' % (a + 1, b + 1, c + 1) for a, b, c in f))
    return ''.join(parts)


def write_obj(filename, verts, faces, decimal_places=None, *, verts_uvs=None, faces_uvs=None, texture=None):
    """Write `filename` as save_obj does.  With verts_uvs (Vt, 2), faces_uvs (F, 3) and an (H, W, 3) uint8 `texture` (already
    quantised, host memory) the .obj gets the material header and `vt` records, and `{stem}.mtl` and `{stem}.png` are
    written beside it."""
    path = Path(filename)
    textured = verts_uvs is not None and faces_uvs is not None and texture is not None
    with open(filename, 'w') as fh:
        if textured:
            fh.write(f'\nmtllib {path.stem}.mtl\nusemtl mesh\n\n')
        fh.write(obj_records(verts, faces, decimal_places, *((verts_uvs, faces_uvs) if textured else ())))
    if textured:
        write_png(path.with_suffix('.png'), texture)
        with open(path.with_suffix('.mtl'), 'w') as fh:
            fh.write(f'newmtl mesh\nmap_Kd {path.stem}.png\n')


def write_png(path, texture):
    from PIL import Image
    texture = np.asarray(texture)
    if texture.dtype != np.uint8 or texture.ndim != 3 or texture.shape[2] != 3:
        raise ValueError(f'write_png: expected an (H, W, 3) uint8 texture, got {texture.dtype} {texture.shape}')
    Image.fromarray(texture).save(path, format='PNG')
