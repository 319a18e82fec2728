"""CPU: the OBJ export without a GPU.  The writer against the files the reference's own save_obj wrote
(tests/golden/obj_export.npz, byte for byte); the atlas packer and the UV remap; the atlas kernel's per-texel math
(differentiable-blocksworld_b200/csrc/dbw_export_math.cuh) compiled for the host (tests/host_math/dbw_export_host.cpp,
g++ -ffp-contract=off) against numpy's quantisation and a map-by-map composition; and the argument checks of the C-ABI and of
dbw_b200.export, which all fail before anything reaches a device.  The kernel itself is tested in tests/test_obj_export_gpu.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests._obj_export_ref import compose_atlas, read_obj, sample_bilinear
from tests.golden.make_obj_export_golden import CASES

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = np.load(os.path.join(HERE, 'golden', 'obj_export.npz'))
CSRC = os.path.join(ROOT, 'differentiable-blocksworld_b200', 'csrc')
ATLAS_THREADS = int(re.search(r'ATLAS_THREADS = (\d+);', open(os.path.join(CSRC, 'dbw_export.cu')).read()).group(1))

# (h, w) of the maps of shipped scene shapes: background and ground S x S (S = TS, or 2 TS with txt_bkg_upscale: 2 for the
# background), blocks TS x (p_left + TS + p_right)
SCENES = {
    'dtu_10_blocks': [(256, 256), (256, 256)] + [(256, 279)] * 10,
    'upscaled_bkg': [(512, 512), (256, 256)] + [(256, 279)] * 4,
    'stress_50_blocks': [(256, 256), (256, 256)] + [(256, 279)] * 50,
    'ts32': [(32, 32), (32, 32)] + [(32, 35)] * 3,
    'no_blocks': [(64, 64), (64, 64)],
    'one_map': [(1, 1)],
    'mixed': [(3, 40), (17, 2), (1, 1), (9, 9), (40, 3), (2, 17), (5, 1), (1, 5), (30, 30)],
}


@pytest.fixture(scope='module')
def hm():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_export_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror',
                    os.path.join(HERE, 'host_math', 'dbw_export_host.cpp'), '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.hm_quantise.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]
    L.hm_quantise.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _quantise(hm, x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(x.shape, np.uint8)
    hm.hm_quantise(x.size, _p(x), _p(out))
    return out


def _numpy_quantise(x):
    return (np.asarray(x, np.float32) * np.float32(255.0)).astype(np.uint8)


def _host_atlas(hm, maps, layout, cta_texels=ATLAS_THREADS):
    from dbw_b200._lib import DbwAtlasJob
    maps = [np.ascontiguousarray(m, np.float32) for m in maps]
    jobs = (DbwAtlasJob * len(maps))(*[DbwAtlasJob(m.ctypes.data, m.shape[0], m.shape[1], x0, y0, cw, ch)
                                       for m, (x0, y0), (cw, ch) in zip(maps, layout.origins, layout.cells)])
    atlas = np.full((layout.height, layout.width, 3), 0xA5, np.uint8)       # every texel must be overwritten
    hm.hm_atlas(jobs, len(maps), layout.width, cta_texels, _p(atlas))
    return atlas


# ------------------------------------------------------------------ the file format, against the reference's own writer
@pytest.mark.parametrize('name', list(CASES))
def test_writer_reproduces_the_references_files(hm, name, tmp_path):
    from dbw_b200 import export
    from PIL import Image
    textured, dp = CASES[name][3], CASES[name][4]
    g = {k: GOLDEN[f'{name}/{k}'] for k in ('verts', 'faces', 'verts_uvs', 'faces_uvs', 'texture_map')}
    obj = tmp_path / f'{name}.obj'
    kw = dict(verts_uvs=g['verts_uvs'], faces_uvs=g['faces_uvs'], texture=_quantise(hm, g['texture_map'])) if textured else {}
    export.write_obj(obj, g['verts'], g['faces'], dp, **kw)
    assert obj.read_bytes() == GOLDEN[f'{name}/obj'].tobytes()
    if textured:
        assert (tmp_path / f'{name}.mtl').read_bytes() == GOLDEN[f'{name}/mtl'].tobytes()
        assert np.array_equal(_quantise(hm, g['texture_map']), GOLDEN[f'{name}/png'])      # the kernel's quantisation
        assert np.array_equal(np.asarray(Image.open(tmp_path / f'{name}.png')), GOLDEN[f'{name}/png'])
    else:
        assert not (tmp_path / f'{name}.mtl').exists() and not (tmp_path / f'{name}.png').exists()


@pytest.mark.parametrize('name', [n for n, c in CASES.items() if not c[3]])
def test_untextured_mesh_is_written_as_geometry_only(name, tmp_path):
    """save_mesh_as_obj of a Meshes without TexturesUV needs no device: the reference's untextured file"""
    from dbw_b200 import Meshes, export
    v, f = torch.from_numpy(GOLDEN[f'{name}/verts']), torch.from_numpy(GOLDEN[f'{name}/faces'])
    export.save_mesh_as_obj(Meshes(v[None], f[None]), tmp_path / 'm.obj', decimal_places=CASES[name][4])
    assert (tmp_path / 'm.obj').read_bytes() == GOLDEN[f'{name}/obj'].tobytes()


@pytest.mark.parametrize('name', ['textured', 'wide', 'one_face'])
def test_load_obj_reads_the_textured_format(hm, name, tmp_path):
    """geometry.load_obj (and so dtu_eval.evaluate_mesh(path)) takes `f a/at ..` by its vertex index and skips the header's
    blank lines; the unterminated last face still counts"""
    from dbw_b200 import export, geometry
    g = {k: GOLDEN[f'{name}/{k}'] for k in ('verts', 'faces', 'verts_uvs', 'faces_uvs', 'texture_map')}
    export.write_obj(tmp_path / 'm.obj', g['verts'], g['faces'], verts_uvs=g['verts_uvs'], faces_uvs=g['faces_uvs'],
                     texture=_quantise(hm, g['texture_map']))
    verts, faces = geometry.load_obj(str(tmp_path / 'm.obj'))
    assert np.array_equal(faces.numpy(), g['faces'])
    want = np.array([[float('%f' % x) for x in r] for r in g['verts'].tolist()], np.float32)
    assert np.array_equal(verts.numpy(), want)
    assert sum(1 for l in open(tmp_path / 'm.obj') if l.startswith('f ')) == len(g['faces'])
    head, v, vt, fv, ft = read_obj(tmp_path / 'm.obj')
    assert head == ['', 'mtllib m.mtl', 'usemtl mesh', ''] and np.array_equal(ft, g['faces_uvs'])


# ------------------------------------------------------------------ packer and UV remap
def _rects(layout, sizes):
    """(x, y, w, h) of each map's rectangle with its gutter"""
    return [(x0 - 1, y0 - 1, w + 2, h + 2) for (x0, y0), (h, w) in zip(layout.origins, sizes)]


def _overlap(a, b):
    return a[0] < b[0] + b[2] and b[0] < a[0] + a[2] and a[1] < b[1] + b[3] and b[1] < a[1] + a[3]


@pytest.mark.parametrize('scene', list(SCENES))
def test_packer_layout(scene):
    import math
    from dbw_b200.export import atlas_layout
    sizes = SCENES[scene]
    lay = atlas_layout(sizes)
    assert lay == atlas_layout(list(sizes))                                         # deterministic
    area = sum((h + 2) * (w + 2) for h, w in sizes)
    assert lay.width == max(max(w + 2 for _, w in sizes), math.ceil(math.sqrt(area)))
    rects = _rects(lay, sizes)
    cells = [(x0 - 1, y0 - 1, cw, ch) for (x0, y0), (cw, ch) in zip(lay.origins, lay.cells)]
    for r, c in zip(rects, cells):
        assert 0 <= r[0] and 0 <= r[1] and r[0] + r[2] <= lay.width and r[1] + r[3] <= lay.height   # gutters inside
        assert c[:2] == r[:2] and c[2] >= r[2] and c[3] >= r[3]                                   # cell holds its rectangle
        assert c[0] + c[2] <= lay.width and c[1] + c[3] <= lay.height
    for i in range(len(rects)):
        for j in range(i):
            assert not _overlap(rects[i], rects[j]) and not _overlap(cells[i], cells[j]), (i, j)
    assert sum(c[2] * c[3] for c in cells) == lay.width * lay.height                 # the cells tile the atlas
    # shelves: left to right in map order, a new shelf when the next rectangle does not fit, height = sum of shelf heights
    shelf_tops = sorted({r[1] for r in rects})
    shelf_h = [max(r[3] for r in rects if r[1] == t) for t in shelf_tops]
    assert shelf_tops == list(np.cumsum([0] + shelf_h[:-1])) and lay.height == sum(shelf_h)
    for a, b in zip(rects, rects[1:]):
        if b[1] == a[1]:
            assert b[0] == a[0] + a[2]
        else:
            assert b[0] == 0 and a[0] + a[2] + b[2] > lay.width and b[1] > a[1]


@pytest.mark.parametrize('scene', list(SCENES))
def test_remap_lands_texel_centres_on_the_atlas_texels(scene):
    """the map UV that samples texel (row s, column x) exactly, u = x / (w - 1) and v = 1 - s / (h - 1), remaps to the UV that
    samples the atlas exactly at its copy (x0 + x, y0 + s), to float64 rounding"""
    from dbw_b200.export import atlas_layout, remap_uvs
    sizes = SCENES[scene]
    lay = atlas_layout(sizes)
    for k, (h, w) in enumerate(sizes):
        s, x = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
        u = x / max(w - 1, 1)
        v = 1 - s / max(h - 1, 1)
        uv = np.stack([u, v], -1).reshape(-1, 1, 2).repeat(3, 1)
        out = remap_uvs(uv, np.full(len(uv), k), sizes, lay)[:, 0]
        cols, rows = out[:, 0] * (lay.width - 1), (1 - out[:, 1]) * (lay.height - 1)
        x0, y0 = lay.origins[k]
        assert np.abs(cols - (x0 + x.reshape(-1))).max() <= 1e-9 and np.abs(rows - (y0 + s.reshape(-1))).max() <= 1e-9


@pytest.mark.parametrize('scene', ['ts32', 'mixed', 'no_blocks', 'one_map'])
def test_atlas_samples_equal_map_samples(scene):
    """sampling the (float) atlas at remapped UVs == sampling each map at its own UVs, with the renderer's addressing, for UVs
    inside, on the edges of and outside [0, 1] (clamped): a flip, a wrong origin or swapped u / v changes whole regions"""
    from dbw_b200.export import atlas_layout, remap_uvs
    sizes = SCENES[scene]
    g = np.random.default_rng(7)
    maps = [g.random((h, w, 3)) for h, w in sizes]
    lay = atlas_layout(sizes)
    atlas = compose_atlas(maps, lay)
    n = 3000
    fmap = g.integers(0, len(sizes), n)
    uv = g.uniform(-0.2, 1.2, (n, 3, 2))
    uv[:50] = g.integers(0, 2, (50, 3, 2))                                          # corners and edges exactly
    got = sample_bilinear(atlas, remap_uvs(uv, fmap, sizes, lay).reshape(-1, 2))
    want = np.concatenate([sample_bilinear(maps[k], uv[i]) for i, k in enumerate(fmap)])
    assert np.abs(got - want).max() <= 1e-9


def test_packer_refuses_empty_input():
    from dbw_b200.export import atlas_layout
    with pytest.raises(ValueError):
        atlas_layout([])
    with pytest.raises(ValueError):
        atlas_layout([(0, 4)])


# ------------------------------------------------------------------ the kernel's math on the host
def test_quantisation_equals_numpy_around_every_boundary(hm):
    """(uint8)(x * 255.f) == (x * 255.0).astype(np.uint8) for every float32 within 64 ulps of each k / 255 in [0, 1], and on
    a million uniform draws"""
    k = (np.arange(256, dtype=np.float64) / 255).astype(np.float32)
    xs = [k]
    up, down = k.copy(), k.copy()
    for _ in range(64):
        up, down = np.nextafter(up, np.float32(2)), np.nextafter(down, np.float32(-1))
        xs += [up, down]
    x = np.concatenate(xs + [np.random.default_rng(0).random(1 << 20, dtype=np.float32)])
    x = x[(x >= 0) & (x <= 1)]
    assert np.array_equal(_quantise(hm, x), _numpy_quantise(x))
    assert np.array_equal(_quantise(hm, x), (torch.from_numpy(x) * 255.0).numpy().astype(np.uint8))
    # outside [0, 1] (no map of the scene has such values) the kernel saturates
    odd = np.float32([-1.0, -0.0, 1.0001, 2.0, np.inf, -np.inf, np.nan])
    assert _quantise(hm, odd).tolist() == [0, 0, 255, 255, 255, 0, 0]


def test_source_texel_covers_rectangle_and_gutter(hm):
    h, w = 3, 5
    want = np.pad(np.arange(h * w).reshape(h, w), 1, mode='edge')
    got = np.array([[hm.hm_source_texel(r, c, h, w) for c in range(w + 4)] for r in range(h + 4)])
    assert np.array_equal(got[:h + 2, :w + 2], want)
    assert (got[h + 2:] == -1).all() and (got[:, w + 2:] == -1).all()


@pytest.mark.parametrize('cta_texels', [ATLAS_THREADS, 37, 1])
@pytest.mark.parametrize('scene', ['ts32', 'mixed', 'no_blocks', 'one_map'])
def test_host_kernel_body_composes_the_atlas(hm, scene, cta_texels):
    """the kernel's per-thread body, run for every (CTA, thread) of the launch, == numpy's quantisation of each map placed at
    its layout origin with edge-copy gutters and zeros elsewhere; cells that end inside a CTA and CTAs that start a cell are
    both exercised (cta_texels that do not divide the cells)"""
    from dbw_b200.export import atlas_layout
    sizes = SCENES[scene]
    g = np.random.default_rng(11)
    maps = [g.random((h, w, 3), dtype=np.float32) for h, w in sizes]
    maps[0][0, 0] = [0.0, 1.0, np.float32(1 / 255)]
    lay = atlas_layout(sizes)
    got = _host_atlas(hm, maps, lay, cta_texels)
    assert np.array_equal(got, compose_atlas([_numpy_quantise(m) for m in maps], lay))


# ------------------------------------------------------------------ C-ABI and Python refusals
def test_atlas_job_struct_layout(tmp_path):
    from dbw_b200._lib import DbwAtlasJob
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(DbwAtlasJob));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DbwAtlasJob, {f}));' for f, _ in DbwAtlasJob._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines + ['  return 0;', '}']))
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(tmp_path / 'a')],
                   check=True)
    got = dict(l.split() for l in subprocess.run([str(tmp_path / 'a')], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(DbwAtlasJob) == 32
    for f, _ in DbwAtlasJob._fields_:
        assert int(got[f]) == getattr(DbwAtlasJob, f).offset, f


def test_c_abi_refuses_bad_tables_before_any_launch():
    from dbw_b200 import _lib
    from dbw_b200._lib import DbwAtlasJob
    from dbw_b200.export import atlas_layout
    L = _lib.lib()
    assert L.dbw_texture_atlas_workspace_bytes(0) == 0 and L.dbw_texture_atlas_workspace_bytes(3) == 3 * 40
    fake, ws = 256, ctypes.c_void_p(512)                                          # never dereferenced: the checks fail first
    sizes = [(4, 6), (5, 3), (2, 2)]
    lay = atlas_layout(sizes)

    def table(edit=None):
        rows = [[fake, h, w, x0, y0, cw, ch] for (h, w), (x0, y0), (cw, ch) in zip(sizes, lay.origins, lay.cells)]
        if edit:
            edit(rows)
        return (DbwAtlasJob * len(rows))(*[DbwAtlasJob(*r) for r in rows])

    def call(jobs, n=3, H=lay.height, W=lay.width, ws_bytes=1 << 20, atlas=ctypes.c_void_p(1024)):
        return L.dbw_texture_atlas_u8(jobs, n, H, W, atlas, ws, ws_bytes, None)

    assert call(None) != 0 and b'null' in L.dbw_last_error()
    assert call(table(), atlas=None) != 0 and b'null' in L.dbw_last_error()
    assert call(table(), n=0) != 0
    assert call(table(), H=0) != 0 and b'atlas size' in L.dbw_last_error()
    assert call(table(), ws_bytes=3 * 40 - 1) != 0 and b'workspace' in L.dbw_last_error()
    assert call(table(lambda r: r[1].__setitem__(0, None))) != 0 and b'no map' in L.dbw_last_error()
    assert call(table(lambda r: r[0].__setitem__(5, 7))) != 0 and b'does not hold' in L.dbw_last_error()    # cell narrower than w + 2
    assert call(table(lambda r: r[0].__setitem__(3, 0))) != 0 and b'does not hold' in L.dbw_last_error()    # gutter off the atlas
    assert call(table(lambda r: r[2].__setitem__(3, r[0][3]) or r[2].__setitem__(4, r[0][4]))) != 0
    assert b'overlap' in L.dbw_last_error()
    assert call(table(), n=2) != 0 and b'tile' in L.dbw_last_error()              # the third cell left uncovered
    assert call(table(), W=lay.width + 1) != 0


def test_python_refuses_cpu_maps():
    from dbw_b200 import Meshes, TexturesUV
    from dbw_b200._lib import DbwError
    from dbw_b200.export import save_mesh_as_obj, texture_atlas
    with pytest.raises(DbwError, match='CUDA'):
        texture_atlas([torch.rand(4, 4, 3)])
    with pytest.raises(ValueError):
        texture_atlas([])
    txt = TexturesUV(torch.rand(1, 4, 4, 3), torch.zeros(1, 1, 3, dtype=torch.long), torch.zeros(1, 1, 2))
    mesh = Meshes(torch.rand(1, 3, 3), torch.tensor([[[0, 1, 2]]]), txt)
    with pytest.raises(DbwError, match='no CPU fallback'):
        save_mesh_as_obj(mesh, '/nonexistent/never_written.obj')
