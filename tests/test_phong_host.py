"""CPU checks of Phong shading: the math of csrc/dbw_shade_math.cuh compiled for the host against the float64 restatement of
PyTorch3D (oracle/phong.py) -- vertex normals on closed and degenerate meshes, diffuse and specular for every light type --,
the C-ABI's struct layout and refusals, the lights and materials the renderer passes, and the eye_light setup of the view
helpers (the renderer each one builds, the refusals of a given R and of anything that is not a mesh)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from dbw_b200 import views as V
from dbw_b200 import Renderer
from dbw_b200.renderer import phong_shading
from oracle import dbw_path as D
from oracle import phong as P
from oracle import pt3d

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope='module')
def hs():
    src = os.path.join(HERE, 'host_math', 'dbw_shade_host.cpp')
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_shade_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', src, '-o', so], check=True)
    L = ctypes.CDLL(so)
    L.hs_vertex_normals.restype = L.hs_phong.restype = None
    L.hs_sizeof_shading.restype = ctypes.c_size_t
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def vertex_face_list(faces, n_verts):
    """the list dbw_vertex_face_list builds: each vertex's faces in ascending order, one entry per corner on the vertex"""
    faces = np.asarray(faces, np.int64)
    corner_v = faces.reshape(-1)
    order = np.argsort(corner_v, kind='stable')                    # corners by vertex, then by corner index (= by face)
    vf_faces = (order // 3).astype(np.int32)
    vf_end = np.cumsum(np.bincount(corner_v, minlength=n_verts)).astype(np.int32)
    return vf_end, vf_faces


def _meshes():
    ico_v, ico_f = pt3d.ico_sphere(2)
    cube_v, cube_f = D.get_cube()
    g = torch.Generator().manual_seed(0)
    # a zero-area face (two equal corners, then three collinear ones) and a vertex no face uses
    deg_v = torch.cat([cube_v, torch.tensor([[0.3, 0.2, 0.1], [0.5, 0.5, 0.5], [1.0, 1.0, 1.0], [7., 7., 7.]])])
    n = len(cube_v)
    deg_f = torch.cat([cube_f, torch.tensor([[0, 0, 1], [n + 1, n + 2, 0]])])
    noisy_v = ico_v * (1 + 0.2 * torch.rand(len(ico_v), 1, generator=g))
    return {'icosphere': (ico_v, ico_f), 'cube': (cube_v, cube_f), 'degenerate': (deg_v, deg_f), 'noisy_icosphere': (noisy_v, ico_f)}


@pytest.mark.parametrize('name', ['icosphere', 'cube', 'degenerate', 'noisy_icosphere'])
def test_vertex_normals_match_float64(hs, name):
    verts, faces = _meshes()[name]
    v32 = np.ascontiguousarray(verts.numpy(), np.float32)
    f32 = np.ascontiguousarray(faces.numpy(), np.int32)
    vf_end, vf_faces = vertex_face_list(f32, len(v32))
    out = np.empty_like(v32)
    hs.hs_vertex_normals(len(v32), _p(v32), _p(f32), _p(vf_end), _p(vf_faces), _p(out))
    ref = P.vertex_normals(torch.from_numpy(v32).double(), faces.long()).numpy()
    assert np.abs(out - ref).max() < 1e-6
    lengths = np.linalg.norm(out, axis=1)
    used = np.bincount(f32.reshape(-1), minlength=len(v32)) > 0
    if name == 'degenerate':
        assert not used[-1] and np.all(out[-1] == 0)                # a vertex without faces keeps a zero normal
    assert np.allclose(lengths[used], 1, atol=1e-6)
    if name in ('icosphere', 'cube'):                               # closed convex meshes centred at 0: normals point outwards
        assert np.all((out * v32).sum(1) > 0)


def test_vertex_face_list_definition():
    faces = np.array([[0, 1, 2], [2, 1, 3], [3, 3, 0]], np.int32)
    vf_end, vf_faces = vertex_face_list(faces, 5)
    assert vf_end.tolist() == [2, 4, 6, 9, 9]
    assert vf_faces.tolist() == [0, 2, 0, 1, 0, 1, 1, 2, 2]


def _shading(name, **kw):
    lights = {'name': name}
    lights.update({k: v for k, v in kw.items() if k != 'materials'})
    return lights, kw.get('materials')


def _phong_ref(lights, materials, texel, normal, point, R, T):
    """(ka La + kd diffuse) * texel + ks specular of single fragments, in float64 through oracle/phong.py"""
    name, L, M, shininess = P.light_terms(lights, materials)
    t, n, p = (torch.from_numpy(x).double() for x in (texel, normal, point))
    R, T = torch.from_numpy(R).double(), torch.from_numpy(T).double()
    ambient = M['ambient_color'] * L['ambient_color']
    if name == 'ambient':
        return (ambient * t).numpy()
    cam = -(T[None] @ R.t())[0]
    direction = L['direction'][None] @ R.t() if name == 'directional' else L['location'] - p
    d = P.diffuse(n, L['diffuse_color'], direction)
    s = P.specular(p, n, direction, L['specular_color'], cam, shininess)
    return ((ambient + M['diffuse_color'] * d) * t + M['specular_color'] * s).numpy()


LIGHT_CASES = [
    ('ambient', {}),
    ('ambient', {'ambient_color': [[0.3, 0.6, 0.9]]}),
    ('directional', {}),
    ('directional', {'direction': [[1, 0.25, -1]], 'ambient_color': [[0.7] * 3], 'diffuse_color': [[0.4] * 3],
                     'specular_color': [[0.] * 3]}),
    ('directional', {'direction': [[0.2, -1, 0.4]], 'specular_color': [[0.5, 0.2, 0.9]], 'materials': {'shininess': 5}}),
    ('directional', {'materials': {'shininess': 0}}),                 # alpha = 0 under the power: pow(0, 0) = 1
    ('point', {}),
    ('point', {'location': [[0.5, 2.0, -1.5]], 'diffuse_color': [[0.9, 0.1, 0.4]],
               'materials': {'shininess': 12.5, 'ambient_color': [[0.2, 0.3, 0.4]], 'diffuse_color': [[0.8, 0.7, 0.6]],
                             'specular_color': [[0.5, 1.0, 0.25]]}}),
    ('point', {'materials': {'shininess': 0}}),
]


@pytest.mark.parametrize('case', LIGHT_CASES, ids=[f'{c[0]}-{i}' for i, c in enumerate(LIGHT_CASES)])
def test_phong_lighting_matches_float64(hs, case):
    name, kw = case
    lights, materials = _shading(name, **kw)
    g = np.random.default_rng(1)
    n = 4096
    texel = g.random((n, 3), dtype=np.float32)
    normal = g.standard_normal((n, 3)).astype(np.float32) * np.float32(0.8)          # interpolated normals are not unit
    point = (g.random((n, 3), dtype=np.float32) - np.float32(0.5)) * np.float32(2)
    R = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(2)))[0]
    R = (R * torch.linalg.det(R)).numpy().astype(np.float32)
    T = np.array([0.1, -0.2, 2.7], np.float32)
    # a quarter of the normals face away from the light (no diffuse, no specular), some point straight at it
    sh = phong_shading(lights, materials)
    out = np.empty_like(texel)
    hs.hs_phong(ctypes.byref(sh), n, _p(texel), _p(normal), _p(point), _p(np.ascontiguousarray(R)), _p(T), _p(out))
    ref = _phong_ref(lights, materials, texel, normal, point, R, T)
    assert np.abs(out - ref).max() < 2e-5, np.abs(out - ref).max()
    if name != 'ambient':
        _, L, _, _ = P.light_terms(lights, materials)
        l = (L['direction'][None] @ torch.from_numpy(R).double().t()).numpy() if name == 'directional' else L['location'].numpy() - point
        back = (normal * l).sum(-1) <= 0
        assert back.mean() > 0.2
        t = texel[back]
        M = P.light_terms(lights, materials)[2]
        amb = (M['ambient_color'] * L['ambient_color']).numpy()
        if float(dict(materials or {}).get('shininess', 64)) != 0:     # back-facing: ambient only
            assert np.allclose(out[back], amb * t, atol=1e-6)
        else:                                                           # ... plus pow(0, 0) * specular
            assert np.allclose(out[back], amb * t + (M['specular_color'] * L['specular_color']).numpy(), atol=1e-6)


def test_light_defaults_follow_pytorch3d():
    sh = phong_shading({'name': 'directional'})
    assert sh.light == 1 and list(sh.ambient_color) == pytest.approx([0.5] * 3) and list(sh.diffuse_color) == pytest.approx([0.3] * 3)
    assert list(sh.specular_color) == pytest.approx([0.2] * 3) and list(sh.direction) == [0., 1., 0.]
    assert list(sh.ka) == list(sh.kd) == list(sh.ks) == [1., 1., 1.] and sh.shininess == 64
    amb = phong_shading({})
    assert amb.light == 0 and list(amb.ambient_color) == [1., 1., 1.] and list(amb.diffuse_color) == list(amb.specular_color) == [0.] * 3
    pt = phong_shading({'name': 'point', 'location': ((1., 2., 3.),)})
    assert pt.light == 2 and list(pt.direction) == [1., 2., 3.]
    with pytest.raises(NotImplementedError):
        phong_shading({'name': 'spot'})


# ------------------------------------------------------------------ C-ABI
def test_phong_struct_layout_matches_the_c_compiler(tmp_path, hs):
    from dbw_b200 import _lib
    gcc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else shutil.which('gcc')
    if gcc is None:
        pytest.skip('no C compiler')
    cls = _lib.DbwPhongShading
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "dbw_render.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(DbwPhongShading));']
    lines += [f'  printf("{f} %zu\\n", offsetof(DbwPhongShading, {f}));' for f, _ in cls._fields_]
    lines += ['  printf("codes %d %d %d\\n", DBW_LIGHT_AMBIENT, DBW_LIGHT_DIRECTIONAL, DBW_LIGHT_POINT);', '  return 0;', '}']
    (tmp_path / 'l.c').write_text('\n'.join(lines))
    subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'l.c'), '-o',
                    str(tmp_path / 'l')], check=True)
    got = dict(l.split(' ', 1) for l in subprocess.run([str(tmp_path / 'l')], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got['size']) == ctypes.sizeof(cls) == hs.hs_sizeof_shading() == 4 + 21 * 4 + 4
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    assert [int(x) for x in got['codes'].split()] == [_lib.LIGHTS[k] for k in ('ambient', 'directional', 'point')]


def test_phong_entry_points_refuse_bad_arguments_without_a_gpu():
    from dbw_b200 import _lib
    from dbw_b200.renderer import make_settings
    L = _lib.lib()
    assert {'dbw_vertex_face_list', 'dbw_vertex_normals', 'dbw_render_forward_phong'} <= set(_lib.EXPORTS)

    def settings(K=1, sigma=0.0, H=64):
        return make_settings(2, H, 48, K, 10, 8, 1, 0, (1., 1., 0., 0.), sigma, 0.0, None, (0., 0., 0.), n_map_floats=48)
    sh = phong_shading({'name': 'directional'})
    p = ctypes.c_void_p(16)

    def call(s, factor, shading=sh, out=p, bkg=None, rgb8=None, world=p):
        return L.dbw_render_forward_phong(ctypes.byref(s), *([p] * 9), world, p, ctypes.byref(shading) if shading is not None else None,
                                          factor, bkg, 1, out, rgb8, p, 1 << 20, None)
    for s, factor, kw, why in [(settings(K=2), 1, {}, 'hard'), (settings(sigma=1e-4), 4, {}, 'hard'), (settings(), 2, {}, 'factor'),
                               (settings(H=62), 4, {}, 'multiples'), (settings(), 1, {'bkg': p}, 'factor 4'),
                               (settings(), 1, {'out': None}, 'out_rgba'), (settings(), 4, {'out': None}, 'both NULL'),
                               (settings(), 1, {'shading': None}, 'shading'), (settings(), 1, {'world': None}, 'verts_world')]:
        assert call(s, factor, **kw) != 0 and why in L.dbw_last_error().decode(), why
    bad = phong_shading({})
    bad.light = 7
    assert call(settings(), 1, shading=bad) != 0 and 'light type' in L.dbw_last_error().decode()
    s = settings()
    s.save_fragment_state = 1
    assert call(s, 1) != 0 and 'save_fragment_state' in L.dbw_last_error().decode()
    assert L.dbw_vertex_face_list(None, 4, 0, None, None, None) != 0 and 'n_verts' in L.dbw_last_error().decode()
    assert L.dbw_vertex_face_list(None, 4, 3, None, None, None) != 0 and 'null' in L.dbw_last_error().decode()
    assert L.dbw_vertex_normals(None, None, 3, None, None, None, None) != 0 and 'null' in L.dbw_last_error().decode()


# ------------------------------------------------------------------ Renderer and views
def test_soft_phong_is_refused_before_any_render():
    for kw in ({'sigma': 1e-4, 'faces_per_pixel': 1}, {'sigma': 0, 'faces_per_pixel': 10}):
        r = Renderer(16, shading_type='phong', lights={'name': 'directional'}, **kw)
        with pytest.raises(NotImplementedError, match='soft phong'):
            r(None, torch.eye(3)[None], torch.zeros(1, 3))


class _Mesh:
    textures = None

    def get_mesh_verts_faces(self, i):
        raise AssertionError('the setup does not read the mesh')

    def to(self, device):
        return self


def test_eye_light_setup_of_the_rotated_views():
    base = {'faces_per_pixel': 10, 'z_clip': 0.001, 'cameras': {'name': 'perspective'}, 'background_color': (1, 1, 1)}
    _, rend, R, T, _ = V._rotated_setup(_Mesh(), 5, 30, 2.5, None, None, None, None, dict(base), True, 'cpu')
    kw = rend.init_kwargs
    assert kw['lights'] == V.EYE_LIGHT_ROTATED and kw['shading_type'] == 'phong' and kw['faces_per_pixel'] == 1
    assert V.EYE_LIGHT_ROTATED == {'name': 'directional', 'direction': [[0, 0, -1]], 'ambient_color': [[0.6, 0.6, 0.6]],
                                   'diffuse_color': [[0.4, 0.4, 0.4]], 'specular_color': [[0., 0., 0.]]}
    assert {k: kw[k] for k in ('z_clip', 'cameras', 'background_color')} == {k: base[k] for k in ('z_clip', 'cameras', 'background_color')}
    assert rend.img_size == (256, 256) and R.shape == (5, 3, 3)
    _, plain, *_ = V._rotated_setup(_Mesh(), 5, 30, 2.5, None, None, None, None, dict(base), False, 'cpu')
    assert plain.shading_type == 'raw' and plain.faces_per_pixel == 10
    # a lit renderer is kept as it is
    lit = Renderer((24, 32), shading_type='flat', lights={'name': 'directional'}, sigma=0, faces_per_pixel=1)
    _, kept, *_ = V._rotated_setup(_Mesh(), 5, 30, 2.5, None, None, None, lit, None, True, 'cpu')
    assert kept.shading_type == 'flat' and kept.light_kwargs == {'name': 'directional'} and kept.img_size == (24, 32)


def test_eye_light_setup_of_the_trajectory_views():
    rend = Renderer((20, 28), faces_per_pixel=7)
    _, out, _ = V._views_setup(_Mesh(), None, rend, None, True, 'cpu', None)
    kw = out.init_kwargs
    assert kw['lights'] == V.EYE_LIGHT_VIEWS and kw['shading_type'] == 'phong' and kw['faces_per_pixel'] == 1
    assert V.EYE_LIGHT_VIEWS == {'name': 'directional', 'direction': [[1, 0.25, -1]], 'ambient_color': [[0.7, 0.7, 0.7]],
                                 'diffuse_color': [[0.4, 0.4, 0.4]], 'specular_color': [[0., 0., 0.]]}
    assert out.img_size == (20, 28)
    _, same, _ = V._views_setup(_Mesh(), None, rend, None, False, 'cpu', None)
    assert same is rend
    _, default, _ = V._views_setup(_Mesh(), None, None, None, True, 'cpu', None)
    assert default.img_size == (256, 256) and default.shading_type == 'phong'


def test_rotated_views_refuse_eye_light_with_a_given_R():
    with pytest.raises(NotImplementedError, match='given R'):
        V.render_rotated_views(_Mesh(), eye_light=True, R=torch.eye(3))
    with pytest.raises(NotImplementedError, match='given R'):
        V.save_mesh_as_video(_Mesh(), 'unused.mp4', eye_light=True, R=torch.eye(3))
    # without eye_light, a given R is the reference's rotation of the turntable
    _, _, R, _, _ = V._rotated_setup(_Mesh(), 4, 30, 2.5, torch.eye(3), None, None, None, None, False, 'cpu')
    assert R.shape == (4, 3, 3)


@pytest.mark.parametrize('eye_light', [False, True])
def test_view_helpers_refuse_what_is_not_a_mesh(eye_light):
    """checked before a renderer or a device is set up: no CUDA device is needed to get the refusal"""
    R, T = torch.eye(3)[None], torch.zeros(1, 3)
    calls = [lambda m: V.render_views(m, R, T, eye_light=eye_light), lambda m: V.render_rotated_views(m, eye_light=eye_light),
             lambda m: V.save_trajectory_as_video(m, 'unused.mp4', R, T, eye_light=eye_light),
             lambda m: V.save_mesh_as_video(m, 'unused.mp4', eye_light=eye_light)]
    for call in calls:
        for bad in (None, torch.zeros(4, 3)):
            with pytest.raises(NotImplementedError, match='is not implemented'):
                call(bad)
