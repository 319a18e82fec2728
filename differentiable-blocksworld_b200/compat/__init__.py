"""Import shims that let the reference's UNMODIFIED `src/trainer.py`, `src/optimizer.py`, `src/scheduler.py` and
`src/utils/*` load on a machine without PyTorch3D / toolz / lpips / seaborn / matplotlib / imageio / trimesh / open3d /
iopath (SURVEY.md 8b "Caveat", 8f rank 3).

    import dbw_b200.compat as compat
    compat.install()                                   # registers stand-ins ONLY for modules that are not importable
    sys.path.insert(0, '/path/to/reference/src')
    import model, dbw_b200.dbw as b200
    model.create_model = b200.create_model             # INTEGRATION.md A; then `import trainer`

What is real: `toolz`'s five dict helpers, the PyTorch3D containers / constructors the model surface hands to the trainer
(`Meshes`, `TexturesUV`, `join_meshes_as_*`, `ico_sphere`, `SubdivideMeshes`, the 6D-rotation transforms -- all this repo's
own implementations), the point-cloud ops of the reference's 3-D evaluation (`knn_points` / `knn_gather` on the sm_90a
k-NN kernels, the chamfer helpers and `chamfer_distance`, `sample_points_from_meshes`: dbw_b200/pointcloud.py), the
look-at cameras `look_at_view_transform` / `look_at_rotation` (dbw_b200/views.py), the two `seaborn` / `matplotlib.colors`
calls behind the block colour map (`utils/plot.py:77-87`).
`load_ply` for point clouds (dtu_eval's PLY reader: the reference's DTUDataset reads its ground truth through it).
Everything else the reference imports at module load but only calls on its export / evaluation paths (PLY writing, OBJ I/O, the
SVD ICP, `Pointclouds`, Open3D, video writing, plotting, LPIPS weights) is a named placeholder that raises
`NotImplementedError` when CALLED: the control plane stays out of scope (SURVEY 8), the import graph is satisfied."""
import colorsys
import importlib
import importlib.util
import sys
import types

import numpy as np
import torch
from torch import nn

from .. import geometry as G
from .. import pointcloud as PC
from .. import views as V
from ..structures import Meshes, TexturesUV, join_meshes_as_batch, join_meshes_as_scene


def _placeholder(qualname):
    """a callable / base class that exists by name and fails loudly when used"""
    class _Missing(nn.Module):
        def __init__(self, *a, **k):
            raise NotImplementedError(f'{qualname} is a placeholder of dbw_b200.compat: this dependency of the reference is not '
                                      f'installed and its call sites (export / evaluation paths) are outside the render hot path')
    _Missing.__name__ = _Missing.__qualname__ = qualname.rsplit('.', 1)[-1]
    return _Missing


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__dict__['__dbw_compat__'] = True
    if '.' in name:                                   # make `import a.b.c` and `a.b.c` attribute access both work
        parent, leaf = name.rsplit('.', 1)
        setattr(_ensure(parent), leaf, m)
    sys.modules[name] = m
    return m


def _ensure(name):
    if name in sys.modules:
        return sys.modules[name]
    return _module(name)


def _importable(name):
    if name in sys.modules:
        return not getattr(sys.modules[name], '__dbw_compat__', False)
    try:
        return importlib.util.find_spec(name) is not None
    except (ImportError, ValueError):
        return False


# ------------------------------------------------------------------ toolz (real)
def _toolz():
    def merge(*dicts):
        if len(dicts) == 1 and not isinstance(dicts[0], dict):
            dicts = dicts[0]
        out = {}
        for d in dicts:
            out.update(d)
        return out
    _module('toolz', merge=merge,
            valmap=lambda f, d: {k: f(v) for k, v in d.items()}, keymap=lambda f, d: {f(k): v for k, v in d.items()},
            valfilter=lambda f, d: {k: v for k, v in d.items() if f(v)}, keyfilter=lambda f, d: {k: v for k, v in d.items() if f(k)})


# ------------------------------------------------------------------ pytorch3d (containers real, the rest placeholders)
class SubdivideMeshes(nn.Module):
    """pytorch3d.ops.SubdivideMeshes on this repo's Meshes: 1 -> 4 split of every face (geometry.subdivide_mesh)"""

    def forward(self, meshes, feats=None):
        out = [G.subdivide_mesh(*meshes.get_mesh_verts_faces(i)) for i in range(len(meshes))]
        return Meshes([v for v, _ in out], [f for _, f in out])


def _ico_sphere(level=0, device=None):
    v, f = G.ico_sphere(level)
    m = Meshes(v[None], f[None])
    return m.to(device) if device is not None else m


def _load_ply(f, *, path_manager=None):
    """pytorch3d.io.load_ply for point clouds (the reference's DTU ground truth, dtu.py:47): (verts (V, 3) float32, faces (0, 3)
    int64), on dtu_eval's PLY reader.  A file with faces is refused rather than returned without them."""
    from ..dtu_eval import read_ply
    with open(f, 'rb') as fh:
        head = fh.read(1 << 16).split(b'end_header')[0].decode('ascii', 'replace').split('\n')
    if any(l.split()[:2] == ['element', 'face'] and int(l.split()[2]) > 0 for l in head if len(l.split()) >= 3):
        raise NotImplementedError(f'dbw_b200.compat load_ply reads point clouds; {f} has faces')
    return torch.from_numpy(read_ply(f)).float(), torch.zeros(0, 3, dtype=torch.int64)


def _pytorch3d():
    P = lambda n: _placeholder(f'pytorch3d.{n}')
    _module('pytorch3d', __version__='0.7.1+dbw_b200.compat')
    _module('pytorch3d.structures', Meshes=Meshes, Pointclouds=P('structures.Pointclouds'),
            join_meshes_as_scene=join_meshes_as_scene, join_meshes_as_batch=join_meshes_as_batch)
    _module('pytorch3d.structures.meshes', Meshes=Meshes, join_meshes_as_scene=join_meshes_as_scene,
            join_meshes_as_batch=join_meshes_as_batch)
    _module('pytorch3d.structures.utils', packed_to_list=lambda x, split: list(x.split(split, dim=0)))
    _module('pytorch3d.utils', ico_sphere=_ico_sphere)
    _module('pytorch3d.transforms', rotation_6d_to_matrix=G.rotation_6d_to_matrix, matrix_to_rotation_6d=G.matrix_to_rotation_6d,
            random_rotations=lambda n, dtype=None, device=None: G.random_rotations(n).to(device=device, dtype=dtype or torch.float32))
    _module('pytorch3d.ops', SubdivideMeshes=SubdivideMeshes, sample_points_from_meshes=PC.sample_points_from_meshes,
            iterative_closest_point=P('ops.iterative_closest_point'), knn_points=PC.knn_points, knn_gather=PC.knn_gather)
    _module('pytorch3d.ops.subdivide_meshes', SubdivideMeshes=SubdivideMeshes)
    _module('pytorch3d.ops.knn', knn_points=PC.knn_points, knn_gather=PC.knn_gather)
    _module('pytorch3d.io', save_ply=P('io.save_ply'), load_ply=_load_ply, save_obj=P('io.save_obj'),
            load_obj=P('io.load_obj'), load_objs_as_meshes=P('io.load_objs_as_meshes'))
    _module('pytorch3d.io.utils', _open_file=P('io.utils._open_file'))
    _module('pytorch3d.loss', mesh_normal_consistency=P('loss.mesh_normal_consistency'), chamfer_distance=PC.chamfer_distance)
    _module('pytorch3d.loss.chamfer', chamfer_distance=PC.chamfer_distance,
            _validate_chamfer_reduction_inputs=PC._validate_chamfer_reduction_inputs,
            _handle_pointcloud_input=PC._handle_pointcloud_input)
    names = ['FoVPerspectiveCameras', 'PerspectiveCameras', 'RasterizationSettings', 'MeshRenderer', 'MeshRasterizer', 'BlendParams',
             'DirectionalLights', 'PointLights', 'AmbientLights', 'TexturesVertex',
             'SoftPhongShader', 'HardPhongShader', 'SoftSilhouetteShader', 'Materials']
    _module('pytorch3d.renderer', TexturesUV=TexturesUV, look_at_view_transform=V.look_at_view_transform,
            look_at_rotation=V.look_at_rotation, **{n: P(f'renderer.{n}') for n in names})
    _module('pytorch3d.renderer.mesh')
    _module('pytorch3d.renderer.mesh.shader', SoftPhongShader=P('renderer.mesh.shader.SoftPhongShader'))
    _module('pytorch3d.renderer.mesh.shading', phong_shading=P('phong_shading'), flat_shading=P('flat_shading'),
            gouraud_shading=P('gouraud_shading'))
    _module('pytorch3d.renderer.cameras', _get_sfm_calibration_matrix=P('renderer.cameras._get_sfm_calibration_matrix'))


# ------------------------------------------------------------------ lpips (structure real, ImageNet weights absent)
class LPIPS(nn.Module):
    """Stand-in for lpips.LPIPS (lpips==0.1.4, environment.yml:29).  The learned perceptual metric needs VGG16 ImageNet weights
    and LPIPS' linear heads, neither of which is on this machine: constructing the network raises unless
    `dbw_b200.compat.LPIPS_FACTORY` has been set to a callable returning an nn.Module with the same
    `forward(in0, in1, normalize=False)` contract (tests install a small random-weight conv net)."""

    def __init__(self, net='vgg', **kwargs):
        super().__init__()
        if LPIPS_FACTORY is None:
            raise NotImplementedError('lpips is not installed (no VGG16 / LPIPS weights here): set dbw_b200.compat.LPIPS_FACTORY')
        self.net = LPIPS_FACTORY(net=net, **kwargs)
        for p in self.net.parameters():
            p.requires_grad_(False)

    def forward(self, in0, in1, normalize=False):
        return self.net(in0, in1, normalize=normalize)


LPIPS_FACTORY = None


# ------------------------------------------------------------------ seaborn / matplotlib.colors (the block colour map only)
def _hls_palette(n_colors=6, h=0.01, l=0.6, s=0.65):
    hues = (np.linspace(0, 1, int(n_colors) + 1)[:-1] + h) % 1
    return [colorsys.hls_to_rgb(float(hi), l, s) for hi in hues]


class _LinearSegmentedColormap:
    def __init__(self, anchors, N=256):
        anchors = np.asarray(anchors, dtype=np.float64)
        xs = np.linspace(0.0, 1.0, len(anchors))
        self.lut = np.stack([np.interp(np.linspace(0.0, 1.0, N), xs, anchors[:, c]) for c in range(3)], axis=1)
        self.N = N

    @classmethod
    def from_list(cls, name, colors, N=256):
        return cls(colors, N)

    def __call__(self, values):
        v = np.asarray(values, dtype=np.float64)
        idx = np.clip((v * self.N).astype(np.int64), 0, self.N - 1)
        idx = np.where(v == 1.0, self.N - 1, idx)
        return np.concatenate([self.lut[idx], np.ones(idx.shape + (1,))], axis=-1)


def _plotting():
    def color_palette(palette=None, n_colors=None, **k):
        if palette == 'hls':
            return _hls_palette(n_colors or 6)
        raise NotImplementedError(f'seaborn.color_palette({palette!r}) is not provided by dbw_b200.compat (plotting is out of scope)')
    if not _importable('seaborn'):
        _module('seaborn', color_palette=color_palette, axes_style=_placeholder('seaborn.axes_style'))
    if not _importable('matplotlib'):
        named = {'gold': (1.0, 215.0 / 255.0, 0.0)}
        _module('matplotlib')
        _module('matplotlib.colors', to_rgb=lambda c: named[c] if isinstance(c, str) else tuple(c)[:3],
                LinearSegmentedColormap=_LinearSegmentedColormap)
        _module('matplotlib.pyplot', subplots=_placeholder('matplotlib.pyplot.subplots'), figure=_placeholder('matplotlib.pyplot.figure'))


def install(verbose=False):
    """Register the stand-ins for every module of the list that cannot be imported here.  Idempotent; a real installation
    of a package always wins.  Returns the names that were shimmed."""
    done = []
    table = [('toolz', _toolz), ('pytorch3d', _pytorch3d),
             ('lpips', lambda: _module('lpips', LPIPS=LPIPS)),
             ('imageio', lambda: _module('imageio', mimsave=_placeholder('imageio.mimsave'), imread=_placeholder('imageio.imread'),
                                         get_writer=_placeholder('imageio.get_writer'))),
             ('iopath', lambda: (_module('iopath'), _module('iopath.common'),
                                 _module('iopath.common.file_io', PathManager=_placeholder('iopath.common.file_io.PathManager')))),
             ('trimesh', lambda: (_module('trimesh', Trimesh=_placeholder('trimesh.Trimesh'), load=_placeholder('trimesh.load')),
                                  _module('trimesh.voxel'),
                                  _module('trimesh.voxel.creation', voxelize=_placeholder('trimesh.voxel.creation.voxelize')))),
             ('open3d', lambda: _module('open3d'))]
    for name, make in table:
        if not _importable(name):
            make()
            done.append(name)
    _plotting()
    done += [n for n in ('seaborn', 'matplotlib') if getattr(sys.modules.get(n), '__dbw_compat__', False)]
    try:                                              # utils/image.py:22 uses the constant Pillow 10 removed
        from PIL import Image
        if not hasattr(Image, 'ANTIALIAS'):
            Image.ANTIALIAS = Image.LANCZOS
    except ImportError:
        pass
    if verbose:
        print(f'[dbw_b200.compat] stand-ins installed for: {", ".join(done) or "nothing"}')
    return done
