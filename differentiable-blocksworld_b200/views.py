"""The reference's rotating-view and trajectory renders and their writers (src/model/renderer.py:290-414,
src/utils/image.py:61-115), with PyTorch3D's look-at cameras.

Every frame is VizMeshRenderer's (hard render at 4H x 4W, box-filtered 4x4), made by `Renderer.render_viz`: the resolving
kernel never writes the 16x sample image, so a chunk of frames costs its H x W outputs plus the scene's face records.
With eye_light=True an unlit renderer is swapped for a Phong-shaded one lit from the camera, as in the reference.
Chunks are sized by a byte budget (CHUNK_BYTES, or `chunk_bytes=`) instead of the reference's fixed 10 frames; the frames
do not depend on the chunk size.  Videos are written with OpenCV (`mp4v`, RGB -> BGR), GIFs with PIL."""
import math
from copy import deepcopy
from pathlib import Path

import numpy as np
import torch
from torch.nn import functional as F

from .renderer import Renderer

VIZ_IMG_SIZE = 256              # renderer.py:19
DIRECTION_LIGHT = [1, 0.25, -1]
MAX_GIF_SIZE = 256              # src/utils/image.py:19
CHUNK_BYTES = 1 << 30           # device bytes one chunk of frames may take


# ------------------------------------------------------------------ cameras (PyTorch3D conventions: X_cam = X_world @ R + T)
def _broadcast(*args, device='cpu'):
    """PyTorch3D's convert_to_tensors_and_broadcast: float32 tensors with a leading batch dimension, expanded to the largest"""
    ts = []
    for a in args:
        t = a.to(device=device, dtype=torch.float32) if torch.is_tensor(a) else torch.tensor(a, dtype=torch.float32, device=device)
        ts.append(t.view(1) if t.dim() == 0 else t)
    N = max(t.shape[0] for t in ts)
    for t in ts:
        if t.shape[0] not in (1, N):
            raise ValueError(f'Got non-broadcastable sizes {[t.shape[0] for t in ts]}')
    return [t.expand(N, *t.shape[1:]) for t in ts]


def look_at_rotation(camera_position, at=((0, 0, 0),), up=((0, 1, 0),), device='cpu'):
    """(N,3,3) rotations of cameras at camera_position looking at `at`, with `up` mapped to +y: the camera's +z axis points to
    `at` and its +x axis to the left of the image (columns of R are the camera axes in world coordinates)"""
    camera_position, at, up = _broadcast(camera_position, at, up, device=device)
    for t, n in zip((camera_position, at, up), ('camera_position', 'at', 'up')):
        if t.shape[-1] != 3:
            raise ValueError(f'Expected arg {n} to have shape (N, 3); got {tuple(t.shape)}')
    z_axis = F.normalize(at - camera_position, eps=1e-5)
    x_axis = F.normalize(torch.cross(up, z_axis, dim=1), eps=1e-5)
    y_axis = F.normalize(torch.cross(z_axis, x_axis, dim=1), eps=1e-5)
    is_close = torch.isclose(x_axis, torch.tensor(0.0, device=x_axis.device), atol=5e-3).all(dim=1, keepdim=True)
    if is_close.any():            # `up` parallel to the viewing direction
        x_axis = torch.where(is_close, F.normalize(torch.cross(y_axis, z_axis, dim=1), eps=1e-5), x_axis)
    return torch.cat((x_axis[:, None], y_axis[:, None], z_axis[:, None]), dim=1).transpose(1, 2)


def camera_position_from_spherical_angles(distance, elevation, azimuth, degrees=True, device='cpu'):
    """d (cos e sin a, sin e, cos e cos a): azimuth about +y from +z, elevation towards +y"""
    dist, elev, azim = _broadcast(distance, elevation, azimuth, device=device)
    if degrees:
        elev, azim = math.pi / 180.0 * elev, math.pi / 180.0 * azim
    return torch.stack([dist * torch.cos(elev) * torch.sin(azim), dist * torch.sin(elev),
                        dist * torch.cos(elev) * torch.cos(azim)], dim=1).view(-1, 3)


def look_at_view_transform(dist=1.0, elev=0.0, azim=0.0, degrees=True, eye=None, at=((0, 0, 0),), up=((0, 1, 0),), device='cpu'):
    """(R (N,3,3), T (N,3)) of cameras at spherical position (dist, elev, azim) around `at` -- or at `eye` -- looking at `at`,
    all arguments broadcast over N"""
    if eye is not None:
        eye, at, up = _broadcast(eye, at, up, device=device)
        C = eye
    else:
        dist, elev, azim, at, up = _broadcast(dist, elev, azim, at, up, device=device)
        C = camera_position_from_spherical_angles(dist, elev, azim, degrees=degrees, device=device) + at
    R = look_at_rotation(C, at, up, device=device)
    T = -torch.bmm(R.transpose(1, 2), C[:, :, None])[:, :, 0]
    return R, T


def get_circle_traj(dist=1, a_scale=15, e_scale=15, N_views=50):
    """N_views cameras on a small loop around the view direction -z (renderer.py:411-414): azimuth -180 + a_scale cos t,
    elevation e_scale sin t"""
    azim = torch.cos(torch.linspace(0, 2, N_views + 1) * np.pi)[:-1] * a_scale - 180
    elev = torch.sin(torch.linspace(0, 2, N_views + 1) * np.pi)[:-1] * e_scale
    return look_at_view_transform(dist, azim=azim, elev=elev)


# ------------------------------------------------------------------ frames
# the lights of the eye_light renders (renderer.py:303-305 and :345-348): a directional light fixed to the camera, no specular
EYE_LIGHT_ROTATED = {'name': 'directional', 'direction': [[0, 0, -1]], 'ambient_color': [[0.6, 0.6, 0.6]],
                     'diffuse_color': [[0.4, 0.4, 0.4]], 'specular_color': [[0., 0., 0.]]}
EYE_LIGHT_VIEWS = {'name': 'directional', 'direction': [DIRECTION_LIGHT], 'ambient_color': [[0.7, 0.7, 0.7]],
                   'diffuse_color': [[0.4, 0.4, 0.4]], 'specular_color': [[0., 0., 0.]]}


def _eye_light(renderer, img_size, lights):
    """the reference's eye_light swap: an unlit (ambient) renderer is replaced by a Phong-shaded, single-layer one with the
    given lights and its other settings; a lit renderer is kept"""
    if renderer.light_kwargs.get('name', 'ambient') != 'ambient':
        return renderer
    kwargs = renderer.init_kwargs
    kwargs['lights'] = deepcopy(lights)
    kwargs['shading_type'] = 'phong'
    kwargs['faces_per_pixel'] = 1
    return Renderer(img_size, **kwargs)


def _check_mesh(mesh, who):
    """the helpers render a Meshes (one joined scene): anything else is refused before a renderer or a device is set up --
    NotImplementedError, as for the other input structures dbw_b200 does not provide for (pointcloud.py)"""
    if not (hasattr(mesh, 'get_mesh_verts_faces') and hasattr(mesh, 'textures')):
        raise NotImplementedError(f'{who}: rendering a {type(mesh).__name__} is not implemented (pass a Meshes with TexturesUV)')


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError('rendering views needs a CUDA device (there is no CPU fallback)')
    return torch.device('cuda:0')


def _fit_bkg(bkg, img_size):
    """bkg (3,H',W') bilinearly resized to the frames' (H, W) when it differs (renderer.py:318-320)"""
    if bkg is not None and tuple(bkg.shape[-2:]) != tuple(img_size):
        bkg = F.interpolate(bkg.reshape(-1, *bkg.shape[-3:])[:1], size=tuple(img_size), mode='bilinear', align_corners=False)[0]
    return bkg


def _chunks(renderer, mesh, n, chunk_bytes):
    """[start, stop) ranges of at most as many frames as chunk_bytes of device memory hold (at least one)"""
    per = max(1, (chunk_bytes or CHUNK_BYTES) // renderer.viz_bytes(mesh, 1))
    return [(k, min(k + per, n)) for k in range(0, n, per)]


def _view_frames(mesh, R, T, renderer, bkg=None, K=None, with_edges=False, linewidth=1, edge_colors=None, clamp=False,
                 u8=False, chunk_bytes=None):
    """yields, per chunk of views, the device frames: (B,4,H,W) float RGBA -- RGB composited over bkg (3,H,W) when given,
    after the clamp to [0, 1] when `clamp` -- or, with u8, the (B,H,W,3) uint8 frames `save_video` would make of its RGB"""
    dev = mesh.device
    R, T = R.to(dev), T.to(dev)
    K = K.reshape(-1, 4, 4).to(dev) if K is not None else None
    for a, b in _chunks(renderer, mesh, len(R), chunk_bytes):
        Kc = K if K is None or len(K) == 1 else K[a:b]
        fast = u8 and not with_edges and not (clamp and bkg is not None)
        if fast:                 # composite and conversion inside the kernel
            yield renderer.render_viz(mesh, R[a:b], T[a:b], K=Kc, bkg=bkg, frames_u8=True)[1]
            continue
        res = renderer.render_viz(mesh, R[a:b], T[a:b], K=Kc)
        if with_edges:
            rgb, alpha = res.split([3, 1], dim=1)
            colors = edge_colors.repeat(b - a, 1) if torch.is_tensor(edge_colors) else edge_colors
            res = torch.cat([renderer.draw_edges(rgb, mesh, R=R[a:b], T=T[a:b], linewidth=linewidth, colors=colors, K=Kc), alpha], 1)
        if clamp:
            res = res.clamp(0, 1)
        if bkg is not None:
            rgb, alpha = res.split([3, 1], dim=1)
            res = torch.cat([rgb * alpha + (1 - alpha) * bkg.to(dev), alpha], dim=1)
        yield _to_u8(res[:, :3]) if u8 else res


def _to_u8(rgb):
    """(B,3,H,W) float -> (B,H,W,3) uint8 as save_video converts (src/utils/image.py:98)"""
    return (rgb * 255).permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8)


def _rotated_setup(mesh, n_views, elev, dist, R, T, bkg, renderer, rend_kwargs, eye_light, device):
    _check_mesh(mesh, 'render_rotated_views')
    if eye_light and R is not None:
        raise NotImplementedError('render_rotated_views: eye_light=True with a given R (as in the reference)')
    img_size = VIZ_IMG_SIZE if renderer is None else renderer.img_size
    device = _device() if device is None else device
    rend_kwargs = {} if rend_kwargs is None else rend_kwargs
    if renderer is not None:          # a fresh renderer with the given one's settings and camera (renderer.py:297-300)
        rend_kwargs = renderer.init_kwargs
        rend_kwargs.setdefault('cameras', {})['K'] = renderer.cameras.K
    renderer = Renderer(img_size, **rend_kwargs)
    if eye_light:
        renderer = _eye_light(renderer, img_size, EYE_LIGHT_ROTATED)
    renderer = renderer.to(device)
    elev, dist = 0 if R is not None else elev, 0 if T is not None else dist
    R = R.to(device) if R is not None else torch.eye(3, device=device)
    T = T.to(device) if T is not None else torch.zeros(3, device=device)
    azim = torch.linspace(-180, 180, n_views)
    R_view = look_at_view_transform(dist=1, elev=elev, azim=azim, device=device)[0]
    T_view = torch.tensor([[0., 0., dist]], device=device).expand(len(R_view), -1)
    return mesh.to(device), renderer, R_view @ R, T_view + T, _fit_bkg(bkg, renderer.img_size)


@torch.no_grad()
def render_rotated_views(mesh, n_views=50, elev=30, dist=2.5, R=None, T=None, bkg=None, renderer=None, rend_kwargs=None,
                         eye_light=False, device=None, chunk_bytes=None):
    """(n_views,3,H,W) CPU frames of the mesh turning around +y, clamped to [0, 1] and composited over bkg (renderer.py:290-327)"""
    mesh, renderer, R, T, bkg = _rotated_setup(mesh, n_views, elev, dist, R, T, bkg, renderer, rend_kwargs, eye_light, device)
    return torch.cat([f[:, :3].cpu() for f in _view_frames(mesh, R, T, renderer, bkg, clamp=True, chunk_bytes=chunk_bytes)])


def _views_setup(mesh, img_size, renderer, rend_kwargs, eye_light, device, bkg):
    _check_mesh(mesh, 'render_views')
    device = _device() if device is None else device
    if renderer is None:
        renderer = Renderer(img_size or VIZ_IMG_SIZE, **({} if rend_kwargs is None else rend_kwargs))
    if eye_light:
        renderer = _eye_light(renderer, renderer.img_size, EYE_LIGHT_VIEWS)
    mesh, renderer = mesh.to(device), renderer.to(device)
    return mesh, renderer, _fit_bkg(bkg, renderer.img_size)


@torch.no_grad()
def render_views(mesh, R, T, img_size=None, bkg=None, renderer=None, rend_kwargs=None, with_edges=False, linewidth=1,
                 edge_colors=None, eye_light=False, with_alpha=False, device=None, K=None, chunk_bytes=None):
    """(N,3,H,W) CPU frames of the mesh seen from R (N,3,3), T (N,3) (renderer.py:330-380): with_edges draws the face edges
    (Renderer.draw_edges, edge_colors one colour or one per face); bkg (3,H,W) is composited under them; with_alpha returns
    (N,4,H,W) RGBA before any composite.  K: (1,4,4) or (N,4,4) per-view intrinsics."""
    mesh, renderer, bkg = _views_setup(mesh, img_size, renderer, rend_kwargs, eye_light, device, bkg)
    frames = _view_frames(mesh, R, T, renderer, None if with_alpha else bkg, K=K, with_edges=with_edges, linewidth=linewidth,
                          edge_colors=edge_colors, chunk_bytes=chunk_bytes)
    out = torch.cat([f.cpu() for f in frames])
    return out if with_alpha else out[:, :3]


# ------------------------------------------------------------------ writers
def _frames_u8(imgs_or_path, in_ext='jpg'):
    """(N,H,W,3) uint8 array of a (N,3,H,W) float tensor, a list of images, or a directory of numbered `in_ext` files"""
    from PIL import Image
    if isinstance(imgs_or_path, (str, Path)):
        files = sorted(Path(imgs_or_path).glob(f'*.{in_ext}'), key=lambda p: int(p.stem))
        return np.stack([np.asarray(Image.open(f).convert('RGB')) for f in files])
    if torch.is_tensor(imgs_or_path):
        return _to_u8(imgs_or_path.detach().float()).cpu().numpy()
    return np.stack([np.asarray(_to_pil(i)) for i in imgs_or_path])


def _to_pil(arr):
    """src/utils/image.py:convert_to_img for a (3,H,W) / (1,3,H,W) tensor, an array or an image"""
    from PIL import Image
    if isinstance(arr, Image.Image):
        return arr
    if torch.is_tensor(arr):
        arr = (arr[0] if arr.dim() == 4 else arr).detach().cpu().permute(1, 2, 0).numpy()
    if np.issubdtype(arr.dtype, np.floating):
        arr = arr.clip(0, 1) * 255
    return Image.fromarray(arr.astype(np.uint8)).convert('RGB')


class VideoWriter:
    """mp4 (`mp4v`, RGB frames in, BGR to OpenCV).  MPEG-4 part 2 codes 4:2:0 chroma, so frames of odd height or width are
    padded by one edge row / column: the file is (H + H % 2) x (W + W % 2)."""

    def __init__(self, path, fps=24):
        import cv2
        self.cv2, self.path, self.fps, self.vw, self.count = cv2, str(path), fps, None, 0

    def write(self, frames):
        """frames: (N,H,W,3) uint8 RGB (array or tensor)"""
        frames = frames.cpu().numpy() if torch.is_tensor(frames) else np.asarray(frames)
        h, w = frames.shape[1:3]
        frames = np.pad(frames, ((0, 0), (0, h % 2), (0, w % 2), (0, 0)), mode='edge')
        if self.vw is None:
            self.vw = self.cv2.VideoWriter(self.path, self.cv2.VideoWriter_fourcc(*'mp4v'), self.fps, (frames.shape[2], frames.shape[1]))
            if not self.vw.isOpened():
                raise RuntimeError(f'OpenCV cannot open {self.path} for writing (mp4v)')
        for f in frames:
            self.vw.write(np.ascontiguousarray(f[..., ::-1]))
        self.count += len(frames)

    def close(self):
        if self.vw is not None:
            self.vw.release()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def save_video(imgs_or_path, name, in_ext='jpg', as_gif=False, fps=24, quality=10):
    """src/utils/image.py:90-115 through OpenCV: written next to the image directory when given one, else at `name`.
    `quality` (an imageio / ffmpeg setting) has no OpenCV counterpart and is ignored."""
    frames = _frames_u8(imgs_or_path, in_ext)
    out = (Path(imgs_or_path).parent if isinstance(imgs_or_path, (str, Path)) else Path('.')) / name
    with VideoWriter(out, fps) as vw:
        vw.write(frames)
    if as_gif:
        save_gif(list(frames), out.with_suffix('.gif'), size=None, total_sec=len(frames) / fps, autodecimate=False)


def save_gif(imgs_or_path, name, in_ext='jpg', size=MAX_GIF_SIZE, total_sec=10, autodecimate=True):
    """src/utils/image.py:61-87: adaptive-palette frames, at most ~250 kept, fitted inside size x size, total_sec in all"""
    from PIL import Image
    if isinstance(imgs_or_path, (str, Path)):
        path = Path(imgs_or_path)
        files = sorted(path.glob(f'*.{in_ext}'), key=lambda p: int(p.stem))
        imgs = [Image.open(f).convert('P', palette=Image.ADAPTIVE) for f in files]
    else:
        imgs, path = [_to_pil(i).convert('P', palette=Image.ADAPTIVE) for i in imgs_or_path], Path('.')
    if len(imgs) == 0:
        return
    if autodecimate:
        step = len(imgs) // 250
        if step > 1:
            imgs = imgs[::step]
    if size is not None:
        size = (size, size) if isinstance(size, int) else tuple(size)
        if size != imgs[0].size:
            ratio = float(min(s1 / s2 for s1, s2 in zip(size, imgs[0].size)))
            new = round(ratio * imgs[0].size[0]), round(ratio * imgs[0].size[1])
            imgs = [i.resize(new, resample=Image.LANCZOS) for i in imgs]
    tpf = int(total_sec * 1000 / len(imgs))
    imgs[0].save(path.parent / name, optimize=False, save_all=True, append_images=imgs[1:], duration=tpf, loop=0)


def save_mesh_as_gif(mesh, filename, n_views=50, elev=30, dist=2.732, R=None, T=None, bkg=None, renderer=None, rend_kwargs=None,
                     eye_light=False):
    save_gif(render_rotated_views(mesh, n_views, elev, dist, R=R, T=T, bkg=bkg, renderer=renderer, rend_kwargs=rend_kwargs,
                                  eye_light=eye_light), filename)


@torch.no_grad()
def save_mesh_as_video(mesh, filename, n_views=240, elev=30, dist=2.732, R=None, T=None, bkg=None, renderer=None,
                       rend_kwargs=None, eye_light=False, chunk_bytes=None):
    """render_rotated_views + save_video, streamed: each chunk's uint8 frames go to the encoder as they are made"""
    mesh, renderer, R, T, bkg = _rotated_setup(mesh, n_views, elev, dist, R, T, bkg, renderer, rend_kwargs, eye_light, None)
    with VideoWriter(filename) as vw:
        for f in _view_frames(mesh, R, T, renderer, bkg, clamp=True, u8=True, chunk_bytes=chunk_bytes):
            vw.write(f)


def save_trajectory_as_gif(mesh, filename, R, T, bkg=None, renderer=None, rend_kwargs=None, with_edges=False, linewidth=1,
                           edge_colors=None, eye_light=False):
    save_gif(render_views(mesh, R, T, bkg=bkg, renderer=renderer, rend_kwargs=rend_kwargs, with_edges=with_edges,
                          linewidth=linewidth, edge_colors=edge_colors, eye_light=eye_light), filename)


@torch.no_grad()
def save_trajectory_as_video(mesh, filename, R, T, bkg=None, renderer=None, rend_kwargs=None, with_edges=False, linewidth=1,
                             edge_colors=None, eye_light=False, K=None, chunk_bytes=None):
    """render_views + save_video, streamed chunk by chunk.  K: (1,4,4) or (N,4,4) per-view intrinsics"""
    mesh, renderer, bkg = _views_setup(mesh, None, renderer, rend_kwargs, eye_light, None, bkg)
    with VideoWriter(filename) as vw:
        for f in _view_frames(mesh, R, T, renderer, bkg, K=K, with_edges=with_edges, linewidth=linewidth,
                              edge_colors=edge_colors, u8=True, chunk_bytes=chunk_bytes):
            vw.write(f)
