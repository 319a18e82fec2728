"""Training views served from device memory: the reference's loaders (src/dataset/__init__.py:9-26, dtu.py:58-68, bmvs.py:49-59)
with no host work per step.

    views = DeviceViews.from_dataset(ds, device)       # decode and resize once
    loader = DeviceLoader(views, batch_size=4, shuffle=True)
    for inp, labels in loader: ...                      # the batches DataLoader(ds, 4, shuffle=True) gives, already on the device

DeviceViews.from_dataset has two paths.  The reference's DTU / BlendedMVS shape (`input_files`, `view_ids`, `KRT`, `img_size` and a
transform that is exactly Compose([Resize(img_size), ToTensor()])) is the fast one: each file is decoded once on the host with
PIL, as the reference decodes it, uploaded in chunks and resized on the device by dbw_resample_u8 (Pillow's bilinear resampler,
bit for bit); the views stay resident as uint8.  Any other map-style dataset yielding ({'imgs', 'K', 'R', 'T'}, labels) is read
through ds[i] once per item and kept as it came.  A batch is one dbw_gather_views launch: the images (x / 255, correctly rounded,
as ToTensor divides), K, R and T of B views picked by indices on the device.

DeviceLoader makes the global-RNG draws of torch's DataLoader (the iterator's base seed, then the RandomSampler's seed) and uses
torch's own samplers, so the batch order and the RNG state after every epoch are those of DataLoader(ds, batch_size, shuffle), or
of a DistributedSampler with rank and world_size.  labels['points'] is min(1e5, P) points of the ground-truth cloud per view,
a uniformly drawn subset without duplicates from a keyed permutation (dbw_subsample_points, keyed by the epoch's base seed, the
batch and the view).  It replaces the reference's per-item torch.randperm, whose stream it does not reproduce; no training
step reads it."""
import ctypes

import numpy as np
import torch
from torch.utils.data import BatchSampler, DistributedSampler, RandomSampler, SequentialSampler

from . import _lib
from ._lib import DbwError, check

N_POINTS = int(1e5)                    # the reference's labels['points'] size (dtu.py:66)
CAMERA_KEYS = ('K', 'R', 'T')


def _vp(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _words(t):
    """32-bit words per leading-dimension entry of a contiguous tensor of 4- or 8-byte elements"""
    if t.element_size() not in (4, 8):
        raise DbwError(f'device views: {t.dtype} tensors cannot be gathered (4- or 8-byte elements only)')
    return t[0].numel() * t.element_size() // 4


def _require_cuda(device):
    device = torch.device(device)
    if device.type != 'cuda':
        raise DbwError('device views live on a CUDA device (there is no CPU fallback)')
    return torch.device('cuda', torch.cuda.current_device() if device.index is None else device.index)


def resample_u8(src, size):
    """Pillow's Image.resize((w, h), BILINEAR) of (N, H, W, 3) uint8 CUDA images to size (h, w), bit for bit"""
    if src.dim() != 4 or src.shape[-1] != 3 or src.dtype != torch.uint8 or not src.is_cuda:
        raise DbwError(f'resample_u8: expected (N, H, W, 3) uint8 CUDA images, got {tuple(src.shape)} {src.dtype} on {src.device}')
    n, in_h, in_w, _ = src.shape
    out_h, out_w = (int(s) for s in size)
    src = src.contiguous()
    L = _lib.lib()
    nbytes = ctypes.c_size_t(0)
    check(L.dbw_resample_u8_workspace_bytes(n, in_h, in_w, out_h, out_w, ctypes.byref(nbytes)), 'dbw_resample_u8_workspace_bytes')
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=src.device)
    dst = torch.empty(n, out_h, out_w, 3, dtype=torch.uint8, device=src.device)
    check(L.dbw_resample_u8(n, in_h, in_w, _vp(src), out_h, out_w, _vp(dst), _vp(ws), ws.numel(), _stream(src.device)),
          'dbw_resample_u8')
    return dst


def is_reference_transform(ds):
    """ds.transform is exactly Compose([Resize(ds.img_size), ToTensor()]) with bilinear interpolation (dtu.py:70-72)"""
    from torchvision.transforms import Compose, InterpolationMode, Resize, ToTensor
    t = getattr(ds, 'transform', None)
    if type(t) is not Compose or len(t.transforms) != 2:
        return False
    r, tt = t.transforms
    size = getattr(ds, 'img_size', None)
    return (type(r) is Resize and type(tt) is ToTensor and isinstance(r.size, (list, tuple)) and size is not None
            and [int(s) for s in r.size] == [int(s) for s in size] and len(size) == 2
            and r.interpolation == InterpolationMode.BILINEAR and r.max_size is None)


def _has_fast_path(ds):
    return all(hasattr(ds, a) for a in ('input_files', 'view_ids', 'KRT', 'img_size')) and is_reference_transform(ds)


class DeviceViews:
    """A split's views resident on one CUDA device, in the item order of the dataset they were read from.  `name`, `tag`,
    `img_size`, `pc_gt` and `scale_mat` are those the trainer reads (src/trainer.py:41,81,256-258), the last two on the device."""

    def __init__(self, item_views, device, imgs_u8=None, imgs=None, cameras=None, pc_gt=None, scale_mat=None, img_size=None,
                 name=None, tag=None):
        self.item_views = torch.as_tensor(item_views, dtype=torch.int64).reshape(-1)        # item i -> resident view
        self.device = torch.device(device)
        self.imgs_u8, self.imgs, self.cameras = imgs_u8, imgs, cameras or {}
        if imgs_u8 is not None:
            self.n_views, self.height, self.width = imgs_u8.shape[:3]
        elif imgs is not None:
            self.n_views, self.height, self.width = len(imgs), imgs.shape[2], imgs.shape[3]
        else:                                                   # an empty split (the reference's nerfstudio 'val')
            self.n_views = 0
            self.height, self.width = (int(s) for s in img_size) if img_size is not None else (0, 0)
        self.pc_gt, self.scale_mat = pc_gt, scale_mat
        self.img_size, self.name, self.tag = img_size, name, tag

    def __len__(self):
        return len(self.item_views)

    @classmethod
    def from_dataset(cls, ds, device, chunk=8):
        """the views of every item of `ds`, read once.  The reads leave the global RNG as they found it: items that draw from it
        (the reference's per-item randperm) would otherwise advance it in this process, where DataLoader's workers do not."""
        device = _require_cuda(device)
        with torch.random.fork_rng(devices=[]):
            return cls._from_dataset(ds, device, chunk)

    @classmethod
    def _from_dataset(cls, ds, device, chunk):
        meta = dict(img_size=getattr(ds, 'img_size', None), name=getattr(ds, 'name', None), tag=getattr(ds, 'tag', None))
        for k in ('pc_gt', 'scale_mat'):
            v = getattr(ds, k, None)
            meta[k] = torch.as_tensor(v).to(device).contiguous() if v is not None else None
        if _has_fast_path(ds):
            return cls._from_files(ds, device, chunk, meta)
        return cls._from_items(ds, device, meta)

    @classmethod
    def _from_files(cls, ds, device, chunk, meta):
        from PIL import Image
        ids = [int(ds.view_ids[i]) for i in range(len(ds))]
        if not ids:
            return cls([], device, **meta)
        files = sorted(set(ids))
        pos = {f: j for j, f in enumerate(files)}
        h, w = (int(s) for s in ds.img_size)
        views = torch.empty(len(files), h, w, 3, dtype=torch.uint8, device=device)
        pending = []

        def flush(j_end):
            if pending:
                raw = torch.from_numpy(np.stack(pending)).pin_memory().to(device, non_blocking=True)
                views[j_end - len(pending):j_end] = resample_u8(raw, (h, w))
                pending.clear()
        for j, f in enumerate(files):
            with Image.open(ds.input_files[f]) as im:
                a = np.asarray(im.convert('RGB'))
            if pending and (a.shape != pending[0].shape or len(pending) == chunk):
                flush(j)
            pending.append(a)
        flush(len(files))
        cams = [torch.stack([torch.as_tensor(ds.KRT[f][c]) for f in files]).to(device).contiguous() for c in range(3)]
        return cls([pos[f] for f in ids], device, imgs_u8=views, cameras=dict(zip(CAMERA_KEYS, cams)), **meta)

    @classmethod
    def _from_items(cls, ds, device, meta):
        items = [ds[i][0] for i in range(len(ds))]
        if not items:
            return cls([], device, **meta)
        keys = set(items[0])
        if keys != {'imgs', *CAMERA_KEYS}:
            raise ValueError(f"DeviceViews: items must be ({{'imgs', 'K', 'R', 'T'}}, labels), got keys {sorted(keys)}")
        stack = lambda k: torch.stack([torch.as_tensor(it[k]) for it in items]).to(device).contiguous()
        imgs = stack('imgs')
        if imgs.dim() != 4 or imgs.shape[1] != 3 or imgs.dtype != torch.float32:
            raise ValueError(f'DeviceViews: expected (3, H, W) float32 images, got {tuple(imgs.shape[1:])} {imgs.dtype}')
        if meta['img_size'] is None:
            meta['img_size'] = tuple(imgs.shape[2:])
        return cls(range(len(items)), device, imgs=imgs, cameras={k: stack(k) for k in CAMERA_KEYS}, **meta)

    def empty_batch(self, batch):
        """fresh (uninitialised) tensors of a batch of `batch` views, in the reference's key order"""
        out = {'imgs': torch.empty(batch, 3, self.height, self.width, dtype=torch.float32, device=self.device)}
        for k, v in self.cameras.items():
            out[k] = torch.empty((batch,) + tuple(v.shape[1:]), dtype=v.dtype, device=self.device)
        return out

    def check_batch(self, out, batch):
        """refuse `out` unless it holds contiguous imgs / K / R / T buffers of a `batch`-view batch on this device"""
        want = {'imgs': ((batch, 3, self.height, self.width), torch.float32)}
        want.update({k: ((batch,) + tuple(v.shape[1:]), v.dtype) for k, v in self.cameras.items()})
        for k, (shape, dtype) in want.items():
            o = out.get(k)
            if o is None or tuple(o.shape) != shape or o.dtype != dtype or o.device != self.device or not o.is_contiguous():
                raise DbwError(f"device views: out['{k}'] must be a contiguous {dtype} tensor of shape {shape} on {self.device}")

    def launch_gather(self, views, out):
        """one dbw_gather_views launch into buffers check_batch accepted: out['imgs'|'K'|'R'|'T'][b] = view views[b] (views:
        int64 CUDA tensor of resident view indices, read on the device, so the launch can be captured in a graph)"""
        if views.dtype != torch.int64 or not views.is_cuda or not views.is_contiguous():
            raise DbwError('device views: view indices must be a contiguous int64 CUDA tensor')
        fields = [(self.cameras[k], out[k]) for k in CAMERA_KEYS]
        if self.imgs is not None:
            fields.append((self.imgs, out['imgs']))
        table = (_lib.DbwGatherField * len(fields))(*[_lib.DbwGatherField(s.data_ptr(), d.data_ptr(), _words(s)) for s, d in fields])
        u8 = self.imgs_u8
        check(_lib.lib().dbw_gather_views(self.n_views, len(views), _vp(views), _vp(u8) if u8 is not None else None, self.height,
                                          self.width, _vp(out['imgs']), table, len(fields), _stream(self.device)), 'dbw_gather_views')
        return out

    def gather(self, views):
        """a fresh batch of the resident views `views` (int64 CUDA tensor)"""
        return self.launch_gather(views, self.empty_batch(len(views)))

    def points(self, views, seed, step, n=N_POINTS):
        """(B, min(n, P), ...) ground-truth points per view: the first entries of the permutation keyed by (seed, step, view)"""
        pc = self.pc_gt
        B = len(views)
        m = min(int(n), len(pc))
        out = torch.empty((B, m) + tuple(pc.shape[1:]), dtype=pc.dtype, device=self.device)
        if m == 0:
            return out
        check(_lib.lib().dbw_subsample_points(len(pc), _words(pc), _vp(pc), self.n_views, B, _vp(views),
                                              ctypes.c_uint64(seed % 2 ** 64), ctypes.c_uint64(step % 2 ** 64), m, _vp(out),
                                              _stream(self.device)), 'dbw_subsample_points')
        return out


class DeviceLoader:
    """The iteration of DataLoader(views' dataset, batch_size, shuffle) -- or, with rank and world_size, of DataLoader(...,
    sampler=DistributedSampler(dataset, world_size, rank, shuffle)) -- over resident views: the same batches in the same order
    and the same global-RNG draws, each batch fresh device tensors from one gather launch.  points=False leaves labels empty."""

    def __init__(self, views, batch_size=1, shuffle=False, rank=None, world_size=None, points=True):
        self.dataset, self.batch_size, self.shuffle, self.points = views, int(batch_size), bool(shuffle), points
        items = range(len(views))
        if rank is not None:
            self.sampler = DistributedSampler(items, num_replicas=world_size, rank=rank, shuffle=self.shuffle)
        else:
            self.sampler = RandomSampler(items) if self.shuffle else SequentialSampler(items)
        self.batch_sampler = BatchSampler(self.sampler, self.batch_size, drop_last=False)

    def __len__(self):
        return len(self.batch_sampler)

    def index_batches(self):
        """(base seed, iterator over the batches' item indices): the draws DataLoader.__iter__ makes -- the base seed now from
        the global RNG, the sampler's seed at the first batch"""
        base_seed = int(torch.empty((), dtype=torch.int64).random_().item())
        return base_seed, iter(self.batch_sampler)

    def __iter__(self):
        seed, batches = self.index_batches()
        return self._batches(seed, batches)

    def _batches(self, seed, batches):
        V = self.dataset
        for step, items in enumerate(batches):
            idx = V.item_views[torch.as_tensor(items, dtype=torch.int64)].pin_memory().to(V.device, non_blocking=True)
            inp = V.gather(idx)
            labels = {'points': V.points(idx, seed, step)} if self.points and V.pc_gt is not None else {}
            yield inp, labels


def create_train_val_test_loader(cfg, rank=None, world_size=None, get_dataset=None, device=None):
    """src/dataset/__init__.py:9-26 on resident views: the reference's datasets (from its `get_dataset`), the same batch sizes,
    shuffling and sampler, each split decoded and resized once onto `device` (default: the current CUDA device)."""
    if get_dataset is None:
        raise TypeError('create_train_val_test_loader: pass the dataset factory (the reference\'s dataset.get_dataset)')
    kwargs = cfg['dataset']
    name = kwargs.pop('name')                                  # as the reference does: cfg['dataset'] loses its name
    device = torch.device('cuda') if device is None else device
    train, val, test = (DeviceViews.from_dataset(get_dataset(name)(split=s, **kwargs), device) for s in ('train', 'val', 'test'))
    bs = cfg['training']['batch_size']
    if rank is not None:
        train_loader = DeviceLoader(train, bs, shuffle=True, rank=rank, world_size=world_size)
    else:
        train_loader = DeviceLoader(train, bs, shuffle=True)
    val_loader, test_loader = DeviceLoader(val, bs), DeviceLoader(test, bs)
    print(f"Dataset '{name}' init on {train.device}: kwargs={kwargs}, n_train={len(train)}, n_val={len(val)}, "
          f"n_test={len(test)}, bs={bs}")
    return train_loader, val_loader, test_loader
