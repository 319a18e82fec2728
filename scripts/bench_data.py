"""What serving the training views from device memory (dbw_b200.data) buys over the reference's loading path, on synthetic
files written to a temporary directory: 49 PNGs at 1600x1200 resized to 400x300 (the DTU shape) and 64 JPEGs at 768x576
resized to 384x288 (the BlendedMVS shape).  The dataset class has the reference's item semantics (src/dataset/dtu.py:58-72): PIL
open / convert, torchvision Compose([Resize, ToTensor]), and a torch.randperm over a 2.5 M-point ground-truth cloud.

  loader     batches/s of DataLoader(batch 4, shuffle, n_workers=4, pin_memory=True), each batch copied to the device, against
             DeviceLoader (host wall time over whole epochs, ending in a synchronise)
  load       the one-time cost: PIL decode of every file, PIL's resize of the decoded images on the host against
             dbw_resample_u8 on the device (CUDA events, upload excluded), and DeviceViews.from_dataset end to end (torchvision
             imported beforehand, as a trainer's datasets import it)
  step       training iterations/s of a GraphedStep(optimizer=BucketAdam) at 4 x 300x400 (bench scene: 10 blocks, TS 256) fed by
             each loader, and with the gather captured inside the step (run(items=...))
  kernels    registers and spills of the data kernels (cuobjdump -res-usage of the library)

--check asserts that the resident views equal ds[i][0]['imgs'] and that a shuffled epoch of DeviceLoader equals DataLoader's
bit for bit (imgs, K, R, T).  Prints one JSON line with the card's name and power limit.

    python scripts/bench_data.py [--check] [--epochs 2] [--steps 40]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time
from copy import deepcopy
from functools import cached_property

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CFG = {'mesh': {'n_blocks': 10, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 256},
       'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
       'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                      'decouple_rendering': True, 'opacity_noise': 0.1},
       'loss': {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1}}
OPT = {'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}
WORKLOADS = {'dtu': dict(n=49, ext='png', raw=(1200, 1600), img_size=(300, 400)),
             'bmvs': dict(n=64, ext='jpg', raw=(576, 768), img_size=(288, 384))}
N_CLOUD, BS = 2_500_000, 4


class RefDataset(torch.utils.data.Dataset):
    """the reference's item: decode, Compose([Resize, ToTensor]), the view's KRT, a randperm subsample of the cloud"""
    name, tag = 'bench', 'synthetic'

    def __init__(self, files, img_size, pc_gt):
        from dbw_b200.synthetic import ring_cameras
        self.input_files, self.img_size, self.pc_gt = files, tuple(img_size), pc_gt
        self.view_ids = list(range(len(files)))
        R, T, K = ring_cameras(len(files), jitter=0.2)
        self.KRT = [(K.clone(), R[i], T[i]) for i in range(len(files))]

    def __len__(self):
        return len(self.view_ids)

    def __getitem__(self, i):
        idx = self.view_ids[i]
        imgs = self.transform(Image.open(self.input_files[idx]).convert('RGB'))
        K, R, T = self.KRT[idx]
        indices = torch.randperm(len(self.pc_gt))[:int(1e5)]
        return {'imgs': imgs, 'K': K, 'R': R, 'T': T}, {'points': self.pc_gt[indices]}

    @cached_property
    def transform(self):
        from torchvision.transforms import Compose, Resize, ToTensor
        return Compose([Resize(self.img_size), ToTensor()])


def write_files(root, n, ext, raw):
    h, w = raw
    yy, xx = np.mgrid[:h, :w]
    rng = np.random.default_rng(0)
    files = []
    for i in range(n):
        base = np.stack([(xx * 255) // w, (yy * 255) // h, ((xx // 7 + yy // 5 + 13 * i) * 9) % 256], -1)
        img = np.clip(base + rng.integers(-24, 25, (h, w, 3)), 0, 255).astype(np.uint8)
        path = os.path.join(root, f'{i:03d}.{ext}')
        Image.fromarray(img).save(path, **({'quality': 95} if ext == 'jpg' else {}))
        files.append(path)
    return files


def sync_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def host_loader(ds):
    from torch.utils.data import DataLoader
    return DataLoader(ds, batch_size=BS, shuffle=True, num_workers=4, pin_memory=True)


def to_dev(inp):
    return {k: v.to('cuda', non_blocking=True) for k, v in inp.items()}


def loader_rate(make_iter, epochs):
    def run():
        n = 0
        for _ in range(epochs):
            for inp, labels in make_iter():
                n += 1
        return n
    t, n = sync_time(run)
    return n / t


def load_costs(ds, views_cls):
    from dbw_b200.data import resample_u8
    t0 = time.perf_counter()
    decoded = []
    for f in ds.input_files:
        with Image.open(f) as im:
            decoded.append(np.asarray(im.convert('RGB')))
    t_decode = time.perf_counter() - t0
    h, w = ds.img_size
    t0 = time.perf_counter()
    host = [np.asarray(Image.fromarray(a).resize((w, h), Image.BILINEAR)) for a in decoded]
    t_host = time.perf_counter() - t0
    raw = torch.from_numpy(np.stack(decoded)).cuda()
    resample_u8(raw, (h, w))                                     # warm-up
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    dev = resample_u8(raw, (h, w))
    e1.record()
    torch.cuda.synchronize()
    same = bool(np.array_equal(dev.cpu().numpy(), np.stack(host)))
    del raw
    t_views, _ = sync_time(lambda: views_cls.from_dataset(ds, 'cuda'))
    return {'decode_ms': 1e3 * t_decode, 'host_resize_ms': 1e3 * t_host, 'device_resize_ms': e0.elapsed_time(e1),
            'from_dataset_ms': 1e3 * t_views, 'device_resize_equals_pil': same}


def step_rates(ds, views, steps):
    import dbw_b200  # noqa: F401
    from dbw_b200.data import DeviceLoader
    from dbw_b200.dbw import DifferentiableBlocksWorld
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel

    def full_batches(make):
        while True:
            for inp, _ in make():
                if len(inp['imgs']) == BS:
                    yield inp

    def rate(run_one, it):
        for _ in range(3):
            run_one(next(it))
        t, _ = sync_time(lambda: [run_one(next(it)) for _ in range(steps)])
        return steps / t

    def fresh(views_arg=None):
        torch.manual_seed(0)
        model = DifferentiableBlocksWorld(tuple(ds.img_size), **deepcopy(CFG)).to(torch.device('cuda:0')).train()
        example = views.gather(torch.zeros(BS, dtype=torch.int64, device='cuda'))
        return GraphedStep(ViewParallel(model, seed=0), example, BS, optimizer=create_optimizer(OPT, model), views=views_arg)

    out = {}
    step = fresh()
    out['host_loader_steps_per_s'] = rate(lambda inp: step.run(to_dev(inp)), full_batches(lambda: host_loader(ds)))
    dl = DeviceLoader(views, BS, shuffle=True, points=False)
    out['device_loader_steps_per_s'] = rate(lambda inp: step.run(inp), full_batches(lambda: dl))
    step = fresh(views)

    def items():
        while True:
            _, batches = dl.index_batches()
            for b in batches:
                if len(b) == BS:
                    yield b
    out['captured_gather_steps_per_s'] = rate(lambda b: step.run(items=b), items())
    return out


def kernel_resources():
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    lib = os.path.join(ROOT, 'differentiable-blocksworld_b200', 'libdbw_render.so')
    text = subprocess.run([cuobjdump, '-res-usage', lib], check=True, capture_output=True, text=True).stdout
    res = {}
    for name, reg, stack in re.findall(r'Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)', text):
        m = re.search(r'(resample_u8_kernelILb[01]E|gather_views_kernel|subsample_points_kernel)', name)
        if m:
            res[m.group(1).replace('ILb0E', '<vertical>').replace('ILb1E', '<horizontal>')] = {'registers': int(reg),
                                                                                                'stack_bytes': int(stack)}
    return res


def check(ds, views):
    from torch.utils.data import DataLoader
    from dbw_b200.data import DeviceLoader
    got = views.gather(views.item_views.cuda())
    for i in range(len(ds)):
        for k, v in ds[i][0].items():
            assert torch.equal(got[k][i].cpu(), v), ('resident view', i, k)
    torch.manual_seed(3)
    ref = [inp for inp, _ in DataLoader(ds, batch_size=BS, shuffle=True, num_workers=4)]
    state = torch.get_rng_state()
    torch.manual_seed(3)
    mine = [inp for inp, _ in DeviceLoader(views, BS, shuffle=True)]
    assert torch.equal(state, torch.get_rng_state()), 'global RNG state after the epoch'
    assert len(ref) == len(mine)
    for a, b in zip(mine, ref):
        for k in b:
            assert torch.equal(a[k].cpu(), b[k]), ('batch', k)
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--check', action='store_true')
    ap.add_argument('--epochs', type=int, default=2, help='epochs of each loader timed')
    ap.add_argument('--steps', type=int, default=40, help='training iterations timed per feed')
    ap.add_argument('--workloads', nargs='+', default=list(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_data.py needs a GPU')
    import dbw_b200  # noqa: F401
    import torchvision.transforms  # noqa: F401     a trainer has imported it with its datasets; its first import is seconds
    from dbw_b200.data import DeviceLoader, DeviceViews
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    result = {'gpu': q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(),
              'kernels': kernel_resources()}
    g = torch.Generator().manual_seed(0)
    cloud = torch.rand(N_CLOUD, 3, generator=g)
    with tempfile.TemporaryDirectory() as tmp:
        for name in args.workloads:
            W = WORKLOADS[name]
            root = os.path.join(tmp, name)
            os.makedirs(root)
            ds = RefDataset(write_files(root, W['n'], W['ext'], W['raw']), W['img_size'], cloud)
            r = {'views': W['n'], 'raw': W['raw'], 'img_size': W['img_size'], 'load': load_costs(ds, DeviceViews)}
            views = DeviceViews.from_dataset(ds, 'cuda')
            if args.check:
                r['check'] = check(ds, views)
            r['host_loader_batches_per_s'] = loader_rate(lambda: ((to_dev(i), l) for i, l in host_loader(ds)), args.epochs)
            dl = DeviceLoader(views, BS, shuffle=True)
            r['device_loader_batches_per_s'] = loader_rate(lambda: iter(dl), max(args.epochs, 20))
            if tuple(W['img_size']) == (300, 400):
                r.update(step_rates(ds, views, args.steps))
            result[name] = r
            print(name, json.dumps(r), file=sys.stderr, flush=True)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
