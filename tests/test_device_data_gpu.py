"""GPU: training views served from device memory (dbw_b200.data, csrc/dbw_data.cu) against the reference's own loading path --
PIL decode, torchvision Compose([Resize, ToTensor]), torch's DataLoader -- on PNG and JPEG files this module writes.  Resident
views and batches must equal the host's bit for bit, the batch order and global-RNG state those of DataLoader, training fed by
either loader the same (eagerly, through GraphedStep, and with the gather captured inside the step), labels['points'] a
deterministic subset without duplicates, and batches fresh tensors."""
from copy import deepcopy
from functools import cached_property

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
IMG_SIZE = (48, 64)
# raw sizes (h, w): PNGs of one size and JPEGs of another, so the upload chunks split where the size changes
RAW = [('png', (120, 160))] * 7 + [('jpg', (96, 128))] * 5


def _write_files(root):
    files = []
    rng = np.random.default_rng(0)
    for i, (ext, (h, w)) in enumerate(RAW):
        yy, xx = np.mgrid[:h, :w]
        base = np.stack([xx * 255 // w, yy * 255 // h, (xx + yy + 17 * i) % 256], -1)
        img = np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
        path = root / f'{i:03d}.{ext}'
        Image.fromarray(img).save(path, quality=90) if ext == 'jpg' else Image.fromarray(img).save(path)
        files.append(str(path))
    return files


class RefViews(torch.utils.data.Dataset):
    """the reference's DTU / BlendedMVS item semantics (src/dataset/dtu.py:58-72): PIL open / convert, Compose([Resize,
    ToTensor]), the KRT of the view, and a randperm subsample of the ground-truth cloud"""
    name, tag = 'synthetic_files', 'scan0'

    def __init__(self, files, view_ids=None, img_size=IMG_SIZE, n_points=3000, cam_dtype=torch.float32, length=None, k_jitter=0.01):
        from dbw_b200.synthetic import ring_cameras
        self.input_files, self.img_size = files, tuple(img_size)
        self.view_ids = list(range(len(files))) if view_ids is None else list(view_ids)
        R, T, K = ring_cameras(len(files), jitter=0.3, seed=3)
        K = K.clone()
        self.KRT = [((K * (1 + k_jitter * i)).float(), R[i].to(cam_dtype), T[i].to(cam_dtype)) for i in range(len(files))]
        i = torch.arange(n_points, dtype=torch.float32)
        self.pc_gt = torch.stack([i, 2 * i, -i], 1)              # point j is (j, 2j, -j): its index can be read back
        self.scale_mat = torch.eye(4, dtype=torch.float64)
        self.length = length

    def __len__(self):
        return len(self.view_ids) if self.length is None else min(self.length, len(self.view_ids))

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


class ItemsOnly(torch.utils.data.Dataset):
    """the same items behind no file attributes: DeviceViews must take the generic path"""

    def __init__(self, ds):
        self.ds, self.img_size, self.pc_gt = ds, ds.img_size, ds.pc_gt

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        return self.ds[i]


@pytest.fixture(scope='module')
def files(tmp_path_factory):
    return _write_files(tmp_path_factory.mktemp('views'))


def _views(ds):
    from dbw_b200.data import DeviceViews
    return DeviceViews.from_dataset(ds, DEV)


def _cpu(batch):
    return {k: v.cpu() for k, v in batch.items()}


def _bits_equal(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ------------------------------------------------------------------ the resize kernel
@pytest.mark.parametrize('in_hw,out_hw', [((1200, 1600), (300, 400)), ((576, 768), (288, 384)), ((97, 131), (31, 45)),
                                          ((30, 40), (64, 81)), ((40, 50), (1, 17)), ((60, 80), (60, 33)), ((60, 80), (21, 80)),
                                          ((45, 45), (45, 45)), ((1000, 3), (999, 5)), ((1000, 10), (999, 5))])
def test_resample_kernel_matches_pillow(in_hw, out_hw):
    from dbw_b200.data import resample_u8
    rng = np.random.default_rng(in_hw[0] + out_hw[1])
    imgs = rng.integers(0, 256, (3,) + in_hw + (3,), dtype=np.uint8)
    got = resample_u8(torch.from_numpy(imgs).to(DEV), out_hw).cpu().numpy()
    for k in range(3):
        want = np.asarray(Image.fromarray(imgs[k]).resize(out_hw[::-1], Image.BILINEAR))
        np.testing.assert_array_equal(got[k], want)


# ------------------------------------------------------------------ resident views
@pytest.mark.parametrize('path', ['fast', 'generic'])
@pytest.mark.parametrize('cam_dtype', [torch.float32, torch.float64])
def test_resident_views_equal_the_datasets_items(files, path, cam_dtype):
    ref = RefViews(files, view_ids=[3, 0, 11, 7, 7, 5, 9], cam_dtype=cam_dtype)           # repeats and a JPEG / PNG mix
    ds = ref if path == 'fast' else ItemsOnly(ref)
    V = _views(ds)
    assert (V.imgs_u8 is not None) == (path == 'fast')
    assert len(V) == len(ref) and tuple(V.img_size) == IMG_SIZE
    got = _cpu(V.gather(V.item_views.to(DEV)))
    for i in range(len(ref)):
        want = ref[i][0]
        assert list(got) == list(want)
        for k in want:
            assert _bits_equal(got[k][i], want[k]), (path, i, k)
    assert torch.equal(V.pc_gt.cpu(), ref.pc_gt)


# ------------------------------------------------------------------ batches against DataLoader
def _host_epochs(ds, bs, shuffle, epochs, sampler=None):
    # workers: the reference's items draw their randperm there, so the main process's RNG sees only the loader's own draws
    from torch.utils.data import DataLoader
    loader = DataLoader(ds, batch_size=bs, shuffle=shuffle if sampler is None else False, sampler=sampler, num_workers=2)
    out = []
    for e in range(epochs):
        if sampler is not None:
            sampler.set_epoch(e)
        out.append(([_cpu(inp) for inp, _ in loader], torch.get_rng_state()))
    return out


def _device_epochs(V, bs, shuffle, epochs, **kw):
    from dbw_b200.data import DeviceLoader
    loader = DeviceLoader(V, bs, shuffle=shuffle, **kw)
    out = []
    for e in range(epochs):
        if 'rank' in kw:
            loader.sampler.set_epoch(e)
        out.append(([_cpu(inp) for inp, _ in loader], torch.get_rng_state()))
    return out


@pytest.mark.parametrize('shuffle,bs,dist', [(True, 4, None), (False, 4, None), (True, 5, (1, 2)), (True, 3, (2, 3))])
def test_batches_equal_dataloaders_for_three_epochs(files, shuffle, bs, dist):
    from torch.utils.data import DistributedSampler
    ds = RefViews(files, view_ids=range(11), cam_dtype=torch.float64)       # 11 items: every last batch is partial
    V = _views(ds)
    kw = {} if dist is None else dict(rank=dist[0], world_size=dist[1])
    sampler = None if dist is None else DistributedSampler(ds, num_replicas=dist[1], rank=dist[0], shuffle=shuffle)
    torch.manual_seed(11)
    want = _host_epochs(ds, bs, shuffle, 3, sampler)
    torch.manual_seed(11)
    got = _device_epochs(V, bs, shuffle, 3, **kw)
    for (gb, gs), (wb, ws) in zip(got, want):
        assert len(gb) == len(wb)
        for g, w in zip(gb, wb):
            assert list(g) == list(w)
            for k in w:
                assert _bits_equal(g[k], w[k]), k
        assert torch.equal(gs, ws)
    if shuffle and dist is None:
        assert len(gb[-1]['imgs']) == 11 % bs and not all(torch.equal(a['R'], b['R']) for a, b in zip(got[0][0], got[1][0]))


# ------------------------------------------------------------------ labels['points']
@pytest.mark.parametrize('P', [1, 3000, 250_000])
def test_points_are_distinct_in_range_and_deterministic(files, P):
    from dbw_b200.data import DeviceLoader
    V = _views(RefViews(files, n_points=P))

    def epoch(seed):
        torch.manual_seed(seed)
        return [labels['points'].cpu() for _, labels in DeviceLoader(V, 4, shuffle=True)]
    a, b, c = epoch(1), epoch(1), epoch(2)
    n = min(P, 100_000)
    for pts in a:
        assert pts.shape == (len(pts), n, 3)
        idx = pts[..., 0].long()
        assert torch.equal(pts, torch.stack([idx, 2 * idx, -idx], -1).float())       # whole rows of the cloud
        assert idx.min() >= 0 and idx.max() < P
        for row in idx:
            assert len(torch.unique(row)) == n
        if P > 1:
            assert not torch.equal(idx[0], idx[1])                                      # every view draws its own subset
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    if P > 1:
        assert not all(torch.equal(x, y) for x, y in zip(a, c))


def test_points_false_leaves_labels_empty(files):
    from dbw_b200.data import DeviceLoader
    assert all(labels == {} for _, labels in DeviceLoader(_views(RefViews(files)), 4, points=False))


# ------------------------------------------------------------------ batches are fresh tensors
def test_viz_samples_taken_from_the_first_batch_survive_iteration(files):
    """src/trainer.py:61-64 keeps slices of the first val batch"""
    from dbw_b200.data import DeviceLoader
    loader = DeviceLoader(_views(RefViews(files)), 4, shuffle=True)
    samples, labels = next(iter(loader))
    viz = {k: v.to(DEV)[:4] for k, v in samples.items()}
    keep = {k: v.clone() for k, v in viz.items()}
    for _ in range(3):
        for inp, _ in loader:
            inp['imgs'].add_(1)
    assert all(torch.equal(viz[k], keep[k]) for k in keep)


# ------------------------------------------------------------------ training fed by either loader
CFG = {
    'mesh': {'n_blocks': 5, 'S_world': 0.5, 'R_world': [115, 0, 0], 'txt_size': 32},
    'renderer': {'faces_per_pixel': 10, 'cameras': {'name': 'perspective'}, 'detach_bary': True, 'z_clip': 0.001},
    'rend_optim': {'coarse_learning': 1500, 'decimate_txt': 750, 'decimate_factor': 8, 'kill_blocks': True,
                   'decouple_rendering': True, 'opacity_noise': 0.1},
    'loss': {'rgb_weight': 1, 'parsimony_weight': 0.01, 'tv_weight': 0.1, 'overlap_weight': 1},
}
OPT = {'training': {'optimizer': {'name': 'adam', 'lr': 0.005, 'texture': {'lr': 0.05}}}}
SEED, BS, STEPS = 5, 3, 10


def _model():
    import dbw_b200  # noqa: F401
    from dbw_b200.dbw import DifferentiableBlocksWorld
    torch.manual_seed(SEED)
    return DifferentiableBlocksWorld(IMG_SIZE, **deepcopy(CFG)).to(DEV).train()


def _close(a, b, tol):
    return (a - b).norm().item() <= tol * b.norm().item() + 1e-12


def _batches(kind, ds, V):
    """STEPS full batches in the loader's order, across epochs"""
    from torch.utils.data import DataLoader
    from dbw_b200.data import DeviceLoader
    loader = DataLoader(ds, BS, shuffle=True, num_workers=2) if kind == 'host' else DeviceLoader(V, BS, shuffle=True)
    while True:
        for inp, _ in loader:
            yield inp


def _items(V):
    """the item indices of the same batches (DeviceLoader.index_batches), for the captured gather"""
    from dbw_b200.data import DeviceLoader
    loader = DeviceLoader(V, BS, shuffle=True)
    while True:
        _, batches = loader.index_batches()
        yield from batches


def _train(mode, kind, ds, V):
    from dbw_b200.graph import GraphedStep
    from dbw_b200.losses import OVERLAP_N_POINTS
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    torch.manual_seed(SEED)
    model = _model()
    opt = create_optimizer(OPT, model)
    torch.manual_seed(123)                                   # the loaders' draws start from here in every run
    losses, seen = [], []
    if mode == 'eager':
        gen = torch.Generator(device=DEV).manual_seed(SEED)
        noise, overlap = torch.zeros_like(model.alpha_logit), torch.zeros(model.n_blocks, OVERLAP_N_POINTS, 3, device=DEV)
        it = _batches(kind, ds, V)
        for _ in range(STEPS):
            inp = {k: v.to(DEV) for k, v in next(it).items()}
            seen.append(_cpu(inp))
            noise.normal_(generator=gen)
            overlap.uniform_(generator=gen)
            model.opacity_noise_buffer, model.overlap_samples_buffer, model.noise_generator = noise, overlap, None
            opt.zero_grad()
            out = model(inp, None)
            out['total'].backward()
            opt.step()
            losses.append(out['total'].item())
    else:
        if mode == 'graphed':
            it = _batches(kind, ds, V)
            first = {k: v.to(DEV) for k, v in next(it).items()}
            step = GraphedStep(ViewParallel(model, seed=SEED), first, BS, optimizer=opt)
            pending = [first]
        else:                                                # the gather captured inside the step
            it = _items(V)
            pending = [next(it)]                             # the loader's draws before the capture, as in the other runs
            step = GraphedStep(ViewParallel(model, seed=SEED), V.gather(torch.zeros(BS, dtype=torch.int64, device=DEV)), BS,
                               optimizer=opt, views=V)
        for _ in range(STEPS):
            if mode == 'graphed':
                inp = pending.pop() if pending else {k: v.to(DEV) for k, v in next(it).items()}
                out = step.run(inp)
            else:
                out = step.run(items=pending.pop() if pending else next(it))
            seen.append(_cpu(step.static_inp))
            losses.append(out['total'].item())
    return losses, {n: p.detach().clone() for n, p in model.named_parameters()}, seen


@pytest.mark.parametrize('mode', ['eager', 'graphed', 'captured_gather'])
def test_ten_training_steps_match_the_host_loader(files, mode):
    ds = RefViews(files, k_jitter=0)                         # without per-view intrinsics the first batch's K serves every view
    V = _views(ds)
    ref_losses, ref_params, ref_seen = _train('eager' if mode == 'eager' else 'graphed', 'host', ds, V)
    losses, params, seen = _train(mode, 'device', ds, V)
    for a, b in zip(seen, ref_seen):                          # the same inputs, bit for bit, at every step
        assert all(_bits_equal(a[k], b[k]) for k in b)
    # the raster backward accumulates with atomics: two runs of the same training differ in their last bits
    # (tests/test_optim_gpu.py::_same_training)
    assert all(abs(x - y) <= 1e-4 * abs(y) + 1e-7 for x, y in zip(losses, ref_losses)), (losses, ref_losses)
    for n in ref_params:
        assert _close(params[n], ref_params[n], 1e-3), n
    assert any(not torch.equal(ref_params[n], p) for n, p in _model().named_parameters())         # training moved them


def test_graphed_step_refuses_mixed_inputs(files):
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    V = _views(RefViews(files))
    model = _model()
    step = GraphedStep(ViewParallel(model, seed=SEED), V.gather(torch.zeros(BS, dtype=torch.int64, device=DEV)), BS,
                       optimizer=create_optimizer(OPT, model), views=V)
    with pytest.raises(ValueError):
        step.run(V.gather(torch.zeros(BS, dtype=torch.int64, device=DEV)))
    with pytest.raises(ValueError):
        step.run(items=[0, 1])


# ------------------------------------------------------------------ empty splits and the global RNG while loading
class EmptySplit(torch.utils.data.Dataset):
    """the reference's nerfstudio 'val' split: no items and no attributes"""

    def __len__(self):
        return 0

    def __getitem__(self, i):
        raise IndexError(i)


def test_an_empty_split_loads_and_yields_nothing(files):
    from torch.utils.data import DataLoader
    from dbw_b200.data import DeviceLoader
    V = _views(EmptySplit())
    loader = DeviceLoader(V, 4)
    assert len(V) == 0 and len(loader) == 0
    torch.manual_seed(5)
    assert list(loader) == []
    got = torch.get_rng_state()
    torch.manual_seed(5)
    assert list(DataLoader(EmptySplit(), batch_size=4)) == []
    assert torch.equal(got, torch.get_rng_state())


def test_create_loaders_with_an_empty_val_split(files):
    from dbw_b200.data import DeviceLoader, create_train_val_test_loader

    def get_dataset(name):
        assert name == 'nerfstudio'
        return lambda split, **kw: EmptySplit() if split == 'val' else ItemsOnly(RefViews(files, **kw))
    cfg = {'dataset': {'name': 'nerfstudio', 'img_size': IMG_SIZE}, 'training': {'batch_size': 4}}
    train, val, test = create_train_val_test_loader(cfg, get_dataset=get_dataset, device=DEV)
    assert all(isinstance(x, DeviceLoader) for x in (train, val, test))
    assert len(train) == 3 and len(val) == 0 and len(test) == 3 and list(val) == []
    assert 'name' not in cfg['dataset']                        # popped, as the reference's create_train_val_test_loader does


@pytest.mark.parametrize('path', ['fast', 'generic'])
def test_loading_leaves_the_global_rng_alone(files, path):
    """the items' own draws (randperm) happen in DataLoader's workers, never in the trainer's process"""
    ref = RefViews(files)
    torch.manual_seed(3)
    before = torch.get_rng_state()
    V = _views(ref if path == 'fast' else ItemsOnly(ref))
    assert (V.imgs_u8 is not None) == (path == 'fast')
    assert torch.equal(before, torch.get_rng_state())


def test_generic_path_batches_and_rng_equal_dataloaders(files):
    """views built between the seed and the epochs, as Trainer.__init__ builds its loaders before create_model"""
    ds = ItemsOnly(RefViews(files, view_ids=range(11), cam_dtype=torch.float64))
    torch.manual_seed(11)
    want = _host_epochs(ds, 4, True, 3)
    torch.manual_seed(11)
    got = _device_epochs(_views(ds), 4, True, 3)
    for (gb, gs), (wb, ws) in zip(got, want):
        assert len(gb) == len(wb)
        for g, w in zip(gb, wb):
            assert all(_bits_equal(g[k], w[k]) for k in w)
        assert torch.equal(gs, ws)


def test_captured_gather_takes_items_as_a_cuda_tensor(files):
    from dbw_b200.graph import GraphedStep
    from dbw_b200.optim import create_optimizer
    from dbw_b200.parallel import ViewParallel
    V = _views(RefViews(files, k_jitter=0))
    model = _model()
    step = GraphedStep(ViewParallel(model, seed=SEED), V.gather(torch.zeros(BS, dtype=torch.int64, device=DEV)), BS,
                       optimizer=create_optimizer(OPT, model), views=V)
    step.run(items=torch.tensor([4, 1, 9], device=DEV))
    want = V.gather(V.item_views[[4, 1, 9]].to(DEV))
    assert all(torch.equal(step.static_inp[k], want[k]) for k in want)
