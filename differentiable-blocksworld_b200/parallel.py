"""View-sharded data parallelism for one optimisation step (new functionality: the reference has no distributed path
that runs, SURVEY.md section 0 item 5 and section 8e).

Views of a step are independent given the replicated scene parameters, so they shard with NO data-path collective:
rank r renders a contiguous range of the B views (or of their 16-row bands) and back-propagates into its own gradients;
ONE all-reduce(SUM) per step over NVLink / NVSwitch then gives every rank the full gradient -- either of a single flat
fp32 bucket of the parameter gradients after the backward (about 9.4 MB for 10 blocks with 256^2 textures), or, while the
textures are box-decimated, of the scene tensors' gradients inside the backward (GradSumPoint: about 0.21 MB).
Correctness conditions handled here:
  * the RGB loss is a MEAN over all B views (dbw.py:367): each rank divides by the GLOBAL pixel count
    (model.n_total_views), so the SUM of the per-rank gradients is the gradient of the global mean;
  * view-independent terms (parsimony / TV / overlap, dbw.py:373-405) are computed identically on every rank: divided by
    the world size before a leaf SUM, counted once when the SUM happens at the scene tensors (they do not pass through it);
  * the opacity noise (dbw.py:300-301) and the overlap sample points (dbw.py:393) come from a generator that every
    rank seeds identically at every step.
Camera poses that require grad (ViewParallel(max_pose_views=N)): the step renders its shard from slices of full-batch pose
leaves, so each rank's pose gradient is a (B, 12) block with zeros on the views it did not render; that block rides in the same
one collective as the scene's gradients (the tail of the leaf bucket, or through the GradSumPoint), and the sum is handed on
to the caller's R / T with one small eager backward.  Intrinsics that require grad (ViewParallel(max_pose_views=N,
intrinsics=True)) ride the same way: a (B, 4) leaf of (fx, fy, px, py) per view after the poses, handed on to the caller's K."""
import ctypes

import torch
import torch.distributed as dist

from . import _lib


def shard_views(n_views, world_size, rank):
    """Contiguous, balanced view ranges: the first n_views % world_size ranks get one extra view (49 -> 7,6,6,6,6,6,6,6)."""
    base, extra = divmod(n_views, world_size)
    start = rank * base + min(rank, extra)
    return slice(start, start + base + (1 if rank < extra else 0))


def refuse_camera_gradients(inp, who, intrinsics_only=False):
    """Camera poses or intrinsics that require grad are refused rather than silently left without a gradient: under view or
    row-band sharding a rank holds only partial per-view sums of them, and a captured graph's static input buffers do not carry
    a gradient back to the caller's tensors.  intrinsics_only: the step carries pose gradients, but not intrinsics gradients."""
    for k in (('K',) if intrinsics_only else ('R', 'T', 'K')):
        v = inp.get(k) if inp is not None else None
        if torch.is_tensor(v) and v.requires_grad:
            how = ('construct its ViewParallel with max_pose_views >= the views of a step and intrinsics=True' if k == 'K' else
                   'construct its ViewParallel with max_pose_views >= the views of a step')
            raise RuntimeError(f"{who}: inp['{k}'] requires grad, but this step was not built for its gradient: {how}, detach "
                               f"it, or call the model directly")


def wants_pose_gradients(inp):
    """inp's camera poses or intrinsics require grad"""
    return inp is not None and any(torch.is_tensor(inp.get(k)) and inp[k].requires_grad for k in ('R', 'T', 'K'))


def wants_intrinsics_gradients(inp):
    return inp is not None and torch.is_tensor(inp.get('K')) and inp['K'].requires_grad


def camera_leaves(poses):
    """the leaves of pose_leaves()'s (R, T, views, intrinsics or None) that take a gradient, in bucket order"""
    return [q for q in (poses[0], poses[1], poses[3]) if q is not None]


def intrinsics_matrix(intr):
    """(B,4) (fx, fy, px, py) -> a (B,4,4) K holding them where renderer.intrinsics_of reads them (other entries 0: unread)"""
    fx, fy, px, py = intr.unbind(1)
    z = torch.zeros_like(fx)              # built on the device: no host copy inside a captured step
    return torch.stack([fx, z, px, z, z, fy, py, z, z, z, z, z, z, z, z, z], -1).view(-1, 4, 4)


def pose_backward(inp, grads):
    """continue the step's summed camera gradients (g_R (B,3,3), g_T (B,3)[, g_intrinsics (B,4)]) into the caller's graph behind
    inp['R'] / inp['T'] (/ inp['K'], through its fx, fy, px, py entries)"""
    from .renderer import intrinsics_of
    pairs = [(inp[k], g) for k, g in zip(('R', 'T'), grads) if torch.is_tensor(inp.get(k)) and inp[k].requires_grad]
    if len(grads) > 2 and wants_intrinsics_gradients(inp):
        pairs.append((intrinsics_of(inp['K']), grads[2]))
    if pairs:
        torch.autograd.backward([t for t, _ in pairs], [g.to(t.dtype) for t, g in pairs])


ROW_BAND = 16          # rows per shardable band: the tallest raster tile (16 x 16, the K <= 4 forward), so tiles stay whole


def shard_row_bands(n_views, height, world_size, rank, band=ROW_BAND):
    """Balanced sharding at (view, row band) granularity: the n_views * ceil(height / band) bands of a step, in (view, row)
    order, are cut into world_size contiguous runs whose lengths differ by at most one band (49 views of 400 rows over 8
    ranks: 153 or 154 bands of 16 rows each, i.e. 6.12 views per rank instead of 7 for the largest whole-view shard).
    Returns this rank's pieces as [(view, row_begin, row_end)], one per view it touches."""
    per_view = -(-height // band)
    total = n_views * per_view
    base, extra = divmod(total, world_size)
    start = rank * base + min(rank, extra)
    stop = start + base + (1 if rank < extra else 0)
    pieces = []
    for v in range(start // per_view, -(-stop // per_view) if stop > start else start // per_view):
        b0, b1 = max(start, v * per_view) - v * per_view, min(stop, (v + 1) * per_view) - v * per_view
        if b1 > b0:
            pieces.append((v, b0 * band, min(b1 * band, height)))
    return pieces


class PeerAllReduce:
    """The hand-written NVLink all-reduce of csrc/dbw_comm.cu (include/dbw_render.h dbw_comm_*): every rank exports its
    arena with a CUDA IPC handle, the handles are all-gathered once through torch.distributed, and from then on an
    all-reduce is ONE kernel launch on the current stream -- capturable inside the step's CUDA graph, no NCCL involved."""

    def __init__(self, max_floats, device, group=None):
        L = _lib.lib()
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.handle = ctypes.c_void_p()
        _lib.check(L.dbw_comm_create(self.world, self.rank, max_floats, ctypes.byref(self.handle)), 'dbw_comm_create')
        ptr = ctypes.c_void_p()
        _lib.check(L.dbw_comm_buffer(self.handle, ctypes.byref(ptr)), 'dbw_comm_buffer')

        class _Arena:          # zero-copy view of the arena's bucket as a tensor (CUDA array interface)
            __cuda_array_interface__ = {'shape': (int(max_floats),), 'typestr': '<f4', 'data': (ptr.value, False), 'version': 3,
                                        'strides': None}
        self._arena = _Arena()
        self.flat = torch.as_tensor(self._arena, device=device)      # the bucket the gradients are gathered into
        mine = (ctypes.c_ubyte * 64)()
        _lib.check(L.dbw_comm_ipc_handle(self.handle, mine), 'dbw_comm_ipc_handle')
        t = torch.tensor(list(mine), dtype=torch.uint8, device=device)
        gathered = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(gathered, t, group=group)
        blob = bytes(torch.cat(gathered).cpu().tolist())
        _lib.check(L.dbw_comm_connect(self.handle, blob), 'dbw_comm_connect')
        dist.barrier(group)

    def all_reduce(self, flat):
        _lib.check(_lib.lib().dbw_comm_all_reduce(self.handle, ctypes.c_void_p(flat.data_ptr()), flat.numel(),
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'dbw_comm_all_reduce')

    def error(self):
        out = ctypes.c_int32(0)
        _lib.check(_lib.lib().dbw_comm_error(self.handle, ctypes.byref(out)), 'dbw_comm_error')
        return out.value

    def close(self):
        if self.handle:
            _lib.lib().dbw_comm_destroy(self.handle)
            self.handle = ctypes.c_void_p()


class _GradSumFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, point, *tensors):
        ctx.point = point
        return tuple(t.view_as(t) for t in tensors)

    @staticmethod
    def backward(ctx, *grads):
        return (None, *ctx.point.sum_over_ranks(grads))


class GradSumPoint:
    """Data-parallel gradient reduction INSIDE the backward, at the scene tensors instead of at the leaves: `point(*tensors)` is the
    identity in the forward; in the backward the tensors' gradients are packed into the peer-memory bucket (one gather kernel),
    summed over the ranks by ONE dbw_comm_all_reduce launch, and handed on as views of the bucket.  The model routes everything
    its two raster passes differentiate through one point -- both passes' vertices, the block opacities, and the textures as their
    box-decimated CELLS (scene_ops.scene_texture_cells) -- so what lies before the point (texture-cell / geometry / opacity
    backward kernels: deterministic, no atomics) turns GLOBAL gradients into leaf gradients, identically on every rank, and no
    leaf all-reduce follows.  While textures are decimated 8x (the first `decimate_txt` iterations, src/model/dbw.py:276-279,
    331-334) the cells hold 64x fewer values than the texture parameters: ~0.21 MB per step (float4 cells) instead of ~9.4 MB on the DTU shape."""

    def __init__(self, peer):
        self.peer = peer
        self.pose_leaves = None          # (R (B,3,3), T (B,3), views, intrinsics (B,4) or None): full-batch camera leaves that ride through the point
        self._cameras = self._K = None

    def __call__(self, *tensors):
        if self.pose_leaves is None:
            return _GradSumFn.apply(self, *tensors)
        views = self.pose_leaves[2]
        leaves = camera_leaves(self.pose_leaves)
        out = _GradSumFn.apply(self, *tensors, *leaves)
        out, cams = out[:len(tensors)], out[len(tensors):]
        self._cameras = (cams[0][views], cams[1][views])
        self._K = intrinsics_matrix(cams[2][views]) if len(cams) > 2 else None
        return tuple(out)

    def ride(self, poses):
        """poses = (R, T, views, intrinsics or None) or None: from the next call on, the camera leaves pass through the point with
        the scene tensors, so their gradients join the same one exchange; the model then renders from cameras() / intrinsics()"""
        self.pose_leaves, self._cameras, self._K = poses, None, None

    def intrinsics(self, K):
        """the per-view K a model renders its shard from: this rank's slice of the point's intrinsics output when intrinsics
        leaves ride along, `K` (the model's own choice) otherwise"""
        if self.pose_leaves is None or self.pose_leaves[3] is None:
            return K
        if self._K is None:
            raise RuntimeError('GradSumPoint.intrinsics() before the point was called on the scene tensors')
        return self._K

    def cameras(self, inp):
        """the (R, T) a model renders its shard from, read after it has called the point: this rank's slices of the point's pose
        outputs when pose leaves ride along, inp's own poses otherwise"""
        if self.pose_leaves is None:
            return inp['R'], inp['T']
        if self._cameras is None:
            raise RuntimeError('GradSumPoint.cameras() before the point was called on the scene tensors')
        return self._cameras

    def sum_over_ranks(self, grads):
        n = sum(g.numel() for g in grads)
        n_pad = (n + 3) // 4 * 4
        if n_pad > self.peer.flat.numel():
            raise RuntimeError(f'{n_pad} gradient floats exceed the peer-memory bucket ({self.peer.flat.numel()})')
        buf = self.peer.flat[:n_pad]
        with torch.no_grad():
            torch.cat([g.reshape(-1).float() for g in grads], out=buf[:n])
            self.peer.all_reduce(buf)
        out, o = [], 0
        for g in grads:
            out.append(buf[o:o + g.numel()].view_as(g))
            o += g.numel()
        return out


class GradBucket:
    """All parameter gradients as views into one flat buffer -> a single all-reduce per step."""

    def __init__(self, params, peer_factory=None, min_floats=0, max_pose_views=0, intrinsics=False):
        """peer_factory(n_floats, device) -> PeerAllReduce or None: when given and successful, the flat buffer IS the peer-memory
        arena's bucket (csrc/dbw_comm.cu) and all_reduce() is its kernel; else a plain tensor and torch.distributed.
        min_floats: capacity the arena needs for its other user (GradSumPoint).
        max_pose_views: room for the pose gradients of that many views (12 floats each: the B x 9 entries of g_R, then the
        B x 3 of g_T) after the parameter gradients, gathered and all-reduced with them.
        intrinsics: 4 more floats per pose view, for the B x 4 intrinsics gradients after g_T"""
        self.params = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        ref = self.params[0]
        self.n = n
        n_pad = (n + 3) // 4 * 4                     # padded: 128-bit all-reduce lanes
        n_all = n_pad + (16 if intrinsics else 12) * int(max_pose_views)
        self.peer = peer_factory(max(n_all, (int(min_floats) + 3) // 4 * 4), ref.device) if peer_factory is not None else None
        if self.peer is not None:
            self.peer.flat.zero_()
            self._all = self.peer.flat[:n_all]
        else:
            self._all = torch.zeros(n_all, dtype=ref.dtype, device=ref.device)
        self.flat = self._all[:n_pad]               # the parameter gradients; the pose region follows it
        self._zeros = {}
        self.received = None                         # per parameter: the last backward() produced a gradient for it
        off, self.views = 0, []
        for p in self.params:
            self.views.append(self.flat[off:off + p.numel()].view_as(p))
            p.grad = self.views[-1]
            off += p.numel()

    def zero_(self):
        """the classic protocol: zero the bucket and make the .grad attributes its views again (a backward(gather=False) leaves
        autograd's own tensors there), so that a plain loss.backward() accumulates into the bucket"""
        self.flat.zero_()
        for p, v in zip(self.params, self.views):
            p.grad = v

    def backward(self, total, gather=True, poses=()):
        """Back-propagate `total` and leave every parameter's gradient in the flat bucket with ONE gather kernel: the
        parameters enter the backward without .grad, so autograd hands over each gradient tensor as it is (no zero-fill
        of the bucket, no accumulate-add per parameter); a single cat then writes them into the flat buffer and the
        .grad attributes become the bucket views again.  CUDA-graph capturable.  gather=False stops after the backward:
        the .grad attributes are autograd's own tensors and the flat buffer is not written (no collective reads it).
        poses: the step's camera leaves (R (B,3,3), T (B,3)[, intrinsics (B,4)]); the same cat writes their gradients into the
        pose region"""
        for p in (*self.params, *poses):
            p.grad = None
        total.backward()
        self.received = [p.grad is not None for p in self.params]      # before the gather gives every parameter a bucket view
        if not gather:
            return
        pieces = [(p.grad if p.grad is not None else self._zero(p.numel())).reshape(-1) for p in self.params]
        n = self.n                                       # a None gradient: unused in this phase (e.g. frozen opacities)
        if poses:
            if self.flat.numel() > n:
                pieces.append(self._zero(self.flat.numel() - n))
            pieces += [(q.grad if q.grad is not None else self._zero(q.numel())).reshape(-1) for q in poses]
            n = self.flat.numel() + sum(q.numel() for q in poses)
        with torch.no_grad():
            torch.cat(pieces, out=self._all[:n])
        for p, v in zip(self.params, self.views):
            p.grad = v
        o = self.flat.numel()
        for q in poses:
            q.grad = self._all[o:o + q.numel()].view_as(q)
            o += q.numel()

    def _zero(self, n):
        if n not in self._zeros:
            self._zeros[n] = torch.zeros(n, dtype=self.flat.dtype, device=self.flat.device)
        return self._zeros[n]

    def grads_flat(self):
        """the gradients as one flat vector in bucket order, whichever way the last backward left them"""
        return torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in self.params])

    def all_reduce(self, group=None, pose_views=0, intrinsics=False):
        """sum the bucket over the ranks; pose_views: the pose gradients of that many views ride in the same collective
        (intrinsics: and their intrinsics gradients)"""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            buf = self._all[:self.flat.numel() + (16 if intrinsics else 12) * pose_views]
            if self.peer is not None:
                self.peer.all_reduce(buf)
            else:
                dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)

    @property
    def nbytes(self):
        return self.flat.numel() * self.flat.element_size()


class ViewParallel:
    """Wraps a model whose `forward(inp, labels)` returns a dict of losses incl. 'total' (the DBW contract,
    src/trainer.py:141-143) and which exposes `n_total_views` and `noise_generator` attributes."""

    VIEW_KEYS = ('imgs', 'R', 'T', 'K')

    def __init__(self, model, group=None, seed=227391, row_bands=False, collective='nccl', reduce_at='auto', gather_grads=None,
                 peer_factory=None, max_pose_views=0, intrinsics=False):
        """collective: 'nccl' (torch.distributed all_reduce; also what gloo groups use), 'p2p' (the NVLink peer-memory kernel
        of csrc/dbw_comm.cu, CUDA-graph capturable) or 'auto' (p2p if it initialises on this node, else nccl).
        reduce_at: 'leaf' (all-reduce the parameter gradients after the backward), 'scene' (sum the gradients of the scene
        tensors inside the backward, GradSumPoint: needs the peer-memory collective; applies while the model's textures are
        decimated on its fused-loss path, see can_sum_gradients_at_scene_tensors) or 'auto' (scene whenever it applies,
        leaf otherwise -- decided per step).
        gather_grads: gather the gradients into bucket.flat (and make the .grad attributes views of it) after every backward;
        None: only when a leaf all-reduce reads the bucket (world > 1 and no reduction inside the backward) -- otherwise the
        .grad attributes are autograd's own tensors and bucket.grads_flat() concatenates them on demand.
        peer_factory(n_floats, device) -> object with `.flat` (the bucket) and `.all_reduce(prefix_of_flat)`: replaces the
        peer-memory arena (tests run the scene-level reduction over gloo with it).
        max_pose_views: 0 refuses camera poses that require grad; N > 0 reserves 12 N floats of the bucket / arena and accepts
        them on steps of at most N views.  Such a step takes FULL-BATCH inputs (all views' imgs, K, R, T, identical on every
        rank) and leaves the gradient of the global loss with respect to all B views' poses in the caller's graph, the same
        on every rank (pose_step).
        intrinsics: with max_pose_views = N > 0, reserve 4 N more floats and accept a K (B,4,4) that requires grad likewise: its
        (fx, fy, px, py) entries receive the gradient of the global loss (the model renders such a step per view)"""
        self.model, self.group, self.seed = model, group, seed
        self.max_pose_views = int(max_pose_views)
        self.intrinsics = bool(intrinsics) and self.max_pose_views > 0
        if intrinsics and not self.intrinsics:
            raise ValueError('ViewParallel: intrinsics=True needs max_pose_views > 0 (the views whose gradients it reserves room for)')
        cam_floats = (16 if self.intrinsics else 12) * self.max_pose_views
        self.reduce_at, self.gather_grads = reduce_at, gather_grads
        self.row_bands = row_bands          # shard at (view, row band) granularity (needs the model's fused-loss path)
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world_size = dist.get_world_size(group) if dist.is_initialized() else 1
        def arena_factory(n_floats, device):
            if not (self.world_size > 1 and collective in ('p2p', 'auto') and device.type == 'cuda'):
                return None
            try:
                return PeerAllReduce(n_floats, device, group)
            except Exception as exc:          # e.g. no peer access between the GPUs of this node
                if collective == 'p2p':
                    raise
                print(f'[dbw_b200] peer-memory all-reduce unavailable ({exc}); using NCCL')
                return None

        want_point = reduce_at in ('scene', 'auto') and hasattr(model, 'grad_sum_floats')
        self.bucket = GradBucket(model.parameters(), peer_factory or arena_factory,
                                 model.grad_sum_floats() + cam_floats if want_point else 0, self.max_pose_views, self.intrinsics)
        self.sum_point = GradSumPoint(self.bucket.peer) if (want_point and self.bucket.peer is not None) else None
        if reduce_at == 'scene' and self.sum_point is None and self.world_size > 1:
            raise RuntimeError("reduce_at='scene' needs the peer-memory collective (collective='p2p' or 'auto') and a model with grad_sum_floats()")
        self._step = 0
        self.collective_name = 'none (1 rank)' if self.world_size == 1 else 'ncclAllReduce'
        if self.bucket.peer is not None:
            self.collective_name = 'hand-written NVLink peer-memory push kernel (dbw_comm_all_reduce), inside the CUDA graph'

    @property
    def graph_capturable_collective(self):
        return self.bucket.peer is not None

    def shard(self, inp):
        """this rank's part of a batch: whole views, or -- with row_bands -- the views it touches plus `rows` (B_local, 2):
        the [row_begin, row_end) of each that it renders (the model hands them to the kernels, dbw_render.h view_rows)"""
        B = len(inp['imgs'])
        sl, rows = self.views(B, inp['imgs'].shape[-2])
        out = self.take(inp, sl, B)
        if rows is not None:
            out['rows'] = rows.to(inp['imgs'].device)          # where the kernels read them: beside the images
        return out, B

    def views(self, n_views, height):
        """this rank's views of a step (a slice) and, with row_bands, the (B_local, 2) rows it renders of each (else None)"""
        if self.row_bands and self.world_size > 1:
            pieces = shard_row_bands(n_views, height, self.world_size, self.rank)
            idx = [v for v, _, _ in pieces]
            sl = slice(idx[0], idx[-1] + 1) if idx else slice(0, 0)
            return sl, torch.tensor([[a, b] for _, a, b in pieces], dtype=torch.int32).reshape(-1, 2)
        return shard_views(n_views, self.world_size, self.rank), None

    def take(self, inp, views, n_views):
        """inp with every per-view tensor of the n_views-view step sliced to `views`"""
        out = dict(inp)
        for k in self.VIEW_KEYS:
            if k in inp and torch.is_tensor(inp[k]) and inp[k].shape[:1] == (n_views,):
                out[k] = inp[k][views]
        return out

    def check_pose_views(self, inp, who):
        """a step whose poses require grad: refused unless this wrapper reserved room for at least its B views"""
        if self.max_pose_views == 0:
            refuse_camera_gradients(inp, who)
        if not self.intrinsics:
            refuse_camera_gradients(inp, who, intrinsics_only=True)
        B = len(inp['imgs'])
        if B > self.max_pose_views:
            raise ValueError(f'{who}: a step of {B} views with camera-pose gradients, but the ViewParallel reserved room for '
                             f'max_pose_views={self.max_pose_views}')
        for k, shape in (('R', (B, 3, 3)), ('T', (B, 3)), ('K', (B, 4, 4))):
            if k == 'K' and not wants_intrinsics_gradients(inp):
                continue
            if tuple(inp[k].shape) != shape:
                raise ValueError(f"{who}: with camera-pose gradients inp['{k}'] is the full batch {shape}, got {tuple(inp[k].shape)}")

    def pose_leaves(self, inp):
        """(R, T, views, intrinsics): leaves holding the values of inp's full-batch poses -- and, when inp['K'] requires grad, of
        its (B,4) (fx, fy, px, py), else None -- which the step renders its shard from"""
        from .renderer import intrinsics_of
        B = len(inp['imgs'])
        leaf = lambda t: t.detach().to(torch.float32, copy=True).requires_grad_(True)
        intr = leaf(intrinsics_of(inp['K'])) if wants_intrinsics_gradients(inp) else None
        return leaf(inp['R']), leaf(inp['T']), self.views(B, inp['imgs'].shape[-2])[0], intr

    @staticmethod
    def pose_grads(poses):
        return [q.grad if q.grad is not None else torch.zeros_like(q) for q in camera_leaves(poses)]

    def _sync_rng(self, device):
        g = getattr(self.model, 'noise_generator', None)
        if g is None or g.device != torch.device(device):
            g = torch.Generator(device=device)
            self.model.noise_generator = g
        g.manual_seed(self.seed + self._step)      # identical on every rank, fresh every step

    def reduces_inside_backward(self, inp):
        """this step's gradients are summed over the ranks inside the backward, at the scene tensors (GradSumPoint)"""
        return self.sum_point is not None and self.model.can_sum_gradients_at_scene_tensors(inp['imgs'])

    def local_step(self, inp, labels, n_total_views, collective=True, poses=None):
        """forward + backward over this rank's shard.  Returns (losses, reduced): reduced = the gradients are already the
        sum over ranks (the GradSumPoint ran inside the backward); otherwise a leaf all-reduce of the bucket is due.
        collective=False on a step that would reduce inside the backward leaves LOCAL gradients (timing breakdowns only).
        poses: (R, T, views) of pose_leaves(): the shard renders from R[views], T[views]; the leaves' (B-row) gradients go
        through the GradSumPoint with the scene tensors, or into the bucket's pose region for the leaf all-reduce."""
        if poses is None:
            refuse_camera_gradients(inp, 'ViewParallel')
        inside = self.reduces_inside_backward(inp)
        self.model.n_total_views = n_total_views
        self.model.grad_sum_point = self.sum_point if (inside and collective) else None
        if poses is not None:
            R, T, views, intr = poses
            if self.model.grad_sum_point is not None:          # the model renders from sum_point.cameras() / intrinsics()
                self.sum_point.ride(poses)
                inp = dict(inp, R=R.detach()[views], T=T.detach()[views])
                if intr is not None and 'K' in inp:
                    inp['K'] = inp['K'].detach()
            else:
                inp = dict(inp, R=R[views], T=T[views])
                if intr is not None:                             # a K that requires grad: the model renders per view
                    inp['K'] = intrinsics_matrix(intr[views])
        try:
            losses = self.model(inp, labels)
            gather = self.gather_grads if self.gather_grads is not None else (self.world_size > 1 and not inside)
            self.bucket.backward(self.weighted_total(losses, len(inp['imgs']), n_total_views, replicated_everywhere=inside),
                                 gather=gather, poses=camera_leaves(poses) if poses is not None else ())
        finally:
            self.model.grad_sum_point = None
            if self.sum_point is not None:
                self.sum_point.ride(None)
        return losses, inside and collective

    def forward_backward(self, inp, labels=None, already_sharded=False, n_total_views=None, all_reduce=True):
        """local forward -> backward -> ONE all-reduce (inside the backward or after it).  Returns the (local) loss dict.
        With poses that require grad (max_pose_views > 0) inp is the full batch; the pose gradient of the global loss is
        back-propagated into the caller's graph behind inp['R'] / inp['T'] before returning."""
        full, poses = inp, None
        if wants_pose_gradients(inp):
            self.check_pose_views(inp, 'ViewParallel')
            if already_sharded:
                raise ValueError('ViewParallel: a step with camera-pose gradients takes the full batch (already_sharded=False)')
            poses = self.pose_leaves(inp)
        if not already_sharded:
            inp, n_total_views = self.shard(inp)
        self._sync_rng(inp['imgs'].device)
        self._step += 1
        losses, reduced = self.local_step(inp, labels, n_total_views, collective=all_reduce, poses=poses)
        if all_reduce and not reduced:
            self.bucket.all_reduce(self.group, pose_views=n_total_views if poses is not None else 0,
                                   intrinsics=poses is not None and poses[3] is not None)
        if poses is not None:
            pose_backward(full, self.pose_grads(poses))
        return losses

    def weighted_total(self, losses, n_local_views, n_total_views, replicated_everywhere=False):
        """the scalar each rank back-propagates: its share of the per-view terms + the replicated terms (regularisers:
        identical on every rank) at 1/world when a leaf all-reduce will sum them, at 1 when no leaf all-reduce follows"""
        shared = [v for k, v in losses.items() if k not in ('rgb', 'perceptual', 'total')]
        total = losses['rgb'] if 'rgb' in losses else 0.
        if 'perceptual' in losses:
            total = total + losses['perceptual'] * (n_local_views / float(n_total_views))
        if shared:
            total = total + sum(shared) / (1 if replicated_everywhere else self.world_size)
        return total
