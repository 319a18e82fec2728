"""View-sharded data parallelism for one optimisation step (new functionality: the reference has no distributed path
that runs, SURVEY.md section 0 item 5 and section 8e).

Views of a step are independent given the replicated scene parameters, so they shard with NO data-path collective:
rank r renders a contiguous range of the B views (or of their 16-row bands) and back-propagates into its own gradients;
ONE all-reduce(SUM) per step over NVLink / NVSwitch then gives every rank the full gradient -- either of a single flat
fp32 bucket of the parameter gradients after the backward (about 9.4 MB for 10 blocks with 256^2 textures), or, while the
textures are box-decimated, of the scene tensors' gradients inside the backward (GradSumPoint: about 0.16 MB).
Correctness conditions handled here:
  * the RGB loss is a MEAN over all B views (dbw.py:367): each rank divides by the GLOBAL pixel count
    (model.n_total_views), so the SUM of the per-rank gradients is the gradient of the global mean;
  * view-independent terms (parsimony / TV / overlap, dbw.py:373-405) are computed identically on every rank: divided by
    the world size before a leaf SUM, counted once when the SUM happens at the scene tensors (they do not pass through it);
  * the opacity noise (dbw.py:300-301) and the overlap sample points (dbw.py:393) come from a generator that every
    rank seeds identically at every step."""
import ctypes

import torch
import torch.distributed as dist

from . import _lib


def shard_views(n_views, world_size, rank):
    """Contiguous, balanced view ranges: the first n_views % world_size ranks get one extra view (49 -> 7,6,6,6,6,6,6,6)."""
    base, extra = divmod(n_views, world_size)
    start = rank * base + min(rank, extra)
    return slice(start, start + base + (1 if rank < extra else 0))


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
    331-334) the cells hold 64x fewer values than the texture parameters: ~0.15 MB per step instead of ~9.4 MB on the DTU shape."""

    def __init__(self, peer):
        self.peer = peer

    def __call__(self, *tensors):
        return _GradSumFn.apply(self, *tensors)

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

    def __init__(self, params, peer_factory=None, min_floats=0):
        """peer_factory(n_floats, device) -> PeerAllReduce or None: when given and successful, the flat buffer IS the peer-memory
        arena's bucket (csrc/dbw_comm.cu) and all_reduce() is its kernel; else a plain tensor and torch.distributed.
        min_floats: capacity the arena needs for its other user (GradSumPoint)"""
        self.params = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        ref = self.params[0]
        self.n = n
        n_pad = (n + 3) // 4 * 4                     # padded: 128-bit all-reduce lanes
        self.peer = peer_factory(max(n_pad, (int(min_floats) + 3) // 4 * 4), ref.device) if peer_factory is not None else None
        if self.peer is not None:
            self.peer.flat.zero_()
            self.flat = self.peer.flat[:n_pad]
        else:
            self.flat = torch.zeros(n_pad, dtype=ref.dtype, device=ref.device)
        self._zeros = {}
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

    def backward(self, total, gather=True):
        """Back-propagate `total` and leave every parameter's gradient in the flat bucket with ONE gather kernel: the
        parameters enter the backward without .grad, so autograd hands over each gradient tensor as it is (no zero-fill
        of the bucket, no accumulate-add per parameter); a single cat then writes them into the flat buffer and the
        .grad attributes become the bucket views again.  CUDA-graph capturable.  gather=False stops after the backward:
        the .grad attributes are autograd's own tensors and the flat buffer is not written (no collective reads it)."""
        for p in self.params:
            p.grad = None
        total.backward()
        if not gather:
            return
        pieces = []
        for p in self.params:
            g = p.grad
            if g is None:                                # unused in this phase (e.g. opacities once they are frozen)
                if id(p) not in self._zeros:
                    self._zeros[id(p)] = torch.zeros(p.numel(), dtype=self.flat.dtype, device=self.flat.device)
                g = self._zeros[id(p)]
            pieces.append(g.reshape(-1))
        with torch.no_grad():
            torch.cat(pieces, out=self.flat[:self.n])
        for p, v in zip(self.params, self.views):
            p.grad = v

    def grads_flat(self):
        """the gradients as one flat vector in bucket order, whichever way the last backward left them"""
        return torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in self.params])

    def all_reduce(self, group=None):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            if self.peer is not None:
                self.peer.all_reduce(self.flat)
            else:
                dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)

    @property
    def nbytes(self):
        return self.flat.numel() * self.flat.element_size()


class ViewParallel:
    """Wraps a model whose `forward(inp, labels)` returns a dict of losses incl. 'total' (the DBW contract,
    src/trainer.py:141-143) and which exposes `n_total_views` and `noise_generator` attributes."""

    VIEW_KEYS = ('imgs', 'R', 'T', 'K')

    def __init__(self, model, group=None, seed=227391, row_bands=False, collective='nccl', reduce_at='auto', gather_grads=None,
                 peer_factory=None):
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
        peer-memory arena (tests run the scene-level reduction over gloo with it)"""
        self.model, self.group, self.seed = model, group, seed
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
        self.bucket = GradBucket(model.parameters(), peer_factory or arena_factory, model.grad_sum_floats() if want_point else 0)
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
        out = dict(inp)
        if self.row_bands and self.world_size > 1:
            pieces = shard_row_bands(B, inp['imgs'].shape[-2], self.world_size, self.rank)
            idx = [v for v, _, _ in pieces]
            sl = slice(idx[0], idx[-1] + 1) if idx else slice(0, 0)
            out['rows'] = torch.tensor([[a, b] for _, a, b in pieces], dtype=torch.int32).reshape(-1, 2)
        else:
            sl = shard_views(B, self.world_size, self.rank)
        for k in self.VIEW_KEYS:
            if k in inp and torch.is_tensor(inp[k]) and inp[k].shape[:1] == (B,):
                out[k] = inp[k][sl]
        return out, B

    def _sync_rng(self, device):
        g = getattr(self.model, 'noise_generator', None)
        if g is None or g.device != torch.device(device):
            g = torch.Generator(device=device)
            self.model.noise_generator = g
        g.manual_seed(self.seed + self._step)      # identical on every rank, fresh every step

    def reduces_inside_backward(self, inp):
        """this step's gradients are summed over the ranks inside the backward, at the scene tensors (GradSumPoint)"""
        return self.sum_point is not None and self.model.can_sum_gradients_at_scene_tensors(inp['imgs'])

    def local_step(self, inp, labels, n_total_views, collective=True):
        """forward + backward over this rank's shard.  Returns (losses, reduced): reduced = the gradients are already the
        sum over ranks (the GradSumPoint ran inside the backward); otherwise a leaf all-reduce of the bucket is due.
        collective=False on a step that would reduce inside the backward leaves LOCAL gradients (timing breakdowns only)."""
        inside = self.reduces_inside_backward(inp)
        self.model.n_total_views = n_total_views
        self.model.grad_sum_point = self.sum_point if (inside and collective) else None
        try:
            losses = self.model(inp, labels)
            gather = self.gather_grads if self.gather_grads is not None else (self.world_size > 1 and not inside)
            self.bucket.backward(self.weighted_total(losses, len(inp['imgs']), n_total_views, replicated_everywhere=inside),
                                 gather=gather)
        finally:
            self.model.grad_sum_point = None
        return losses, inside and collective

    def forward_backward(self, inp, labels=None, already_sharded=False, n_total_views=None, all_reduce=True):
        """local forward -> backward -> ONE all-reduce (inside the backward or after it).  Returns the (local) loss dict."""
        if not already_sharded:
            inp, n_total_views = self.shard(inp)
        self._sync_rng(inp['imgs'].device)
        self._step += 1
        losses, reduced = self.local_step(inp, labels, n_total_views, collective=all_reduce)
        if all_reduce and not reduced:
            self.bucket.all_reduce(self.group)
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
