"""Whole-step CUDA graph: zero the gradient bucket, build the scene, render both passes, composite + loss, and
back-propagate to every leaf parameter -- captured once on static buffers and replayed per step.  The step is a few
hundred kernel launches of 2-100 us each (scene construction, two rasterization passes, their backward, the
reductions); replaying them as one graph removes the launch gaps and the Python/autograd dispatch that otherwise cost
more than the kernels themselves.  Requires the model's static-topology mode (dbw.py): no host synchronisation and no
shape that depends on parameter values inside forward().

Camera-pose gradients (a ViewParallel built with max_pose_views > 0, and poses that require grad in example_inp): the inputs
are the full batch; the step keeps this rank's slice of the per-view inputs and the full-batch poses as static LEAF buffers
that require grad, renders from their slices inside the graph, and after each replay back-propagates the (summed) pose
gradient into the caller's graph behind run()'s inp['R'] / inp['T'] -- a small eager backward outside the graph.

The parameter update (GraphedStep(optimizer=BucketAdam)): the optimiser's one launch (optim.py) is captured after the point
where the gradients are final -- the captured all-reduce, or the backward when the sum happens inside it or there is one rank
-- so one replay is one training iteration.  Every rank applies the same elementwise update to the same summed gradients.  The
learning rates are read on the device: a scheduler changes them between replays without a new capture.

Per-view intrinsics (model.set_per_view_intrinsics(True)): inp['K'] is one of the static inputs, copied in before each replay, so
a batch with other intrinsics is rendered with them without a new capture.  Intrinsics gradients (a ViewParallel built with
intrinsics=True, and a K that requires grad in example_inp): (fx, fy, px, py) of the full batch become one more static leaf
beside the poses, and its summed gradient is back-propagated into the caller's K after the replay.

Captured gather (GraphedStep(views=data.DeviceViews)): the step's inputs are gathered from views resident on the device by a
launch captured at the head of the graph, from a static buffer of B view indices.  run(items=...) writes the B dataset item
indices of the batch there, one small host-to-device copy, and replays: no image crosses the bus.  The inputs are then exactly
those DeviceLoader would have handed to run(inp).  Not combined with camera-pose gradients."""
import torch

from .optim import BucketAdam
from .parallel import (camera_leaves, pose_backward, refuse_camera_gradients, wants_intrinsics_gradients, wants_pose_gradients)
from .renderer import intrinsics_of


class GraphedStep:
    def __init__(self, view_parallel, example_inp, n_total_views, warmup=3, capture_all_reduce=None, generator=None, optimizer=None,
                 views=None):
        self.vp, self.model = view_parallel, view_parallel.model
        if optimizer is not None and not isinstance(optimizer, BucketAdam):
            raise TypeError('GraphedStep: only an optim.BucketAdam can be captured (its launch reads rates and counters on the device)')
        self.optimizer = optimizer
        self.pose = None                   # (R, T, views): static full-batch pose leaves and this rank's views of them
        if wants_pose_gradients(example_inp):
            view_parallel.check_pose_views(example_inp, 'GraphedStep')
            if n_total_views != len(example_inp['imgs']):
                raise ValueError('GraphedStep: with camera-pose gradients example_inp is the full batch of n_total_views views')
            self.pose = view_parallel.pose_leaves(example_inp)
            example_inp = {k: v for k, v in view_parallel.shard(example_inp)[0].items() if k not in self._leaf_keys}
        # The gradient all-reduce is captured INTO the graph when it is the peer-memory kernel (a plain launch).  An
        # ncclAllReduce is issued right after the replay instead: captured, it hung on 2 GPUs with this image's NCCL (round 1).
        if capture_all_reduce is None:
            capture_all_reduce = view_parallel.graph_capturable_collective
        self.capture_all_reduce = capture_all_reduce and view_parallel.world_size > 1
        if optimizer is not None and view_parallel.world_size > 1 and not self.capture_all_reduce:
            raise RuntimeError('GraphedStep: with an optimizer the gradient sum must be captured too (capture_all_reduce=True, the '
                               'peer-memory collective): a collective issued after the replay would come after the update')
        self.n_total = n_total_views
        dev = example_inp['imgs'].device
        self.static_inp = {k: v.clone() for k, v in example_inp.items()}
        self.views, self.view_index = views, None
        if views is not None:
            if self.pose is not None:
                raise ValueError('GraphedStep: a captured gather (views=...) cannot be combined with camera-pose gradients')
            if set(self.static_inp) != {'imgs', 'K', 'R', 'T'}:
                raise ValueError(f"GraphedStep: with views=..., example_inp holds exactly imgs, K, R and T, got {sorted(self.static_inp)}")
            self.view_index = torch.zeros(len(self.static_inp['imgs']), dtype=torch.int64, device=dev)
            views.check_batch(self.static_inp, len(self.view_index))     # refuses buffers whose shapes or dtypes differ
        self.model.n_total_views = n_total_views
        # random inputs of a step are pre-drawn into buffers OWNED BY THIS STEP (a graph captures addresses): the opacity
        # noise (dbw.py:300-301) and the overlap term's sample points (dbw.py:393).  `generator` is shared by the steps of a
        # PipelinedGraphedStep so that consecutive steps draw consecutive numbers; every rank seeds it identically.
        self.noise_buf = torch.zeros_like(self.model.alpha_logit)
        from .losses import OVERLAP_N_POINTS
        self.overlap_buf = (torch.zeros(self.model.n_blocks, OVERLAP_N_POINTS, 3, device=dev)
                            if 'overlap' in self.model.loss_weights else None)
        self.gen = generator
        if self.gen is None:
            self.gen = torch.Generator(device=dev)
            self.gen.manual_seed(self.vp.seed)
        self.model._install_cameras(self.static_inp)          # the one-off host read of the intrinsics happens here
        self.segment_table = optimizer.new_segment_table() if optimizer is not None else None
        self._capture(warmup=warmup)

    def _phase(self):
        """what the captured control flow depends on: the training-schedule switches of dbw.py:210-212,276,331-334"""
        m = self.model
        frozen = self.optimizer.captured_constants() if self.optimizer is not None else ()      # a capture holds them by value
        return (m.training, m.is_live('coarse_learning'), m.is_live('decimate_txt'), m.is_live('kill_blocks'), m.per_view_intrinsics,
                *frozen)

    def _bind_buffers(self):
        self.model.opacity_noise_buffer, self.model.overlap_samples_buffer = self.noise_buf, self.overlap_buf
        self.model.noise_generator = None          # nothing draws inside the captured region

    def _capture(self, warmup=1):
        self.phase = self._phase()
        self._bind_buffers()
        # the parameters (and their AccumulateGrad nodes) were created on the default stream, the capture runs on a side
        # stream: intended, and ordered by the wait_stream calls below -- silence autograd's stream-mismatch warning
        _warn_off = getattr(torch.autograd.graph, 'set_warn_on_accumulate_grad_stream_mismatch', None)
        if _warn_off is not None:
            _warn_off(False)
        side = torch.cuda.Stream()                 # eager run(s) of the new control flow first (lazy state, allocator warm-up)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._body()
        torch.cuda.current_stream().wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.losses = self._body()
        # the gradient tensors THIS capture writes (bucket views when the gradients are gathered, else tensors of the graph's
        # private pool): another GraphedStep on the same model (PipelinedGraphedStep) leaves its own in the .grad attributes
        self.grads = [p.grad for p in self.vp.bucket.params]
        if self.optimizer is not None:
            # the records the captured launch reads, written now that the capture has fixed the gradients' addresses; a parameter
            # is active when this phase's backward gave it a gradient (torch.optim skips a .grad that is None: hard opacities
            # leave alpha_logit alone, whereas the bucket's zeros would keep moving it on old momentum)
            got = {id(p) for p, r in zip(self.vp.bucket.params, self.vp.bucket.received) if r}
            self.optimizer.write_segments(self.segment_table, [p.grad for p in self.optimizer.params],
                                          active=[id(p) in got for p in self.optimizer.params])
        self.pose_grads = self.vp.pose_grads(self.pose) if self.pose is not None else None

    def _body(self):
        if self.views is not None:
            self.views.launch_gather(self.view_index, self.static_inp)
        losses, reduced = self.vp.local_step(self.static_inp, None, self.n_total, collective=self.capture_all_reduce, poses=self.pose)
        self.inside = self.vp.reduces_inside_backward(self.static_inp)      # the collective sits INSIDE the backward (parallel.GradSumPoint)
        if self.capture_all_reduce and not reduced:
            self.vp.bucket.all_reduce(self.vp.group, pose_views=self._pose_views, intrinsics=self._intrinsics_leaf)
        if self.optimizer is not None and torch.cuda.is_current_stream_capturing():      # the warm-up runs must not train
            self.optimizer.launch(self.segment_table)
        return losses

    @property
    def _pose_views(self):
        return self.n_total if self.pose is not None else 0

    @property
    def _intrinsics_leaf(self):
        return self.pose is not None and self.pose[3] is not None

    @property
    def _leaf_keys(self):
        """the inputs held as static leaves rather than copied into static inputs"""
        return ('R', 'T', 'K') if self._intrinsics_leaf else ('R', 'T')

    def check_poses(self, inp):
        """poses (and K) in `inp` must require grad exactly when this step was captured with their gradients"""
        if inp is None or not any(k in inp for k in ('R', 'T', 'K')):
            return
        if self.pose is None and wants_pose_gradients(inp):
            if self.vp.max_pose_views == 0:
                refuse_camera_gradients(inp, 'GraphedStep')
            raise RuntimeError('GraphedStep: these cameras require grad, but the step was captured with cameras that do not; '
                               'build the step from an example whose cameras require grad')
        if 'K' in inp and wants_intrinsics_gradients(inp) != self._intrinsics_leaf:
            if not self.vp.intrinsics:
                refuse_camera_gradients(inp, 'GraphedStep', intrinsics_only=True)
            raise RuntimeError(f"GraphedStep: inp['K'].requires_grad is {wants_intrinsics_gradients(inp)}, but the step was captured "
                               f"with {self._intrinsics_leaf}; build the step from an example whose K matches")
        if self.pose is not None and not wants_pose_gradients(inp):
            raise RuntimeError('GraphedStep: the step was captured with cameras that require grad, but these do not')

    def staged(self, inp):
        """[(static buffer, value)] for the tensors of `inp` that a run copies into the static inputs: with pose gradients,
        this rank's slice of the full-batch per-view tensors; the poses themselves are not among them (load_poses)"""
        if self.pose is not None:
            inp = self.vp.take({k: v for k, v in inp.items() if k not in self._leaf_keys}, self.pose[2], self.n_total)
        return [(self.static_inp[k], v) for k, v in inp.items() if k in self.static_inp]

    def load_poses(self, inp, non_blocking=True):
        """copy inp's full-batch poses (and intrinsics) into the static camera leaves (on the current stream)"""
        with torch.no_grad():
            for k, leaf in zip(('R', 'T'), self.pose[:2]):
                if k in inp:
                    leaf.copy_(inp[k].detach(), non_blocking=non_blocking)
            if self._intrinsics_leaf and 'K' in inp:
                self.pose[3].copy_(intrinsics_of(inp['K'].detach()), non_blocking=non_blocking)

    def run(self, inp=None, non_blocking=True, all_reduce=True, items=None):
        """inp: optional dict of (host or device) tensors for this step, copied into the static buffers.
        all_reduce=False skips the collective when it is issued after the replay (a captured one always runs).
        With an optimizer the replay also applies the update, at the learning rates param_groups hold now.
        With pose gradients, inp holds the full batch, and the summed pose gradient is back-propagated into the graph
        behind inp['R'] / inp['T'] (without them, it stays in the static leaves' .grad).
        items: with views=..., the dataset item indices of this step's batch, gathered inside the graph (a host sequence or
        tensor; a CUDA tensor is read back to the host first, a synchronisation)."""
        self.check_poses(inp)
        if self.views is not None and inp is not None:
            raise ValueError('GraphedStep: this step gathers its inputs inside the graph; pass run(items=...), not inp')
        if items is not None:
            if self.views is None:
                raise ValueError('GraphedStep: run(items=...) needs a step built with views=... (a captured gather)')
            idx = self.views.item_views[torch.as_tensor(items, dtype=torch.int64).cpu()]
            if idx.shape != self.view_index.shape:
                raise ValueError(f'GraphedStep: {len(idx)} items, but the step was captured for {len(self.view_index)} views')
            self.view_index.copy_(idx.pin_memory(), non_blocking=non_blocking)
        if self.optimizer is not None and not all_reduce and self.vp.world_size > 1:
            raise RuntimeError('GraphedStep: run(all_reduce=False) with an optimizer would update from gradients that are not summed')
        if inp is not None:
            if self.pose is not None:
                self.load_poses(inp, non_blocking)
            for buf, v in self.staged(inp):
                buf.copy_(v, non_blocking=non_blocking)
        if self._phase() != self.phase:          # a schedule milestone was crossed (coarse -> fine, decimation off): re-capture
            self._capture()
        self._bind_buffers()                       # eager code in between (evaluation, another GraphedStep) may have re-pointed them
        self.noise_buf.normal_(generator=self.gen)                      # identical on every rank (same seed, same count)
        if self.overlap_buf is not None:
            self.overlap_buf.uniform_(generator=self.gen)
        if self.optimizer is not None:
            self.optimizer.prepare_replay()
        self.graph.replay()
        for p, g in zip(self.vp.bucket.params, self.grads):
            p.grad = g
        if self.pose is not None:
            for q, g in zip(camera_leaves(self.pose), self.pose_grads):
                q.grad = g
        if not self.capture_all_reduce and all_reduce and self.vp.world_size > 1:
            if self.inside:
                raise RuntimeError('this step sums its gradients inside the backward (parallel.GradSumPoint) but was captured '
                                   'with capture_all_reduce=False: its gradients are local and cannot be reduced afterwards')
            self.vp.bucket.all_reduce(self.vp.group, pose_views=self._pose_views, intrinsics=self._intrinsics_leaf)
        if self.pose is not None and inp is not None:
            pose_backward(inp, self.pose_grads)
        return self.losses


class PipelinedGraphedStep:
    """Two GraphedSteps on alternating static input buffers: while step i replays, the inputs of step i+1 are copied
    host->device on a side stream (what a prefetching DataLoader does for src/trainer.py:141).  `run(host_inp)` returns
    the losses of the step that consumed `host_inp`.  Poses that require grad are NOT prefetched: an optimiser step may
    change them between the prefetch and the step that consumes them, so they are copied into that step's static leaves on
    the current stream right before its replay."""

    def __init__(self, view_parallel, example_inp, n_total_views, capture_all_reduce=None, optimizer=None):
        if wants_pose_gradients(example_inp):
            view_parallel.check_pose_views(example_inp, 'PipelinedGraphedStep')
        gen = torch.Generator(device=example_inp['imgs'].device)
        gen.manual_seed(view_parallel.seed)
        self.steps = [GraphedStep(view_parallel, example_inp, n_total_views, capture_all_reduce=capture_all_reduce, generator=gen,
                                  optimizer=optimizer)
                      for _ in range(2)]
        self.copy_stream = torch.cuda.Stream()
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]      # inputs of buffer b have landed
        self.free = [torch.cuda.Event(), torch.cuda.Event()]       # buffer b has been consumed by its replay
        self.i = 0
        self.primed = False

    def _stage(self, b, host_inp):
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.free[b])
            for buf, v in self.steps[b].staged(host_inp):
                buf.copy_(v, non_blocking=True)
            self.ready[b].record(self.copy_stream)

    def run(self, host_inp, next_host_inp=None, all_reduce=True):
        """consume `host_inp` (staged now unless it was prefetched as the previous call's `next_host_inp`) and
        prefetch `next_host_inp` for the following call."""
        for x in (host_inp, next_host_inp):
            self.steps[0].check_poses(x)
        b = self.i % 2
        cur = torch.cuda.current_stream()
        if not self.primed:
            self.free[0].record(cur)
            self.free[1].record(cur)
            self._stage(b, host_inp)
            self.primed = True
        if next_host_inp is not None:
            self._stage(1 - b, next_host_inp)
        else:
            self.primed = False
        cur.wait_event(self.ready[b])
        poses = None
        if self.steps[b].pose is not None:          # the poses as they are now, not as they were at the prefetch
            poses = {k: host_inp[k] for k in self.steps[b]._leaf_keys if k in host_inp}
        losses = self.steps[b].run(poses, all_reduce=all_reduce)
        self.free[b].record(cur)
        self.i += 1
        return losses


class GraphedModel:
    """A captured step with its optimiser, behind the call sequence of the reference's training loop (src/trainer.py:137-147:
    `optimizer.zero_grad(); loss = model(inp, labels); loss['total'].backward(); optimizer.step()`), which cannot call
    step.run().  The call replays the step, update included; the `total` it returns back-propagates into nothing, and the
    BucketAdam skips the step() call that follows.  Everything else (train(), step(), predict(), state_dict(), ...) is the
    wrapped model's."""

    def __init__(self, step):
        if step.optimizer is None:
            raise ValueError('GraphedModel: the step must be built with an optimizer')
        self.graphed_step, self.model = step, step.model

    def __getattr__(self, name):
        if name in ('model', 'graphed_step'):          # not set yet (copying, unpickling): no delegation to a missing model
            raise AttributeError(name)
        return getattr(self.model, name)

    def __call__(self, inp, labels=None):
        step = self.graphed_step
        if not self.model.training:
            raise RuntimeError('GraphedModel: the captured step is a training iteration; call the model itself to evaluate')
        if len(inp['imgs']) != len(step.static_inp['imgs']):
            raise ValueError(f"GraphedModel: a batch of {len(inp['imgs'])} views, but the step was captured for "
                             f"{len(step.static_inp['imgs'])} (drop the last, smaller batch of an epoch)")
        losses = dict(step.run(inp))
        step.optimizer.skip_next_step()
        losses['total'] = losses['total'].detach().clone().requires_grad_(True)      # a leaf: backward() reaches no parameter
        return losses
