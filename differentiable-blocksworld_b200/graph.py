"""Whole-step CUDA graph: zero the gradient bucket, build the scene, render both passes, composite + loss, and
back-propagate to every leaf parameter -- captured once on static buffers and replayed per step.  The step is a few
hundred kernel launches of 2-100 us each (scene construction, two rasterization passes, their backward, the
reductions); replaying them as one graph removes the launch gaps and the Python/autograd dispatch that otherwise cost
more than the kernels themselves.  Requires the model's static-topology mode (dbw.py): no host synchronisation and no
shape that depends on parameter values inside forward()."""
import torch

from .parallel import refuse_camera_gradients


class GraphedStep:
    def __init__(self, view_parallel, example_inp, n_total_views, warmup=3, capture_all_reduce=None, generator=None):
        refuse_camera_gradients(example_inp, 'GraphedStep')
        self.vp, self.model = view_parallel, view_parallel.model
        # The gradient all-reduce is captured INTO the graph when it is the peer-memory kernel (a plain launch).  An
        # ncclAllReduce is issued right after the replay instead: captured, it hung on 2 GPUs with this image's NCCL (round 1).
        if capture_all_reduce is None:
            capture_all_reduce = view_parallel.graph_capturable_collective
        self.capture_all_reduce = capture_all_reduce and view_parallel.world_size > 1
        self.n_total = n_total_views
        dev = example_inp['imgs'].device
        self.static_inp = {k: v.clone() for k, v in example_inp.items()}
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
        self._capture(warmup=warmup)

    def _phase(self):
        """what the captured control flow depends on: the training-schedule switches of dbw.py:210-212,276,331-334"""
        m = self.model
        return (m.training, m.is_live('coarse_learning'), m.is_live('decimate_txt'), m.is_live('kill_blocks'))

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

    def _body(self):
        losses, reduced = self.vp.local_step(self.static_inp, None, self.n_total, collective=self.capture_all_reduce)
        self.inside = self.vp.reduces_inside_backward(self.static_inp)      # the collective sits INSIDE the backward (parallel.GradSumPoint)
        if self.capture_all_reduce and not reduced:
            self.vp.bucket.all_reduce(self.vp.group)
        return losses

    def run(self, inp=None, non_blocking=True, all_reduce=True):
        """inp: optional dict of (host or device) tensors for this step, copied into the static buffers.
        all_reduce=False skips the collective when it is issued after the replay (a captured one always runs)."""
        refuse_camera_gradients(inp, 'GraphedStep')
        if inp is not None:
            for k, v in inp.items():
                if k in self.static_inp:
                    self.static_inp[k].copy_(v, non_blocking=non_blocking)
        if self._phase() != self.phase:          # a schedule milestone was crossed (coarse -> fine, decimation off): re-capture
            self._capture()
        self._bind_buffers()                       # eager code in between (evaluation, another GraphedStep) may have re-pointed them
        self.noise_buf.normal_(generator=self.gen)                      # identical on every rank (same seed, same count)
        if self.overlap_buf is not None:
            self.overlap_buf.uniform_(generator=self.gen)
        self.graph.replay()
        for p, g in zip(self.vp.bucket.params, self.grads):
            p.grad = g
        if not self.capture_all_reduce and all_reduce and self.vp.world_size > 1:
            if self.inside:
                raise RuntimeError('this step sums its gradients inside the backward (parallel.GradSumPoint) but was captured '
                                   'with capture_all_reduce=False: its gradients are local and cannot be reduced afterwards')
            self.vp.bucket.all_reduce(self.vp.group)
        return self.losses


class PipelinedGraphedStep:
    """Two GraphedSteps on alternating static input buffers: while step i replays, the inputs of step i+1 are copied
    host->device on a side stream (what a prefetching DataLoader does for src/trainer.py:141).  `run(host_inp)` returns
    the losses of the step that consumed `host_inp`."""

    def __init__(self, view_parallel, example_inp, n_total_views, capture_all_reduce=None):
        refuse_camera_gradients(example_inp, 'PipelinedGraphedStep')
        gen = torch.Generator(device=example_inp['imgs'].device)
        gen.manual_seed(view_parallel.seed)
        self.steps = [GraphedStep(view_parallel, example_inp, n_total_views, capture_all_reduce=capture_all_reduce, generator=gen)
                      for _ in range(2)]
        self.copy_stream = torch.cuda.Stream()
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]      # inputs of buffer b have landed
        self.free = [torch.cuda.Event(), torch.cuda.Event()]       # buffer b has been consumed by its replay
        self.i = 0
        self.primed = False

    def _stage(self, b, host_inp):
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.free[b])
            for k, v in host_inp.items():
                if k in self.steps[b].static_inp:
                    self.steps[b].static_inp[k].copy_(v, non_blocking=True)
            self.ready[b].record(self.copy_stream)

    def run(self, host_inp, next_host_inp=None, all_reduce=True):
        """consume `host_inp` (staged now unless it was prefetched as the previous call's `next_host_inp`) and
        prefetch `next_host_inp` for the following call."""
        refuse_camera_gradients(host_inp, 'PipelinedGraphedStep')
        refuse_camera_gradients(next_host_inp, 'PipelinedGraphedStep')
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
        losses = self.steps[b].run(all_reduce=all_reduce)
        self.free[b].record(cur)
        self.i += 1
        return losses
