"""Adam over all of a model's parameters as ONE kernel launch (csrc/dbw_optim.cu, include/dbw_render.h "Optimiser"), with the
learning rates and the step counters read on the device -- so the launch can sit inside a captured training step
(graph.GraphedStep(optimizer=...)) and replay with whatever rates a scheduler has set since.

`BucketAdam` is a torch.optim.Optimizer with torch.optim.Adam's constructor, semantics (amsgrad=False, maximize=False: a
parameter whose .grad is None is left alone, moments and step count included) and state-dict format, so the reference's
schedulers (src/scheduler.py) drive its `param_groups[g]['lr']` and its trainer's checkpoints (src/trainer.py:84-108) load in
both directions between the two classes.  `create_optimizer` has the signature of the reference's factory (src/optimizer.py:6).
There is no CPU path: the state lives where the parameters live, and step() on anything but CUDA tensors raises."""
import ctypes
from copy import deepcopy

import torch

from . import _lib

# what torch.optim.Adam keeps in a param group besides lr / betas / eps / weight_decay: carried (at these values) so that a
# state dict of this class loads into torch.optim.Adam and back without a key missing on either side
_TORCH_ADAM_GROUP_KEYS = dict(amsgrad=False, maximize=False, foreach=None, capturable=False, differentiable=False, fused=None,
                              decoupled_weight_decay=False)


class BucketAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0., amsgrad=False, *, maximize=False):
        self.params = None
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                      **dict(_TORCH_ADAM_GROUP_KEYS, amsgrad=amsgrad, maximize=maximize)))
        self._check_groups()
        self.params = [p for g in self.param_groups for p in g['params']]
        self._group_of = [gi for gi, g in enumerate(self.param_groups) for _ in g['params']]
        if len(self.params) > _lib.ADAM_MAX_SEGMENTS or len(self.param_groups) > _lib.ADAM_MAX_GROUPS:
            raise ValueError(f'BucketAdam: at most {_lib.ADAM_MAX_SEGMENTS} parameter tensors in {_lib.ADAM_MAX_GROUPS} groups '
                             f'(got {len(self.params)} in {len(self.param_groups)})')
        dev = self.params[0].device
        for p in self.params:
            if p.dtype != torch.float32 or p.device != dev or not p.is_contiguous():
                raise ValueError('BucketAdam: parameters must be contiguous fp32 tensors on one device')
        # both moments in one flat buffer each, every parameter's share starting at a multiple of four floats (float4 lanes)
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.n_total = sum(p.numel() for p in self.params)
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        self.steps = torch.zeros(len(self.params), dtype=torch.int64, device=dev)
        self.lr = torch.zeros(len(self.param_groups), dtype=torch.float32, device=dev)
        self._lr_uploaded = None
        for i, (p, o) in enumerate(zip(self.params, offs)):
            self.state[p] = {'step': self.steps[i], 'exp_avg': self.exp_avg[o:o + p.numel()].view_as(p),
                             'exp_avg_sq': self.exp_avg_sq[o:o + p.numel()].view_as(p)}
        self._table = self.new_segment_table()
        self._table_key = None
        self._applied_by_replay = False

    def add_param_group(self, param_group):
        if self.params is not None:
            raise RuntimeError('BucketAdam: the parameter groups are fixed at construction (the state is one flat buffer)')
        super().add_param_group(param_group)

    def _check_groups(self):
        for g in self.param_groups:
            if g['amsgrad'] or g['maximize']:
                raise NotImplementedError('BucketAdam: amsgrad=True and maximize=True are not implemented')
            b1, b2 = g['betas']
            if not (0. <= b1 < 1. and 0. <= b2 < 1. and g['eps'] >= 0. and g['weight_decay'] >= 0. and float(g['lr']) >= 0.):
                raise ValueError(f"BucketAdam: invalid hyper-parameters lr={g['lr']} betas={g['betas']} eps={g['eps']} "
                                 f"weight_decay={g['weight_decay']}")

    # ------------------------------------------------------------------ the launch and what it reads
    def new_segment_table(self):
        """device storage for the DbwAdamSegment records of this optimiser's parameters (fill it with write_segments)"""
        return torch.zeros(len(self.params) * ctypes.sizeof(_lib.DbwAdamSegment), dtype=torch.uint8, device=self.params[0].device)

    def write_segments(self, table, grads, active=None):
        """upload the segment records for the gradient tensors `grads` (one per parameter in param_groups order, or None) into
        `table`, asynchronously on the current stream.  active: per parameter; default: the gradient is not None"""
        self._require_cuda()
        recs = (_lib.DbwAdamSegment * len(self.params))()
        for i, (p, g) in enumerate(zip(self.params, grads)):
            on = g is not None and (active is None or bool(active[i]))
            if on and (g.dtype != torch.float32 or g.device != p.device or g.shape != p.shape or g.layout != torch.strided
                       or not g.is_contiguous()):
                raise ValueError('BucketAdam: gradients must be dense contiguous fp32 tensors of their parameter\'s shape and device')
            st = self.state[p]
            recs[i] = _lib.DbwAdamSegment(p.data_ptr(), g.data_ptr() if on else 0, st['exp_avg'].data_ptr(),
                                          st['exp_avg_sq'].data_ptr(), p.numel(), self._group_of[i], int(on))
        # a fresh pinned tensor per upload: the host allocator keeps it until the copy has run, so nothing waits and a later
        # upload cannot overwrite bytes an earlier copy has yet to read
        table.copy_(torch.frombuffer(bytearray(recs), dtype=torch.uint8).pin_memory(), non_blocking=True)

    def captured_constants(self):
        """what a captured launch freezes (the groups travel by value): a change of these needs a new capture; `lr` does not"""
        return tuple((float(g['betas'][0]), float(g['betas'][1]), float(g['eps']), float(g['weight_decay'])) for g in self.param_groups)

    def refresh_lr(self):
        """make the device learning rates those of param_groups (an asynchronous copy on the current stream, only on a change)"""
        lrs = tuple(float(g['lr']) for g in self.param_groups)
        if lrs != self._lr_uploaded:
            self._require_cuda()
            self.lr.copy_(torch.tensor(lrs, dtype=torch.float32).pin_memory(), non_blocking=True)
            self._lr_uploaded = lrs

    def launch(self, table):
        """dbw_adam_step on the current stream over the segments of `table`; capturable (reads lr and the counters on the device)"""
        self._require_cuda()
        groups = (_lib.DbwAdamGroup * len(self.param_groups))(*[_lib.DbwAdamGroup(*c) for c in self.captured_constants()])
        _lib.check(_lib.lib().dbw_adam_step(table.data_ptr(), len(self.params), self.n_total, groups, len(groups),
                                            self.lr.data_ptr(), self.steps.data_ptr(),
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'dbw_adam_step')

    def _require_cuda(self):
        if not self.params[0].is_cuda:
            raise _lib.DbwError('BucketAdam: the update is a CUDA kernel and the parameters are not CUDA tensors (there is no CPU path)')

    # ------------------------------------------------------------------ torch.optim.Optimizer
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._applied_by_replay:          # graph.GraphedModel: the replay this iteration's forward ran has applied the update
            self._applied_by_replay = False
            return loss
        grads = [p.grad for p in self.params]
        key = tuple(g.data_ptr() if g is not None else 0 for g in grads)
        if key != self._table_key:           # the .grad tensors changed identity: new addresses for the kernel
            self.write_segments(self._table, grads)
            self._table_key = key
        self.refresh_lr()
        self.launch(self._table)
        return loss

    def prepare_replay(self):
        """before the replay of a captured step that contains this optimiser's launch: the rates the replay will read.  Counts
        as an optimiser step for the schedulers' step-order check."""
        self.refresh_lr()
        self._opt_called = True

    def skip_next_step(self):
        """the update of this iteration has been applied by a replay: the next step() call does nothing"""
        self._applied_by_replay = True

    def state_dict(self):
        """torch.optim.Adam's format: state[i] = {'step' (fp32 scalar on the host), 'exp_avg', 'exp_avg_sq'} for the parameters
        that have taken a step, indexed in param_groups order; copies, not views of the flat buffers (one host read)"""
        steps = self.steps.tolist()
        state = {i: {'step': torch.tensor(float(t), dtype=torch.float32), 'exp_avg': self.state[p]['exp_avg'].clone(),
                     'exp_avg_sq': self.state[p]['exp_avg_sq'].clone()}
                 for i, (p, t) in enumerate(zip(self.params, steps)) if t > 0}
        groups, i = [], 0
        for g in self.param_groups:
            packed = {k: v for k, v in g.items() if k != 'params'}
            packed['params'] = list(range(i, i + len(g['params'])))
            i += len(g['params'])
            groups.append(packed)
        return {'state': state, 'param_groups': groups}

    @torch.no_grad()
    def load_state_dict(self, state_dict):
        """from this class or from torch.optim.Adam (same groups, same parameter shapes).  A parameter without an entry has
        taken no step: zero moments, step 0."""
        saved = state_dict['param_groups']
        if len(saved) != len(self.param_groups) or any(len(s['params']) != len(g['params']) for s, g in zip(saved, self.param_groups)):
            raise ValueError("loaded state dict contains parameter groups that don't match the optimizer's")
        if any(s.get('amsgrad') or s.get('maximize') for s in saved):
            raise NotImplementedError('BucketAdam: amsgrad=True and maximize=True are not implemented')
        ids = [i for s in saved for i in s['params']]
        steps = []
        for i, p in zip(ids, self.params):
            entry, st = state_dict['state'].get(i), self.state[p]
            if entry is not None and entry['exp_avg'].shape != p.shape:
                raise ValueError(f'loaded optimiser state of parameter {i} has shape {tuple(entry["exp_avg"].shape)}, not {tuple(p.shape)}')
            for k in ('exp_avg', 'exp_avg_sq'):
                st[k].zero_() if entry is None else st[k].copy_(entry[k])
            steps.append(0 if entry is None else int(float(entry['step'])))
        self.steps.copy_(torch.tensor(steps, dtype=torch.int64))
        for s, g in zip(saved, self.param_groups):
            g.update({k: deepcopy(v) for k, v in s.items() if k != 'params'})
        self._check_groups()


def create_optimizer(cfg, model):
    """optimiser factory with the reference's signature (src/optimizer.py:6): cfg['training']['optimizer'] = {name: adam,
    <Adam options>, texture: {<options of the group of the parameters whose name starts with 'texture'>}}"""
    kwargs = deepcopy(cfg['training']['optimizer'] or {})
    name = kwargs.pop('name', None)
    if name != 'adam':
        raise NotImplementedError(f"optimizer '{name}': only 'adam' has a kernel here")
    texture = kwargs.pop('texture', None)
    if texture is None:
        return BucketAdam(model.parameters(), **kwargs)
    named = list(model.named_parameters())
    return BucketAdam([{'params': [p for n, p in named if not n.startswith('texture')]},
                       {'params': [p for n, p in named if n.startswith('texture')], **texture}], **kwargs)
