"""Fused Adam (+ optional mean-teacher EMA) over the flat parameter arena.

Drop-in for ``torch.optim.Adam(model.parameters(), lr, betas)`` as the reference uses it
(base_adaptor.py:126: eps 1e-8, no weight decay, no amsgrad) with the arithmetic of torch's single-tensor
Adam, but one kernel launch for all 169 tensors (``dboa_adam_ema``), optionally folding
``update_teacher`` (base_adaptor.py:193-201) into the same sweep.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import ptr, stream


def _find_owner(params):
    for p in params:
        owner = getattr(p, '_dboa_owner', None)
        if owner is not None:
            return owner()
    raise RuntimeError('FusedAdam needs the parameters of a dynaboa_b200 HMR model (flat arena)')


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, model=None):
        params = list(params)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
        if model is None:
            model = _find_owner(params)
        self.model = getattr(model, 'module', model)          # accept the MAML wrapper
        self.m = torch.zeros_like(self.model.arena)
        self.v = torch.zeros_like(self.model.arena)
        self.step_count = 0
        self.pre_step_hook = None                              # e.g. the data-parallel gradient all-reduce (dist.attach)
        self.grad_sync = None                                  # dist.BucketedGradSync: all-reduce overlapped with the backward
        self.reduced = False                                   # the gradient of the coming step has already been all-reduced
        self.gscale = 1.0                                      # g * gscale inside the sweep (1 / world under data parallelism)
        self.wait_before_write = []                            # events of side-stream readers of the weights (Adaptor.predict_async)
        self.scalars = None                                    # device block of step_captured's scalars (write_scalars)

    def _gather_grads(self):
        """Make sure every ``p.grad`` lives in the flat gradient arena (autograd may have re-created them)."""
        model = self.model
        had = model._grad_arena is not None
        stale = [(p, p.grad) for p in model._param_list] if not had else None
        g = model.grad_arena()
        views = model._lay.views(g)
        if not had:
            for (p, old), view in zip(stale, views):
                if old is not None:
                    view.copy_(old)
        else:
            for p, view in zip(model._param_list, views):
                if p.grad is None:
                    view.zero_()
                    p.grad = view
                elif p.grad.data_ptr() != view.data_ptr():
                    view.copy_(p.grad)
                    p.grad = view
        return g

    def zero_grad(self, set_to_none=False):
        g = self.model.grad_arena()
        _lib.call('dboa_fill_zero', ptr(g), g.numel() * 4, stream())

    @torch.no_grad()
    def step(self, closure=None, teacher=None, alpha=0.0):
        if closure is not None:
            raise NotImplementedError('closures are not used on the DynaBOA path')
        g = self._gather_grads()
        if self.reduced:                                       # bucketed all-reduce in flight on the communication stream
            torch.cuda.current_stream().wait_stream(self.grad_sync.comm)
            self.reduced = False
        elif self.pre_step_hook is not None:
            self.pre_step_hook(g)
        if self.wait_before_write:                             # a side stream may still be reading the weights this step overwrites
            cur = torch.cuda.current_stream()
            for ev in self.wait_before_write:
                cur.wait_event(ev)
            self.wait_before_write = []
        grp = self.param_groups[0]
        self.step_count += 1
        t = None if teacher is None else teacher.arena
        _lib.call('dboa_adam_ema_scaled', ptr(self.model.arena), ptr(g), ptr(self.m), ptr(self.v), ptr(t), self.model.arena.numel(),
                  float(grp['lr']), float(grp['betas'][0]), float(grp['betas'][1]), float(grp['eps']), self.step_count, float(alpha),
                  float(self.gscale), stream())

    # ---- the same step split for a CUDA graph: scalars written eagerly before each replay, the sweep captured once
    def write_scalars(self, alpha):
        """Advance ``step_count`` and write the fp32 scalars of its sweep (``dboa_adam_scalars``, the arithmetic of ``step``) to
        the device block that ``step_captured`` reads; an asynchronous copy on the current stream."""
        grp = self.param_groups[0]
        self.step_count += 1
        host = torch.empty(_lib.ADAM_SCALARS, dtype=torch.float32, pin_memory=True)
        _lib.call('dboa_adam_scalars', ptr(host), float(grp['lr']), float(grp['betas'][0]), float(grp['betas'][1]), float(grp['eps']),
                  self.step_count, float(alpha), float(self.gscale))
        if self.scalars is None:
            self.scalars = torch.empty(_lib.ADAM_SCALARS, dtype=torch.float32, device=self.m.device)
        self.scalars.copy_(host, non_blocking=True)

    @torch.no_grad()
    def step_captured(self, read_event, teacher=None):
        """``step`` for a graph capture: waits for the latest record of ``read_event`` (made outside the graph by the side-stream
        readers of the weights) and sweeps with the scalars of the ``scalars`` block, both at replay time.  No gradient
        all-reduce."""
        g = self._gather_grads()
        _lib.call('dboa_stream_wait_external', stream(), C.c_void_p(read_event.cuda_event))
        t = None if teacher is None else teacher.arena
        _lib.call('dboa_adam_ema_dev', ptr(self.model.arena), ptr(g), ptr(self.m), ptr(self.v), ptr(t), self.model.arena.numel(),
                  ptr(self.scalars), stream())


def ema_update(teacher, model, alpha):
    """teacher <- alpha * teacher + (1 - alpha) * model over the flat arenas (reference base_adaptor.py:193-201)."""
    model = getattr(model, 'module', model)
    _lib.call('dboa_ema_update', ptr(teacher.arena), ptr(model.arena), model.arena.numel(), float(alpha), stream())
