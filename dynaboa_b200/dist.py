"""Data-parallel adaptation over streaming frames (SURVEY.md §8e): one process per GPU, every rank holds a
full replica of theta / Adam state / teacher and adapts on its own frame (or its own video stream); the only
exchange step is ONE all-reduce (mean) of the flat fp32 outer gradient (107.9 MB) per outer update, plus a
3-float all-reduce so that every rank takes the same ``dynamic_boa`` branch.

The reference has no distributed code; this is the CUDA-native addition.  Semantics: per-rank inner SGD step,
rank-averaged outer gradient -- NOT identical to the reference at ``--batch_size R`` (which takes one inner step
on the batch-mean loss); ``mode='replicas'`` (no collective, R independent videos) is the exact-semantics mode.
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's environment; returns (rank, world, local_rank)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        # the bucketed all-reduce runs UNDER the backward: NCCL's channel count trades link bandwidth against the SMs it takes
        # from the backward kernels
        os.environ.setdefault('NCCL_MAX_NCHANNELS', '16')
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_range(n_items, rank, world):
    """Contiguous shard [lo, hi) of ``n_items`` for ``rank`` (first ranks take the remainder)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def make_grad_sync(world, group=None):
    """Hook for ``FusedAdam.pre_step_hook``: all-reduce(sum) of the flat gradient arena, then 1/world (one blocking
    collective after the backward: the path the autograd driver uses; ``attach`` installs the overlapped variant)."""
    if world <= 1:
        return None

    def sync(flat_grad):
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
        flat_grad.mul_(1.0 / world)
    return sync


class BucketedGradSync:
    """Overlaps the all-reduce of the outer gradient with the backward that produces it (SURVEY.md §8e).

    ``dboa_hmr_backward`` completes the gradient arena head -> layer4 -> layer3 -> ... -> stem; armed through
    ``dboa_hmr_backward_buckets`` it records one event per bucket (layer4 + head: 74 MB, layer3: 28 MB, the rest: 6 MB) as
    soon as every kernel writing that span is ordered.  ``after_backward`` makes a communication stream wait for each event
    and all-reduce (sum) that span of the flat arena, so only the last, smallest bucket is exposed after the backward; the
    mean (1 / world) is folded into the Adam sweep (``FusedAdam.gscale``), which waits for the communication stream."""

    def __init__(self, world, device, group=None):
        from . import _lib
        self.world, self.group = world, group
        self.comm = torch.cuda.Stream(device=device)
        self.events = [torch.cuda.Event() for _ in range(3)]
        for ev in self.events:
            ev.record()                                    # forces creation of the cudaEvent_t handed to the library
        lib = _lib.load()
        self.bounds = [(lib.dboa_hmr_bucket_offset(k), lib.dboa_hmr_bucket_offset(k - 1)) for k in range(3)]

    def arm(self):
        from . import _lib
        import ctypes as C
        _lib.call('dboa_hmr_backward_buckets', *[C.c_void_p(ev.cuda_event) for ev in self.events])

    def after_backward(self, flat_grad):
        for ev, (lo, hi) in zip(self.events, self.bounds):
            self.comm.wait_event(ev)
            with torch.cuda.stream(self.comm):
                dist.all_reduce(flat_grad[lo:hi], op=dist.ReduceOp.SUM, group=self.group)
        flat_grad.record_stream(self.comm)


def attach(adaptor, world, group=None):
    """Turn ``adaptor`` into one rank of a data-parallel run: the fused path (``Adaptor.adapt``) all-reduces the outer
    gradient bucket by bucket under the upper-level backward, the autograd path (``Adaptor.adaptation``) with one collective
    before the optimiser step; both leave the 1 / world to the Adam sweep, and ``cal_feature_diff`` all-reduces its sums."""
    if world <= 1:
        return None
    opt = adaptor.optimizer
    opt.gscale = 1.0 / world
    adaptor.dp_group = group
    sync = None
    if os.environ.get('DBOA_DP_BUCKETS', '1') != '0':          # 0: one all-reduce after the backward (A/B reference of the overlap)
        sync = BucketedGradSync(world, adaptor.device, group)
    opt.grad_sync = sync

    def hook(flat_grad):                                   # autograd path / any step the bucketed path did not cover
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    opt.pre_step_hook = hook
    return sync


def allreduce_cosine_terms(dot, na2, nb2, group=None):
    """Sum (a.b, |a|^2, |b|^2) over ranks so that the dynamic-loop decision is identical everywhere and equals
    the reference's batch-level ``cal_feature_diff`` (it flattens across the batch, base_adaptor.py:215)."""
    t = torch.stack([dot, na2, nb2]) if torch.is_tensor(dot) else torch.tensor([dot, na2, nb2], dtype=torch.float64)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t[0] / (t[1].sqrt().clamp_min(1e-12) * t[2].sqrt().clamp_min(1e-12))


def max_over_ranks(value, device=None):
    """MAX all-reduce of a python float (timings are reported as the max over ranks)."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device if device is not None else 'cpu')
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
