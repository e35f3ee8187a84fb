"""Oracle of the data-parallel mode (test infrastructure only; SURVEY.md §8e "CPU emulation of R ranks").

The reference has no distributed code.  The CUDA implementation shards independent frame streams over ranks: every rank
holds a replica of theta / Adam state / teacher, takes its OWN inner SGD step(s) on its own frame, and the outer gradient is
the mean over ranks (one all-reduce); under ``dynamic_boa`` the (a.b, |a|^2, |b|^2) sums of every feature are summed over the
ranks before the cosine is formed, which is the reference's batch-level decision (``cal_feature_diff`` flattens across the
batch, base_adaptor.py:215).  This module restates exactly that with R ``OracleAdaptor`` replicas in lock step (one thread
per rank, barriers at the two exchange points), so the GPU test can compare every rank's trajectory with it.  It is NOT the
reference at ``--batch_size R`` (one inner step on the batch-mean loss), see SURVEY.md §8e.
"""
import threading

import torch


class _Exchange:
    def __init__(self, R):
        self.R, self.bar, self.slots = R, threading.Barrier(R), [None] * R

    def all_reduce(self, rank, value, mean=False):
        self.slots[rank] = value
        self.bar.wait()
        total = self.slots[0].clone()
        for r in range(1, self.R):                 # fixed order on every rank -> identical replicas
            total = total + self.slots[r]
        self.bar.wait()
        return total / self.R if mean else total


def run(make_oracle, streams, n_frames):
    """``make_oracle(rank)`` -> OracleAdaptor; ``streams[rank][t]`` -> batch.  Returns per-rank lists of adaptation records
    plus the oracles (for final predictions / theta)."""
    R = len(streams)
    ex = _Exchange(R)
    oracles = [make_oracle(r) for r in range(R)]
    records = [[] for _ in range(R)]
    errors = []

    def worker(rank):
        ora = oracles[rank]

        def grad_hook(o):
            names = list(o.theta.keys())
            flat = torch.cat([o.theta[k].grad.flatten() for k in names])
            flat = ex.all_reduce(rank, flat, mean=True)
            off = 0
            for k in names:
                n = o.theta[k].numel()
                o.theta[k].grad.copy_(flat[off:off + n].view_as(o.theta[k]))
                off += n
        ora.grad_hook = grad_hook
        ora.cos_hook = lambda terms: ex.all_reduce(rank, terms)
        try:
            for t in range(n_frames):
                ora.global_step, ora.fit_losses = t, {}
                records[rank].append(ora.adaptation(streams[rank][t], with_inference=False))
        except Exception as e:      # noqa: BLE001 - surfaced to the caller; a dead rank must not leave the others in a barrier
            errors.append(e)
            ex.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(R)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        raise errors[0]
    return records, oracles
