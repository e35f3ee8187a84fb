"""What the timing scripts share: the card line, three ways of timing a region, the synthetic asset directory, device frames,
the reset of a single-video ``Adaptor`` between videos, and the posed SMPL mesh of tests/harness.py.  A plain module: the
scripts run with scripts/ on sys.path."""
import os
import subprocess
import sys
import tempfile
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(REPO, 'tests'), REPO):
    if _p not in sys.path:
        sys.path.insert(0, _p)
from harness import fetch, posed_smpl_mesh, stream  # noqa: E402,F401

# what card() reports: a number measured on the GPU is worth something only with the card's name and power limit beside it
CARD_FIELDS = 'name, power limit, SM clock, max SM clock'


def card():
    """The card's name, power limit, SM clock and max SM clock from nvidia-smi, or the device name where it cannot be asked."""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        out = q.stdout.strip() if q.returncode == 0 else ''
    except (OSError, subprocess.SubprocessError):
        out = ''
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def timed_window(fn, ts):
    """ms between one CUDA event before ``fn(t)`` for every t in `ts` and one after."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in ts:
        fn(t)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def timed_each(fn, n):
    """Mean ms of fn(t) over t < n, each call between two CUDA events and followed by a device sync."""
    total = 0.0
    for t in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(t)
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
    return total / n


def timed_once(fn):
    """(CUDA-event ms, host-clock ms) of one call of fn, from a synchronised device to the end of its last kernel."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3


def asset_dir(prefix, n_exemplars=None):
    """A new temporary directory with the synthetic assets under data/, made the data root.  Returns the directory."""
    from dynaboa_b200 import config, synthetic
    work = tempfile.mkdtemp(prefix=prefix)
    synthetic.write_asset_dir(os.path.join(work, 'data'), **({} if n_exemplars is None else {'n_exemplars': n_exemplars}))
    config.set_data_root(os.path.join(work, 'data'))
    return work


def device_frames(n_videos, n):
    """frames[g][t]: frame t of ``SyntheticStream(rank=g)`` on the device, for g < n_videos and t < n."""
    return [[fetch(s[t]) for t in range(n)] for s in (stream(g, n) for g in range(n_videos))]


def snapshot(ad):
    return ad.model.module.arena.clone(), ad.teacher.arena.clone()


def restart(ad, snap):
    """Give a single-video Adaptor a new video: theta and teacher from `snap` (``snapshot``), zero Adam moments and step count,
    an empty history."""
    ad.model.module.arena.copy_(snap[0])
    ad.teacher.arena.copy_(snap[1])
    ad.optimizer.m.zero_(); ad.optimizer.v.zero_(); ad.optimizer.step_count = 0
    ad.history = {}
