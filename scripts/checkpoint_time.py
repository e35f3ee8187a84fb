"""What a pool checkpoint costs at C2 (``MultiVideoAdaptor.save`` / ``load``, DESIGN.md section 11).  Prints the card and its
power limit, then one JSON line per pool width G (1 and 8):

- ``stall_ms``: host time ``save(wait=False)`` takes between two frames: forming the records, enqueuing the device-to-host
  copies into pinned buffers and starting the background write (the adapting stream is not synchronised);
- ``durable_ms``: wall time from the start of ``save`` until the checkpoint's manifest is on disk;
- ``frame_ms`` / ``frame_ms_during_write``: the pool frame alone, and a frame enqueued while the previous checkpoint is written;
- ``load_ms``: ``load`` of that checkpoint into a fresh pool, ending in a device synchronise;
- ``bytes``: the size of the checkpoint.  Each figure is the median of `reps` checkpoints taken after `warmup` frames.

    python scripts/checkpoint_time.py [--warmup 4] [--reps 3] [--out FILE]"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, fetch, stream


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--warmup', type=int, default=4)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('checkpoint_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config, state
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = asset_dir('dboa_ckpt_')
    n = args.warmup + 2 * args.reps + 2
    opts = lambda name: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    print(f'card ({CARD_FIELDS}): {card()}', flush=True)
    lines = []
    for G in (1, 8):
        mv = MultiVideoAdaptor(opts(f'g{G}'), G)
        streams = [stream(g, n) for g in range(G)]
        frame = lambda t: mv.adapt([fetch(s[t]) for s in streams])

        def timed_frame(t):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            frame(t)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3
        t = 0
        for _ in range(args.warmup):
            frame(t)
            t += 1
        root = tempfile.mkdtemp(prefix='dboa_ckpt_dir_', dir=work)
        stall, durable, plain, during = [], [], [], []
        for _ in range(args.reps):
            plain.append(timed_frame(t))
            t += 1
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mv.save(root, wait=False)
            stall.append((time.perf_counter() - t0) * 1e3)
            during.append(timed_frame(t))
            t += 1
            mv._writer.wait()
            durable.append((time.perf_counter() - t0) * 1e3)
        path, man = state.latest(root)
        size = sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
        del mv
        torch.cuda.empty_cache()
        fresh = MultiVideoAdaptor(opts(f'load{G}'), G)
        loads = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fresh.load(root)
            torch.cuda.synchronize()
            loads.append((time.perf_counter() - t0) * 1e3)
        del fresh
        torch.cuda.empty_cache()
        shutil.rmtree(root, ignore_errors=True)
        med = lambda v: round(statistics.median(v), 2)
        line = dict(workload='c2', G=G, stall_ms=med(stall), durable_ms=med(durable), frame_ms=med(plain), frame_ms_during_write=med(during),
                    load_ms=med(loads), bytes=size, reps=args.reps)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
