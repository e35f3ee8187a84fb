"""Slots of ``MultiVideoAdaptor`` at C2 on one GPU.  Prints the card, its power limit and SM clock, then one JSON line per
measurement:

(a) occupancy: G = 8 slots with n = 1..8 of them active (the others None), ms per step from CUDA events over `frames` steps after
    `warmup` untimed ones, next to single-video ``Adaptor.adapt``;
(b) pool: `videos` ``SyntheticStream``s with seeded lengths in [4, 40] through G = 8 slots, each slot refilled with ``start`` as
    soon as its video ends, against the same videos through ``Adaptor.adapt`` one after another.  Adapted frames per second of
    wall time, ending in a device synchronise; the first `warmup` frames of each arm run once before the timed pass.

    python scripts/multivideo_pool_time.py [--frames 12] [--warmup 3] [--videos 24] [--seed 0] [--out FILE]"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(n):
        fn(t)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--videos', type=int, default=24)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_pool_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config, synthetic
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    G = 8
    work = tempfile.mkdtemp(prefix='dboa_pool_')
    synthetic.write_asset_dir(os.path.join(work, 'data'))
    config.set_data_root(os.path.join(work, 'data'))
    opts = lambda name, n: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    fetch = lambda s, t: {k: v.cuda() if torch.is_tensor(v) else v for k, v in s[t].items()}
    info = card()
    print(f'card (name, power limit, SM clock, max SM clock): {info}', flush=True)
    rows = []

    # (a) occupancy
    n = args.warmup + args.frames
    streams = [synthetic.SyntheticStream(length=n, batch_size=1, rank=g) for g in range(G)]
    frames = [[fetch(s, t) for s in streams] for t in range(n)]
    ad = Adaptor(opts('single', n))
    ad.fused_eval = 'none'

    def single(t):
        ad.global_step = t
        ad.adapt(frames[t][0])
    for t in range(args.warmup):
        single(t)
    single_ms = timed(lambda t: single(args.warmup + t), args.frames) / args.frames
    occ = {}
    for k in range(1, G + 1):
        mv = MultiVideoAdaptor(opts(f'occ{k}', n), G)
        step = lambda t: mv.adapt([frames[t][g] if g < k else None for g in range(G)])
        for t in range(args.warmup):
            step(t)
        occ[k] = timed(lambda t: step(args.warmup + t), args.frames) / args.frames
        del mv
        torch.cuda.empty_cache()
    r = {'measurement': 'occupancy', 'workload': 'c2', 'G': G, 'steps': args.frames, 'single_video_ms_per_frame': round(single_ms, 3),
         'ms_per_step': {str(k): round(v, 3) for k, v in occ.items()},
         'adapted_frames_per_s': {str(k): round(1000.0 * k / v, 1) for k, v in occ.items()}}
    print(json.dumps(r), flush=True)
    rows.append(r)

    # (b) pool
    rng = random.Random(args.seed)
    lengths = [rng.randint(4, 40) for _ in range(args.videos)]
    vstreams = [synthetic.SyntheticStream(length=L, batch_size=1, rank=100 + i) for i, L in enumerate(lengths)]
    vframes = [[fetch(s, t) for t in range(L)] for s, L in zip(vstreams, lengths)]

    def pool(mv):
        queue, slot, done, steps = list(range(args.videos)), [None] * G, 0, 0
        for g in range(G):
            if queue:
                mv.start(g)
                slot[g] = [queue.pop(0), 0]
        while any(s is not None for s in slot):
            mv.adapt([vframes[s[0]][s[1]] if s is not None else None for s in slot])
            steps += 1
            for g, s in enumerate(slot):
                if s is None:
                    continue
                s[1] += 1
                done += 1
                if s[1] == lengths[s[0]]:
                    slot[g] = None
                    if queue:
                        mv.start(g)
                        slot[g] = [queue.pop(0), 0]
        return done, steps

    def sequential(ad):
        snap = (ad.model.module.arena.clone(), ad.teacher.arena.clone())
        done = 0
        for v, L in enumerate(lengths):
            ad.model.module.arena.copy_(snap[0]); ad.teacher.arena.copy_(snap[1])
            ad.optimizer.m.zero_(); ad.optimizer.v.zero_(); ad.optimizer.step_count = 0
            ad.history = {}
            for t in range(L):
                ad.global_step = t
                ad.adapt(vframes[v][t])
                done += 1
        return done

    mv = MultiVideoAdaptor(opts('pool_warm', 40), G)
    for t in range(args.warmup):
        mv.adapt([frames[t][g] for g in range(G)])
    del mv
    mv = MultiVideoAdaptor(opts('pool', 40), G)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pool_frames, pool_steps = pool(mv)
    torch.cuda.synchronize()
    pool_s = time.perf_counter() - t0
    del mv
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    seq_frames = sequential(ad)
    torch.cuda.synchronize()
    seq_s = time.perf_counter() - t0
    r = {'measurement': 'pool', 'workload': 'c2', 'G': G, 'videos': args.videos, 'lengths': lengths, 'adapted_frames': pool_frames,
         'pool': {'steps': pool_steps, 'seconds': round(pool_s, 3), 'adapted_frames_per_s': round(pool_frames / pool_s, 1)},
         'sequential': {'seconds': round(seq_s, 3), 'adapted_frames_per_s': round(seq_frames / seq_s, 1)},
         'speedup': round(seq_s / pool_s, 3)}
    print(json.dumps(r), flush=True)
    rows.append(r)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
