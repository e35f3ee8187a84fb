"""Slots of ``MultiVideoAdaptor`` at C2 on one GPU.  Prints the card, its power limit and SM clock, then one JSON line per
measurement:

(a) occupancy: G = 8 slots with n = 1..8 of them active (the others None), ms per step from CUDA events over `frames` steps after
    `warmup` untimed ones, next to single-video ``Adaptor.adapt``;
(b) pool: `videos` ``SyntheticStream``s with seeded lengths in [4, 40] through G = 8 slots by ``MultiVideoAdaptor.run``, each
    slot refilled as soon as its video ends, against the same videos through ``Adaptor.adapt`` one after another.  Adapted frames per second of
    wall time, ending in a device synchronise; the first `warmup` frames of each arm run once before the timed pass.

    python scripts/multivideo_pool_time.py [--frames 12] [--warmup 3] [--videos 24] [--seed 0] [--out FILE]"""
import argparse
import json
import random
import sys
import time

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, device_frames, fetch, restart, snapshot, stream, timed_window


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
    from dynaboa_b200 import config
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    G = 8
    work = asset_dir('dboa_pool_')
    opts = lambda name, n: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []

    # (a) occupancy
    n = args.warmup + args.frames
    frames = [list(f) for f in zip(*device_frames(G, n))]                    # frames[t][g]
    ad = Adaptor(opts('single', n))
    ad.fused_eval = 'none'

    def single(t):
        ad.global_step = t
        ad.adapt(frames[t][0])
    for t in range(args.warmup):
        single(t)
    single_ms = timed_window(single, range(args.warmup, n)) / args.frames
    occ = {}
    for k in range(1, G + 1):
        mv = MultiVideoAdaptor(opts(f'occ{k}', n), G)
        step = lambda t: mv.adapt([frames[t][g] if g < k else None for g in range(G)])
        for t in range(args.warmup):
            step(t)
        occ[k] = timed_window(step, range(args.warmup, n)) / args.frames
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
    vstreams = [stream(100 + i, L) for i, L in enumerate(lengths)]
    vframes = [[fetch(s[t]) for t in range(L)] for s, L in zip(vstreams, lengths)]

    def pool(mv):
        steps = mv.global_step
        done = sum(r['frames'] for r in mv.run(vframes))       # fused_eval 'none': adaptation only
        return done, mv.global_step - steps

    def sequential(ad):
        snap = snapshot(ad)
        done = 0
        for v, L in enumerate(lengths):
            restart(ad, snap)
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
