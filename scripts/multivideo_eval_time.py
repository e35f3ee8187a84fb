"""Cost of evaluating the videos of a ``MultiVideoAdaptor`` pool.  Prints the card (name, power limit, SM clock, max SM clock),
then one JSON line per measurement, ms per pool frame from CUDA events over `frames` frames after `warmup` untimed ones:

- C2, G in `groups`, every slot active, with ``fused_eval`` 'none', 'final' and 'all';
- the same G videos one after another through ``Adaptor.adapt`` with ``fused_eval = 'final'`` (ms per G frames);
- C5 (``dynamic_loop=True``) at G = `c5_groups` with 'none' and 'all'.

The videos are ``SyntheticStream(rank=g)``, fetched to the device before anything is timed.

    python scripts/multivideo_eval_time.py [--frames 12] [--warmup 3] [--groups 1 4 8 16] [--c5-groups 4] [--out FILE]"""
import argparse
import json
import sys

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, device_frames, restart, snapshot, timed_window


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 4, 8, 16])
    ap.add_argument('--c5-groups', type=int, default=4)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_eval_time.py needs a GPU')
    from bench import N_EXEMPLARS, WORKLOADS, default_options
    from dynaboa_b200 import config
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = asset_dir('dboa_eval_', n_exemplars=N_EXEMPLARS)
    n = args.warmup + args.frames
    opts = lambda name, w: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS[w])
    Gmax = max(args.groups + [args.c5_groups])
    frames = device_frames(Gmax, n)                                           # frames[g][t]
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []

    def pool_ms(G, mode, w):
        mv = MultiVideoAdaptor(opts(f'{w}_{G}_{mode}', w), G, dynamic_loop=(w == 'c5'))
        mv.fused_eval = mode
        step = lambda t: mv.adapt([frames[g][t] for g in range(G)])
        for t in range(args.warmup):
            step(t)
        ms = timed_window(step, range(args.warmup, n)) / args.frames
        mv.records(0)
        del mv
        torch.cuda.empty_cache()
        return ms

    def sequential_ms(G):
        ad = Adaptor(opts(f'seq_{G}', 'c2'))
        ad.fused_eval = 'final'
        snap = snapshot(ad)
        total = 0.0
        for g in range(G):
            restart(ad, snap)

            def step(t):
                ad.global_step = t
                ad.adapt(frames[g][t])
            for t in range(args.warmup):
                step(t)
            total += timed_window(step, range(args.warmup, n))
        del ad
        torch.cuda.empty_cache()
        return total / args.frames

    pool_ms(1, 'all', 'c2'), sequential_ms(1)              # untimed: what the first pool and adaptor of the process pay
    for G in args.groups:
        ms = {mode: pool_ms(G, mode, 'c2') for mode in ('none', 'final', 'all')}
        seq = sequential_ms(G)
        r = {'workload': 'c2', 'G': G, 'frames': args.frames, 'pool_ms_per_frame': {k: round(v, 2) for k, v in ms.items()},
             'sequential_final_ms_per_G_frames': round(seq, 2),
             'final_over_none': round(ms['final'] / ms['none'], 3), 'all_over_none': round(ms['all'] / ms['none'], 3),
             'sequential_over_pool_final': round(seq / ms['final'], 3)}
        print(json.dumps(r), flush=True)
        rows.append(r)
    G = args.c5_groups
    ms = {mode: pool_ms(G, mode, 'c5') for mode in ('none', 'all')}
    r = {'workload': 'c5', 'G': G, 'frames': args.frames, 'pool_ms_per_frame': {k: round(v, 2) for k, v in ms.items()},
         'all_over_none': round(ms['all'] / ms['none'], 3)}
    print(json.dumps(r), flush=True)
    rows.append(r)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
