"""Per-video hyperparameters at C2 on one GPU.  Prints the card, its power limit and SM clock, then one JSON line per measurement:

(a) frame: for G = 4 and 8, ms per pool frame of a uniform pool (no hparams) and of a pool whose slots all carry different values
    of every PER_VIDEO key, alternated `rounds` times in one run, each window `frames` pool frames between CUDA events after
    `warmup` untimed ones;
(b) sweep: for G = 4 and 8, the per-video Adam + EMA sweep (dboa_adam_ema_groups, every video at its own step count) over
    G * P floats, in GB/s of the 9 x 4 bytes each float moves, from CUDA events over `reps` launches, 2 x `rounds` windows.

    python scripts/multivideo_hparams_time.py [--frames 12] [--warmup 3] [--rounds 3] [--reps 50] [--out FILE]"""
import argparse
import ctypes as C
import json
import sys

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, device_frames, timed_window

FACTORS = (1.5, 0.7, 1.3, 0.8, 1.2, 0.9, 1.1, 0.6)


def hparams_of(o, g):
    """Slot g's values of every PER_VIDEO key, distinct between slots and from ``o``."""
    f = FACTORS[g % len(FACTORS)]
    hp = {k: getattr(o, k) * f for k in ('lr', 'fastlr', 's2dloss_weight', 'shape_prior_weight', 'pose_prior_weight', 'teacherloss_weight',
                                          'motionloss_weight', 'labelloss_weight', 'cos_sim_threshold')}
    hp.update(beta1=0.4 + 0.02 * g, beta2=0.85 + 0.01 * g, alpha=0.05 + 0.02 * g, optim_steps=2 + g)
    return hp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_hparams_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import _lib, config
    from dynaboa_b200._lib import stream
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = asset_dir('dboa_hparams_')
    n = args.warmup + args.frames
    opts = lambda name: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []

    # (a) pool frames, uniform and per-video pools alternated
    for G in (4, 8):
        frames = [list(f) for f in zip(*device_frames(G, n))]                 # frames[t][g]
        ms = {'uniform': [], 'per_video': []}
        for r in range(args.rounds):
            for arm in ('uniform', 'per_video'):
                o = opts(f'{arm}{G}_{r}')
                mv = MultiVideoAdaptor(o, G)
                for g in range(G):
                    mv.start(g, hparams=hparams_of(o, g) if arm == 'per_video' else None)
                step = lambda t: mv.adapt(frames[t])
                for t in range(args.warmup):
                    step(t)
                ms[arm].append(timed_window(step, range(args.warmup, n)) / args.frames)
                del mv, step
                torch.cuda.empty_cache()
        row = {'measurement': 'frame', 'workload': 'c2', 'G': G, 'frames': args.frames,
               'ms_per_pool_frame': {k: [round(x, 3) for x in v] for k, v in ms.items()},
               'ratio_of_means': round(sum(ms['per_video']) / sum(ms['uniform']), 4)}
        print(json.dumps(row), flush=True)
        rows.append(row)

    # (b) the Adam + EMA sweep over G * P floats
    P = int(_lib.load().dboa_hmr_arena_floats())
    for G in (4, 8):
        t = [torch.randn(G * P, device='cuda') * 1e-3 for _ in range(5)]          # theta, grad, m, v, teacher
        t[3].abs_()
        table = (C.c_float * (G * _lib.ADAM_SCALARS))()
        one = (C.c_float * _lib.ADAM_SCALARS)()
        for g in range(G):
            _lib.call('dboa_adam_scalars', one, 3e-6 * FACTORS[g], 0.5, 0.9, 1e-8, 1 + g, 0.1, 1.0)
            table[g * _lib.ADAM_SCALARS:(g + 1) * _lib.ADAM_SCALARS] = one[:]
        ptrs = [x.data_ptr() for x in t]
        sweep = lambda i: _lib.call('dboa_adam_ema_groups', *ptrs, P, table, G, (1 << G) - 1, stream())
        for i in range(5):
            sweep(i)
        gbs = []
        for r in range(2 * args.rounds):
            ms = timed_window(sweep, range(args.reps)) / args.reps
            gbs.append(round(9 * 4 * G * P / (ms * 1e-3) / 1e9, 1))
        row = {'measurement': 'sweep', 'G': G, 'floats': G * P, 'bytes_per_float': 36, 'GB_per_s': gbs}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del t
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
