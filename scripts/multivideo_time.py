"""Aggregate adapted frames/s of G videos at C2 on one GPU: ``MultiVideoAdaptor.adapt`` (one frame of every video per call,
every network pass grouped) against G single-video ``Adaptor.adapt`` runs done one after another.  Prints the card, its power
limit and one JSON line per G.

    python scripts/multivideo_time.py [--groups 1 2 4 8 16] [--frames 12] [--warmup 3] [--out FILE]

CUDA events around `frames` frames of every video after `warmup` untimed ones; the two arms run back to back per G.  Teacher
dropout stays live, as in bench.py's C2 workload."""
import argparse
import json
import sys

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, device_frames, timed_window


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 2, 4, 8, 16])
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = asset_dir('dboa_mv_')
    n = args.warmup + args.frames
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []
    for G in args.groups:
        opts = lambda g: default_options(expdir=work, expname=f'g{G}_{g}', model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
        frames = [list(f) for f in zip(*device_frames(G, n))]                # frames[t][g]
        mv = MultiVideoAdaptor(opts(0), G)
        for t in range(args.warmup):
            mv.adapt(frames[t])
        grouped_ms = timed_window(lambda t: mv.adapt(frames[t]), range(args.warmup, n))
        del mv
        torch.cuda.empty_cache()
        singles = []
        for g in range(G):
            ad = Adaptor(opts(g))
            ad.fused_eval = 'none'
            singles.append(ad)

        def seq(t):
            for g, ad in enumerate(singles):
                ad.global_step = t
                ad.adapt(frames[t][g])
        for t in range(args.warmup):
            seq(t)
        seq_ms = timed_window(seq, range(args.warmup, n))
        del singles
        torch.cuda.empty_cache()
        r = {'G': G, 'workload': 'c2', 'frames_per_video': args.frames,
             'grouped': {'ms_per_step': round(grouped_ms / args.frames, 3), 'adapted_frames_per_s': round(1000.0 * G * args.frames / grouped_ms, 1)},
             'sequential': {'ms_per_step': round(seq_ms / args.frames, 3), 'adapted_frames_per_s': round(1000.0 * G * args.frames / seq_ms, 1)}}
        r['speedup'] = round(seq_ms / grouped_ms, 3)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
