"""Aggregate adapted frames/s of G videos at C2 on one GPU: ``MultiVideoAdaptor.adapt`` (one frame of every video per call,
every network pass grouped) against G single-video ``Adaptor.adapt`` runs done one after another.  Prints the card, its power
limit and one JSON line per G.

    python scripts/multivideo_time.py [--groups 1 2 4 8 16] [--frames 12] [--warmup 3] [--out FILE]

CUDA events around `frames` frames of every video after `warmup` untimed ones; the two arms run back to back per G.  Teacher
dropout stays live, as in bench.py's C2 workload."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
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
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 2, 4, 8, 16])
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config, synthetic
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = tempfile.mkdtemp(prefix='dboa_mv_')
    synthetic.write_asset_dir(os.path.join(work, 'data'))
    config.set_data_root(os.path.join(work, 'data'))
    n = args.warmup + args.frames
    info = card()
    print(f'card: {info}', flush=True)
    rows = []
    for G in args.groups:
        opts = lambda g: default_options(expdir=work, expname=f'g{G}_{g}', model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
        streams = [synthetic.SyntheticStream(length=n, batch_size=1, rank=g) for g in range(G)]
        frames = [[{k: v.cuda() if torch.is_tensor(v) else v for k, v in s[t].items()} for s in streams] for t in range(n)]
        mv = MultiVideoAdaptor(opts(0), G)
        for t in range(args.warmup):
            mv.adapt(frames[t])
        grouped_ms = timed(lambda t: mv.adapt(frames[args.warmup + t]), args.frames)
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
        seq_ms = timed(lambda t: seq(args.warmup + t), args.frames)
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
