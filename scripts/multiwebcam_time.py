"""Cost of serving several webcam streams from one GPU with ``MultiWebcamAdaptor``.  Prints the card (name, power limit, SM
clock, max SM clock), then one JSON line per G in `groups`:

- pool: ms per tick of ``MultiWebcamAdaptor.online_adaptation`` on G host frames (1280x720 uint8 numpy) and their detections,
  from the host frames to the result dictionaries: a CUDA event before the call, one after it, then a device sync;
- sequential: the same G streams through G ``WebcamAdaptor.online_adaptation`` calls, one after another (ms per G frames);
- input side alone: ``MultiWebcamAdaptor.input_side`` (host boxes, frame uploads, one grouped crop and one grouped keypoint
  call) against G ``WebcamAdaptor.dataprocess`` calls (one ``crop`` and one ``j2d_processing`` each).

Options: the reference webcam script's defaults (dynaboa_webcam.py:339-371) with ``use_boa=1``, the bilevel step the pool
groups: one inner step, mean teacher, motion term at interval 5, no dynamic loop.  Detections are seeded synthetic OpenPose
joints around a person-sized box, so every stream has a person in view on every tick.

    python scripts/multiwebcam_time.py [--ticks 20] [--warmup 6] [--groups 1 2 4 8] [--out FILE]"""
import argparse
import json
import sys
from types import SimpleNamespace

import numpy as np
import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, timed_each


def streams(G, n, seed=0):
    """frames[t][g] (720, 1280, 3) uint8 and dets[t][g] (1, 25, 3) of G cameras over n ticks."""
    rng = np.random.default_rng(seed)
    frames = [[rng.integers(0, 256, size=(720, 1280, 3), dtype=np.uint8) for _ in range(G)] for _ in range(n)]
    centre = rng.uniform([400, 250], [880, 470], size=(G, 2))
    dets = [[np.concatenate([centre[g] + rng.uniform(-150, 150, size=(25, 2)), rng.uniform(0, 1, size=(25, 1))], 1)[None]
             for g in range(G)] for _ in range(n)]
    return frames, dets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ticks', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=6)
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 2, 4, 8])
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multiwebcam_time.py needs a GPU')
    from dynaboa_b200 import config
    from dynaboa_b200.webcam import MultiWebcamAdaptor, WebcamAdaptor
    work = asset_dir('dboa_webcam_')
    opts = lambda name: SimpleNamespace(expdir=work, expname=name, tensorboard=0, model_file=config.BASE_MODEL, seed=22, lr=3e-6, beta1=0.5,
                                        beta2=0.9, use_boa=1, fastlr=8e-6, s2dloss_weight=10.0, shape_prior_weight=2e-6,
                                        pose_prior_weight=1e-4, use_meanteacher=1, alpha=0.1, teacherloss_weight=0.1, use_motion=1,
                                        interval=5, motionloss_weight=0.8, dynamic_boa=0, cos_sim_threshold=3.1e-4, optim_steps=7,
                                        test_basemodel=0)
    n = args.warmup + args.ticks
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []
    for G in args.groups:
        frames, dets = streams(G, n, seed=G)
        mv = MultiWebcamAdaptor(opts(f'pool{G}'), G)
        for t in range(args.warmup):
            mv.online_adaptation(frames[t], dets[t])
        pool = timed_each(lambda t: mv.online_adaptation(frames[args.warmup + t], dets[args.warmup + t]), args.ticks)
        side = timed_each(lambda t: mv.input_side(frames[args.warmup + t], dets[args.warmup + t]), args.ticks)
        del mv
        torch.cuda.empty_cache()
        singles = [WebcamAdaptor(opts(f'single{G}_{g}')) for g in range(G)]

        def seq(t):
            for g, ad in enumerate(singles):
                ad.online_adaptation(frames[t][g], dets[t][g])
        for t in range(args.warmup):
            seq(t)
        sequential = timed_each(lambda t: seq(args.warmup + t), args.ticks)

        def seq_side(t):
            for g, ad in enumerate(singles):
                ad.dataprocess(frames[args.warmup + t][g], dets[args.warmup + t][g][0], scaleFactor=1.2)
        side_seq = timed_each(seq_side, args.ticks)
        del singles
        torch.cuda.empty_cache()
        r = {'G': G, 'ticks': args.ticks, 'pool_ms_per_tick': round(pool, 2), 'sequential_ms_per_G_frames': round(sequential, 2),
             'sequential_over_pool': round(sequential / pool, 3), 'input_side_pool_ms': round(side, 3),
             'input_side_sequential_ms': round(side_seq, 3), 'input_side_sequential_over_pool': round(side_seq / side, 3)}
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
