"""Per-slot checkpoints on one GPU.  Prints the card (name, power limit, SM clock, max SM clock), then one JSON line per
measurement:

(a) start: the host stall of ``start(g, model=path)`` -- read, checks, digest, upload, theta / teacher reset -- for a checkpoint
    no slot holds yet and for one already in the device store, from a synchronised device to the end of the call's last copy
    (host clock), `reps` calls each;
(b) frame: ms per C2 pool frame at G = 4 and 8 with every slot on the pool's checkpoint and with every slot on a checkpoint of
    its own, alternated `rounds` times, each window `frames` pool frames between CUDA events after `warmup` untimed ones.  The
    adaptation calls are the same in both arms, so the two should be equal;
(c) webcam: ms per ``MultiWebcamAdaptor.adapt_processed`` tick with ``test_basemodel=1`` at G = 1, 4 and 8, every stream on the
    pool's checkpoint (one forward of the pool's arena) against one checkpoint per stream (one grouped forward over the stack of
    base arenas), alternated `rounds` times, each a CUDA event before and after every tick and a device sync.

    python scripts/slot_models_time.py [--frames 12] [--warmup 3] [--rounds 3] [--reps 5] [--out FILE]"""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

import torch

from gpu_timing import CARD_FIELDS, asset_dir, card, device_frames, timed_each, timed_window


def write_models(work, n):
    """n checkpoints of different weights (synthetic base models at seeds 101..) in the reference format."""
    from dynaboa_b200 import synthetic
    paths = []
    for i in range(n):
        paths.append(os.path.join(work, f'model{i}.pt'))
        torch.save(synthetic.make_basemodel(101 + i), paths[-1])
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('slot_models_time.py needs a GPU')
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    work = asset_dir('dboa_slot_models_')
    n = args.warmup + args.frames
    paths = write_models(work, max(8, args.reps))
    opts = lambda name: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    rows = []

    # (a) the host stall of start(g, model=path)
    mv = MultiVideoAdaptor(opts('start'), 2)
    mv.start(1, model=paths[-1])                                         # the pool digest and the first upload out of the way
    stall = {'new': [], 'in_store': []}
    for i in range(args.reps):
        for arm, g, path in (('new', 0, paths[i]), ('in_store', 1, paths[-1])):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mv.start(g, model=path)
            torch.cuda.synchronize()
            stall[arm].append(round((time.perf_counter() - t0) * 1e3, 1))
    row = {'measurement': 'start', 'ms': stall}
    print(json.dumps(row), flush=True)
    rows.append(row)
    del mv
    torch.cuda.empty_cache()

    # (b) C2 pool frames, one checkpoint against one per slot
    for G in (4, 8):
        frames = [list(f) for f in zip(*device_frames(G, n))]             # frames[t][g]
        ms = {'pool_checkpoint': [], 'own_checkpoints': []}
        for r in range(args.rounds):
            for arm in ms:
                mv = MultiVideoAdaptor(opts(f'{arm}{G}_{r}'), G)
                for g in range(G):
                    mv.start(g, model=paths[g] if arm == 'own_checkpoints' else None)
                step = lambda t: mv.adapt(frames[t])
                for t in range(args.warmup):
                    step(t)
                ms[arm].append(timed_window(step, range(args.warmup, n)) / args.frames)
                del mv, step
                torch.cuda.empty_cache()
        row = {'measurement': 'frame', 'workload': 'c2', 'G': G, 'frames': args.frames,
               'ms_per_pool_frame': {k: [round(x, 3) for x in v] for k, v in ms.items()},
               'ratio_of_means': round(sum(ms['own_checkpoints']) / sum(ms['pool_checkpoint']), 4)}
        print(json.dumps(row), flush=True)
        rows.append(row)

    # (c) webcam ticks with the base model shown beside the adapted one
    cam = lambda name: SimpleNamespace(expdir=work, expname=name, tensorboard=0, model_file=config.BASE_MODEL, seed=22, lr=3e-6, beta1=0.5,
                                       beta2=0.9, use_boa=1, fastlr=8e-6, s2dloss_weight=10.0, shape_prior_weight=2e-6,
                                       pose_prior_weight=1e-4, use_meanteacher=1, alpha=0.1, teacherloss_weight=0.1, use_motion=1,
                                       interval=5, motionloss_weight=0.8, dynamic_boa=0, cos_sim_threshold=3.1e-4, optim_steps=7,
                                       test_basemodel=1)
    for G in (1, 4, 8):
        frames = device_frames(G, n)
        images = [torch.cat([frames[g][t]['image'] for g in range(G)]) for t in range(n)]
        kps = [torch.cat([frames[g][t]['smpl_j2d'] for g in range(G)]) for t in range(n)]
        ms = {'pool_checkpoint': [], 'own_checkpoints': []}
        for r in range(args.rounds):
            for arm in ms:
                mv = MultiWebcamAdaptor(cam(f'cam_{arm}{G}_{r}'), G)
                for g in range(G):
                    mv.start(g, model=paths[g] if arm == 'own_checkpoints' else None)
                for t in range(args.warmup):
                    mv.adapt_processed(images[t], kps[t])
                ms[arm].append(timed_each(lambda t: mv.adapt_processed(images[args.warmup + t], kps[args.warmup + t]), args.frames))
                del mv
                torch.cuda.empty_cache()
        row = {'measurement': 'webcam', 'G': G, 'ticks': args.frames, 'test_basemodel': 1,
               'ms_per_tick': {k: [round(x, 3) for x in v] for k, v in ms.items()},
               'ratio_of_means': round(sum(ms['own_checkpoints']) / sum(ms['pool_checkpoint']), 4)}
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
