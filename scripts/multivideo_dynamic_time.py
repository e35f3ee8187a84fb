"""The per-video dynamic loop of ``MultiVideoAdaptor(..., dynamic_loop=True)`` at C5 (``bench.py``'s c5 flags: 3 inner steps,
retrieval with 8 exemplars, ``cos_sim_threshold`` 2e-5, ``optim_steps`` 7, teacher dropout live).  Prints the card and its power
limit, then one JSON line per G in {1, 2, 4, 8}:

- grouped: G videos (``SyntheticStream(rank=g)``) in one pool, every slot active, `frames` timed pool frames after `warmup`
  untimed ones (from frame `warmup` on the motion term is live);
- sequential: the same G videos one after another through ``Adaptor.adapt``, the same frames timed;
- ms per pool frame (grouped) and per G frames (sequential), adapted frames/s, from CUDA events;
- per pool frame of the timed part: the mean and maximum trip count over the videos, and the host syncs of the feature tests
  (1 + the longest loop), against the sum over the videos of 1 + their loop lengths for the sequential runs;
- how many (video, frame) trip counts differ between the grouped and the sequential runs.

Both arms draw the same teacher masks and retrieval seeds per (video, frame).

    python scripts/multivideo_dynamic_time.py [--frames 8] [--warmup 6] [--groups 1 2 4 8] [--out FILE]"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=6)
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 2, 4, 8])
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('multivideo_dynamic_time.py needs a GPU')
    from bench import N_EXEMPLARS, WORKLOADS, default_options
    from dynaboa_b200 import config, synthetic
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    work = tempfile.mkdtemp(prefix='dboa_dyn_')
    synthetic.write_asset_dir(os.path.join(work, 'data'), n_exemplars=N_EXEMPLARS)
    config.set_data_root(os.path.join(work, 'data'))
    n = args.warmup + args.frames
    opts = lambda name: default_options(expdir=work, expname=name, model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c5'])
    cap = opts('x').optim_steps
    Gmax = max(args.groups)
    streams = [synthetic.SyntheticStream(length=n, batch_size=1, rank=g) for g in range(Gmax)]
    frames = [[{k: v.cuda() if torch.is_tensor(v) else v for k, v in s[t].items()} for t in range(n)] for s in streams]
    # teacher keep-masks per (video, frame, teacher forward), made before anything is timed
    gen = torch.Generator().manual_seed(0)
    masks = {(g, t, c): ((torch.rand(3, 2, 1, 1024, generator=gen) >= 0.5).float() * 2.0).cuda()
             for g in range(Gmax) for t in range(n) for c in range(1 + cap)}
    seed = lambda g, t: 7919 * g + t
    info = card()
    print(f'card (name, power limit): {info}', flush=True)

    def timed(fn, ts):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for t in ts:
            fn(t)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    single = Adaptor(opts('single'))
    single.fused_eval = 'none'
    snap = (single.model.module.arena.clone(), single.teacher.arena.clone())
    rows = []
    for G in args.groups:
        # grouped
        mv = MultiVideoAdaptor(opts(f'pool{G}'), G, dynamic_loop=True)
        calls = [0] * G
        cur = {'t': 0}

        def provider(g, B, dev):
            m = masks[(g, cur['t'], min(calls[g], cap))]
            calls[g] += 1
            return m

        mv.mask_provider = provider

        def pool_step(t):
            cur['t'] = t
            for g in range(G):
                calls[g] = 0
                mv.rngs[g].seed(seed(g, t))
            mv.adapt([frames[g][t] for g in range(G)])
        for t in range(args.warmup):
            pool_step(t)
        pool_ms = timed(pool_step, range(args.warmup, n))
        pool_trips = [rec[args.warmup:] for rec in mv.optim_step_record]
        del mv
        torch.cuda.empty_cache()
        # sequential
        seq_ms, seq_trips = 0.0, []
        for g in range(G):
            ad = single
            ad.model.module.arena.copy_(snap[0])
            ad.teacher.arena.copy_(snap[1])
            ad.optimizer.m.zero_(); ad.optimizer.v.zero_(); ad.optimizer.step_count = 0
            ad.history, ad.optim_step_record, ad.feat_sims = {}, [], {}

            def one(t, g=g, ad=ad):
                c = {'i': 0}

                def prov(B, dev):
                    m = masks[(g, t, min(c['i'], cap))]
                    c['i'] += 1
                    return m
                ad.teacher.mask_provider = prov
                random.seed(seed(g, t))
                ad.global_step, ad.fit_losses = t, {}
                ad.adapt(frames[g][t])
            for t in range(args.warmup):
                one(t)
            seq_ms += timed(one, range(args.warmup, n))
            seq_trips.append(list(ad.optim_step_record[args.warmup:]))
        F = args.frames
        loops = lambda trips: [[min(x, cap) for x in r] for r in trips]
        pl, sl = loops(pool_trips), loops(seq_trips)
        pool_syncs = [1 + max(pl[g][t] for g in range(G)) for t in range(F)]
        seq_syncs = [sum(1 + sl[g][t] for g in range(G)) for t in range(F)]
        r = {'workload': 'c5', 'G': G, 'timed_frames': F, 'warmup_frames': args.warmup,
             'grouped': {'ms_per_pool_frame': round(pool_ms / F, 2), 'adapted_frames_per_s': round(1000.0 * G * F / pool_ms, 2),
                         'trips_mean_per_frame': [round(sum(pool_trips[g][t] for g in range(G)) / G, 2) for t in range(F)],
                         'trips_max_per_frame': [max(pool_trips[g][t] for g in range(G)) for t in range(F)],
                         'feature_test_syncs_per_frame': pool_syncs},
             'sequential': {'ms_per_G_frames': round(seq_ms / F, 2), 'adapted_frames_per_s': round(1000.0 * G * F / seq_ms, 2),
                            'feature_test_syncs_per_frame': seq_syncs},
             'speedup': round(seq_ms / pool_ms, 3),
             'trip_counts_differing': sum(pool_trips[g][t] != seq_trips[g][t] for g in range(G) for t in range(F)),
             'trip_counts_compared': G * F, 'trips_grouped': pool_trips, 'trips_sequential': seq_trips}
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
