#!/usr/bin/env python
"""Where the time of a C2 frame (bench.py's workload) goes, and what replaying it as a CUDA graph (Adaptor.adapt) changes.

    python scripts/step_graph_time.py [--frames K] [--pairs P] [--out FILE]

Per arm (eager: DBOA_STEP_GRAPH off; graph), alternated P times in one process, from the same weights:
* host enqueue per frame: perf_counter around ``adapt`` + ``predict_async`` issued on an idle device (no sync inside);
* device time per frame: CUDA events around K pipelined frames, as bench.py times them.
Then one torch.profiler run of each arm: the summed duration of the device activity of the frames against the wall span
they cover (the rest are gaps between launches).  Prints the card line with every number; ``--out`` also writes them as JSON."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gpu_timing import asset_dir, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=100)
    ap.add_argument('--pairs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import adaptor, config, synthetic
    torch.cuda.set_device(0)
    work = asset_dir('dboa_step_graph_')
    prelude, n = 12, 12 + args.frames
    opts = default_options(expdir=work, expname='t', model_file=config.BASE_MODEL, synthetic_frames=n, **WORKLOADS['c2'])
    ad = adaptor.Adaptor(opts)
    ad.fused_eval = 'none'
    stream = synthetic.SyntheticStream(length=n, batch_size=1)
    frames = [{k: stream[t][k].cuda() for k in ('image', 'smpl_j2d')} for t in range(n)]
    snap = (ad.model.module.arena.clone(), ad.teacher.arena.clone())

    def frame(t):
        ad.global_step, ad.fit_losses = t, {}
        ad.adapt(frames[t])
        ad.predict_async(frames[t]['image'])

    def restart(graph):
        adaptor.STEP_GRAPH = graph
        ad.model.module.arena.copy_(snap[0]); ad.teacher.arena.copy_(snap[1])
        ad.optimizer.m.zero_(); ad.optimizer.v.zero_(); ad.optimizer.step_count = 0
        ad.reset_records()
        for t in range(prelude):
            frame(t)
        torch.cuda.synchronize()

    def measure(graph):
        restart(graph)
        host = []
        for t in range(prelude, n):                       # one frame at a time on an idle device: the enqueue cost alone
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            frame(t)
            host.append((time.perf_counter() - t0) * 1e3)
        restart(graph)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for t in range(prelude, n):
            frame(t)
        torch.cuda.current_stream().wait_stream(ad.output_stream)
        e1.record()
        e1.synchronize()
        return statistics.median(host), e0.elapsed_time(e1) / args.frames

    line = card()
    rows = []
    for p in range(args.pairs):
        for graph in (False, True):
            h, d = measure(graph)
            rows.append({'arm': 'graph' if graph else 'eager', 'pair': p, 'host_enqueue_ms': h, 'device_ms_per_frame': d})
            print(f'[{line}] pair {p} {rows[-1]["arm"]:5s}: host enqueue {h:.2f} ms/frame, device {d:.2f} ms/frame', flush=True)

    from torch.profiler import ProfilerActivity, profile
    trace = {}
    for graph in (False, True):
        restart(graph)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for t in range(prelude, prelude + 10):
                frame(t)
            torch.cuda.synchronize()
        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        busy = sum(e.time_range.elapsed_us() for e in ev) / 1e3
        span = (max(e.time_range.end for e in ev) - min(e.time_range.start for e in ev)) / 1e3
        arm = 'graph' if graph else 'eager'
        trace[arm] = {'device_activities': len(ev), 'busy_ms_per_frame': busy / 10, 'span_ms_per_frame': span / 10}
        print(f'[{line}] profiler {arm}: {len(ev) / 10:.0f} device activities/frame, summed duration {busy / 10:.2f} ms/frame over a '
              f'span of {span / 10:.2f} ms/frame (both streams)', flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump({'card': line, 'fields': 'name, power limit, SM clock, max SM clock', 'rows': rows, 'profiler': trace}, f, indent=1)


if __name__ == '__main__':
    main()
