"""In-situ kernel timeline of one adapted frame (workload C2) through CUPTI (torch.profiler).

ncu serialises kernels and flushes caches between replays, so its per-launch durations are cold and say nothing
about the gaps between launches.  This script records the running step instead: for every kernel its start and
duration on the device, from which it prints (a) per-kernel-name count / total / mean, (b) the busy time of the
device versus the span of the frame (the rest is launch gaps / dependencies), (c) how much of the span has two or
more kernels in flight (stream overlap).  Writes traces/trace_<tag>.json (summary) next to the table.

    python scripts/trace_step.py --tag r02 [--region frame|forward|fwdbwd]
"""
import argparse
import json
import os
import sys
import tempfile
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

ap = argparse.ArgumentParser()
ap.add_argument('--region', default='frame', choices=['frame', 'forward', 'fwdbwd'])
ap.add_argument('--tc', type=int, default=-1)
ap.add_argument('--tag', default='trace')
ap.add_argument('--batch', type=int, default=1)
args = ap.parse_args()

from bench import WORKLOADS, default_options  # noqa: E402
from dynaboa_b200 import _lib, config, hmr as hmr_mod, synthetic  # noqa: E402
from dynaboa_b200.adaptor import Adaptor  # noqa: E402

lib = _lib.load()
if args.tc >= 0:
    lib.dboa_set_tensor_core_conv(args.tc)
work = tempfile.mkdtemp(prefix='dboa_trace_')
synthetic.write_asset_dir(os.path.join(work, 'data'))
config.set_data_root(os.path.join(work, 'data'))
opts = default_options(expdir=work, expname='trace', model_file=config.BASE_MODEL, synthetic_frames=12, **WORKLOADS['c2'])
ad = Adaptor(opts)
ad.fused_eval = 'none'
stream = synthetic.SyntheticStream(length=12, batch_size=1)
frames = [{k: v.cuda() if torch.is_tensor(v) else v for k, v in stream[t].items()} for t in range(12)]
model = ad.model.module


def region():
    if args.region == 'frame':
        ad.global_step = 9
        ad.adapt(frames[9])
        ad.predict(frames[9]['image'])
    else:
        rot, shape, cam, _, _ = hmr_mod.raw_forward(model.arena, model._buffers, X, None, TAPE)
        if args.region == 'fwdbwd':
            hmr_mod.raw_backward(model.arena, TAPE, args.batch, False, torch.ones_like(rot), torch.ones_like(shape), torch.ones_like(cam), GA)


if args.region == 'frame':
    for t in range(9):
        ad.global_step, ad.fit_losses = t, {}
        ad.adapt(frames[t])
else:
    X = frames[0]['image'].repeat(args.batch, 1, 1, 1)
    TAPE = torch.empty(hmr_mod.tape_floats(args.batch), device='cuda')
    GA = torch.zeros_like(model.arena)
    for _ in range(3):
        region()
torch.cuda.synchronize()
import time  # noqa: E402
t0 = time.perf_counter()
region()
t1 = time.perf_counter()
torch.cuda.synchronize()
t2 = time.perf_counter()
print(f'cpu issue time of the region: {(t1 - t0) * 1e3:.2f} ms; until device idle: {(t2 - t0) * 1e3:.2f} ms')
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    region()
    torch.cuda.synchronize()

evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total >= 0
       and not e.name.lower().startswith('memcpy') and not e.name.lower().startswith('memset')]
copies = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
          and (e.name.lower().startswith('memcpy') or e.name.lower().startswith('memset'))]
iv = sorted((e.time_range.start, e.time_range.end) for e in evs + copies)
span = iv[-1][1] - iv[0][0]
busy, overlap, cur_end = 0.0, 0.0, iv[0][0]
points = sorted([(s, 1) for s, _ in iv] + [(e, -1) for _, e in iv])
depth, last = 0, points[0][0]
for tpt, d in points:
    if depth >= 1:
        busy += tpt - last
    if depth >= 2:
        overlap += tpt - last
    depth += d
    last = tpt
by = defaultdict(lambda: [0, 0.0])
for e in evs:
    name = e.name.split('(')[0].split('<')[0].replace('void ', '').replace('dboa::', '')
    by[name][0] += 1
    by[name][1] += e.time_range.end - e.time_range.start
rows = sorted(by.items(), key=lambda kv: -kv[1][1])
tot = sum(v[1] for v in by.values())
print(f'region={args.region} kernels={len(evs)} copies={len(copies)} span={span:.0f}us busy={busy:.0f}us ({busy / span:.1%}) '
      f'overlap>=2={overlap:.0f}us sum_kernel={tot:.0f}us')
print(f'{"kernel":48s} {"n":>5s} {"total_us":>10s} {"mean_us":>9s} {"share":>7s}')
for k, (n, t) in rows[:40]:
    print(f'{k[:48]:48s} {n:5d} {t:10.1f} {t / n:9.2f} {t / tot:7.1%}')
os.makedirs(os.path.join(REPO, 'traces'), exist_ok=True)
with open(os.path.join(REPO, 'traces', f'trace_{args.tag}_{args.region}.json'), 'w') as f:
    json.dump({'region': args.region, 'kernels': len(evs), 'span_us': span, 'busy_us': busy, 'overlap_us': overlap,
               'by_kernel': [{'name': k, 'n': n, 'total_us': t, 'mean_us': t / n} for k, (n, t) in rows]}, f, indent=1)
