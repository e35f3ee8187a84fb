"""Per-layer timing of the three convolution products (forward, data gradient, weight gradient) of the HMR backbone at
batch B, for the fp32 CUDA-core kernels and the wgmma TF32x3 kernel, through the C ABI.

Each shape is launched `iters` times back to back on one stream (inputs stay in L2, as inside the running step);
the figure is the mean time per launch in microseconds, launch gaps included.  The stand-alone tensor-core entry points are
launched without programmatic dependent launch unless DBOA_CABI_PDL=1 (which this script sets: chains of the same kernel on
fixed weights are safe); DBOA_PDL=0 switches PDL off everywhere.

    python scripts/conv_microbench.py [--batch 1] [--iters 60]
"""
import argparse
import os
import sys

os.environ.setdefault('DBOA_CABI_PDL', '1')

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from dynaboa_b200 import _lib as L  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=1)
ap.add_argument('--iters', type=int, default=60)
args = ap.parse_args()
B = args.batch
lib = L.load()
lib.dboa_set_tensor_core_conv(2)

# (H_in, Cin, Cout, k, stride, pad, count in the network)
SHAPES = [
    (56, 64, 64, 1, 1, 0, 1), (56, 64, 64, 3, 1, 1, 3), (56, 64, 256, 1, 1, 0, 4), (56, 256, 64, 1, 1, 0, 2),
    (56, 256, 128, 1, 1, 0, 1), (56, 128, 128, 3, 2, 1, 1), (28, 128, 512, 1, 1, 0, 4), (56, 256, 512, 1, 2, 0, 1),
    (28, 512, 128, 1, 1, 0, 3), (28, 128, 128, 3, 1, 1, 3),
    (28, 512, 256, 1, 1, 0, 1), (28, 256, 256, 3, 2, 1, 1), (14, 256, 1024, 1, 1, 0, 6), (28, 512, 1024, 1, 2, 0, 1),
    (14, 1024, 256, 1, 1, 0, 5), (14, 256, 256, 3, 1, 1, 5),
    (14, 1024, 512, 1, 1, 0, 1), (14, 512, 512, 3, 2, 1, 1), (7, 512, 2048, 1, 1, 0, 3), (14, 1024, 2048, 1, 2, 0, 1),
    (7, 2048, 512, 1, 1, 0, 2), (7, 512, 512, 3, 1, 1, 2),
]


def timeit(fn):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / args.iters


ws = torch.empty(8 << 20, device='cuda')
tot = {k: 0.0 for k in ('fwd32', 'fwdtc', 'dg32', 'dgtc', 'wg32', 'wgtc')}
print(f'batch {B}; us per launch  (PDL={os.environ.get("DBOA_PDL", "1")})')
print(f'{"Hin":>4s} {"Cin":>5s} {"Cout":>5s} k s  n | {"fwd32":>7s} {"fwdTC":>7s} | {"dgrad32":>7s} {"dgradTC":>7s} | {"wgrad32":>7s} {"wgradTC":>7s}')
for (H, Cin, Cout, k, s, p, cnt) in SHAPES:
    Ho = (H + 2 * p - k) // s + 1
    K = k * k * Cin
    x = torch.randn(B, H, H, Cin, device='cuda')
    w = torch.randn(Cout, K, device='cuda') * 0.05
    y = torch.empty(B, Ho, Ho, Cout, device='cuda')
    dy = torch.randn(B, Ho, Ho, Cout, device='cuda')
    dx = torch.empty_like(x)
    dw = torch.zeros_like(w)
    a = (B, H, H, Cin, Cout, k, s, p, K)
    st = L.stream()
    r = {}
    r['fwd32'] = timeit(lambda: L.call('dboa_conv2d_fwd', L.ptr(x), L.ptr(w), L.ptr(y), *a, L.ptr(ws), ws.numel(), st))
    r['fwdtc'] = timeit(lambda: L.call('dboa_conv2d_tc_fwd', L.ptr(x), L.ptr(w), L.ptr(y), *a, st))
    r['dg32'] = timeit(lambda: L.call('dboa_conv2d_dgrad', L.ptr(dy), L.ptr(w), L.ptr(dx), *a, 0, L.ptr(ws), ws.numel(), st))
    r['dgtc'] = timeit(lambda: L.call('dboa_conv2d_tc_dgrad', L.ptr(dy), L.ptr(w), L.ptr(dx), *a, 0, st))
    r['wg32'] = timeit(lambda: L.call('dboa_conv2d_wgrad', L.ptr(dy), L.ptr(x), L.ptr(dw), *a, L.ptr(ws), ws.numel(), st))
    r['wgtc'] = timeit(lambda: L.call('dboa_conv2d_tc_wgrad', L.ptr(dy), L.ptr(x), L.ptr(dw), *a, st))
    for kk in tot:
        tot[kk] += r[kk] * cnt
    print(f'{H:4d} {Cin:5d} {Cout:5d} {k} {s} {cnt:2d} | {r["fwd32"]:7.2f} {r["fwdtc"]:7.2f} | {r["dg32"]:7.2f} {r["dgtc"]:7.2f} | '
          f'{r["wg32"]:7.2f} {r["wgtc"]:7.2f}')
print('network totals (us, weighted by layer count): ' + ', '.join(f'{k}={v:.0f}' for k, v in tot.items()))
