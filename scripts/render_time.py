"""Time of one mesh overlay (dboa_render_overlay) at 1920 x 1080: the synthetic SMPL mesh posed by an HMR forward of the
synthetic base model, 1x and 4x sampled.  Whole call with CUDA events after warm-up, then the time of each of its kernels
(vertex, normals, face set-up, scan, raster, resolve) from torch.profiler in a separate pass.  Prints the card (name, power
limit, SM clocks) with the numbers.  The synthetic mesh has random faces -- many very large triangles -- so it is a worst case
for fill, not what a real SMPL mesh costs.

    python scripts/render_time.py [--iters 50]
"""
import argparse
import json

import torch

from gpu_timing import asset_dir, card, posed_smpl_mesh, timed_window
from dynaboa_b200 import render  # noqa: E402  (importable once gpu_timing has put the repository on sys.path)

KERNELS = ('render_vertex_kernel', 'render_normal_kernel', 'render_face_kernel', 'render_scan_kernel', 'render_raster_kernel',
           'render_resolve_kernel')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'render_time.py needs a GPU'
    asset_dir('dboa_render_time_')
    verts, faces, cam4 = posed_smpl_mesh()
    W, H = 1920, 1080
    img = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda()
    name = card()
    for samples in (1, 4):
        def call():
            return render.draw(img, verts, faces, cam4, color=(205 / 255, 129 / 255, 98 / 255), samples=samples)
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        call_ms = timed_window(lambda _: call(), range(args.iters)) / args.iters
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                call()
            torch.cuda.synchronize()
        per = {k: 0.0 for k in KERNELS}
        for ev in prof.key_averages():
            for k in KERNELS:
                if k in ev.key:
                    per[k] += ev.device_time_total / 1000.0 / args.iters
        covered = int((render.draw(img, verts, faces, cam4, samples=samples, face_ids=True)[1] >= 0).any(2).sum())
        print(json.dumps({'card': name, 'W': W, 'H': H, 'samples': samples, 'NV': int(verts.shape[0]), 'NF': int(len(faces)),
                          'covered_pixels': covered, 'call_ms': round(call_ms, 4),
                          'kernel_ms': {k.replace('render_', '').replace('_kernel', ''): round(v, 4) for k, v in per.items()}}))


if __name__ == '__main__':
    main()
