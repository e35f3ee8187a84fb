"""Time of one mesh overlay (dboa_render_overlay) at 1920 x 1080: the synthetic SMPL mesh posed by an HMR forward of the
synthetic base model, 1x and 4x sampled.  Whole call with CUDA events after warm-up, then the time of each of its kernels
(vertex, normals, face set-up, scan, raster, resolve) from torch.profiler in a separate pass.  Prints the card's name and
power limit with the numbers.  The synthetic mesh has random faces -- many very large triangles -- so it is a worst case
for fill, not what a real SMPL mesh costs.

    python scripts/render_time.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from dynaboa_b200 import config, render, synthetic  # noqa: E402
from dynaboa_b200.hmr import hmr  # noqa: E402
from dynaboa_b200.smpl import SMPL  # noqa: E402

KERNELS = ('render_vertex_kernel', 'render_normal_kernel', 'render_face_kernel', 'render_scan_kernel', 'render_raster_kernel',
           'render_resolve_kernel')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'render_time.py needs a GPU'
    work = tempfile.mkdtemp(prefix='dboa_render_time_')
    synthetic.write_asset_dir(os.path.join(work, 'data'))
    config.set_data_root(os.path.join(work, 'data'))
    m = hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict({k.replace('module.', ''): v for k, v in synthetic.make_basemodel()['model'].items()}, strict=True)
    m.eval()
    x = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    with torch.no_grad():
        rot, shape, _ = m(x)
        verts = SMPL(config.SMPL_MODEL_DIR, create_transl=False).cuda()(
            betas=shape, body_pose=rot[:, 1:], global_orient=rot[:, 0].unsqueeze(1), pose2rot=False).vertices[0].contiguous()
    faces = render.get_smpl_faces()
    W, H = 1920, 1080
    cam4 = render.convert_crop_cam_to_orig_img(np.array([[0.9, 0.05, 0.1]]), np.array([[900.0, 560.0, 400.0]]), W, H)[0]
    img = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda()
    name = card()
    for samples in (1, 4):
        def call():
            return render.draw(img, verts, faces, cam4, color=(205 / 255, 129 / 255, 98 / 255), samples=samples)
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        call_ms = e0.elapsed_time(e1) / args.iters
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
