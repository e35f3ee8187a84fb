"""Grouped mesh overlay (dboa_render_overlay_groups) against the same meshes drawn by one dboa_render_overlay call each.

A webcam pool tick of G streams draws 2 G meshes: per stream the adapted and the base mesh, each over its own copy of the
stream's frame.  For G in {1, 2, 4, 8, 16}, frames of 640 x 480, 1280 x 720 and 1920 x 1080, 1 and 4 samples and two meshes
(the synthetic SMPL mesh posed by an HMR forward of the synthetic base model -- its faces join random vertices, so it is a
worst case for fill -- and the closed UV sphere of tests/harness.py), the two ways are alternated in one process
after warm-up.  Each round is timed with CUDA events and with the host clock, both from the first launch to the end of the
last kernel; the medians over the rounds are printed with the card (name, power limit, SM clocks).

    python scripts/render_groups_time.py [--rounds 15] [--sizes 640x480,1280x720,1920x1080] [--streams 1,2,4,8,16]
"""
import argparse
import json

import numpy as np
import torch

from gpu_timing import asset_dir, card, posed_smpl_mesh, timed_once
from dynaboa_b200 import render  # noqa: E402  (importable once gpu_timing has put the repository on sys.path)
from harness import sphere  # noqa: E402


def tick(G, W, H, verts, seed):
    """2 G entries: stream g's frame twice, the adapted mesh (205, 129, 98) and the base mesh (100, 100, 200) with two crop
    cameras around a box in the middle of the frame."""
    rng = np.random.default_rng(seed)
    imgs, vs, cams, cols = [], [], [], []
    for g in range(G):
        img = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed + g)).cuda()
        box = np.array([[W * rng.uniform(0.4, 0.6), H * rng.uniform(0.4, 0.6), 0.7 * H]])
        for col in ((205, 129, 98), (100, 100, 200)):
            cam = np.array([[rng.uniform(0.8, 1.0), rng.uniform(-0.05, 0.05), rng.uniform(0.0, 0.15)]])
            imgs.append(img)
            vs.append(verts)
            cams.append(render.convert_crop_cam_to_orig_img(cam, box, W, H)[0])
            cols.append(np.array(col) / 255)
    return imgs, vs, cams, cols


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=15)
    ap.add_argument('--sizes', default='640x480,1280x720,1920x1080')
    ap.add_argument('--streams', default='1,2,4,8,16')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'render_groups_time.py needs a GPU'
    sv, sf = sphere()
    asset_dir('dboa_render_groups_time_')
    meshes = {'smpl': posed_smpl_mesh()[:2], 'sphere': (torch.from_numpy(sv).cuda(), sf)}
    name = card()
    sizes = [tuple(int(x) for x in s.split('x')) for s in args.sizes.split(',')]
    for mesh, (verts, faces) in meshes.items():
        for W, H in sizes:
            for samples in (1, 4):
                for G in [int(g) for g in args.streams.split(',')]:
                    imgs, vs, cams, cols = tick(G, W, H, verts, 1000 * G + W)

                    def singles():
                        return [render.draw(i, v, faces, c, color=col, samples=samples) for i, v, c, col in zip(imgs, vs, cams, cols)]

                    def grouped():
                        return render.draw_groups(imgs, vs, faces, cams, cols, samples=samples)
                    a, b = singles(), grouped()
                    assert all(torch.equal(x, y) for x, y in zip(a, b))
                    for _ in range(3):
                        singles()
                        grouped()
                    t_single, t_group = [], []
                    for _ in range(args.rounds):
                        t_single.append(timed_once(singles))
                        t_group.append(timed_once(grouped))
                    s_ev, s_wall = np.median([t[0] for t in t_single]), np.median([t[1] for t in t_single])
                    g_ev, g_wall = np.median([t[0] for t in t_group]), np.median([t[1] for t in t_group])
                    print(json.dumps({'card': name, 'mesh': mesh, 'W': W, 'H': H, 'samples': samples, 'streams': G, 'meshes': 2 * G,
                                      'single_ms': round(float(s_ev), 3), 'grouped_ms': round(float(g_ev), 3),
                                      'single_wall_ms': round(float(s_wall), 3), 'grouped_wall_ms': round(float(g_wall), 3),
                                      'speedup_wall': round(float(s_wall / g_wall), 2)}), flush=True)


if __name__ == '__main__':
    main()
