"""Cost of adapting G Internet videos with ``MultiInternetAdaptor.run`` against G ``InternetAdaptor.excute(fused=True)`` runs one
after another.  Prints the card (name, power limit, SM clock, max SM clock), then one JSON line per (G, save_res):

- pool_fps / sequential_fps: adapted frames per second, from the start of ``run`` (or of the first ``excute``) to the last
  file on disk and a device sync, host clock;
- decode / upload / encode shares: host time spent decoding frames (cv2, on the I/O threads), uploading them (main thread) and
  encoding and writing PNGs and Pred files (I/O threads), each over the pool's wall time (the threads overlap the main thread,
  so the shares may add up to more than 1).

The G sequences are synthetic 1920 x 1080 PNG frames generated from a seed into a temporary directory, in the reference's npz
layout.  Options: run_on_internet.sh's flags (retrieval, mix-training, dynamic loop at 3.1e-4, shape prior 2e-4).  With
save_res 1 the sequential runs draw every frame as the reference driver's ``inference`` does (``BaseAdaptor.save_results``).

    python scripts/multiinternet_time.py [--frames 12] [--groups 1 4 8] [--out FILE]"""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

from gpu_timing import CARD_FIELDS, asset_dir, card

INTERNET = dict(motionloss_weight=0.8, retrieval=1, dynamic_boa=1, optim_steps=7, cos_sim_threshold=3.1e-4, shape_prior_weight=2e-4,
                pose_prior_weight=1e-4)


def write_sequences(root, G, n, seed=0):
    """G sequences of n 1080 x 1920 frames under root, one npz each (``s<g>.npz``), frames in root/images."""
    import cv2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    rng = np.random.default_rng(seed)
    for g in range(G):
        base = cv2.resize(cv2.GaussianBlur(rng.uniform(0, 255, size=(135, 240, 3)).astype(np.float32), (0, 0), 2), (1920, 1080))
        names, centers, scales, parts = [], [], [], []
        for t in range(n):
            frame = np.clip(np.roll(base, 4 * t, axis=1) + rng.normal(0, 2, base.shape), 0, 255).astype(np.uint8)
            names.append(f's{g}_{t:04d}.png')
            cv2.imwrite(os.path.join(root, 'images', names[-1]), frame)
            c = np.array([960.0, 540.0]) + rng.uniform(-100, 100, size=2)
            s = 2.6 * rng.uniform(0.95, 1.05)
            centers.append(c); scales.append(s)
            parts.append(np.concatenate([c + rng.uniform(-110, 110, size=(49, 2)) * s, np.ones((49, 1))], 1))
        np.savez(os.path.join(root, f's{g}.npz'), imgname=np.array(names), center=np.stack(centers), scale=np.array(scales),
                 part=np.stack(parts))


def options(work, name, save_res):
    from dynaboa_b200 import config
    from oracle import adaptor_ref
    o = vars(adaptor_ref.default_options(**INTERNET))
    o.update(expdir=work, expname=name, tensorboard=0, cache_results=1, model_file=config.BASE_MODEL, dataset='internet',
             save_res=save_res, seq_seed=22)
    return SimpleNamespace(**o)


def drawing_adaptor():
    """``InternetAdaptor`` whose ``inference`` also draws with ``save_res`` (reference dynaboa_internet.py:142-168)."""
    from dynaboa_b200 import constants
    from dynaboa_b200.adaptor import InternetAdaptor

    class Drawing(InternetAdaptor):
        def inference(self, batch, model, need_feature=False):
            import joblib
            model.eval()
            with torch.no_grad():
                out = model(batch['image'], need_feature)
                rot, shape, cam = out[0], out[1], out[2]
                verts = self.decode_smpl_params(rot, shape)['vts']
            cam_t = torch.stack([cam[:, 1], cam[:, 2], 2 * 5000. / (constants.IMG_RES * cam[:, 0] + 1e-9)], dim=-1)
            joblib.dump({'verts': verts.cpu().numpy(), 'cam': cam_t.cpu().numpy(), 'rotmat': rot.cpu().numpy(), 'beta': shape.cpu().numpy()},
                        os.path.join(self.exppath, 'result', f'Pred_{self.global_step}.pt'))
            if self.options.save_res:
                self.save_results(verts, cam, batch['image'], batch['imgname'], batch['bbox'], prefix='Pred')
            zero = np.zeros(rot.shape[0], np.float32)
            return (zero, zero, 0.0, out[3]) if need_feature else (zero, zero, 0.0)
    return Drawing


class Clock:
    """Host seconds spent inside wrapped functions, summed over threads."""

    def __init__(self):
        self.s = {}

    def wrap(self, key, fn):
        def timed(*a, **k):
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                self.s[key] = self.s.get(key, 0.0) + time.perf_counter() - t0
        return timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--groups', type=int, nargs='+', default=[1, 4, 8])
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    out = os.path.abspath(args.out) if args.out else None      # before the chdir below
    if not torch.cuda.is_available():
        sys.exit('multiinternet_time.py needs a GPU')
    from dynaboa_b200 import internet
    from dynaboa_b200.datasets import internet_videos
    work = asset_dir('dboa_internet_')
    os.chdir(work)                                          # save_results writes demo.obj into the working directory
    info = card()
    print(f'card ({CARD_FIELDS}): {info}', flush=True)
    Drawing = drawing_adaptor()
    rows = []
    for G in args.groups:
        root = tempfile.mkdtemp(prefix=f'seq{G}_', dir=work)
        write_sequences(root, G, args.frames, seed=G)
        vids = internet_videos(root)
        for save_res in (0, 1):
            tag = f'G{G}_r{save_res}'
            mv = internet.MultiInternetAdaptor(options(work, f'pool_{tag}', save_res), G, dynamic_loop=True)
            mv.run([vids[0]], os.path.join(work, f'warm_{tag}'))                # warm-up: every shape of a tick
            clock = Clock()
            decode, upload, writer = internet.decode, mv._upload, mv.writer
            internet.decode = clock.wrap('decode', decode)
            mv._upload = clock.wrap('upload', upload)
            writer.pred, writer.image = clock.wrap('encode', writer.pred), clock.wrap('encode', writer.image)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mv.run(vids, os.path.join(work, f'out_{tag}'))
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            internet.decode = decode
            del mv
            torch.cuda.empty_cache()
            seq = 0.0
            for g in range(G):
                one = os.path.join(root, f'one{g}')
                if not os.path.exists(one):
                    os.makedirs(one)
                    os.symlink(os.path.join(root, 'images'), os.path.join(one, 'images'))
                    os.symlink(os.path.join(root, f's{g}.npz'), os.path.join(one, f's{g}.npz'))
                os.environ['DYNABOA_INTERNET_ROOT'] = one
                ad = Drawing(options(work, f'seq_{tag}_{g}', save_res))
                if g == 0:
                    ad.excute(max_frames=2, fused=True)                          # warm-up
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                ad.excute(fused=True)
                torch.cuda.synchronize()
                seq += time.perf_counter() - t1
                del ad
                torch.cuda.empty_cache()
            frames = G * args.frames
            r = {'G': G, 'save_res': save_res, 'frames': frames, 'pool_fps': round(frames / wall, 2),
                 'sequential_fps': round(frames / seq, 2), 'pool_over_sequential': round(seq / wall, 3),
                 'decode_share': round(clock.s.get('decode', 0.0) / wall, 3), 'upload_share': round(clock.s.get('upload', 0.0) / wall, 3),
                 'encode_share': round(clock.s.get('encode', 0.0) / wall, 3)}
            print(json.dumps(r), flush=True)
            rows.append(r)
    if out:
        with open(out, 'w') as f:
            json.dump({'card': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
