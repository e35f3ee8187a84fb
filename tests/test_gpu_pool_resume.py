"""Saving and resuming the pools (MultiVideoAdaptor.save / load / save_slot / start(g, state=...), run(checkpoint=...), and the
same through MultiInternetAdaptor and MultiWebcamAdaptor), bit for bit against the uninterrupted runs: theta, teacher, Adam
m / v, step and frame counts, upper losses, every record, trip counts and predictions, and byte-identical result files."""
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from harness import FLAGS, MIXED_THRESHOLD, N_FRAMES, PoolRun, bits, fetch, pool_options, state, stream, webcam_pool

pytestmark = pytest.mark.gpu


def same(a, b):
    return torch.equal(bits(a), bits(b))


def same_values(a, b):
    """Records and summaries equal value for value, floats and arrays bit for bit (NaN included), and the pickles of both
    byte-identical (what the result files are written with)."""
    def eq(x, y):
        if isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
            return type(x) is type(y) and x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
        if isinstance(x, float) or isinstance(y, float):
            return type(x) is type(y) and np.float64(x).tobytes() == np.float64(y).tobytes()
        if isinstance(x, dict):
            return type(x) is type(y) and list(x) == list(y) and all(eq(x[k], y[k]) for k in x)
        if isinstance(x, (list, tuple)):
            return type(x) is type(y) and len(x) == len(y) and all(eq(p, q) for p, q in zip(x, y))
        return type(x) is type(y) and x == y
    return eq(a, b) and pickle.dumps(a) == pickle.dumps(b)


def snapshot(mv, g, images):
    return state(mv, g) + [mv.last_upper_loss[g:g + 1].clone()] + [mv.predict(images)[g]['vertices'].clone()]


def check(ta, tb, what):
    assert len(ta) == len(tb)
    for t, (ra, rb) in enumerate(zip(ta, tb)):
        for name, x, y in zip(('theta', 'teacher', 'm', 'v', 'upper loss', 'vertices'), ra, rb):
            assert same(x, y), (what, t, name)


def test_pool_checkpoint_continues_in_a_new_pool(asset_dir, tmp_path, golden):
    """G = 4 at C2, teacher masks from torch's generator: saved after pool frame 3 with slot 2 sitting frames out, then
    continued in the original pool and, from the checkpoint, in a new one."""
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    streams = [stream(10 + g, 8) for g in range(4)]
    idle = {1: [2], 2: [2], 4: [1]}                             # pool frame -> slots that sit it out

    def tick(mv, f):
        batches = [None if g in idle.get(f, []) else fetch(streams[g][mv.video_steps[g]]) for g in range(4)]
        mv.adapt(batches)
        return torch.cat([fetch(streams[g][max(mv.video_steps[g] - 1, 0)])['image'] for g in range(4)])

    def pool(name):
        mv = MultiVideoAdaptor(pool_options(tmp_path, golden, 'c2', name), 4)
        mv.fused_eval = 'final'
        return mv
    ck = str(tmp_path / 'ck')
    a = pool('a')
    for f in range(3):
        tick(a, f)
    a.save(ck)
    ta = []
    for f in range(3, 7):
        images = tick(a, f)
        ta.append([snapshot(a, g, images) for g in range(4)])
    ra = [a.records(g) for g in range(4)]
    del a
    b = pool('b')
    assert b.load(ck) is None                                 # a pool driven by adapt: no run
    assert b.global_step == 3 and b.video_steps == [3, 3, 1, 3]
    tb = []
    for f in range(3, 7):
        images = tick(b, f)
        tb.append([snapshot(b, g, images) for g in range(4)])
    for g in range(4):
        check([x[g] for x in ta], [x[g] for x in tb], g)
        assert same_values(b.records(g), ra[g]), g


@pytest.mark.parametrize('dynamic', [False, True], ids=['c2', 'c5-dynamic'])
def test_a_slot_moves_to_another_slot_and_pool(asset_dir, tmp_path, golden, dynamic):
    """Slot 1 saved after 3 frames and restored into slot 3 of another G = 4 pool: identical to its uninterrupted run (masks
    from mask_provider, as the schedule-invariance tests give them)."""
    tag, extra = ('c5', dict(cos_sim_threshold=MIXED_THRESHOLD)) if dynamic else ('c2', {})
    k, path = 3, str(tmp_path / 'slot1.pt')
    a = PoolRun(pool_options(tmp_path, golden, tag, 'a', **extra), 4, dynamic_loop=dynamic)
    for g in range(4):
        a.start(g, g, stream(g, N_FRAMES))
    for _ in range(k):
        a.step([0, 1, 2, 3])
    a.mv.save_slot(1, path)
    ta = []
    for _ in range(N_FRAMES - k):
        a.step([0, 1, 2, 3])
        ta.append(a.state(1) + [a.mv.last_upper_loss[1:2].clone()])
    rec_a = a.mv.records(1)
    del a
    b = PoolRun(pool_options(tmp_path, golden, tag, 'b', **extra), 4, dynamic_loop=dynamic)
    for g in range(3):
        b.start(g, 20 + g, stream(20 + g, N_FRAMES))
    b.mv.start(3, state=path)
    b.slot[3] = [1, stream(1, N_FRAMES), k]
    assert b.mv.video_steps[3] == k
    tb = []
    for _ in range(N_FRAMES - k):
        b.step([0, 1, 2, 3])
        tb.append(b.state(3) + [b.mv.last_upper_loss[3:4].clone()])
    check(ta, tb, 'slot 1 -> 3')
    rec_b = b.mv.records(3)
    assert same_values(rec_a, rec_b)
    if dynamic:
        assert rec_b['optim_step_record'] and any(rec_b['optim_step_record']), 'the dynamic loop never ran'
    small = PoolRun(pool_options(tmp_path, golden, tag, 'c', **extra), 2, dynamic_loop=dynamic)
    with pytest.raises(ValueError, match='4 slots'):
        small.mv.start(0, state=path)


class Stop(Exception):
    pass


class Cut:
    """The items of `video`, then Stop instead of item k."""

    def __init__(self, video, k):
        self.video, self.k = video, k

    def __iter__(self):
        for t, item in enumerate(self.video):
            if t == self.k:
                raise Stop
            yield item


def tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            with open(os.path.join(d, f), 'rb') as fh:
                out[os.path.relpath(os.path.join(d, f), root)] = fh.read()
    return out


def test_run_resumes_mid_queue(asset_dir, tmp_path, golden):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    lengths = [3, 6, 2, 5, 4, 3]

    def pool(name):
        mv = MultiVideoAdaptor(pool_options(tmp_path, golden, 'c2', name), 4)
        mv.fused_eval = 'final'
        return mv
    videos = [stream(30 + i, n) for i, n in enumerate(lengths)]
    want = pool('straight').run(videos, str(tmp_path / 'out_straight'))
    ck, out = str(tmp_path / 'ck'), str(tmp_path / 'out_resumed')
    cut = list(videos)
    cut[4] = Cut(videos[4], 2)                                 # video 4 starts in slot 2 at tick 2 and stops the run at tick 4
    with pytest.raises(Stop):
        pool('cut').run(cut, out, checkpoint=ck, every=2)
    assert not os.path.exists(os.path.join(out, '4'))
    got = pool('resumed').run(videos, out, checkpoint=ck, every=2)
    assert same_values(got, want)
    a, b = tree(tmp_path / 'out_straight'), tree(out)
    assert sorted(a) == sorted(b) and len(a) == 8 * len(lengths)
    for f in a:
        assert a[f] == b[f], f
    again = pool('again').run(videos, out, checkpoint=ck, every=2)         # a finished run: its summaries, nothing recomputed
    assert same_values(again, want)


# ------------------------------------------------------------------ Internet pool
SPECS = [('v0', (240, 320), 5), ('v1', (360, 480), 3), ('v2', (240, 320), 2), ('v3', (300, 400), 4)]


def write_videos(root):
    import cv2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    for k, (name, (H, W), n) in enumerate(SPECS):
        rng = np.random.default_rng(k + 40)
        base = cv2.resize(cv2.GaussianBlur(rng.uniform(0, 255, size=(H // 8, W // 8, 3)).astype(np.float32), (0, 0), 2), (W, H))
        names, centers, scales, parts = [], [], [], []
        for t in range(n):
            frame = np.clip(np.roll(base, 3 * t, axis=1) + rng.normal(0, 2, base.shape), 0, 255).astype(np.uint8)
            names.append(f'{name}_{t:03d}.png')
            cv2.imwrite(os.path.join(root, 'images', names[-1]), frame[:, :, ::-1])
            center = np.array([W / 2 + rng.uniform(-W / 10, W / 10), H / 2 + rng.uniform(-H / 10, H / 10)])
            scale = H / 2 / 200 * rng.uniform(0.9, 1.1)
            kp = np.concatenate([center + rng.uniform(-45, 45, size=(49, 2)) * scale, (rng.uniform(size=(49, 1)) > 0.1)], 1)
            centers.append(center); scales.append(scale); parts.append(kp)
        np.savez(os.path.join(root, f'{name}.npz'), imgname=np.array(names), center=np.stack(centers), scale=np.array(scales),
                 part=np.stack(parts))


def test_internet_run_resumes_with_identical_files(asset_dir, tmp_path):
    from dynaboa_b200 import config
    from dynaboa_b200.datasets import internet_videos
    from dynaboa_b200.internet import MultiInternetAdaptor
    from oracle import adaptor_ref
    root = str(tmp_path / 'videos')
    write_videos(root)
    vids = internet_videos(root)

    def options(name):
        o = vars(adaptor_ref.default_options(**FLAGS))
        o.update(expdir=str(tmp_path), expname=name, tensorboard=0, cache_results=1, model_file=config.BASE_MODEL, dataset='internet',
                 save_res=1, seq_seed=22)
        return SimpleNamespace(**o)

    class Cut(MultiInternetAdaptor):
        ticks = 5

        def input_side(self, frames):
            Cut.ticks -= 1
            if Cut.ticks < 0:
                raise Stop
            return super().input_side(frames)
    want = MultiInternetAdaptor(options('a'), 2).run(vids, str(tmp_path / 'straight'))
    ck, out = str(tmp_path / 'ck'), str(tmp_path / 'resumed')
    with pytest.raises(Stop):
        Cut(options('b'), 2).run(vids, out, checkpoint=ck, every=2)
    got = MultiInternetAdaptor(options('c'), 2).run(vids, out, checkpoint=ck, every=2)
    assert got == want
    a, b = tree(tmp_path / 'straight'), tree(out)
    assert sorted(a) == sorted(b) and len(a) == 2 * sum(n for _, _, n in SPECS)
    for f in a:
        assert a[f] == b[f], f


def test_webcam_stream_moves_across_pools(asset_dir, tmp_path, golden):
    gd = golden('adapt_webcam')
    frames = [fetch(stream(50, 9)[t]) for t in range(9)]
    other = [fetch(stream(51, 9)[t]) for t in range(9)]
    a = webcam_pool(tmp_path, gd, 2, 'a')
    assert a.motion_lead == 1
    for t in range(6):
        a.adapt_processed([frames[t]['image'], other[t]['image']], [frames[t]['smpl_j2d'], other[t]['smpl_j2d']])
    path = str(tmp_path / 'cam0.pt')
    a.save_slot(0, path)
    ta = []
    for t in range(6, 9):                                       # the motion term is live from the stream's frame 4 on
        res = a.adapt_processed([frames[t]['image'], None], [frames[t]['smpl_j2d'], None])
        ta.append([a.thetas[0].clone(), a.m[0].clone(), res[0]['vts'].clone()])
    b = webcam_pool(tmp_path, gd, 2, 'b')
    b.start(1, state=path)
    assert b.video_steps[1] == 6
    tb = []
    for t in range(6, 9):
        res = b.adapt_processed([None, frames[t]['image']], [None, frames[t]['smpl_j2d']])
        tb.append([b.thetas[1].clone(), b.m[1].clone(), res[1]['vts'].clone()])
    for t, (x, y) in enumerate(zip(ta, tb)):
        for name, p, q in zip(('theta', 'm', 'vertices'), x, y):
            assert same(p, q), (t, name)
    assert 'ul/motion_loss' in b.fit_losses
