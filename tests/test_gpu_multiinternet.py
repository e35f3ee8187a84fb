"""Internet pool (MultiInternetAdaptor) on the GPU, fed from synthetic sequences in the reference's npz layout with frames of
different sizes (240 x 320 up to 1080 x 1920) and lengths (2 to 8).  Teacher masks and retrieval seeds follow the video and its
own frame (harness.video_masks / video_seed), in the pool and in the single-video runs alike.

- Input side: every active staged image row and keypoint row bit-identical to ``Internet_dataset``'s item of that frame; idle
  rows keep a sentinel.
- One video is ``InternetAdaptor.excute(fused=True)``: theta, teacher, Adam moments, trip counts and every Pred_<t>.pt array bit
  for bit, at run_on_internet.sh's flags and at the suite's FLAGS.
- Six videos through four slots: each follows its own single-video run (Pred vertices, rotmat, beta and crop camera within 1e-3
  relative, theta within 4 lr n_outer, equal trip counts); a video's files are byte-identical whether it runs alone in slot 0
  or in slot 2, started mid-run.
- Drawing: each PNG is ``BaseAdaptor.save_results``'s for the pool's own mesh, camera, box and frame (and with a crop camera
  that puts the mesh in view); one grouped overlay call per tick.
- I/O: two runs write byte-identical trees, numbered 0 to n - 1 per video; a writer's exception comes out of ``run``."""
import os
import random
import shutil
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import FLAGS, bits, state, video_masks, video_seed

pytestmark = pytest.mark.gpu
SENTINEL = 0x7fc0dead                  # a NaN payload no kernel writes
# name, (H, W), frames.  Through four slots: slot 2 takes v4 at tick 2 (mid-run), slot 3 takes v5 at tick 3, slot 1 idles from
# tick 4 while v4 still runs.
SPECS = [('v0', (240, 320), 8), ('v1', (1080, 1920), 4), ('v2', (720, 1280), 2), ('v3', (480, 640), 3), ('v4', (600, 800), 4),
         ('v5', (1080, 1920), 6)]
VID = {name: k for k, (name, _, _) in enumerate(SPECS)}
# run_on_internet.sh's flags (save_res set per test)
INTERNET = dict(motionloss_weight=0.8, retrieval=1, dynamic_boa=1, optim_steps=7, cos_sim_threshold=3.1e-4, shape_prior_weight=2e-4,
                pose_prior_weight=1e-4)
# the loop at every frame and far from any threshold: 1 - cos >= 0 > -1, so every frame takes optim_steps + 1 trips
ALWAYS_LOOP = dict(INTERNET, cos_sim_threshold=-1.0, optim_steps=2)


def write_videos(root, specs=SPECS):
    """The sequences of `specs` under root (frames in root/images, one npz per sequence): smooth content drifting sideways, a
    box of about half the frame's height, 49 keypoints inside it (a few with zero confidence)."""
    import cv2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    for name, (H, W), n in specs:
        rng = np.random.default_rng(VID.get(name, 99) + 7)
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


@pytest.fixture(scope='module')
def root(tmp_path_factory):
    r = str(tmp_path_factory.mktemp('internet'))
    write_videos(r)
    return r


def single_root(root, tmp, name):
    """A folder holding video `name` alone (its npz, the shared images), for an ``Internet_dataset`` of that video."""
    d = tmp / f'seq_{name}'
    if not d.exists():
        d.mkdir()
        os.symlink(os.path.join(root, 'images'), d / 'images')
        shutil.copy(os.path.join(root, f'{name}.npz'), d / f'{name}.npz')
    return str(d)


def options(tmp, name, **flags):
    from dynaboa_b200 import config
    from oracle import adaptor_ref
    o = vars(adaptor_ref.default_options(**flags))
    o.update(expdir=str(tmp), expname=name, tensorboard=0, cache_results=1, model_file=config.BASE_MODEL, dataset='internet',
             save_res=flags.get('save_res', 0), seq_seed=22)
    return SimpleNamespace(**o)


def videos(root, names):
    from dynaboa_b200.datasets import internet_videos
    by = {v.name: v for v in internet_videos(root)}
    return [by[n] for n in names]


def pool(tmp, G, name, **flags):
    from dynaboa_b200.internet import MultiInternetAdaptor

    class Pool(MultiInternetAdaptor):
        """Teacher masks and retrieval seeds of the video and frame each slot holds; ``outputs``: the last tick's rotmat,
        betas, crop camera and vertices; ``thetas_at_end[name]``: theta after the video's last frame."""

        def input_side(self, frames):
            self.cur = getattr(self, 'cur', [None] * self.G)
            for g, f in enumerate(frames):
                if f is not None:
                    vid = VID[f[0].name]
                    self.cur[g] = [vid, f[1], 0]
                    self.rngs[g].seed(video_seed(vid, f[1]))
            return super().input_side(frames)

        fixed_cam = None

        def _outputs(self, images, active=None):
            rot, shape, cam, out = super()._outputs(images, active)
            if self.fixed_cam is not None:                       # a crop camera that puts the mesh in view
                cam = torch.tensor([self.fixed_cam] * cam.shape[0], dtype=cam.dtype, device=cam.device)
            self.outputs = rot, shape, cam, out
            ends = getattr(self, 'thetas_at_end', {})
            ends.update({SPECS[self.cur[g][0]][0]: self.thetas[g].clone() for g in self._slots(active)})
            self.thetas_at_end = ends
            return self.outputs

    mv = Pool(options(tmp, name, **flags), G, dynamic_loop=True)

    def provider(g, B, dev):
        c = mv.cur[g]
        c[2] += 1
        return video_masks(c[0], c[1], c[2] - 1).to(dev)
    mv.mask_provider = provider
    return mv


def single(root, tmp, name, monkeypatch, **flags):
    """``InternetAdaptor.excute(fused=True)`` of video `name` alone, with the pool's masks and seeds."""
    from dynaboa_b200.adaptor import InternetAdaptor
    monkeypatch.setenv('DYNABOA_INTERNET_ROOT', single_root(root, tmp, name))
    ad = InternetAdaptor(options(tmp, f'single_{name}', **flags))
    vid, calls = VID[name], [0]

    def provider(B, dev):
        calls[0] += 1
        return video_masks(vid, ad.global_step, calls[0] - 1).to(dev)
    ad.teacher.mask_provider = provider
    adapt = ad.adapt

    def seeded(batch):
        calls[0] = 0
        random.seed(video_seed(vid, ad.global_step))
        return adapt(batch)
    ad.adapt = seeded
    ad.excute(fused=True)
    return ad


def load(path):
    import joblib
    return joblib.load(path)


def crop_cam(cam_t):
    """The crop camera (s, tx, ty) of a Pred file's (tx, ty, depth) camera."""
    c = np.asarray(cam_t, dtype=np.float64)
    return np.stack([2 * 5000. / (224 * c[:, 2]), c[:, 0], c[:, 1]], 1)


def tree(d):
    """{relative path: bytes} of every file under d."""
    out = {}
    for base, _, files in os.walk(d):
        for f in files:
            p = os.path.join(base, f)
            with open(p, 'rb') as fh:
                out[os.path.relpath(p, d)] = fh.read()
    return out


# ------------------------------------------------------------------ input side
@pytest.mark.parametrize('G', [1, 4])
def test_input_side_is_internet_dataset(asset_dir, tmp_path, root, monkeypatch, G):
    from dynaboa_b200.datasets import Internet_dataset
    mv = pool(tmp_path, G, 'mv', **FLAGS)
    monkeypatch.setenv('DYNABOA_INTERNET_ROOT', root)
    ds = Internet_dataset(mv.options)
    vids = videos(root, [n for n, _, _ in SPECS])
    first = np.cumsum([0] + [len(v) for v in vids])            # Internet_dataset concatenates the npz in name order
    ticks = [[(vids[0], 3)]] if G == 1 else [[(vids[1], 0), (vids[5], 2), None, (vids[2], 1)], [None, (vids[3], 2), (vids[0], 7), None]]
    for frames in ticks:
        rows = mv._rows()
        for t in rows.values():
            t.view(torch.int32).fill_(SENTINEL)
        on, imgs, bboxes = mv.input_side(frames)
        torch.cuda.synchronize()
        for g, f in enumerate(frames):
            if f is None:
                assert not (on >> g) & 1 and imgs[g] is None
                assert bool((rows['image'][g].view(torch.int32) == SENTINEL).all()), g
                assert bool((rows['smpl_j2d'][g].view(torch.int32) == SENTINEL).all()), g
                continue
            item = ds[int(first[vids.index(f[0])] + f[1])]
            assert torch.equal(bits(rows['image'][g]), bits(item['image'])), (g, f[0].name, f[1])
            assert torch.equal(bits(rows['smpl_j2d'][g]), bits(item['smpl_j2d'])), (g, f[0].name, f[1])
            assert np.array_equal(bboxes[g][0], item['bbox']), g
            H, W = dict((n, s) for n, s, _ in SPECS)[f[0].name]
            assert imgs[g].shape == (H, W, 3) and imgs[g].dtype == torch.uint8


# ------------------------------------------------------------------ one video
@pytest.mark.parametrize('flags', [INTERNET, FLAGS], ids=['run_on_internet', 'suite'])
def test_one_video_is_the_internet_adaptor(asset_dir, tmp_path, root, monkeypatch, flags):
    name = 'v0'
    n = dict((s[0], s[2]) for s in SPECS)[name]
    mv = pool(tmp_path, 1, 'mv', **flags)
    out = mv.run(videos(root, [name]), str(tmp_path / 'pool'))
    ad = single(root, tmp_path, name, monkeypatch, **flags)
    assert out[0]['name'] == name and out[0]['frames'] == n
    if flags['dynamic_boa']:
        assert out[0]['optim_step_record'] == ad.optim_step_record and len(ad.optim_step_record) == n
    else:
        assert 'optim_step_record' not in out[0]
    for x, y in zip(state(mv, 0), [ad.model.module.arena, ad.teacher.arena, ad.optimizer.m, ad.optimizer.v]):
        assert torch.equal(bits(x), bits(y))
    for t in range(n):
        p = load(tmp_path / 'pool' / name / 'result' / f'Pred_{t}.pt')
        r = load(tmp_path / f'single_{name}' / 'result' / f'Pred_{t}.pt')
        assert list(p) == list(r) == ['verts', 'cam', 'rotmat', 'beta'], t
        for k in r:
            assert p[k].dtype == r[k].dtype and p[k].shape == r[k].shape, (t, k)
            assert np.array_equal(p[k].view(np.int32), r[k].view(np.int32)), (t, k)


# ------------------------------------------------------------------ several videos
def test_six_videos_follow_their_own_runs_and_not_their_slot(asset_dir, tmp_path, root, monkeypatch):
    names = [n for n, _, _ in SPECS]
    lengths = {n: k for n, _, k in SPECS}
    mv = pool(tmp_path, 4, 'mv', save_res=1, **ALWAYS_LOOP)
    out = mv.run(videos(root, names), str(tmp_path / 'pool'))
    assert [o['name'] for o in out] == names and [o['frames'] for o in out] == [lengths[n] for n in names]
    ends = dict(mv.thetas_at_end)
    o = mv.options
    for name in names:
        ad = single(root, tmp_path, name, monkeypatch, **ALWAYS_LOOP)
        rec = out[names.index(name)]['optim_step_record']
        assert rec == ad.optim_step_record == [o.optim_steps + 1] * lengths[name], name
        n_outer = sum(1 + min(s, o.optim_steps) for s in rec)
        assert float((ends[name] - ad.model.module.arena).abs().max()) <= 4 * o.lr * n_outer, name
        for t in range(lengths[name]):
            p = load(tmp_path / 'pool' / name / 'result' / f'Pred_{t}.pt')
            r = load(tmp_path / f'single_{name}' / 'result' / f'Pred_{t}.pt')
            for k in ('verts', 'rotmat', 'beta'):
                assert rel_err(p[k], r[k]) < 1e-3, (name, t, k)
            # Pred's cam is (tx, ty, 2 * 5000 / (224 s)): the depth magnifies the relative error of a small scale s, so the
            # pool tests' bound applies to the crop camera (s, tx, ty) it comes from
            assert rel_err(crop_cam(p['cam']), crop_cam(r['cam'])) < 1e-3, (name, t)
        del ad
        torch.cuda.empty_cache()
    # v4 ran in slot 2 from tick 2 (slot 0 running, slot 1 idle from tick 4, slot 3 refilled at tick 3); alone in slot 0:
    alone = pool(tmp_path, 4, 'alone', save_res=1, **ALWAYS_LOOP)
    assert alone.run(videos(root, ['v4']), str(tmp_path / 'alone'))[0]['frames'] == lengths['v4']
    a, b = tree(tmp_path / 'alone' / 'v4'), tree(tmp_path / 'pool' / 'v4')
    assert sorted(a) == sorted(b) and len(a) == 2 * lengths['v4']
    for k in a:
        assert a[k] == b[k], k


# ------------------------------------------------------------------ drawing
@pytest.mark.parametrize('own_camera', [True, False], ids=['own-camera', 'camera-in-view'])
def test_frames_are_drawn_as_save_results(asset_dir, tmp_path, root, monkeypatch, own_camera):
    import cv2
    from dynaboa_b200 import _lib
    from dynaboa_b200.base_adaptor import BaseAdaptor
    monkeypatch.chdir(tmp_path)                                  # save_results writes demo.obj into the working directory
    calls = []
    call = _lib.call

    def counting(name, *args):
        calls.append(name)
        return call(name, *args)
    monkeypatch.setattr(_lib, 'call', counting)
    mv = pool(tmp_path, 3, 'mv', save_res=1, **FLAGS)
    if not own_camera:
        mv.fixed_cam = (0.9, 0.05, 0.1)
    vids = videos(root, ['v1', 'v3', 'v0'])                     # 1080 x 1920, 480 x 640, 240 x 320
    ref = SimpleNamespace(imgdir=os.path.join(root, 'images'), exppath=str(tmp_path / 'ref'), device=torch.device('cuda'))
    os.makedirs(tmp_path / 'ref' / 'image')
    for t, active in enumerate([0b111, 0b101, 0b010]):
        frames = [(v, t) if (active >> g) & 1 else None for g, v in enumerate(vids)]
        for v in vids:
            os.makedirs(tmp_path / 'pool' / v.name / 'image', exist_ok=True)
            os.makedirs(tmp_path / 'pool' / v.name / 'result', exist_ok=True)
        del calls[:]
        files = mv.tick(frames, str(tmp_path / 'pool'))
        assert calls.count('dboa_render_overlay_groups') == 1, t
        assert [f[0] for f in files] == [g for g in range(3) if (active >> g) & 1]
        mv.write(files)
        rot, shape, cam, out = mv.outputs
        for g, _, pred, png, image in files:
            v = vids[g]
            path, _, _, _, bbox = v.frame(t)
            assert np.array_equal(pred['verts'], out['vts'][g:g + 1].cpu().numpy()) and image.shape == cv2.imread(path).shape
            ref.global_step = t
            BaseAdaptor.save_results(ref, out['vts'][g:g + 1], cam[g:g + 1], None, [os.path.basename(path)], bbox, prefix='Pred')
            want = cv2.imread(str(tmp_path / 'ref' / 'image' / f'Pred_{t}.png'))
            got = cv2.imread(png)
            assert png == str(tmp_path / 'pool' / v.name / 'image' / f'Pred_{t}.png')
            assert got.dtype == want.dtype and got.shape == want.shape, (t, g)
            assert np.array_equal(got, want), (t, g, int((got != want).sum()))
            if not own_camera:
                assert (got != cv2.imread(path)).sum() > 1000, (t, g)   # the mesh is in view


# ------------------------------------------------------------------ I/O
def test_runs_write_identical_complete_trees(asset_dir, tmp_path, root):
    names = ['v2', 'v3', 'v0']
    trees = []
    for r in range(2):
        mv = pool(tmp_path, 2, f'mv{r}', save_res=1, **FLAGS)
        mv.run(videos(root, names), str(tmp_path / f'run{r}'), names=[f'seq_{n}' for n in names])
        trees.append(tree(tmp_path / f'run{r}'))
        del mv
    a, b = trees
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k] == b[k], k
    lengths = {n: k for n, _, k in SPECS}
    want = {os.path.join(f'seq_{n}', sub, f'Pred_{t}.{ext}') for n in names for t in range(lengths[n])
            for sub, ext in (('result', 'pt'), ('image', 'png'))}
    assert set(a) == want


def test_a_writer_error_comes_out_of_run(asset_dir, tmp_path, root):
    from dynaboa_b200.internet import FileWriter

    class Failing(FileWriter):
        def pred(self, path, arrays):
            if path.endswith(os.path.join('v3', 'result', 'Pred_1.pt')):
                raise OSError('disk full')
            super().pred(path, arrays)
    mv = pool(tmp_path, 2, 'mv', **FLAGS)
    mv.writer = Failing()
    with pytest.raises(OSError, match='disk full'):
        mv.run(videos(root, ['v2', 'v3', 'v0']), str(tmp_path / 'out'))
    assert not os.path.exists(tmp_path / 'out' / 'v3' / 'result' / 'Pred_1.pt')
