"""Per-slot checkpoints on the GPU (start(g, model=...), run(..., models=...), DESIGN.md section 10, "Per-slot checkpoints").

- Invariant: a video started from checkpoint X in a pool on checkpoint Y, beside videos on Y and on Z that pause, finish and
  restart, is bit-identical to the same video alone in a pool whose model_file is X (C2, and C5 with the dynamic loop); at
  G = 1, start(0, model=X) is Adaptor(model_file=X).
- Round trip through export_model, start(h) back to the pool's checkpoint, the webcam pool's reload(g).
- The device store: one arena per distinct model, freed with the last slot on it.
- The webcam pool's base outputs per stream, and today's single forward while no active stream has a model of its own.
- The Internet pool's run(models=): each video's Pred files byte-identical to its run alone on its model.
- Saved states: a slot on its own model continues bit for bit, needs its model again, and a resumed run needs its models."""
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import FLAGS, MIXED_THRESHOLD, PoolRun, bits, cam_options, masks_for, pool_options, seed_for, state, stream

pytestmark = pytest.mark.gpu
N = 8


def same(a, b):
    return torch.equal(bits(a), bits(b))


def same_values(a, b):
    """Records equal value for value, floats and arrays bit for bit, and their pickles byte-identical."""
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


@pytest.fixture
def models(tmp_path):
    """Checkpoints X and Z in the reference format (the pool's own, Y, is config.BASE_MODEL)."""
    from dynaboa_b200 import synthetic
    out = {}
    for name, seed in (('X', 5), ('Z', 7)):
        out[name] = str(tmp_path / f'{name}.pt')
        torch.save(synthetic.make_basemodel(seed), out[name])
    return out


def options(tmp_path, golden, tag, name, model_file=None, **extra):
    if tag == 'c5':
        extra.setdefault('cos_sim_threshold', MIXED_THRESHOLD)
    o = pool_options(tmp_path, golden, tag, name, **extra)
    if model_file is not None:
        o.model_file = model_file
    return o


def pool(o, G, gd, dynamic=False):
    return PoolRun(o, G, dynamic_loop=dynamic, masks=lambda vid, t, call: masks_for(vid, t, call, gd), seed=seed_for)


def put(p, g, vid, model=None, state=None):
    p.mv.start(g, model=model, state=state)
    p.slot[g] = [vid, stream(vid, 12), p.mv.video_steps[g]]


def trace(p, g):
    return p.state(g) + [p.mv.last_upper_loss[g:g + 1].clone()]


def check(ta, tb, what):
    assert len(ta) == len(tb)
    for t, (ra, rb) in enumerate(zip(ta, tb)):
        for name, x, y in zip(('theta', 'teacher', 'm', 'v', 'upper loss'), ra, rb):
            assert same(x, y), (what, t, name)


# ------------------------------------------------------------------ invariant
@pytest.mark.parametrize('tag', ['c2', 'c5'])
def test_a_slot_on_its_own_model_is_that_model_alone(asset_dir, tmp_path, golden, models, tag):
    gd, dynamic = golden(f'adapt_{tag}'), tag == 'c5'
    X, Z = models['X'], models['Z']
    mix = pool(options(tmp_path, golden, tag, 'mix'), 4, gd, dynamic)
    put(mix, 0, 1)                                           # Y, finishes after 4 frames
    put(mix, 1, 3, model=Z)
    put(mix, 2, 2, model=X)
    assert mix.mv.slot_model(2)[0] == X and mix.mv.slot_model(0) is None and mix.mv.slot_model(1)[1] != mix.mv.slot_model(2)[1]
    runs = {0: [0, 1, 2], 1: [0, 2], 2: [0, 1, 2, 3], 3: [0, 1, 3], 4: [0, 1, 2, 3]}
    ta = []
    for f in range(9):
        if f == 2:
            put(mix, 3, 4)
        if f == 4:
            put(mix, 0, 5, model=Z)                          # slot 0's video ended: a new one on Z
        run = runs.get(f, [0, 1, 2, 3])
        mix.step(run)
        if 2 in run:
            ta.append(trace(mix, 2))
    assert len(ta) == N and mix.mv.video_steps[2] == N
    alone = pool(options(tmp_path, golden, tag, 'alone', model_file=X), 4, gd, dynamic)
    put(alone, 0, 2)
    tb = []
    for _ in range(N):
        alone.step([0])
        tb.append(trace(alone, 0))
    check(ta, tb, tag)
    ra, rb = mix.mv.records(2), alone.mv.records(0)
    assert same_values(ra, rb)
    if dynamic:
        assert ra['optim_step_record'] and any(ra['optim_step_record']) and ra['feat_sims'], 'the dynamic loop never ran'


def test_one_slot_on_its_own_model_is_the_adaptor_on_it(asset_dir, tmp_path, golden, models):
    from harness import SingleRun
    gd = golden('adapt_c2')
    p = pool(options(tmp_path, golden, 'c2', 'mv'), 1, gd)
    put(p, 0, 0, model=models['X'])
    s = SingleRun(options(tmp_path, golden, 'c2', 'ad', model_file=models['X']), 0,
                  masks=lambda vid, t, call: masks_for(vid, t, call, gd), seed=seed_for)
    ad = s.ad
    assert same(p.mv.theta(0), ad.model.module.arena)
    for t in range(N):
        s.step(t, p.step([0])[0][2])
        assert same(p.mv.last_upper_loss[0], ad.last_upper_loss), t
    assert same(p.mv.theta(0), ad.model.module.arena) and same(p.mv.teachers[0], ad.teacher.arena)


# ------------------------------------------------------------------ round trip, store
def test_exported_model_goes_back_into_a_slot(asset_dir, tmp_path, golden):
    from dynaboa_b200 import layout
    gd = golden('adapt_c2')
    a = pool(options(tmp_path, golden, 'c2', 'a'), 2, gd)
    put(a, 0, 1)
    put(a, 1, 2)
    for _ in range(3):
        a.step([0, 1])
    path = str(tmp_path / 'adapted.pt')
    a.mv.export_model(0, path)
    exported = a.mv.thetas[0].clone()
    b = pool(options(tmp_path, golden, 'c2', 'b'), 3, gd)
    put(b, 0, 3)
    b.step([0])
    other = state(b.mv, 0)
    b.mv.start(2, model=path)
    assert b.mv.slot_model(2) == (path, layout.arena_digest(exported, b.mv.buffers))
    assert same(b.mv.thetas[2], exported) and same(b.mv.teachers[2], exported)
    assert not b.mv.m[2].any() and not b.mv.v[2].any() and b.mv.step_counts[2] == 0
    assert all(same(x, y) for x, y in zip(other, state(b.mv, 0)))
    b.mv.start(2)
    assert b.mv.slot_model(2) is None and not b.mv._store
    assert same(b.mv.thetas[2], b.mv.base.model.module.arena) and same(b.mv.teachers[2], b.mv.base.teacher.arena)


def test_slots_on_one_model_share_one_arena(asset_dir, tmp_path, golden, models):
    from dynaboa_b200 import config, layout
    mv = pool(options(tmp_path, golden, 'c2', 'mv'), 4, golden('adapt_c2')).mv
    torch.cuda.synchronize()

    def held():
        return torch.cuda.memory_stats()['requested_bytes.all.current']
    before = held()
    for g in range(3):
        mv.start(g, model=models['X'])
    torch.cuda.synchronize()
    arena = layout.arena_layout().floats * 4
    assert held() - before == arena
    assert len({mv.slot_model(g) for g in range(3)}) == 1 and len(mv._store) == 1 and mv.slot_model(3) is None
    assert all(same(mv.thetas[g], mv.thetas[0]) for g in range(3)) and not same(mv.thetas[0], mv.thetas[3])
    mv.start(0)
    mv.start(1, model=config.BASE_MODEL)                    # the pool's own weights: the pool's checkpoint, no arena
    assert mv.slot_model(1) is None and len(mv._store) == 1
    mv.start(2, model=models['Z'])
    torch.cuda.synchronize()
    assert len(mv._store) == 1 and held() - before == arena
    mv.start(2)
    torch.cuda.synchronize()
    assert not mv._store and held() == before


# ------------------------------------------------------------------ webcam pool
def cam_inputs(gd, vid, n):
    from dynaboa_b200 import synthetic
    s = synthetic.SyntheticStream(length=n, batch_size=1, rank=vid)
    rng = np.random.default_rng(100 + vid)
    out = []
    for t in range(n):
        kp = torch.zeros(1, 49, 3)
        k25 = gd['kp25'][t % len(gd['kp25'])].copy()
        k25[..., :2] += rng.uniform(-0.05, 0.05, size=k25[..., :2].shape).astype(np.float32)
        kp[:, :25] = torch.from_numpy(k25)
        out.append((s[t]['image'].cuda(), kp.cuda()))
    return out


def cam_tick(mv, ins):
    return mv.adapt_processed([None if x is None else x[0] for x in ins], [None if x is None else x[1] for x in ins])


def test_webcam_reload_returns_to_the_streams_model(asset_dir, tmp_path, golden, models):
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    gd = golden('adapt_webcam')
    mv = MultiWebcamAdaptor(cam_options(tmp_path / 'w', gd), 2, dynamic_loop=True)
    mv.start(0, model=models['X'])
    x = mv.thetas[0].clone()
    ins = [cam_inputs(gd, 1, 4), cam_inputs(gd, 2, 4)]
    for t in range(3):
        cam_tick(mv, [ins[0][t], ins[1][t]])
    assert not same(mv.thetas[0], x)
    other = [mv.thetas[1].clone(), mv.m[1].clone(), mv.v[1].clone()] + ([mv.teachers[1].clone()] if mv.teachers is not None else [])
    mv.reload(0)
    assert same(mv.thetas[0], x) and not mv.m[0].any() and not mv.v[0].any() and mv.step_counts[0] == 0
    if mv.teachers is not None:
        assert same(mv.teachers[0], x)
    assert mv.slot_model(0)[0] == models['X'] and mv.video_steps[0] == 3
    now = [mv.thetas[1], mv.m[1], mv.v[1]] + ([mv.teachers[1]] if mv.teachers is not None else [])
    assert all(same(p, q) for p, q in zip(other, now))


def test_webcam_base_outputs_per_stream(asset_dir, tmp_path, golden, models, monkeypatch):
    from dynaboa_b200 import config, webcam
    from dynaboa_b200.webcam import MultiWebcamAdaptor, WebcamAdaptor
    gd = golden('adapt_webcam')
    calls = []
    forward = webcam.hmr_mod.raw_forward

    def spy(arena, *a, **k):
        calls.append((arena.data_ptr(), k.get('groups', 1), k.get('active')))
        return forward(arena, *a, **k)
    monkeypatch.setattr(webcam.hmr_mod, 'raw_forward', spy)
    mv = MultiWebcamAdaptor(cam_options(tmp_path / 'w', gd, test_basemodel=1, dynamic_boa=0), 3)
    base = mv.base.model.module.arena.data_ptr()
    ins = [cam_inputs(gd, g, 6) for g in range(3)]

    def base_calls():
        """The tick's base-output forwards: those of the pool's arena or of the stack of base arenas."""
        stack = None if mv._base_stack is None else mv._base_stack.data_ptr()
        got = [c for c in calls if c[0] in (base, stack)]
        calls.clear()
        return got
    res = cam_tick(mv, [ins[0][0], ins[1][0], ins[2][0]])
    assert base_calls() == [(base, 1, None)] and mv._base_stack is None               # no stream on a model of its own: today's
    mv.start(0, model=models['X'])
    mv.start(2, model=models['Z'])
    assert mv._base_stack is not None and same(mv._base_stack[1], mv.base.model.module.arena)
    res = cam_tick(mv, [None, ins[1][1], None])
    assert base_calls() == [(base, 1, None)]                                          # the active stream is on the pool's
    res = cam_tick(mv, [ins[0][1], ins[1][2], ins[2][1]])
    assert base_calls() == [(mv._base_stack.data_ptr(), 3, 0b111)]
    for g, path in ((0, models['X']), (1, config.BASE_MODEL), (2, models['Z'])):
        o = cam_options(tmp_path / f's{g}', gd, test_basemodel=1, dynamic_boa=0)
        o.model_file = path
        ad = WebcamAdaptor(o)
        image = ins[g][1 if g != 1 else 2][0]
        with torch.no_grad():
            rot, shape, cam = ad.basemodel(image)
            vts = ad.decode_smpl_params(rot, shape)['vts']
        assert rel_err(res[g]['cam_base'], cam) < 1e-5 and rel_err(res[g]['vts_base'], vts) < 1e-5, g
        del ad
    first = [res[0]['vts_base'].clone(), res[0]['cam_base'].clone()]
    mv.start(2, model=models['X'])                                                      # another stream changes model ...
    res = cam_tick(mv, [ins[0][1], None, ins[2][2]])                                    # ... or sits the tick out
    assert same(res[0]['vts_base'], first[0]) and same(res[0]['cam_base'], first[1])
    mv.start(1, model=models['Z'])
    res = cam_tick(mv, [ins[0][1], ins[1][3], None])
    assert same(res[0]['vts_base'], first[0]) and same(res[0]['cam_base'], first[1])
    calls.clear()
    for g in range(3):
        mv.start(g)
    assert mv._base_stack is None
    cam_tick(mv, [ins[0][4], ins[1][4], ins[2][4]])
    assert base_calls() == [(base, 1, None)]


# ------------------------------------------------------------------ Internet pool
SPECS = [('v0', (240, 320), 3), ('v1', (300, 400), 2), ('v2', (240, 320), 4), ('v3', (240, 320), 2), ('v4', (360, 480), 3),
         ('v5', (240, 320), 2)]


def write_videos(root):
    import cv2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    for k, (name, (H, W), n) in enumerate(SPECS):
        rng = np.random.default_rng(k + 60)
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


def tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            with open(os.path.join(d, f), 'rb') as fh:
                out[os.path.relpath(os.path.join(d, f), root)] = fh.read()
    return out


class VideoMasks:
    """A mask_provider whose teacher masks follow the video (by name) and its own frame, as masks_for draws them."""

    def __init__(self, mv, names):
        self.mv, self.names, self.seen = mv, names, {}

    def __call__(self, g, B, dev):
        vid = int(self.names[self.mv.slot_video[g]][1:]) + 1
        key = (vid, self.mv.video_steps[g])
        call = self.seen.get(key, 0)
        self.seen[key] = call + 1
        return masks_for(vid, key[1], call, None).to(dev)


def test_internet_run_with_a_model_per_video(asset_dir, tmp_path, models):
    from dynaboa_b200 import config
    from dynaboa_b200.datasets import internet_videos
    from dynaboa_b200.internet import MultiInternetAdaptor
    from oracle import adaptor_ref
    root = str(tmp_path / 'videos')
    write_videos(root)
    vids = internet_videos(root)
    assert [v.name for v in vids] == [s[0] for s in SPECS]
    per = [models['X'], None, models['Z'], models['X'], config.BASE_MODEL, models['Z']]

    def make(name, model_file=config.BASE_MODEL):
        o = vars(adaptor_ref.default_options(**FLAGS))
        o.update(expdir=str(tmp_path), expname=name, tensorboard=0, cache_results=1, model_file=model_file, dataset='internet',
                 save_res=0, seq_seed=22)
        return MultiInternetAdaptor(SimpleNamespace(**o), 4)
    mv = make('pool')
    mv.mask_provider = VideoMasks(mv, [v.name for v in vids])
    got = mv.run(vids, str(tmp_path / 'pooled'), models=per)
    assert [s['model'] for s in got] == per and [s['frames'] for s in got] == [n for _, _, n in SPECS]
    pooled = tree(tmp_path / 'pooled')
    assert len(pooled) == sum(n for _, _, n in SPECS)
    for path in (models['X'], models['Z'], config.BASE_MODEL):
        alone = make('alone', model_file=path)
        for i, v in enumerate(vids):
            if (per[i] or config.BASE_MODEL) != path:
                continue
            alone.mask_provider = VideoMasks(alone, [v.name])
            alone.run([v], str(tmp_path / 'alone'))
        del alone
    single = tree(tmp_path / 'alone')
    assert sorted(single) == sorted(pooled)
    for f in pooled:
        assert pooled[f] == single[f], f


# ------------------------------------------------------------------ saved states
def test_slot_state_on_its_own_model(asset_dir, tmp_path, golden, models):
    gd = golden('adapt_c2')
    X, k = models['X'], 3
    a = pool(options(tmp_path, golden, 'c2', 'a'), 4, gd)
    put(a, 1, 6, model=X)
    put(a, 0, 7)
    for _ in range(k):
        a.step([0, 1])
    path, plain = str(tmp_path / 'slot1.pt'), str(tmp_path / 'slot0.pt')
    a.mv.save_slot(1, path)
    a.mv.save_slot(0, plain)
    assert torch.load(path, weights_only=True)['model'] == {'path': X, 'digest': a.mv.slot_model(1)[1]}
    assert 'model' not in torch.load(plain, weights_only=True)                  # a slot on the pool's checkpoint: as before
    ta = []
    for _ in range(N - k):
        a.step([0, 1])
        ta.append(trace(a, 1))
    b = pool(options(tmp_path, golden, 'c2', 'b'), 4, gd)
    put(b, 2, 8)
    b.step([2])
    before = [t.clone() for t in (b.mv.thetas, b.mv.m, b.mv.v, b.mv.teachers)]
    moved = str(tmp_path / 'moved.pt')
    os.rename(X, moved)
    with pytest.raises(ValueError, match='not a readable checkpoint'):
        b.mv.start(3, state=path)                                          # the recorded path is gone
    with pytest.raises(ValueError, match='not the checkpoint the state was adapted from'):
        b.mv.start(3, state=path, model=models['Z'])
    with pytest.raises(ValueError, match='not the checkpoint the state was adapted from'):
        b.mv.start(3, state=plain, model=moved)                            # a state on the pool's checkpoint given another model
    assert all(same(x, y) for x, y in zip(before, (b.mv.thetas, b.mv.m, b.mv.v, b.mv.teachers)))
    put(b, 3, 6, model=moved, state=path)
    assert b.mv.slot_model(3) == (moved, a.mv.slot_model(1)[1]) and b.mv.video_steps[3] == k
    tb = []
    for _ in range(N - k):
        b.step([2, 3])
        tb.append(trace(b, 3))
    check(ta, tb, 'slot 1 -> 3')
    assert same_values(a.mv.records(1), b.mv.records(3))
    b.mv.start(3)                                                          # back to the pool's checkpoint
    assert same(b.mv.thetas[3], b.mv.base.model.module.arena) and not b.mv._store
    put(b, 0, 7, state=plain)                                              # a state file without a model entry loads as before
    assert b.mv.slot_model(0) is None and b.mv.video_steps[0] == k


class Stop(Exception):
    pass


class Cut:
    def __init__(self, video, k):
        self.video, self.k = video, k

    def __iter__(self):
        for t, item in enumerate(self.video):
            if t == self.k:
                raise Stop
            yield item


def test_run_resumes_with_its_models(asset_dir, tmp_path, golden, models):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    lengths = [3, 6, 2, 5, 4, 3]
    per = [models['X'], None, models['Z'], models['X'], None, models['Z']]

    def make(name):
        mv = MultiVideoAdaptor(options(tmp_path, golden, 'c2', name), 4)
        mv.fused_eval = 'final'
        return mv
    videos = [stream(30 + i, n) for i, n in enumerate(lengths)]
    want = make('straight').run(videos, str(tmp_path / 'out_straight'), models=per)
    assert [s['model'] for s in want] == per
    ck, out = str(tmp_path / 'ck'), str(tmp_path / 'out_resumed')
    cut = list(videos)
    cut[4] = Cut(videos[4], 2)
    with pytest.raises(Stop):
        make('cut').run(cut, out, checkpoint=ck, every=2, models=per)
    other = make('other')
    with pytest.raises(ValueError, match='models'):
        other.run(videos, out, checkpoint=ck, every=2, models=[models['Z']] + per[1:])
    with pytest.raises(ValueError, match='models'):
        other.run(videos, out, checkpoint=ck, every=2)
    assert other.global_step == 0 and all(m is None for m in other.slot_models)
    got = make('resumed').run(videos, out, checkpoint=ck, every=2, models=per)
    assert same_values(got, want)
    a, b = tree(tmp_path / 'out_straight'), tree(out)
    assert sorted(a) == sorted(b) and len(a) == 8 * len(lengths)
    for f in a:
        assert a[f] == b[f], f
