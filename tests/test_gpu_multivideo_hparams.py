"""Per-video hyperparameters of a pool on the GPU.

- Kernels: every per-video entry point is bit-identical, on each video's rows, to the uniform call with that video's scalars;
  idle videos' floats keep a sentinel.  G = 1, 2, 7, 64 and sweep lengths that are not a multiple of the block's floats; Adam
  with a distinct step count per video.
- Isolation: a G = 4 pool whose slots carry distinct values of every PER_VIDEO key, one slot starting two frames late, at C2, C3
  and C5.  Video g is bit-identical to video g of a pool in which every slot runs with video g's options: theta, teacher, m, v,
  step count, fit_losses, 2D losses, trip counts, cosines, retrieval picks and (fused_eval='all') its metrics.  The videos
  differ from a pool without hparams.
- Uniform path: hparams equal to the options give the pool without hparams, bit for bit and launch for launch.
- Resume: save_slot / start(g, state=) carries a slot's hparams; contradicting hparams raise.  An interrupted run(..., hparams=,
  checkpoint=) resumes to the uninterrupted run's summaries and result files; a resume with other hparams raises before any slot
  is restored.
- Other pools: a webcam pool (with reload(g) mid-run) and an Internet pool with per-stream hparams, each stream matched against a
  pool run at that stream's own options."""
import ctypes as C
import os
import pickle
from types import SimpleNamespace

import pytest
import torch

from harness import Buf, bits, pool_options, stream

pytestmark = pytest.mark.gpu


def same(a, b):
    return torch.equal(bits(a.contiguous()), bits(b.to(a.device).contiguous()))


def floats(v):
    return (C.c_float * len(v))(*v)


# ------------------------------------------------------------------ kernels
SIZES = [(1, 1028), (2, 4 * 257), (7, 4 * 1000 + 4), (64, 4 * 300 + 8)]


def actives(G):
    every = (1 << G) - 1
    return [every] if G == 1 else [every, every & 0x5555555555555555, 1 << (G - 1)]


@pytest.mark.parametrize('G,n', SIZES)
def test_sgd_groups(G, n):
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import stream as cur
    gen = torch.Generator().manual_seed(G)
    p, g = torch.randn(G * n, generator=gen).cuda(), torch.randn(G * n, generator=gen).cuda()
    lr = [8e-6 * (1 + 0.37 * k) for k in range(G)]
    for active in actives(G):
        out = Buf(n=G * n)
        out.t.fill_(-3.0)
        _lib.call('dboa_sgd_update_groups', p.data_ptr(), g.data_ptr(), out.ptr, floats(lr), n, G, active, cur())
        for k in range(G):
            rows = slice(k * n, (k + 1) * n)
            if (active >> k) & 1:
                one = torch.empty(n, device='cuda')
                _lib.call('dboa_sgd_update', p[rows].data_ptr(), g[rows].data_ptr(), one.data_ptr(), lr[k], n, cur())
                assert same(out.t[rows], one), (G, active, k)
            else:
                assert (out.t[rows] == -3.0).all(), (G, active, k)
        assert out.intact()


@pytest.mark.parametrize('teacher', [True, False])
@pytest.mark.parametrize('G,n', SIZES)
def test_adam_ema_groups(G, n, teacher):
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import stream as cur
    gen = torch.Generator().manual_seed(100 + G)
    init = [torch.randn(G * n, generator=gen).cuda() for _ in range(3)] + [torch.rand(G * n, generator=gen).cuda()]
    init.append(torch.randn(G * n, generator=gen).cuda())          # p, g, m, v, teacher
    rows = (C.c_float * (G * _lib.ADAM_SCALARS))()
    one = (C.c_float * _lib.ADAM_SCALARS)()
    hp = [(3e-6 * (1 + 0.3 * k), 0.5 - 0.004 * k, 0.9 + 0.001 * k, 1 + 3 * k, 0.1 + 0.01 * k) for k in range(G)]   # distinct steps
    for k, (lr, b1, b2, step, alpha) in enumerate(hp):
        _lib.call('dboa_adam_scalars', one, lr, b1, b2, 1e-8, step, alpha, 1.0)
        rows[k * _lib.ADAM_SCALARS:(k + 1) * _lib.ADAM_SCALARS] = one[:]
    for active in actives(G):
        p, g, m, v, t = [x.clone() for x in init]
        tt = t if teacher else None
        _lib.call('dboa_adam_ema_groups', p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), None if tt is None else tt.data_ptr(), n,
                  rows, G, active, cur())
        for k, (lr, b1, b2, step, alpha) in enumerate(hp):
            q = slice(k * n, (k + 1) * n)
            if not (active >> k) & 1:
                for a, b in zip((p, m, v, t), (init[0], init[2], init[3], init[4])):
                    assert same(a[q], b[q]), (G, active, k)
                continue
            r = [x[q].clone() for x in init]
            _lib.call('dboa_adam_ema_scaled', r[0].data_ptr(), r[1].data_ptr(), r[2].data_ptr(), r[3].data_ptr(),
                      r[4].data_ptr() if teacher else None, n, lr, b1, b2, 1e-8, step, alpha, 1.0, cur())
            for a, b in zip((p, m, v, t), (r[0], r[2], r[3], r[4])):
                assert same(a[q], b), (G, active, k)


def rand_rot(n, gen):
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import stream as cur
    aa = (torch.randn(n, 3, generator=gen) * 0.4).cuda()
    R = torch.empty(n, 3, 3, device='cuda')
    _lib.call('dboa_rodrigues', aa.data_ptr(), R.data_ptr(), n, 0, cur())
    return R


@pytest.mark.parametrize('G', [1, 2, 7, 64])
def test_loss_head_and_motion_weights(G):
    """dboa_loss_multi_weights, dboa_pose_prior_groups and dboa_loss_motion_weights against the uniform calls on each video's
    rows with its weights (b = 1 row per video; G = 7 also at b = 3)."""
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import stream as cur
    for b in ([1, 3] if G == 7 else [1]):
        B = G * b
        gen = torch.Generator().manual_seed(G * 10 + b)
        p2d, j3d = (torch.randn(B, 49, 2, generator=gen) * 0.3).cuda(), (torch.randn(B, 49, 3, generator=gen) * 0.3).cuda()
        R, beta = rand_rot(B * 24, gen).view(B, 24, 3, 3), torch.randn(B, 10, generator=gen).cuda()
        kp = torch.cat([torch.randn(B, 49, 2, generator=gen) * 0.5, (torch.rand(B, 49, 1, generator=gen) > 0.3).float()], -1).cuda()
        t_p2d, t_j3d = (torch.randn(B, 49, 2, generator=gen) * 0.3).cuda(), (torch.randn(B, 49, 3, generator=gen) * 0.3).cuda()
        t_beta, t_R = torch.randn(B, 10, generator=gen).cuda(), rand_rot(B * 24, gen).view(B, 24, 3, 3)
        W = [[10.0 * (1 + 0.1 * k), 2e-6 * (1 + k), 0.0, 0.5 + k, 0.25 * k, 1e-4 * k, 0.1 + k, 0.3 * k] for k in range(G)]
        outs = {}
        for who in ['groups'] + list(range(G)):
            rows = slice(None) if who == 'groups' else slice(who * b, (who + 1) * b)
            n = B if who == 'groups' else b
            a = _lib.LossArgsStruct()
            a.B, a.groups = n, (G if who == 'groups' else 1)
            terms = torch.empty(a.groups, 9, device='cuda')
            grads = [torch.full_like(x[rows], float('nan')) for x in (p2d, j3d, R, beta)]
            keep = [x[rows].contiguous() for x in (p2d, j3d, R, beta, kp, t_p2d, t_j3d, t_beta, t_R)]
            for name, x in zip(('p2d', 'j3d', 'R', 'beta', 'kp', 't_p2d', 't_j3d', 't_beta', 't_R'), keep):
                setattr(a, name, x.data_ptr())
            a.terms = terms.data_ptr()
            a.dp2d, a.dj3d, a.dR, a.dbeta = [x.data_ptr() for x in grads]
            a.kp_first, a.kp_count = 25, 24
            if who == 'groups':
                _lib.call('dboa_loss_multi_weights', C.byref(a), floats([x for r in W for x in r]), cur())
            else:
                for i in range(8):
                    a.w[i] = W[who][i]
                _lib.call('dboa_loss_multi', C.byref(a), cur())
            outs[who] = (terms, grads)
        for k in range(G):
            terms, grads = outs['groups']
            rt, rg = outs[k]
            assert same(terms[k], rt[0]), (G, b, k)
            for x, y in zip(grads, rg):
                assert same(x[k * b:(k + 1) * b], y), (G, b, k)
        # motion: the videos whose bit is set, the others keep their rows
        mw = [0.8 * (1 + 0.2 * k) for k in range(G)]
        ph = (torch.randn(B, 49, 2, generator=gen) * 0.3).cuda()
        kh = torch.cat([torch.randn(B, 49, 2, generator=gen) * 0.5, (torch.rand(B, 49, 1, generator=gen) > 0.2).float()], -1).cuda()
        for active in actives(G):
            term, dpa, dph = torch.full((G,), 7.0, device='cuda'), torch.full_like(p2d, 5.0), torch.full_like(p2d, 6.0)
            _lib.call('dboa_loss_motion_weights', p2d.data_ptr(), ph.data_ptr(), kp.data_ptr(), kh.data_ptr(), floats(mw), term.data_ptr(),
                      dpa.data_ptr(), dph.data_ptr(), B, 1, 25, 24, G, active, cur())
            for k in range(G):
                q = slice(k * b, (k + 1) * b)
                if not (active >> k) & 1:
                    assert term[k] == 0 and (dpa[q] == 5.0).all() and (dph[q] == 6.0).all()
                    continue
                t1, d1, d2 = torch.empty(1, device='cuda'), torch.full_like(p2d[q], 5.0), torch.empty_like(p2d[q])
                _lib.call('dboa_loss_motion_active', p2d[q].contiguous().data_ptr(), ph[q].contiguous().data_ptr(), kp[q].contiguous().data_ptr(),
                          kh[q].contiguous().data_ptr(), mw[k], t1.data_ptr(), d1.data_ptr(), d2.data_ptr(), b, 1, 25, 24, 1, 1, cur())
                assert same(term[k:k + 1], t1) and same(dpa[q], d1) and same(dph[q], d2), (G, b, k)


@pytest.mark.parametrize('G', [1, 2, 7, 64])
def test_pose_prior_groups(G):
    """dboa_pose_prior_groups against dboa_pose_prior on each video's rows with its scale w / b (b = 2)."""
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import stream as cur
    from dynaboa_b200.prior import MaxMixturePrior
    pr = MaxMixturePrior(prior_folder=None).cuda()
    b = 2
    B = G * b
    R = rand_rot(B * 24, torch.Generator().manual_seed(G)).view(B, 24, 3, 3)
    scale = [1e-4 * (1 + 0.5 * k) / b for k in range(G)]
    consts = [x.data_ptr() for x in (pr.means, pr.precisions, pr.neg_log_weights)]
    prior_b, dR = torch.full((B,), float('nan'), device='cuda'), torch.full_like(R, float('nan'))
    _lib.call('dboa_pose_prior_groups', R.data_ptr(), *consts, prior_b.data_ptr(), dR.data_ptr(), floats(scale), B, G, cur())
    for k in range(G):
        q = slice(k * b, (k + 1) * b)
        pb, d = torch.empty(b, device='cuda'), torch.empty_like(R[q])
        _lib.call('dboa_pose_prior', R[q].contiguous().data_ptr(), *consts, pb.data_ptr(), d.data_ptr(), scale[k], b, cur())
        assert same(prior_b[q], pb) and same(dR[q], d), (G, k)


# ------------------------------------------------------------------ pools
FACTORS = (1.5, 0.7, 1.3, 0.8)
BETA1, BETA2, ALPHA, STEPS = (0.45, 0.55, 0.6, 0.4), (0.92, 0.88, 0.95, 0.85), (0.15, 0.05, 0.2, 0.12), (3, 2, 5, 4)
SCALED = ('lr', 'fastlr', 's2dloss_weight', 'shape_prior_weight', 'pose_prior_weight', 'teacherloss_weight', 'motionloss_weight',
          'labelloss_weight', 'cos_sim_threshold')


def hparams_of(o, g):
    """Slot g's values of every PER_VIDEO key ``o`` holds, distinct between slots and from ``o``."""
    hp = {k: getattr(o, k) * FACTORS[g] for k in SCALED if hasattr(o, k)}
    hp.update(beta1=BETA1[g], beta2=BETA2[g], alpha=ALPHA[g], optim_steps=STEPS[g])
    return hp


FRAMES, LATE = 3, 3                 # slot LATE starts two pool frames late


def drive(opts, hparams, dynamic_loop, fused_eval='none'):
    """A G = 4 pool over videos 0..3 (FRAMES frames each) with per-video teacher masks and retrieval seeds, slot g starting with
    ``hparams[g]`` (None: none) and slot LATE two pool frames late.  Returns per video its per-frame records and its final state."""
    from harness import PoolRun
    pr = PoolRun(opts, 4, dynamic_loop=dynamic_loop)
    mv = pr.mv
    mv.fused_eval = fused_eval
    recs = {g: [] for g in range(4)}
    for g in range(4):
        mv.start(g, hparams=hparams[g])
        pr.slot[g] = [g, stream(g, FRAMES), 0]
    launches = []
    from dynaboa_b200 import _lib
    lib = _lib.load()
    for f in range(FRAMES + 2):
        run = [g for g in range(4) if (g != LATE or f >= 2) and pr.slot[g][2] < FRAMES]
        before = lib.dboa_launch_count()
        pr.step(run)
        launches.append(lib.dboa_launch_count() - before)
        for g in run:
            fit = {k: (v[g:g + 1].clone() if torch.is_tensor(v) else v) for k, v in mv.fit_losses.items()}
            recs[g].append(dict(fit=fit, lower=[x[g:g + 1].clone() for x in mv.kp2dlosses_lower], steps=mv.optimized_step[g],
                                picks=mv.last_retrieval[g]))
    final = {g: dict(state=[mv.thetas[g].clone(), mv.teachers[g].clone(), mv.m[g].clone(), mv.v[g].clone()], count=mv.step_counts[g],
                     records=mv.records(g)) for g in range(4)}
    del pr, mv
    torch.cuda.empty_cache()
    return recs, final, launches


def assert_same_video(a, b, what):
    recs_a, fin_a = a
    recs_b, fin_b = b
    assert len(recs_a) == len(recs_b), what
    for t, (x, y) in enumerate(zip(recs_a, recs_b)):
        assert set(x['fit']) == set(y['fit']), (what, t)
        for k in x['fit']:
            u, v = x['fit'][k], y['fit'][k]
            assert same(torch.as_tensor(u).float(), torch.as_tensor(v).float()), (what, t, k)
        assert all(same(u, v) for u, v in zip(x['lower'], y['lower'])), (what, t)
        assert x['steps'] == y['steps'] and x['picks'] == y['picks'], (what, t)
    for name, u, v in zip(('theta', 'teacher', 'm', 'v'), fin_a['state'], fin_b['state']):
        assert same(u, v), (what, name)
    assert fin_a['count'] == fin_b['count'], what
    ra, rb = fin_a['records'], fin_b['records']
    assert pickle.dumps(ra) == pickle.dumps(rb), what    # metrics, 2D losses, trip counts and cosines as the host records hold them


@pytest.mark.parametrize('tag', ['c2', 'c3', 'c5'])
def test_each_video_is_the_pool_of_its_own_options(asset_dir, tmp_path, golden, tag):
    from harness import MIXED_THRESHOLD
    over = dict(cos_sim_threshold=MIXED_THRESHOLD) if tag == 'c5' else {}
    opts = pool_options(tmp_path, golden, tag, 'mixed', **over)
    hps = [hparams_of(opts, g) for g in range(4)]
    ev = 'all' if tag == 'c2' else 'none'
    mixed, fin, _ = drive(opts, hps, tag == 'c5', ev)
    plain_recs, plain_fin, _ = drive(opts, [None] * 4, tag == 'c5', ev) if tag != 'c3' else (None, None, None)
    for g in range(4):
        own = pool_options(tmp_path, golden, tag, f'own{g}', **{**over, **hps[g]})
        recs, fin_g, _ = drive(own, [None] * 4, tag == 'c5', ev)
        assert_same_video((mixed[g], fin[g]), (recs[g], fin_g[g]), (tag, g))
        if plain_fin is not None:
            assert not same(fin[g]['state'][0], plain_fin[g]['state'][0]), ('overrides ignored', g)
    if tag == 'c5':                         # cos_sim_threshold and optim_steps reach the loop: some trip counts differ
        trips = lambda recs: [[r['steps'] for r in recs[g]] for g in range(4)]
        assert trips(mixed) != trips(plain_recs)


def test_uniform_hparams_are_the_pool_without_them(asset_dir, tmp_path, golden):
    from dynaboa_b200.multivideo import PER_VIDEO
    opts = pool_options(tmp_path, golden, 'c3', 'u')
    same_hp = {k: getattr(opts, k) for k in PER_VIDEO}
    a, fa, la = drive(opts, [same_hp] * 4, False)
    b, fb, lb = drive(opts, [None] * 4, False)
    assert la == lb
    for g in range(4):
        assert_same_video((a[g], fa[g]), (b[g], fb[g]), g)


def test_slot_state_carries_its_hparams(asset_dir, tmp_path, golden):
    """save_slot after two frames, start(g, state=) in a new pool, two more frames: the uninterrupted video's state; the restored
    slot runs with the saved hparams, and contradicting hparams raise."""
    from harness import PoolRun
    opts = pool_options(tmp_path, golden, 'c2', 'r')
    hps = [hparams_of(opts, g) for g in range(4)]
    s = [stream(g, 4) for g in range(4)]

    def pool():
        pr = PoolRun(opts, 4)
        for g in range(4):
            pr.mv.start(g, hparams=hps[g])
            pr.slot[g] = [g, s[g], 0]
        return pr
    ref = pool()
    for _ in range(4):
        ref.step(range(4))
    want = ref.state(1)
    del ref
    first = pool()
    for _ in range(2):
        first.step(range(4))
    path = str(tmp_path / 'slot1.pt')
    first.mv.save_slot(1, path)
    del first
    second = PoolRun(opts, 4)
    with pytest.raises(ValueError, match='contradict'):
        second.mv.start(2, state=path, hparams=hps[0])
    for g in range(4):
        second.mv.start(g, state=path if g == 2 else None, hparams=None if g == 2 else hps[g])
        second.slot[g] = [g if g != 2 else 1, s[g if g != 2 else 1], 2 if g == 2 else 0]
    assert second.mv.slot_options(2).lr == hps[1]['lr']
    for _ in range(2):
        second.step([2])
    assert all(same(x, y) for x, y in zip(second.state(2), want))


# ------------------------------------------------------------------ resumed runs
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


def test_run_with_hparams_resumes_mid_queue(asset_dir, tmp_path, golden):
    """Six videos with their own hparams through 4 slots, cut at tick 4 and resumed from the checkpoint: the uninterrupted
    run's summaries and result files; resuming with other hparams raises and leaves the pool's slots alone."""
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    lengths = [3, 6, 2, 5, 4, 3]

    def pool(name):
        mv = MultiVideoAdaptor(pool_options(tmp_path, golden, 'c2', name), 4)
        mv.fused_eval = 'final'
        return mv
    o = pool_options(tmp_path, golden, 'c2', 'o')
    hps = [hparams_of(o, i % 4) if i != 3 else None for i in range(len(lengths))]
    videos = [stream(30 + i, n) for i, n in enumerate(lengths)]
    want = pool('straight').run(videos, str(tmp_path / 'out_straight'), hparams=hps)
    plain = pool('plain').run(videos, str(tmp_path / 'out_plain'))
    assert [w['mpjpe'] for w in want] != [w['mpjpe'] for w in plain]
    ck, out = str(tmp_path / 'ck'), str(tmp_path / 'out_resumed')
    cut = list(videos)
    cut[4] = Cut(videos[4], 2)
    with pytest.raises(Stop):
        pool('cut').run(cut, out, checkpoint=ck, every=2, hparams=hps)
    other = pool('other')
    before = other.thetas.clone()
    with pytest.raises(ValueError, match='hparams'):
        other.run(videos, out, checkpoint=ck, every=2, hparams=[None] * len(lengths))
    assert same(other.thetas, before) and other.slot_video == [None] * 4
    got = pool('resumed').run(videos, out, checkpoint=ck, every=2, hparams=hps)
    assert pickle.dumps(got) == pickle.dumps(want)
    a, b = tree(tmp_path / 'out_straight'), tree(out)
    assert sorted(a) == sorted(b) and len(a) == 8 * len(lengths)
    for f in a:
        assert a[f] == b[f], f


# ------------------------------------------------------------------ other pools
def test_webcam_streams_with_their_own_options(asset_dir, tmp_path, golden):
    """Two webcam streams with their own hparams (stream 0 reloaded after frame 3) against pools run at each stream's options."""
    from harness import cam_options, webcam_pool
    from dynaboa_b200 import synthetic
    gd = golden('adapt_webcam')
    o = cam_options(tmp_path / 'o', gd)
    hps = [hparams_of(o, g) for g in range(2)]
    n = 7
    inputs = []
    for g in range(2):
        s = synthetic.SyntheticStream(length=n, batch_size=1, rank=60 + g)
        inputs.append([(s[t]['image'].cuda(), torch.cat([torch.from_numpy(gd['kp25'][t % len(gd['kp25'])]).float().reshape(1, 25, 3),
                                                         torch.zeros(1, 24, 3)], 1).cuda()) for t in range(n)])

    def drive_cam(mv):
        out = []
        for t in range(n):
            res = mv.adapt_processed([inputs[g][t][0] for g in range(2)], [inputs[g][t][1] for g in range(2)])
            if t == 3:
                mv.reload(0)
            out.append([(mv.thetas[g].clone(), mv.m[g].clone(), mv.optim_step_record[g][-1], res[g]['vts'].clone()) for g in range(2)])
        return out
    mv = webcam_pool(tmp_path, gd, 2, 'mixed')
    for g in range(2):
        mv.start(g, hparams=hps[g])
    mixed = drive_cam(mv)
    assert mv.slot_options(0).lr == hps[0]['lr']                     # reload kept the stream's values
    del mv
    for g in range(2):
        ref = drive_cam(webcam_pool(tmp_path, gd, 2, f'own{g}', **hps[g]))
        for t, (x, y) in enumerate(zip(mixed, ref)):
            a, b = x[g], y[g]
            assert same(a[0], b[0]) and same(a[1], b[1]) and a[2] == b[2] and same(a[3], b[3]), (g, t)


SPECS = [('v0', (240, 320), 4), ('v1', (360, 480), 3), ('v2', (240, 320), 2)]


def write_videos(root):
    import cv2
    import numpy as np
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    for k, (name, (H, W), n) in enumerate(SPECS):
        rng = np.random.default_rng(k + 70)
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


def test_internet_videos_with_their_own_options(asset_dir, tmp_path):
    """Three Internet videos with their own hparams through 2 slots: each video's Pred files are those of a pool run at its
    options."""
    from harness import FLAGS
    from dynaboa_b200 import config
    from dynaboa_b200.datasets import internet_videos
    from dynaboa_b200.internet import MultiInternetAdaptor
    from oracle import adaptor_ref
    root = str(tmp_path / 'videos')
    write_videos(root)
    vids = internet_videos(root)

    def options(name, **over):
        o = vars(adaptor_ref.default_options(**FLAGS))
        o.update(expdir=str(tmp_path), expname=name, tensorboard=0, cache_results=1, model_file=config.BASE_MODEL, dataset='internet',
                 seq_seed=22, **over)
        return SimpleNamespace(**o)
    o = options('o')
    hps = [hparams_of(o, i) for i in range(len(vids))]
    MultiInternetAdaptor(options('mixed'), 2).run(vids, str(tmp_path / 'mixed'), hparams=hps)
    MultiInternetAdaptor(options('plain'), 2).run(vids, str(tmp_path / 'plain'))
    mixed, plain = tree(tmp_path / 'mixed'), tree(tmp_path / 'plain')
    for i, v in enumerate(vids):
        MultiInternetAdaptor(options(f'own{i}', **hps[i]), 2).run(vids, str(tmp_path / f'own{i}'))
        own = tree(tmp_path / f'own{i}')
        mine = sorted(f for f in mixed if f.startswith(v.name + os.sep))
        assert mine and mine == sorted(f for f in own if f.startswith(v.name + os.sep))
        for f in mine:
            assert mixed[f] == own[f], f
        assert any(mixed[f] != plain[f] for f in mine), v.name
