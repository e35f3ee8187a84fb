"""The dynamic re-adaptation loop of MultiVideoAdaptor, run per video (``dynamic_loop=True``).

- dboa_cosine_terms_active: each video's sums bit-identical to dboa_cosine_terms on its parts alone (the 15 feature sizes at
  B = G, and lengths that are not multiples of COS_CHUNK), within the fp64 bound of test_cosine_and_retrieval; idle videos'
  NaN inputs are not read and their rows of terms keep a sentinel; groups = 1 is dboa_cosine_terms.
- One video is the single-video loop: theta, teacher, trip counts and every cosine bit-identical to ``Adaptor.adapt``.
- Trajectories: G = 4 at adapt_c5.npz's options (video 0 against the golden, the others against their own single-video runs),
  then G = 4 over 8 frames at MIXED_THRESHOLD, where trip counts differ between videos: each video takes exactly the trip counts
  of its single-video run.
- Schedule invariance with the loop, and two runs bit for bit."""
import ctypes as C
import random

import pytest
import torch

from conftest import rel_err
from test_gpu_adapt import make_options
from test_gpu_multivideo_adapt import masks_for, seed_for
from test_gpu_multivideo_pool import video_masks

pytestmark = pytest.mark.gpu
COS_CHUNK = 256 * 16
SENTINEL = 0x7ff8dead0000beef                  # a NaN payload no kernel writes
# cos_sim_threshold for videos 0..3 (SyntheticStream(rank=g), video_masks, seeds 7919 g + t) at adapt_c5.npz's options over 8
# frames, calibrated once on an H100 80GB HBM3: the single-video loops run different numbers of iterations in frames 1 and 2
# (trip counts [1, 1, 2, 1] and [0, 0, 0, 3]), and the closest of all 1 - cos12 decisions lies 2.1 % from it.
# test_mixed_trip_counts_follow_the_single_video_runs checks both.
MIXED_THRESHOLD = 7e-5
N_FRAMES = 8


# ------------------------------------------------------------------ kernel
def feature_lengths(G):
    """Per-video lengths of the 15 features of the dynamic test at B = G (dboa_hmr_feature_info)."""
    from dynaboa_b200 import _lib
    lib = _lib.load()
    off, nd = C.c_longlong(), C.c_int()
    shp, strd = (C.c_longlong * 4)(), (C.c_longlong * 4)()
    out = []
    for i in range(15):
        _lib.check(lib.dboa_hmr_feature_info(G, i, C.byref(off), C.byref(nd), shp, strd), 'dboa_hmr_feature_info')
        n = 1
        for k in range(nd.value):
            n *= shp[k]
        out.append(n // G)
    return out


ODD = [3 * COS_CHUNK + 17, COS_CHUNK - 1, COS_CHUNK + 1, 1000, 5, 1, 2 * COS_CHUNK]


def sums(a, b, n, groups=None, active=None):
    """dboa_cosine_terms (groups None) or dboa_cosine_terms_active on the device tensors a[i], b[i] (lengths n[i] in total)."""
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import ptr, stream
    k = len(a)
    pa = (C.c_void_p * k)(*[t.data_ptr() for t in a])
    pb = (C.c_void_p * k)(*[t.data_ptr() for t in b])
    ln = (C.c_longlong * k)(*n)
    lib = _lib.load()
    if groups is None:
        part = torch.empty(lib.dboa_cosine_partial_floats(ln, k), device='cuda')
        terms = torch.empty(k, 3, dtype=torch.float64, device='cuda')
        _lib.call('dboa_cosine_terms', pa, pb, ln, k, ptr(part), part.numel(), ptr(terms), stream())
    else:
        part = torch.empty(lib.dboa_cosine_partial_floats_groups(ln, k, groups), device='cuda')
        terms = torch.empty(groups, k, 3, dtype=torch.float64, device='cuda')
        terms.view(torch.int64).fill_(SENTINEL)
        _lib.call('dboa_cosine_terms_active', pa, pb, ln, k, ptr(part), part.numel(), ptr(terms), stream(), groups, active)
    torch.cuda.synchronize()
    return terms


def bits(t):
    return t.contiguous().view(torch.int64)


@pytest.mark.parametrize('kind', ['features', 'odd'])
@pytest.mark.parametrize('G', [1, 2, 4, 8])
def test_each_video_is_the_one_video_call_on_its_parts(G, kind):
    per = feature_lengths(G) if kind == 'features' else ODD
    gen = torch.Generator().manual_seed(7 * G + len(kind))
    A = [torch.randn(G * n, generator=gen) for n in per]
    Bt = [a + 0.05 * torch.randn(a.shape, generator=gen) for a in A]
    a, b = [t.cuda() for t in A], [t.cuda() for t in Bt]
    n = [G * m for m in per]
    every = (1 << G) - 1
    full = sums(a, b, n, G, every)
    for g in range(G):
        s = [slice(g * m, (g + 1) * m) for m in per]
        one = sums([t[q] for t, q in zip(a, s)], [t[q] for t, q in zip(b, s)], per)
        assert torch.equal(bits(full[g]), bits(one)), g
        t = full[g].cpu()
        cos = t[:, 0] / (t[:, 1].sqrt() * t[:, 2].sqrt())
        ref = torch.stack([torch.nn.functional.cosine_similarity(x[q].double(), y[q].double(), dim=0) for x, y, q in zip(A, Bt, s)])
        assert (cos - ref).abs().max().item() < 2e-6, g
    if G == 1:
        assert torch.equal(bits(full[0]), bits(sums(a, b, n)))
        return
    for mask in (1 << (G // 2), every & ~(1 << (G - 1))):        # one active video, and all but one
        ai, bi = [t.clone() for t in a], [t.clone() for t in b]
        for g in range(G):
            if not (mask >> g) & 1:
                for t, m in zip(ai + bi, per + per):
                    t[g * m:(g + 1) * m] = float('nan')
        got = sums(ai, bi, n, G, mask)
        for g in range(G):
            if (mask >> g) & 1:
                assert torch.equal(bits(got[g]), bits(full[g])), (bin(mask), g)
            else:
                assert bool((bits(got[g]) == SENTINEL).all()), (bin(mask), g)


# ------------------------------------------------------------------ adaptor
class Videos:
    """A MultiVideoAdaptor with the dynamic loop whose slots carry (video id, stream, own frame); teacher masks
    ``masks(vid, t, call)`` and retrieval seeds ``seed(vid, t)`` follow the video."""

    def __init__(self, opts, G, masks=video_masks, seed=lambda vid, t: 7919 * vid + t):
        from dynaboa_b200.multivideo import MultiVideoAdaptor
        self.mv = MultiVideoAdaptor(opts, G, dynamic_loop=True)
        self.masks, self.seed = masks, seed
        self.slot, self.calls = [None] * G, [0] * G
        self.mv.mask_provider = self.provider

    def provider(self, g, B, dev):
        vid, _, t = self.slot[g]
        m = self.masks(vid, t, self.calls[g])
        self.calls[g] += 1
        return m.to(dev)

    def start(self, g, vid, stream):
        self.mv.start(g)
        self.slot[g] = [vid, stream, 0]

    def step(self, run):
        """One pool frame: the slots in `run` advance by one frame of their video.  Returns {slot: (vid, own frame, batch)}."""
        batches, done = [None] * self.mv.G, {}
        for g in run:
            vid, s, t = self.slot[g]
            batches[g] = {k: v.cuda() if torch.is_tensor(v) else v for k, v in s[t].items()}
            self.calls[g] = 0
            self.mv.rngs[g].seed(self.seed(vid, t))
            done[g] = (vid, t, batches[g])
        self.mv.adapt(batches)
        for g in run:
            self.slot[g][2] += 1
        return done

    def state(self, g):
        mv = self.mv
        return [mv.thetas[g].clone(), mv.teachers[g].clone(), mv.m[g].clone(), mv.v[g].clone()]


class Single:
    """``Adaptor.adapt`` of one video with the same teacher masks and retrieval seeds."""

    def __init__(self, opts, vid, masks=video_masks, seed=lambda vid, t: 7919 * vid + t):
        from dynaboa_b200.adaptor import Adaptor
        self.ad = Adaptor(opts)
        self.ad.fused_eval = 'none'
        self.vid, self.masks, self.seed = vid, masks, seed

    def step(self, t, batch):
        calls, ad = {'i': 0}, self.ad

        def provider(B, dev):
            m = self.masks(self.vid, t, calls['i'])
            calls['i'] += 1
            return m.to(dev)
        ad.teacher.mask_provider = provider
        random.seed(self.seed(self.vid, t))
        ad.global_step, ad.fit_losses = t, {}
        ad.model.eval()
        ad.adapt(batch)


def c5_options(tmp, golden, name, threshold=None):
    from dynaboa_b200 import config
    o = make_options(tmp / name, str(golden('adapt_c5')['options']), model_file=config.BASE_MODEL)
    assert o.dynamic_boa
    if threshold is not None:
        o.cos_sim_threshold = threshold
    return o


def stream(vid, n):
    from dynaboa_b200 import synthetic
    return synthetic.SyntheticStream(length=n, batch_size=1, rank=vid)


@pytest.mark.parametrize('threshold', [None, MIXED_THRESHOLD], ids=['golden', 'mixed'])
def test_one_video_is_the_single_video_loop(asset_dir, tmp_path, golden, threshold):
    p = Videos(c5_options(tmp_path, golden, 'mv', threshold), 1)
    s = Single(c5_options(tmp_path, golden, 'ad', threshold), 0)
    p.start(0, 0, stream(0, N_FRAMES))
    for t in range(N_FRAMES):
        batch = p.step([0])[0][2]
        s.step(t, batch)
        ad, mv = s.ad, p.mv
        assert mv.optim_step_record[0] == ad.optim_step_record and mv.optimized_step == [ad.optimized_step], t
        assert mv.feat_sims[0][t] == ad.feat_sims[t], t                 # python floats of the float32 cosines: bit for bit
        assert torch.equal(mv.last_upper_loss[0], ad.last_upper_loss), t
        assert float(mv.fit_losses['feat_sim/cos_sim'][0]) == float(ad.fit_losses['feat_sim/cos_sim']), t
    assert torch.equal(p.mv.theta(0), s.ad.model.module.arena)
    assert torch.equal(p.mv.teachers[0], s.ad.teacher.arena)


def compare_outputs(p, done, singles, bound_of, what):
    mv = p.mv
    imgs = torch.cat([done[g][2]['image'] for g in range(mv.G)])
    preds, up = mv.predict(imgs), mv.last_upper_loss.cpu()
    for g, (vid, t, batch) in done.items():
        if vid not in singles:
            continue
        ad = singles[vid].ad
        assert mv.optim_step_record[g] == ad.optim_step_record, (what, vid, t)
        ref_up = float(ad.last_upper_loss)
        assert abs(float(up[g]) - ref_up) <= 1e-3 * abs(ref_up), (what, vid, t, float(up[g]), ref_up)
        ref = ad.predict(batch['image'])
        for k in ('rotmat', 'betas', 'cam', 'joints', 'vertices'):
            assert rel_err(preds[g][k], ref[k].cpu().numpy()) < 1e-3, (what, vid, t, k)
        d, bound = float((mv.theta(g) - ad.model.module.arena).abs().max()), bound_of(g)
        assert d <= bound, (what, vid, t, d, bound)
        assert mv.last_retrieval[g] == ad.last_retrieval, (what, vid, t)
    return preds, up


def test_golden_c5_videos_follow_their_trajectories(asset_dir, tmp_path, golden):
    """G = 4 at adapt_c5.npz's options, where every loop hits the cap: video 0 against the golden to the criteria of
    test_gpu_adapt.run_and_compare, videos 1..3 against their own single-video runs."""
    from oracle.make_golden import sample_indices
    gd = golden('adapt_c5')
    masks = lambda vid, t, call: masks_for(vid, t, call, gd)
    p = Videos(c5_options(tmp_path, golden, 'mv'), 4, masks=masks, seed=seed_for)
    o = p.mv.options
    singles = {g: Single(c5_options(tmp_path, golden, f'v{g}'), g, masks=masks, seed=seed_for) for g in range(1, 4)}
    n_frames = gd['upper_loss'].shape[0]
    for g in range(4):
        p.start(g, g, stream(g, n_frames))
    names = [str(s) for s in gd['param_names']]
    lay = p.mv.base.model.module._lay
    n_outer = [0] * 4
    for t in range(n_frames):
        done = p.step(range(4))
        for g in range(1, 4):
            singles[g].step(t, done[g][2])
        for g in range(4):
            n_outer[g] += 1 + min(p.mv.optim_step_record[g][-1], o.optim_steps)
        preds, up = compare_outputs(p, done, singles, lambda g: 4 * o.lr * n_outer[g], 'c5')
        assert p.mv.optim_step_record[0][-1] == int(gd['dyn_steps'][t]) == o.optim_steps + 1, t
        tol = 2e-4 if t == 0 else 1e-3
        assert abs(float(up[0]) - gd['upper_loss'][t]) <= tol * abs(gd['upper_loss'][t]), t
        q = preds[0]
        assert rel_err(q['rotmat'], gd['rotmat'][t]) < 1e-3 and rel_err(q['betas'], gd['betas'][t]) < 1e-3, t
        assert rel_err(q['cam'], gd['cam'][t]) < 1e-3 and rel_err(q['joints'], gd['joints'][t]) < 1e-3, t
        assert rel_err(q['vertices'][:, ::10], gd['verts_sub'][t]) < 1e-3, t
        views = dict(zip(lay.names, lay.views(p.mv.theta(0).clone())))
        for i, name in enumerate(names):
            idx = sample_indices(name, views[name].numel())
            th = views[name].contiguous().flatten()[idx].double().cpu().numpy()
            assert abs(th - gd['theta_samples'][t][i]).max() <= 4 * o.lr * n_outer[0], (t, name)


def decisions(ad, t):
    """1 - cos12 of every feature test of frame t of a single-video run."""
    return [1 - s[12]['cos'] for s in ad.feat_sims[t]]


def test_mixed_trip_counts_follow_the_single_video_runs(asset_dir, tmp_path, golden):
    """G = 4 over 8 frames (the motion term goes live) at MIXED_THRESHOLD: each video takes exactly the trip counts of its
    single-video run, and its theta stays within 4 lr n_outer of it, n_outer counting that video's own Adam steps."""
    thr = MIXED_THRESHOLD
    p = Videos(c5_options(tmp_path, golden, 'mv', thr), 4)
    o = p.mv.options
    singles = {g: Single(c5_options(tmp_path, golden, f'v{g}', thr), g) for g in range(4)}
    for g in range(4):
        p.start(g, g, stream(g, N_FRAMES))
    n_outer, mixed = [0] * 4, []
    for t in range(N_FRAMES):
        done = p.step(range(4))
        for g in range(4):
            singles[g].step(t, done[g][2])
            for v in decisions(singles[g].ad, t):
                assert abs(v - thr) >= 0.01 * thr, (f'video {g} frame {t}: decision 1 - cos12 = {v:.6e} lies within 1 % of '
                                                    f'MIXED_THRESHOLD = {thr:.3e}: re-calibrate it')
        trips = [singles[g].ad.optim_step_record[-1] for g in range(4)]
        if len({min(n, o.optim_steps) for n in trips}) > 1:              # loops of different lengths: the mask narrows
            mixed.append(t)
        for g in range(4):
            n_outer[g] += 1 + min(trips[g], o.optim_steps)
        compare_outputs(p, done, singles, lambda g: 4 * o.lr * n_outer[g], 'mixed')
        assert p.mv.optimized_step == trips, t
    assert mixed, 'the single-video loops never ran different numbers of iterations in one frame: re-calibrate MIXED_THRESHOLD'


def test_a_looping_video_does_not_depend_on_its_slot_or_schedule(asset_dir, tmp_path, golden):
    """Video X alone in slot 0, against X in slot 2 from pool frame 3 while the other slots run, pause, finish and restart with
    their own trip counts: theta, teacher, m, v, upper loss, trip counts and cosines bit for bit.  A slot that sits a frame out
    keeps its arenas bit for bit."""
    X, thr = 5, MIXED_THRESHOLD
    a = Videos(c5_options(tmp_path, golden, 'a', thr), 4)
    a.start(0, X, stream(X, N_FRAMES))
    traj_a = []
    for _ in range(N_FRAMES):
        a.step([0])
        traj_a.append(a.state(0) + [a.mv.last_upper_loss[0].clone()])
    rec_a = (list(a.mv.optim_step_record[0]), dict(a.mv.feat_sims[0]))
    del a
    b = Videos(c5_options(tmp_path, golden, 'b', thr), 4)
    total = N_FRAMES + 3
    b.start(0, 11, stream(11, total))
    b.start(1, 12, stream(12, total))
    b.start(2, 13, stream(13, 3))
    b.start(3, 14, stream(14, 2))
    traj_b, differs = [], False
    for f in range(total):
        if f == 3:
            b.start(2, X, stream(X, N_FRAMES))
        if f == 4:
            b.start(3, 15, stream(15, total))
        run = [0, 2]
        if f not in (1, 4, 5):                       # slot 1 pauses
            run.append(1)
        if f not in (2, 3):                          # slot 3: video 14 on frames 0-1, idle, video 15 from frame 4
            run.append(3)
        run.sort()
        idle = [g for g in range(4) if g not in run]
        before = {g: b.state(g) for g in idle}
        b.step(run)
        for g in idle:
            assert all(torch.equal(x, y) for x, y in zip(before[g], b.state(g))), (f, g)
            assert b.mv.optimized_step[g] is None, (f, g)
        if f >= 3:
            traj_b.append(b.state(2) + [b.mv.last_upper_loss[2].clone()])
            cap = b.mv.options.optim_steps             # loop iterations of a slot: min(trip count, optim_steps)
            mine = min(b.mv.optimized_step[2], cap)
            differs |= any(min(b.mv.optimized_step[g], cap) != mine for g in run if g != 2)
    assert differs, "X's loop mask never differed from another active slot's: re-calibrate MIXED_THRESHOLD"
    assert (b.mv.optim_step_record[2], b.mv.feat_sims[2]) == rec_a
    for t, (ra, rb) in enumerate(zip(traj_a, traj_b)):
        for name, x, y in zip(('theta', 'teacher', 'm', 'v', 'upper loss'), ra, rb):
            assert torch.equal(x, y), (t, name)


def test_two_runs_are_bit_identical(asset_dir, tmp_path, golden):
    runs = []
    for r in range(2):
        p = Videos(c5_options(tmp_path, golden, f'r{r}', MIXED_THRESHOLD), 4)
        for g in range(4):
            p.start(g, g, stream(g, 4))
        for _ in range(4):
            p.step(range(4))
        torch.cuda.synchronize()
        runs.append((p.mv.thetas.clone(), [list(x) for x in p.mv.optim_step_record]))
        del p
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]
