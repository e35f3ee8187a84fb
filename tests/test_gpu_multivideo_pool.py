"""Slots of MultiVideoAdaptor over the active-video mask of the grouped plan.

- Masked network calls (dboa_hmr_{forward,backward}_active): with the idle videos' image rows, dropout masks, upstream gradients
  and the tape filled with NaN and their gradient arenas with a sentinel, every active video's outputs, tape rows and gradient
  are bit-identical to the unmasked call on finite inputs, and the idle gradient arenas keep the sentinel bytes.  All bits set
  is bit-identical to dboa_hmr_{forward,backward}_groups.
- dboa_loss_motion_active: enabled videos bit-identical to dboa_loss_motion_groups, disabled ones untouched with term 0.
- Schedule invariance: a video's theta, teacher, Adam moments and upper losses do not depend on its slot, its start frame or
  what the other slots do (busy, idle, finished and restarted), bit for bit, at C2 over 8 frames and C3 over 2.
- Semantics: every video of a 6-video pool through 4 slots follows its own single-video Adaptor.adapt run to the criteria of
  test_gpu_adapt, the videos started mid-run included.
- start(g) restores the checkpoint's theta and teacher and zero moments."""
import random

import pytest
import torch

from conftest import rel_err
from harness import PoolRun, SingleRun, bits, hmr_model, inputs, pool_options, stacked, stream

pytestmark = pytest.mark.gpu

# (videos G, samples per video b, tensor-core mode, dropout masks, active mask: an int, or 'seeded')
CONFIGS = [(2, 1, 3, False, 0b01), (2, 8, 0, True, 0b10), (4, 1, 1, True, 0b0100), (4, 8, 2, False, 0b1011),
           (8, 1, 3, True, 'seeded'), (8, 8, 3, False, 0b11101111), (8, 1, 0, False, 0b10000000), (4, 1, 3, False, 'seeded'),
           (8, 2, 1, False, 'seeded')]
IDS = [f'G{g}-b{b}-tc{m}' + ('-masked' if k else '') + f'-{a if isinstance(a, str) else bin(a)}' for g, b, m, k, a in CONFIGS]
SENTINEL = 0x7fc0dead                  # a NaN payload no kernel writes


@pytest.fixture(scope='module')
def model():
    yield from hmr_model()


def call(m, arenas, x, masks, d, G, active, tape_fill, grad):
    from dynaboa_b200.hmr import raw_backward, raw_forward, tape_floats
    B = x.shape[0]
    tape = torch.full((tape_floats(B),), tape_fill, device='cuda')
    out = raw_forward(arenas, m._buffers, x, masks, tape, groups=G, active=active)[:3]
    raw_backward(arenas, tape, B, masks is not None, d[0], d[1], d[2], grad, groups=G, active=active)
    torch.cuda.synchronize()
    return out, tape, grad


def sample_axis(key):
    return {'xc': 1, 'h1pre': 1, 'h1post': 1, 'h2pre': 1, 'h2post': 1, 'params': 1, 'masks': 2}.get(key, 0)


def rows_of(t, axis, s):
    return t[(slice(None),) * axis + (s,)]


@pytest.mark.parametrize('cfg', CONFIGS, ids=IDS)
def test_masked_calls_are_the_unmasked_calls_of_the_active_videos(model, cfg):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import tape_views
    G, b, mode, masked, active = cfg
    B = G * b
    if active == 'seeded':
        gen = random.Random(31 * G + b)
        active = 0
        while active in (0, (1 << G) - 1):
            active = gen.getrandbits(G)
    _lib.load().dboa_set_tensor_core_conv(mode)
    arenas = stacked(model, G, 300 + 10 * G + b + mode)
    x, masks, d = inputs(B, 8000 + 10 * B + mode, masked)
    ref_out, ref_tape, ref_grad = call(model, arenas, x, masks, d, G, None, float('nan'), torch.zeros_like(arenas))
    # the unmasked call is the call with every bit set
    out, tape, grad = call(model, arenas, x, masks, d, G, (1 << G) - 1, float('nan'), torch.zeros_like(arenas))
    for a, c in zip(out, ref_out):
        assert torch.equal(bits(a), bits(c))
    assert torch.equal(bits(tape), bits(ref_tape)) and torch.equal(grad, ref_grad)
    # idle videos: NaN inputs, NaN tape, sentinel gradient arenas
    on = [bool((active >> g) & 1) for g in range(G)]
    sl = [slice(g * b, (g + 1) * b) for g in range(G)]
    xi, mi, di = x.clone(), None if masks is None else masks.clone(), [t.clone() for t in d]
    gi = torch.zeros_like(arenas)
    for g in range(G):
        if not on[g]:
            xi[sl[g]] = float('nan')
            if mi is not None:
                mi[:, :, sl[g]] = float('nan')
            for t in di:
                t[sl[g]] = float('nan')
            gi[g].view(torch.int32).fill_(SENTINEL)
    out, tape, grad = call(model, arenas, xi, mi, di, G, active, float('nan'), gi)
    v, rv = tape_views(tape, B), tape_views(ref_tape, B)
    for g in range(G):
        if not on[g]:
            assert bool((grad[g].view(torch.int32) == SENTINEL).all()), g
            continue
        for a, c in zip(out, ref_out):
            assert torch.equal(bits(a[sl[g]]), bits(c[sl[g]])), g
        assert torch.equal(grad[g], ref_grad[g]), g
        for key, val in v.items():
            ax = sample_axis(key)
            for i, t in enumerate(val if isinstance(val, list) else [val]):
                if t is None:
                    continue
                r = rv[key][i] if isinstance(val, list) else rv[key]
                assert torch.equal(bits(rows_of(t, ax, sl[g])), bits(rows_of(r, ax, sl[g]))), (g, key, i)
    assert any(on) and not all(on)


def test_motion_mask():
    from dynaboa_b200 import _lib
    from dynaboa_b200._lib import ptr, stream
    G, b = 8, 2
    B = G * b
    gen = torch.Generator().manual_seed(11)
    pa, ph = torch.randn(B, 49, 2, generator=gen).cuda(), torch.randn(B, 49, 2, generator=gen).cuda()
    ka, kh = torch.randn(B, 49, 3, generator=gen).cuda(), torch.randn(B, 49, 3, generator=gen).cuda()
    ka[..., 2], kh[..., 2] = (ka[..., 2] > 0).float(), (kh[..., 2] > -0.5).float()
    dpa0 = torch.randn(B, 49, 2, generator=gen).cuda()
    runs = {}
    for active in (None, 0b10110010):
        term, dpa, dph = torch.full((G,), float('nan'), device='cuda'), dpa0.clone(), torch.full_like(pa, 7.0)
        args = (ptr(pa), ptr(ph), ptr(ka), ptr(kh), 0.3, ptr(term), ptr(dpa), ptr(dph), B, 1, 25, 24, G)
        if active is None:
            _lib.call('dboa_loss_motion_groups', *args, stream())
        else:
            _lib.call('dboa_loss_motion_active', *args, active, stream())
        torch.cuda.synchronize()
        runs[active] = term, dpa, dph
    (t0, a0, h0), (t1, a1, h1) = runs[None], runs[0b10110010]
    for g in range(G):
        s = slice(g * b, (g + 1) * b)
        if (0b10110010 >> g) & 1:
            assert torch.equal(t1[g], t0[g]) and torch.equal(a1[s], a0[s]) and torch.equal(h1[s], h0[s]), g
        else:
            assert float(t1[g]) == 0.0 and torch.equal(a1[s], dpa0[s]) and bool((h1[s] == 7.0).all()), g


# ------------------------------------------------------------------ adaptor
@pytest.mark.parametrize('tag,n_frames', [('c2', 8), ('c3', 2)])
def test_a_video_does_not_depend_on_its_slot_or_schedule(asset_dir, tmp_path, golden, tag, n_frames):
    X = 5
    # A: X alone in slot 0 from pool frame 0
    a = PoolRun(pool_options(tmp_path, golden, tag, 'a'), 4)
    a.start(0, X, stream(X, n_frames))
    traj_a = []
    for _ in range(n_frames):
        a.step([0])
        traj_a.append(a.state(0) + [a.mv.last_upper_loss[0].clone()])
    del a
    # B: X in slot 2 from pool frame 3; slot 0 runs one long video, slot 1 pauses, slot 2 first runs a 3-frame video, slot 3
    # finishes a 2-frame video and is refilled at pool frame 4
    b = PoolRun(pool_options(tmp_path, golden, tag, 'b'), 4)
    total = n_frames + 3
    b.start(0, 11, stream(11, total))
    b.start(1, 12, stream(12, total))
    b.start(2, 13, stream(13, 3))
    b.start(3, 14, stream(14, 2))
    traj_b = []
    for f in range(total):
        if f == 3:
            b.start(2, X, stream(X, n_frames))
            st = b.mv
            assert torch.equal(st.thetas[2], st.base.model.module.arena) and torch.equal(st.teachers[2], st.base.teacher.arena)
            assert not st.m[2].any() and not st.v[2].any() and st.video_steps[2] == 0 and st.step_counts[2] == 0
        if f == 4:
            b.start(3, 15, stream(15, total))
        run = [0, 2]
        if f not in (1, 4, 5):                       # slot 1 pauses
            run.append(1)
        if f not in (2, 3):                          # slot 3: video 14 on frames 0-1, idle, video 15 from frame 4
            run.append(3)
        b.step(sorted(run))
        if f >= 3:
            traj_b.append(b.state(2) + [b.mv.last_upper_loss[2].clone()])
    assert len(traj_a) == len(traj_b) == n_frames
    for t, (ra, rb) in enumerate(zip(traj_a, traj_b)):
        for name, x, y in zip(('theta', 'teacher', 'm', 'v', 'upper loss'), ra, rb):
            assert torch.equal(x, y), (tag, t, name)


def test_every_pool_video_follows_its_own_single_video_run(asset_dir, tmp_path, golden):
    lengths = [3, 8, 2, 5, 6, 4]                     # videos 0..5 through 4 slots, each slot refilled when its video ends
    p = PoolRun(pool_options(tmp_path, golden, 'c2', 'pool'), 4)
    o = p.mv.options
    queue = list(range(len(lengths)))
    singles, frames = {}, {}
    for g in range(4):
        vid = queue.pop(0)
        p.start(g, vid, stream(vid, lengths[vid]))
    seen = set()
    while True:
        for g in range(4):                           # refill finished slots
            if p.slot[g] is not None and p.slot[g][2] >= lengths[p.slot[g][0]]:
                p.slot[g] = None
                if queue:
                    vid = queue.pop(0)
                    p.start(g, vid, stream(vid, lengths[vid]))
        run = [g for g in range(4) if p.slot[g] is not None]
        if not run:
            break
        done = p.step(run)
        imgs = torch.cat([done[g][2]['image'] if g in done else torch.zeros(1, 3, 224, 224, device='cuda') for g in range(4)])
        preds = p.mv.predict(imgs)
        up = p.mv.last_upper_loss.cpu()
        for g, (vid, t, batch) in done.items():
            seen.add(vid)
            if vid not in singles:
                singles[vid] = SingleRun(pool_options(tmp_path, golden, 'c2', f'v{vid}'), vid)
            singles[vid].step(t, batch)
            ad = singles[vid].ad
            ref_up = float(ad.last_upper_loss)
            assert abs(float(up[g]) - ref_up) <= 1e-3 * abs(ref_up), (vid, t, float(up[g]), ref_up)
            ref = ad.predict(batch['image'])
            for k in ('rotmat', 'betas', 'cam', 'joints', 'vertices'):
                assert rel_err(preds[g][k], ref[k].cpu().numpy()) < 1e-3, (vid, t, k)
            bound = 4 * o.lr * (t + 1)
            d = float((p.mv.theta(g) - ad.model.module.arena).abs().max())
            assert d <= bound, (vid, t, d, bound)
            frames[vid] = t + 1
    assert seen == set(range(len(lengths))) and all(frames[v] == n for v, n in enumerate(lengths))


def test_start_restores_the_checkpoint(asset_dir, tmp_path, golden):
    p = PoolRun(pool_options(tmp_path, golden, 'c2', 's'), 2)
    for g in range(2):
        p.start(g, g, stream(g, 2))
    for _ in range(2):
        p.step([0, 1])
    mv = p.mv
    assert not torch.equal(mv.thetas[1], mv.base.model.module.arena) and bool(mv.m[1].any())
    before = p.state(0)
    mv.start(1, seed=3)
    assert torch.equal(mv.thetas[1], mv.base.model.module.arena) and torch.equal(mv.teachers[1], mv.base.teacher.arena)
    assert not mv.m[1].any() and not mv.v[1].any()
    assert mv.video_steps[1] == mv.step_counts[1] == 0 and mv.rngs[1].random() == random.Random(3).random()
    assert all(torch.equal(x, y) for x, y in zip(p.state(0), before))
