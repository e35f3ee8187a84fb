"""The grouped HMR plan and every grouped entry point at the pool's full width: 16 to 64 videos, and active masks whose bits
reach 63.  The modules of the grouped calls at G <= 8 (test_gpu_multivideo*.py, test_gpu_step_kernels.py, test_gpu_multiwebcam.py)
hold the same criteria; here the group arithmetic, the split-K sizing of a 64-group grid and the 64-bit masks are exercised.

- Layer parity: every video's convolution outputs, GroupNorm statistics, post-activations, regressor rows and outputs (from the
  GPU's own inputs, read from the tape) and all 169 gradient tensors (oracle/hmr_frozen.py on the GPU's own ReLU / max-pool /
  dropout pattern) against fp64 with that video's own weights, to the bounds of test_gpu_hmr_layers.py, GRAD_L2 per video.  The
  reference takes the 6D -> rotation map at the GPU's own 6D pose: with dropout, some joints' two 6D columns come within a few
  degrees of each other, and the map's derivative then turns the forward's in-bound rounding of the pose into a gradient error
  above GRAD_L2 (1.3e-5 and 2.5e-5 in two of 80 dropout videos; 2.1e-6 and 6.5e-6 with the GPU's point).  For the same reason a
  joint with sin(a1, a2) < ILL_POSED is held to the rotmat bound scaled by sin / ILL_POSED.  Two negative controls (a
  neighbour's weights, a neighbour's samples) must miss the gradient bound by 10x.
- Masks over all 64 bits: with idle videos' inputs NaN, every active video's outputs, tape rows and gradient are bit-identical to
  the all-ones call, and idle gradient arenas keep a sentinel; the all-ones mask is the unmasked ``_groups`` entry.
- Isolation: identical videos in slots 0, 31, 32 and 63 give identical bits, perturbing video 63 or video 0 changes no bit of
  any other video, and two identical calls are bit-identical.
- dboa_cosine_terms_active, dboa_eval_metrics_active, dboa_keypoint_transform_groups and dboa_crop_resize_normalize_groups at 64
  videos under the same masks: active rows equal the one-video calls (and the fp64 references), idle rows are not written."""
import ctypes as C
import json
import math
import random
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from harness import (COS_TOL, CROP_TOL, FWD_TOL, GRAD_L2, GRAD_TOL, TERMS_TOL, bits, crop_kind, crop_oracle, gn_apply, gn_stats,
                     hmr_model, inputs, nchw, rel, scene, stacked, structure, tape_pattern)

pytestmark = pytest.mark.gpu

# (videos G, samples per video b, tensor-core mode, dropout masks)
CONFIGS = [(64, 1, 3, False), (64, 1, 0, False), (64, 1, 2, True), (48, 1, 3, False), (32, 2, 1, False), (16, 4, 3, True)]
IDS = [f'G{g}-b{b}-tc{m}' + ('-masked' if k else '') for g, b, m, k in CONFIGS]
# active masks of 64 videos: the top bit alone, the high word, the two bits either side of the 32-bit boundary, every other bit,
# and one seeded mask
MASKS = [1 << 63, 0xFFFFFFFF00000000, (1 << 31) | (1 << 32), 0x5555555555555555, random.Random(64).getrandbits(64)]
MASK_IDS = ['bit63', 'high-word', 'bits31-32', 'alternate', 'seeded']
ALL = (1 << 64) - 1
SENTINEL = 0x7fc0dead                  # a NaN payload no kernel writes
ILL_POSED = 0.1                        # sin(a1, a2) below which a joint's rotation is ill-conditioned (about 6 degrees)


@pytest.fixture(scope='module')
def model():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield from hmr_model()
    print(f'\nWIDE module: {time.time() - t0:.0f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')


def run(m, arenas, x, masks, d, G, active=None, grad=None):
    """One grouped forward and backward on a NaN-filled tape: (outputs, tape, gradient arenas)."""
    from dynaboa_b200.hmr import raw_backward, raw_forward, tape_floats
    B = x.shape[0]
    tape = torch.full((tape_floats(B),), float('nan'), device='cuda')
    out = raw_forward(arenas, m._buffers, x, masks, tape, groups=G, active=active)[:3]
    grad = torch.zeros_like(arenas) if grad is None else grad
    raw_backward(arenas, tape, B, masks is not None, d[0], d[1], d[2], grad, groups=G, active=active)
    torch.cuda.synchronize()
    return out, tape, grad


def sample_axis(key):
    return {'xc': 1, 'h1pre': 1, 'h1post': 1, 'h2pre': 1, 'h2post': 1, 'params': 1, 'masks': 2}.get(key, 0)


def rows_differ(ra, rb, B):
    """(B,) bool: the samples whose outputs or tape rows differ in any bit between the runs ``ra`` and ``rb``."""
    from dynaboa_b200.hmr import tape_views
    bad = torch.zeros(B, dtype=torch.bool, device='cuda')
    for a, c in zip(ra[0], rb[0]):
        bad |= (bits(a) != bits(c)).reshape(B, -1).any(1)
    va, vb = tape_views(ra[1], B), tape_views(rb[1], B)
    for key, val in va.items():
        pairs = zip(val, vb[key]) if isinstance(val, list) else [(val, vb[key])]
        for a, c in pairs:
            if a is not None:
                bad |= (bits(a) != bits(c)).movedim(sample_axis(key), 0).reshape(B, -1).any(1)
    return bad


def video_views(m, arena):
    """{name: fp64 leaf} of one video's weights, plus the buffers hmr_frozen reads."""
    from dynaboa_b200.hmr import layout
    lay = layout()
    p = {n: w.detach().double().requires_grad_(True) for n, w in zip(lay.names, lay.views(arena.clone()))}
    return p, {k: m._buffers[k].double() for k in ('init_pose', 'init_shape', 'init_cam')}


def gpu_pattern(tape, B, s, masks=None):
    """``tape_pattern`` of the samples ``s`` with the GPU's final 6D pose, where oracle/hmr_frozen.py takes the rotation map."""
    from dynaboa_b200.hmr import tape_views
    return dict(tape_pattern(tape, B, s, masks), pose6d=tape_views(tape, B)['params'][3][s, :144].double())


def frozen_grad(m, arena, x, d, pattern):
    """fp64 gradient {name: tensor} of the samples ``x`` (upstream gradients ``d``) through weights ``arena`` on ``pattern``."""
    from oracle import hmr_frozen
    p, bufs = video_views(m, arena)
    rot, shape, cam, _ = hmr_frozen.forward(x.double(), dict(p, **bufs), pattern)
    ((rot * d[0].double()).sum() + (shape * d[1].double()).sum() + (cam * d[2].double()).sum()).backward()
    return {n: t.grad for n, t in p.items()}


def grad_errors(grad, ref):
    """(worst per-tensor error relative to the tensor's largest fp64 value and its name, whole-arena relative L2)."""
    from dynaboa_b200.hmr import layout
    lay = layout()
    worst, num, den = (0.0, ''), 0.0, 0.0
    for n, gv in zip(lay.names, lay.views(grad.clone())):
        e = rel(gv, ref[n])
        if not e <= worst[0]:
            worst = (e, n)
        num, den = num + float((gv.double() - ref[n]).pow(2).sum()), den + float(ref[n].pow(2).sum())
    return worst, math.sqrt(num / den)


def check_forward(m, arena, v, s, rot, masks, note):
    """Every forward tape entry of the samples ``s`` recomputed in fp64 from the GPU's own inputs (test_gpu_hmr_layers.py)."""
    from dynaboa_b200.hmr import layout
    from oracle import geometry_ref
    lay = layout()
    P = lay.views(arena.clone())                      # views() offsets are absolute: give it a tensor of its own
    geo, blocks = structure()
    block_in = [v['p0'][s]] + [v['a'][bl[2]][s] for bl in blocks[:-1]]
    conv_in = {0: v['x0'][s]}
    for bi, (c1, c2, c3, cd) in enumerate(blocks):
        conv_in.update({c1: block_in[bi], c2: v['a'][c1][s], c3: v['a'][c2][s]})
        if cd is not None:
            conv_in[cd] = block_in[bi]
    ys = {}
    for i, (name, _, _, k, stride, _) in enumerate(geo):
        y = nchw(v['y'][i][s])
        note('y', rel(y, F.conv2d(nchw(conv_in[i]), P[3 * i].double(), stride=stride, padding=k // 2)), name)
        mean, rstd = gn_stats(y)
        st = v['stats'][i][s].double()
        note('stats', float(torch.cat([((st[..., 0] - mean).abs() * rstd).flatten(), (st[..., 1] / rstd - 1).abs().flatten()]).max()), name)
        ys[i] = (y, mean, rstd)

    def gn(i):
        return gn_apply(*ys[i], P[3 * i + 1], P[3 * i + 2])
    note('a', rel(nchw(v['a'][0][s]), torch.relu(gn(0))), 'conv1')
    for bi, (c1, c2, c3, cd) in enumerate(blocks):
        note('a', rel(nchw(v['a'][c1][s]), torch.relu(gn(c1))), geo[c1][0])
        note('a', rel(nchw(v['a'][c2][s]), torch.relu(gn(c2))), geo[c2][0])
        res = gn(cd) if cd is not None else nchw(block_in[bi])
        note('a', rel(nchw(v['a'][c3][s]), torch.relu(gn(c3) + res)), geo[c3][0])
    xf = nchw(v['a'][blocks[-1][2]][s]).mean(dim=(2, 3))
    names = lay.names
    W = {n: P[names.index(n)].double() for n in ('fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias')}
    Wd = torch.cat([P[names.index(n + '.weight')].double() for n in ('decpose', 'decshape', 'deccam')])
    bd = torch.cat([P[names.index(n + '.bias')].double() for n in ('decpose', 'decshape', 'deccam')])
    for it in range(3):
        xc = v['xc'][it][s]
        note('head', rel(xc[:, :2048], xf), f'xc[{it}] pooled')
        assert torch.equal(xc[:, 2048:2205], v['params'][it][s, :157]), f'xc[{it}] params'
        h1 = v['h1pre'][it][s]
        note('head', rel(h1, xc[:, :2205].double() @ W['fc1.weight'].t() + W['fc1.bias']), f'h1pre[{it}]')
        assert torch.equal(v['h1post'][it][s], h1 * masks[it, 0, s] if masks is not None else h1), f'h1post[{it}]'
        h2 = v['h2pre'][it][s]
        note('head', rel(h2, v['h1post'][it][s].double() @ W['fc2.weight'].t() + W['fc2.bias']), f'h2pre[{it}]')
        assert torch.equal(v['h2post'][it][s], h2 * masks[it, 1, s] if masks is not None else h2), f'h2post[{it}]'
        delta = v['h2post'][it][s].double() @ Wd.t() + bd
        note('head', rel(v['params'][it + 1][s, :157], v['params'][it][s, :157].double() + delta, delta.abs().max()), f'params[{it + 1}]')
    # rotmat from the GPU's own 6D pose.  fp32 Gram-Schmidt loses accuracy as 1 / sin(a1, a2), the sine between a joint's two
    # 6D columns: a joint with sin < ILL_POSED is held to the bound scaled by sin / ILL_POSED
    p6 = v['params'][3][s, :144].double()
    ref = geometry_ref.rot6d_to_rotmat(p6).view(-1, 24, 3, 3)
    a1, a2 = p6.view(-1, 24, 3, 2).unbind(-1)
    b1 = a1 / a1.norm(dim=-1, keepdim=True)
    sin = (a2 - (b1 * a2).sum(-1, keepdim=True) * b1).norm(dim=-1) / a2.norm(dim=-1)
    err = (rot[s].double() - ref).abs().amax((-2, -1)) / ref.abs().max()
    note('out', float((err * (sin / ILL_POSED).clamp(max=1)).max()), 'rotmat')


# ------------------------------------------------------------------ 1. every video against fp64 with its own weights
@pytest.mark.parametrize('cfg', CONFIGS, ids=IDS)
def test_every_video_against_fp64_with_its_own_weights(model, cfg):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import tape_views
    G, b, mode, masked = cfg
    B = G * b
    _lib.load().dboa_set_tensor_core_conv(mode)
    m = model
    arenas = stacked(m, G, 100 * G + 10 * b + mode)
    x, masks, d = inputs(B, 4000 + B + mode, masked)
    (rot, shape, cam), tape, grad = run(m, arenas, x, masks, d, G)
    v = tape_views(tape, B)
    worst = {k: (0.0, '') for k in list(FWD_TOL) + ['grad', 'grad_l2']}

    def note(kind, err, where):
        tol = {'grad': GRAD_TOL, 'grad_l2': GRAD_L2}.get(kind) or FWD_TOL[kind]
        assert err <= tol, (kind, where, err)
        if err > worst[kind][0]:
            worst[kind] = (err, where)
    for g in range(G):
        s = slice(g * b, (g + 1) * b)
        check_forward(m, arenas[g], v, s, rot, masks, lambda kind, e, where: note(kind, e, f'video {g} {where}'))
        p3 = v['params'][3][s, :157]
        assert torch.equal(shape[s], p3[:, 144:154]) and torch.equal(cam[s], p3[:, 154:157]), g
        ref = frozen_grad(m, arenas[g], x[s], [t[s] for t in d], gpu_pattern(tape, B, s, masks))
        (e, name), l2 = grad_errors(grad[g], ref)
        note('grad', e, f'video {g} {name}')
        note('grad_l2', l2, f'video {g}')
    print(f'\nWIDE {IDS[CONFIGS.index(cfg)]} worst ' + json.dumps({k: [f'{e:.2e}', w] for k, (e, w) in worst.items()}))


def test_negative_controls_miss_the_gradient_bound(model):
    """The per-video comparison can tell videos apart: video 63's gradient against the fp64 gradient with video 62's weights,
    and video 40's against the fp64 gradient of video 41's samples (image, kink pattern, upstream gradient) with video 40's
    weights, each miss GRAD_L2 by at least 10x."""
    from dynaboa_b200 import _lib
    G, B = 64, 64
    _lib.load().dboa_set_tensor_core_conv(3)
    m = model
    arenas = stacked(m, G, 100 * G + 10 + 3)
    x, masks, d = inputs(B, 4000 + B + 3, False)
    _, tape, grad = run(m, arenas, x, masks, d, G)

    def sample(g):
        s = slice(g, g + 1)
        return x[s], [t[s] for t in d], gpu_pattern(tape, B, s)
    margins = {}
    for name, g, weights, rows in (("video 63 on video 62's weights", 63, 62, 63), ("video 40 on video 41's samples", 40, 40, 41)):
        _, l2 = grad_errors(grad[g], frozen_grad(m, arenas[weights], *sample(rows)))
        margins[name] = l2 / GRAD_L2
    for name, g in (('video 63', 63), ('video 40', 40)):                 # the same comparisons, right: within the bound
        _, l2 = grad_errors(grad[g], frozen_grad(m, arenas[g], *sample(g)))
        assert l2 <= GRAD_L2, (name, l2)
    print('\nWIDE negative controls, relative L2 / GRAD_L2: ' + json.dumps({k: f'{r:.3g}' for k, r in margins.items()}))
    assert all(r >= 10 for r in margins.values()), margins


# ------------------------------------------------------------------ 2. masks across all 64 bits
def groups_call(m, arenas, x, d, G):
    """dboa_hmr_forward_groups / dboa_hmr_backward_groups (every video, no mask argument), as ``run``."""
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import ptr, scratch_for, stream, tape_floats
    B = x.shape[0]
    tape = torch.full((tape_floats(B),), float('nan'), device='cuda')
    o = [torch.empty(B, 24, 3, 3, device='cuda'), torch.empty(B, 10, device='cuda'), torch.empty(B, 3, device='cuda'),
         torch.empty(B, 144, device='cuda')]
    grad = torch.zeros_like(arenas)
    bufs = m._buffers
    _lib.call('dboa_hmr_forward_groups', ptr(arenas), ptr(bufs['init_pose']), ptr(bufs['init_shape']), ptr(bufs['init_cam']), ptr(x), B,
              None, ptr(tape), ptr(scratch_for(B, x.device)), *[ptr(t) for t in o], stream(), G)
    _lib.call('dboa_hmr_backward_groups', ptr(arenas), ptr(tape), B, 0, *[ptr(t) for t in d], ptr(grad), ptr(scratch_for(B, x.device)),
              stream(), G)
    torch.cuda.synchronize()
    return o[:3], tape, grad


@pytest.mark.parametrize('mode', [3, 0], ids=['tc3', 'tc0'])
def test_masks_across_all_64_bits(model, mode):
    from dynaboa_b200 import _lib
    G = B = 64
    _lib.load().dboa_set_tensor_core_conv(mode)
    m = model
    arenas = stacked(m, G, 500 + mode)
    x, _, d = inputs(B, 9000 + mode, False)
    ref = run(m, arenas, x, None, d, G, ALL)
    # every bit set is the unmasked entry (all_videos(64) in the library)
    unmasked = groups_call(m, arenas, x, d, G)
    assert not bool(rows_differ(ref, unmasked, B).any())
    assert all(torch.equal(unmasked[2][g], ref[2][g]) for g in range(G))
    del unmasked
    grad = torch.empty_like(arenas)
    for active, name in zip(MASKS, MASK_IDS):
        on = torch.tensor([(active >> g) & 1 for g in range(G)], dtype=torch.bool, device='cuda')
        assert 0 < int(on.sum()) < G, name
        xi, di = x.clone(), [t.clone() for t in d]
        for t in [xi] + di:
            t[~on] = float('nan')
        grad.zero_()
        grad.view(torch.int32)[~on] = SENTINEL
        res = run(m, arenas, xi, None, di, G, active, grad)
        bad = rows_differ(res, ref, B) & on
        assert not bool(bad.any()), (name, bad.nonzero().flatten().tolist()[:8])
        for g in range(G):
            if (active >> g) & 1:
                assert torch.equal(grad[g], ref[2][g]), (name, g)
            else:
                assert bool((grad[g].view(torch.int32) == SENTINEL).all()), (name, g)
        del res


# ------------------------------------------------------------------ 3. isolation and reproducibility at G = 64
def test_videos_are_isolated_and_reproducible_at_64(model):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import tape_views
    G = B = 64
    _lib.load().dboa_set_tensor_core_conv(3)
    m = model
    arenas = stacked(m, G, 1200)
    x, masks, d = inputs(B, 1300, True)
    twins = (0, 31, 32, 63)                      # the same weights and the same samples
    for g in twins[1:]:
        arenas[g] = arenas[0]
        x[g], masks[:, :, g] = x[0], masks[:, :, 0]
        for t in d:
            t[g] = t[0]
    base = run(m, arenas, x, masks, d, G)
    out, tape, grad = base
    v = tape_views(tape, B)
    rows = [bits(t) for t in out] + [bits(t).movedim(sample_axis(key), 0) for key, val in v.items()
                                     for t in (val if isinstance(val, list) else [val]) if t is not None]
    for g in twins[1:]:
        assert all(torch.equal(t[g], t[0]) for t in rows), g
        assert torch.equal(grad[g], grad[0]), g
    del rows
    again = run(m, arenas, x, masks, d, G)
    assert not bool(rows_differ(again, base, B).any()) and torch.equal(again[2], grad)
    del again
    for p in (63, 0):
        keep = arenas[p].clone()
        arenas[p] = stacked(m, 1, 77 + p)[0]
        pert = run(m, arenas, x, masks, d, G)
        arenas[p] = keep
        diff = rows_differ(pert, base, B)
        assert diff.nonzero().flatten().tolist() == [p], p
        for g in range(G):
            assert torch.equal(pert[2][g], grad[g]) != (g == p), (p, g)
        del pert


# ------------------------------------------------------------------ 4. the other grouped entry points at 64 slots
def feature_lengths(b):
    from dynaboa_b200 import _lib
    lib = _lib.load()
    off, nd = C.c_longlong(), C.c_int()
    shp, strd = (C.c_longlong * 4)(), (C.c_longlong * 4)()
    out = []
    for i in range(15):
        _lib.check(lib.dboa_hmr_feature_info(b, i, C.byref(off), C.byref(nd), shp, strd), 'dboa_hmr_feature_info')
        out.append(math.prod(shp[k] for k in range(nd.value)))
    return out


def cosine_terms(A, B, n, G, active, offset=0):
    """dboa_cosine_terms_active over the pairs (A[i], B[i]) of ``G`` parts of n[i] floats each, from part ``offset`` on:
    (G, pairs, 3) fp64 terms, NaN where unwritten."""
    from dynaboa_b200 import _lib
    lib, k = _lib.load(), len(A)
    pa = (C.c_void_p * k)(*[t.data_ptr() + 4 * offset * c for t, c in zip(A, n)])
    pb = (C.c_void_p * k)(*[t.data_ptr() + 4 * offset * c for t, c in zip(B, n)])
    ln = (C.c_longlong * k)(*[G * c for c in n])
    part = torch.full((lib.dboa_cosine_partial_floats_groups(ln, k, G),), float('nan'), device='cuda')
    terms = torch.full((G, k, 3), float('nan'), dtype=torch.float64, device='cuda')
    _lib.call('dboa_cosine_terms_active', pa, pb, ln, k, _lib.ptr(part), part.numel(), _lib.ptr(terms), _lib.stream(), G, active)
    torch.cuda.synchronize()
    return terms


def test_cosine_terms_at_64_videos():
    G = 64
    n = feature_lengths(1)
    gen = torch.Generator(device='cuda').manual_seed(64)
    noise = torch.logspace(-3, 0, G, device='cuda')[:, None]            # 1 - cos from about 5e-7 to 0.5 across the videos
    A = [torch.randn(G, c, device='cuda', generator=gen) for c in n]
    B = [a + noise * torch.randn(a.shape, device='cuda', generator=gen) for a in A]
    A, B = [t.reshape(-1) for t in A], [t.reshape(-1) for t in B]
    one = torch.cat([cosine_terms(A, B, n, 1, 1, g) for g in range(G)])     # each video's parts alone
    rows = []
    for a, b in zip(A, B):
        a, b = a.double().view(G, -1), b.double().view(G, -1)
        rows.append(torch.stack([(a * b).sum(1), (a * a).sum(1), (b * b).sum(1), (a * b).abs().sum(1)], 1))
    t = torch.stack(rows, 1)
    ref, scale = t[..., :3], torch.stack([t[..., 3], t[..., 1], t[..., 2]], -1)

    def one_minus_cos(u):
        return 1.0 - u[..., 0] / (u[..., 1].sqrt().clamp_min(1e-12) * u[..., 2].sqrt().clamp_min(1e-12))
    err = float(((one - ref).abs() / scale).max())
    dcos = float((one_minus_cos(one) - one_minus_cos(ref)).abs().max())
    assert err <= TERMS_TOL and dcos <= COS_TOL, (err, dcos)
    for active, name in zip([ALL] + MASKS, ['all'] + MASK_IDS):
        got = cosine_terms(A, B, n, G, active)
        for g in range(G):
            if (active >> g) & 1:
                assert torch.equal(bits(got[g]), bits(one[g])), (name, g)
            else:
                assert bool(torch.isnan(got[g]).all()), (name, g)
    print(f'\nWIDE cosines G=64 b=1: terms {err:.2e}, 1 - cos {dcos:.2e}')


def metrics(pred, gt, gtn, J, jmap, groups=None, active=None, out=None):
    """dboa_eval_metrics (groups None) or dboa_eval_metrics_active; ``out`` is written in place when given."""
    from dynaboa_b200 import _lib
    B, NV, NJ = pred.shape[0], pred.shape[1], J.shape[0]
    scratch = torch.full((_lib.load().dboa_eval_scratch_floats(B, NJ),), float('nan'), device='cuda')
    out = torch.empty(B, 3, device='cuda') if out is None else out
    args = (_lib.ptr(pred), _lib.ptr(gt), _lib.ptr(gtn), _lib.ptr(J), NJ, NV, _lib.ptr(jmap), jmap.numel(), _lib.ptr(scratch), _lib.ptr(out), B)
    if groups is None:
        _lib.call('dboa_eval_metrics', *args, _lib.stream())
    else:
        _lib.call('dboa_eval_metrics_active', *args, groups, active, _lib.stream())
    torch.cuda.synchronize()
    return out


def test_eval_metrics_at_64_videos(golden):
    G = 64
    jmap = torch.from_numpy(golden('eval_metrics')['joint_map'].astype(np.int32)).cuda()
    rng = np.random.RandomState(64)
    NV, NJ = 6890, 17
    J = (rng.rand(NJ, NV) ** 12).astype(np.float32)
    J /= J.sum(1, keepdims=True)
    gt = (rng.randn(G, NV, 3) * 0.5).astype(np.float32)
    pred = (gt * 1.1 + rng.randn(G, NV, 3) * 0.08).astype(np.float32)
    gtn = (gt + rng.randn(G, NV, 3) * 0.02).astype(np.float32)
    pred, gt, gtn, J = [torch.from_numpy(t).cuda() for t in (pred, gt, gtn, J)]
    one = torch.cat([metrics(pred[g:g + 1].contiguous(), gt[g:g + 1].contiguous(), gtn[g:g + 1].contiguous(), J, jmap) for g in range(G)])
    for active, name in zip([ALL] + MASKS, ['all'] + MASK_IDS):
        ins = [t.clone() for t in (pred, gt, gtn)]
        for g in range(G):
            if not (active >> g) & 1:
                for t in ins:
                    t[g] = float('nan')
        out = torch.empty(G, 3, device='cuda')
        out.view(torch.int32).fill_(SENTINEL)
        metrics(*ins, J, jmap, G, active, out=out)
        for g in range(G):
            if (active >> g) & 1:
                assert torch.equal(bits(out[g]), bits(one[g])), (name, g)
            else:
                assert bool((bits(out[g]) == SENTINEL).all()), (name, g)


def test_keypoints_at_64_streams():
    from dynaboa_b200 import dataprocess as D
    G = 64
    _, centers, scales = scene(G, 81)
    rng = np.random.default_rng(64)
    det = np.concatenate([rng.uniform(-100, 2000, size=(G, 25, 2)), (rng.uniform(0, 1, size=(G, 25, 1)) > 0.3)], 2)
    kp = torch.from_numpy(det).float().cuda()
    for active, name in zip([ALL] + MASKS, ['all'] + MASK_IDS):
        kin = kp.clone()
        for g in range(G):
            if not (active >> g) & 1:
                kin[g] = float('nan')
        out = torch.empty(G, 49, 3, device='cuda')
        out.view(torch.int32).fill_(SENTINEL)
        D.j2d_processing_groups(kin, centers, scales, out, active)
        torch.cuda.synchronize()
        for g in range(G):
            if not (active >> g) & 1:
                assert bool((out[g].view(torch.int32) == SENTINEL).all()), (name, g)
                continue
            assert torch.equal(bits(out[g, :25]), bits(D.j2d_processing(kp[g], centers[g], scales[g]))), (name, g)
            assert bool((out[g, 25:] == 0).all()) and not torch.signbit(out[g, 25:]).any(), (name, g)


def test_crop_at_64_frames_against_the_oracle():
    from dynaboa_b200 import dataprocess as D
    G = 64
    frames, centers, scales = scene(G, 64)
    kinds = [crop_kind(f, c, s) for f, c, s in zip(frames, centers, scales)]
    assert {k[0] for k in kinds} >= {'inside', 'partial', 'outside'} and {k[1] for k in kinds} >= {'up', 'down'}
    assert {f.dtype for f in frames} == {torch.uint8, torch.float32}
    oracle = [crop_oracle(f, c, s) for f, c, s in zip(frames, centers, scales)]
    worst = {}
    for active, name in zip([ALL] + MASKS, ['all'] + MASK_IDS):
        fr = [f if (active >> g) & 1 else torch.full_like(f, float('nan'), dtype=torch.float32) for g, f in enumerate(frames)]
        out = torch.empty(G, 3, 224, 224, device='cuda')
        out.view(torch.int32).fill_(SENTINEL)
        D.crop_groups(fr, centers, scales, out, active)
        torch.cuda.synchronize()
        host = out.cpu().numpy()
        for g in range(G):
            if not (active >> g) & 1:
                assert bool((out[g].view(torch.int32) == SENTINEL).all()), (name, g)
                continue
            err = float(np.abs(host[g] - oracle[g]).max())
            assert err < CROP_TOL, (name, g, kinds[g], str(frames[g].dtype), err)
            key = f'{kinds[g][0]}-{kinds[g][1]}-{str(frames[g].dtype)[6:]}'
            worst[key] = max(worst.get(key, 0.0), err)
    print('\nWIDE crop G=64 against the oracle, worst by kind: ' + json.dumps({k: f'{e:.1e}' for k, e in sorted(worst.items())}))
