"""The loss head (everything after the HMR network in a forward graph) against fp64, at the batches production runs.

SMPL forward and backward (csrc/smpl.cu), the projection, the GMM pose prior, the multi-term head ``dboa_loss_multi`` and
the motion term are each compared with oracle/loss_head_ref.py evaluated in float64 on the GPU's own fp32 inputs, so each
bound is the rounding of one stage: the synthetic SMPL arrays and the prior's fp32 means / precisions / -log weights are
cast to double as shipped, rotations are the GPU's own (rot6d of random 6-vectors, or ``dboa_rodrigues`` kind 0), and the
pose prior is compared at the mixture component the GPU selected.  The calls are the ones ``fused.py`` makes:
``accumulate`` / ``acc_j`` / ``dR_accumulate`` set, ``groups = G`` with per-video means, the prior scaled by ``w / b``,
and the one-video motion pair whose gradient buffers hold 2 nb rows of which the head writes the first nb.

Tapes, scratch and output buffers are filled with NaN (or a sentinel) before each call, so a region a kernel fails to
write fails its check, and accumulating calls are checked bit for bit against ``base + (the overwriting call)``.

Bounds: errors are max |gpu - ref| over the largest |ref| of the quantity (per video where the call is grouped), terms
and prior values relative to themselves.  Each bound is about 3x the worst measured over this file on an H100 80GB HBM3
(power limit 400 W), which is given beside it."""
import json
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {                          # bound         worst measured
    'smpl_verts': 2e-6,          # 7.6e-7 (B = 7)
    'smpl_joints': 1.2e-6,       # 4.3e-7 (B = 16)
    'smpl_dR': 1.4e-6,           # 4.7e-7 (B = 17)
    'smpl_dbeta': 1.3e-6,        # 4.3e-7 (B = 7)
    'proj_p2d': 5e-7,            # 1.7e-7 (B = 64)
    'proj_dj3d': 3e-7,           # 1.1e-7 (B = 9)
    'proj_dcam': 3.8e-7,         # 1.3e-7 (B = 64)
    'prior_value': 7e-7,         # 2.4e-7 (B = 64), also bounds how far above the fp64 minimum the GPU's choice may lie
    'prior_dR': 9e-7,            # 3.0e-7 (B = 64)
    'gmm_value': 6e-7,           # 2.0e-7 (B = 64)
    'gmm_dpose': 7.5e-7,         # 2.6e-7 (B = 1)
    'head_terms': 1.3e-6,        # 4.6e-7 (labelled, G = 64, b = 1)
    'head_dp2d': 4.8e-7,         # 1.6e-7 (teacher, G = 8, b = 8)
    'head_dj3d': 8e-7,           # 2.7e-7 (labelled, G = 64, b = 1)
    'head_dR': 1.2e-6,           # 4.2e-7 (webcam, G = 64, b = 1)
    'head_dbeta': 4.8e-7,        # 1.6e-7 (teacher, G = 64, b = 1)
    'motion_term': 5e-7,         # 1.7e-7 (G = 8)
    'motion_grad': 4.5e-7,       # 1.5e-7 (G = 64)
    'e2e_terms': 4.7e-7,         # 1.6e-7 (grouped level)
    'e2e_dR': 1.4e-6,            # 6.0e-7 (level_backward, one-video pair, b = 9)
    'e2e_dbeta': 1.7e-6,         # 5.7e-7 (grouped level)
    'e2e_dcam': 1.7e-6,          # 6.3e-7 (level_backward, grouped)
}


def report(name, errs):
    print(f'\nERR {name} ' + json.dumps({k: float(f'{v:.3e}') for k, v in errs.items()}))
    bad = {k: v for k, v in errs.items() if not v <= TOL[k]}
    assert not bad, bad


def finite(e):
    """An error that is NaN (a NaN or unwritten output) as +inf.  Every error below passes through here, because Python's
    max() drops NaN (max(0.0, nan) is 0.0) and a NaN would otherwise vanish before it reached its bound."""
    return e if e == e else math.inf


def rel(a, ref, scale=None):
    """max |a - ref| / max |ref|; +inf for any NaN in ``a``."""
    ref = ref.detach().double().cpu()
    s = float(ref.abs().max()) if scale is None else float(scale)
    d = float((a.detach().double().cpu() - ref).abs().max())
    if s == 0.0:
        return 0.0 if d == 0.0 else math.inf
    return finite(d / s)


def per_video(a, ref, G):
    """``rel`` of each video's rows against that video's own largest reference value; the worst video."""
    a, ref = a.detach().double().cpu().reshape(G, -1), ref.detach().double().cpu().reshape(G, -1)
    return max(rel(a[g], ref[g]) for g in range(G))


def rel_each(a, ref):
    """Largest element-wise relative error (an exact zero must be matched exactly); +inf for any NaN in ``a``."""
    a, ref = a.detach().double().cpu().flatten(), ref.detach().double().cpu().flatten()
    nz = ref != 0
    if not bool(torch.equal(a[~nz], ref[~nz])):
        return math.inf
    return finite(float(((a[nz] - ref[nz]).abs() / ref[nz].abs()).max())) if bool(nz.any()) else 0.0


@pytest.fixture(scope='module')
def env():
    from dynaboa_b200 import _lib, constants as K, synthetic
    from dynaboa_b200.prior import MaxMixturePrior
    from dynaboa_b200.smpl import SMPL
    _lib.load()
    body, extra = synthetic.make_smpl_model('neutral'), synthetic.make_extra_regressors()['J_regressor_extra']
    smpl = SMPL(data=body, extra_regressor=extra).cuda()
    prior = MaxMixturePrior(prior_folder=None).cuda()
    model64 = {k: torch.as_tensor(v, dtype=torch.long if k == 'parents' else torch.float64) for k, v in body.items() if k != 'faces'}
    return SimpleNamespace(
        smpl=smpl, prior=prior,
        smpl64=(model64, torch.as_tensor(extra, dtype=torch.float64), torch.tensor(K.JOINT_MAP_49), torch.tensor(K.SMPL_EXTRA_VERTEX_IDS)),
        consts64=(prior.means.double().cpu(), prior.precisions.double().cpu(), prior.neg_log_weights.double().cpu()))


# ------------------------------------------------------------------ GPU calls
def call(name, *args):
    from dynaboa_b200 import _lib
    _lib.call(name, *args, _lib.stream())


def P(t):
    from dynaboa_b200._lib import ptr
    return ptr(t)


def nan(*shape):
    return torch.full(shape, float('nan'), device='cuda')


def rot6d(n, gen):
    """GPU rotation matrices (n, 3, 3) of random 6-vectors, as the network makes them."""
    x = torch.randn(n, 6, generator=gen).cuda()
    R = nan(n, 3, 3)
    call('dboa_rot6d_fwd', P(x), P(R), n)
    return R


def rodrigues(aa):
    """GPU rotation matrices of axis-angles by the reference's quaternion route (kind 0: the exemplar ground truth)."""
    aa = aa.reshape(-1, 3).float().cuda().contiguous()
    R = nan(aa.shape[0], 3, 3)
    call('dboa_rodrigues', P(aa), P(R), aa.shape[0], 0)
    return R


def smpl_forward(env, betas, R):
    from dynaboa_b200 import _lib
    B = betas.shape[0]
    verts, joints, tape = nan(B, 6890, 3), nan(B, 49, 3), nan(_lib.load().dboa_smpl_tape_floats(B))
    call('dboa_smpl_forward', env.smpl._struct_ref(), P(betas), P(R), B, P(verts), P(joints), P(tape))
    return verts, joints, tape


def smpl_backward(env, R, tape, dj, drot, dbeta, accumulate):
    from dynaboa_b200 import _lib
    B = R.shape[0]
    scratch = nan(_lib.load().dboa_smpl_scratch_floats(B))
    call('dboa_smpl_backward', env.smpl._struct_ref(), P(R), B, P(tape), P(dj), P(scratch), P(drot), P(dbeta), accumulate)


def gpu_prior(env, R, drot=None, scale=1.0):
    B = R.shape[0]
    pb = nan(B)
    p = env.prior
    call('dboa_pose_prior', P(R), P(p.means), P(p.precisions), P(p.neg_log_weights), P(pb), P(drot), float(scale), B)
    return pb


def selected(ll, prior_b):
    """The component each body's GPU prior value belongs to: the fp64 component value closest to it."""
    return (ll.detach() - prior_b.double().cpu()[:, None]).abs().argmin(1)


def d64(t, grad=False):
    t = t.detach().double().cpu()
    return t.requires_grad_(True) if grad else t


# ------------------------------------------------------------------ 1. SMPL
@pytest.mark.parametrize('B', [1, 2, 7, 8, 9, 16, 17, 64])
def test_smpl_forward_backward(env, B):
    from oracle import loss_head_ref as ref
    gen = torch.Generator().manual_seed(100 + B)
    betas = torch.randn(B, 10, generator=gen).cuda()
    R = rot6d(B * 24, gen).view(B, 24, 3, 3)
    dj = torch.randn(B, 49, 3, generator=gen).cuda()
    verts, joints, tape = smpl_forward(env, betas, R)
    b64, R64 = d64(betas, True), d64(R, True)
    v64, j64 = ref.smpl(*env.smpl64, b64, R64)
    (j64 * d64(dj)).sum().backward()
    drot, dbeta = torch.full((B, 24, 3, 3), 3.0, device='cuda'), torch.full((B, 10), 3.0, device='cuda')
    smpl_backward(env, R, tape, dj, drot, dbeta, 0)
    # accumulate = 1 on top of a base of the gradient's own size: exactly base + the overwriting call's result
    base_R = torch.randn(B, 24, 3, 3, generator=gen).cuda() * float(R64.grad.abs().max())
    base_b = torch.randn(B, 10, generator=gen).cuda() * float(b64.grad.abs().max())
    acc_R, acc_b = base_R.clone(), base_b.clone()
    smpl_backward(env, R, tape, dj, acc_R, acc_b, 1)
    torch.cuda.synchronize()
    assert torch.equal(acc_R, base_R + drot) and torch.equal(acc_b, base_b + dbeta), 'accumulate = 1'
    report(f'smpl B={B}', {'smpl_verts': rel(verts, v64), 'smpl_joints': rel(joints, j64), 'smpl_dR': rel(drot, R64.grad),
                           'smpl_dbeta': rel(dbeta, b64.grad)})


def test_smpl_batch_invariance(env):
    """Body b of a B = 64 call (8 blend-shape chunks) is bit-identical to a B = 1 call on that body alone."""
    B = 64
    gen = torch.Generator().manual_seed(164)
    betas = torch.randn(B, 10, generator=gen).cuda()
    R = rot6d(B * 24, gen).view(B, 24, 3, 3)
    dj = torch.randn(B, 49, 3, generator=gen).cuda()
    verts, joints, tape = smpl_forward(env, betas, R)
    drot, dbeta = nan(B, 24, 3, 3), nan(B, 10)
    smpl_backward(env, R, tape, dj, drot, dbeta, 0)
    for b in (0, 1, 7, 8, 9, 15, 16, 33, 56, 63):
        s = slice(b, b + 1)
        v1, j1, t1 = smpl_forward(env, betas[s].contiguous(), R[s].contiguous())
        r1, be1 = nan(1, 24, 3, 3), nan(1, 10)
        smpl_backward(env, R[s].contiguous(), t1, dj[s].contiguous(), r1, be1, 0)
        torch.cuda.synchronize()
        assert torch.equal(v1, verts[s]) and torch.equal(j1, joints[s]), f'forward of body {b}'
        assert torch.equal(r1, drot[s]) and torch.equal(be1, dbeta[s]), f'backward of body {b}'


# ------------------------------------------------------------------ 2. projection
@pytest.mark.parametrize('B', [1, 9, 64])
def test_projection(env, B):
    from oracle import loss_head_ref as ref
    gen = torch.Generator().manual_seed(200 + B)
    cam = torch.stack([torch.rand(B, generator=gen) * 0.6 + 0.7, torch.randn(B, generator=gen) * 0.1,
                       torch.randn(B, generator=gen) * 0.1], 1).cuda()
    j3d = (torch.randn(B, 49, 3, generator=gen) * 0.4).cuda()
    dp = torch.randn(B, 49, 2, generator=gen).cuda()
    p2d = nan(B, 49, 2)
    call('dboa_project_fwd', P(cam), P(j3d), P(p2d), B, 49)
    c64, j64 = d64(cam, True), d64(j3d, True)
    p64 = ref.project(c64, j64)
    (p64 * d64(dp)).sum().backward()
    out = {}
    for acc_j in (0, 1):
        for acc_c in (0, 1):
            bj, bc = torch.randn(B, 49, 3, generator=gen).cuda(), torch.randn(B, 3, generator=gen).cuda()
            dj, dc = bj.clone(), bc.clone()
            call('dboa_project_bwd', P(cam), P(j3d), P(dp), P(dj), P(dc), B, 49, acc_j, acc_c)
            out[acc_j, acc_c] = (bj, bc, dj, dc)
    torch.cuda.synchronize()
    _, _, dj0, dc0 = out[0, 0]
    for (acc_j, acc_c), (bj, bc, dj, dc) in out.items():
        assert torch.equal(dj, bj + dj0 if acc_j else dj0), ('dj3d', acc_j, acc_c)
        assert torch.equal(dc, bc + dc0 if acc_c else dc0), ('dcam', acc_j, acc_c)
    report(f'projection B={B}', {'proj_p2d': rel(p2d, p64), 'proj_dj3d': rel(dj0, j64.grad), 'proj_dcam': rel(dc0, c64.grad)})


# ------------------------------------------------------------------ 3. pose prior
ANGLES = (1e-5, 1e-3, math.pi - 1e-3, math.pi - 1e-5, float(np.float32(math.pi)))


def prior_rotations(B, gen):
    """(B, 24, 3, 3) GPU rotations: random ones, and on 20 of the body joints near-identity, near-pi and pi rotations about
    the three coordinate axes and one random axis (the axis-angle conversion's four branches)."""
    R = rot6d(B * 24, gen).view(B, 24, 3, 3).clone()
    axes = torch.cat([torch.eye(3), F.normalize(torch.randn(1, 3, generator=gen), dim=1)])
    special = rodrigues(torch.stack([a * ax for ax in axes for a in ANGLES]))
    slots = [(b, j) for b in range(B) for j in range(1, 24)]
    for i, k in enumerate(torch.randperm(len(slots), generator=gen)[:special.shape[0]].tolist()):
        R[slots[k]] = special[i]
    return R


def asymmetric(P_, gen):
    """The precisions plus an antisymmetric part of 5 % of each matrix's largest entry: the quadratic form's value is
    unchanged, its gradient 0.5 (P + P^T) d is not P d."""
    A = torch.randn(P_.shape, generator=gen).to(P_.device)
    return (P_ + (A - A.transpose(1, 2)) * 0.05 * P_.abs().amax((1, 2), keepdim=True)).contiguous()


@pytest.mark.parametrize('B', [1, 9, 64])
def test_pose_prior_rotations(env, B):
    from oracle import loss_head_ref as ref
    gen = torch.Generator().manual_seed(300 + B)
    R = prior_rotations(B, gen)
    branches = set(ref.r2aa_branch(d64(R[:, 1:])).tolist())
    assert branches == {0, 1, 2, 3}, branches
    means, prec, nlw = env.consts64
    errs = {'prior_value': 0.0, 'prior_dR': 0.0}
    for Pm in (env.prior.precisions, asymmetric(env.prior.precisions, gen)):
        scale = 1e-4 / max(1, B // 8)                  # w / b, as fused._loss_head scales it
        drot = nan(B, 24, 3, 3)
        pb = nan(B)
        call('dboa_pose_prior', P(R), P(env.prior.means), P(Pm), P(env.prior.neg_log_weights), P(pb), P(drot), scale, B)
        torch.cuda.synchronize()
        R64 = d64(R, True)
        ll = ref.prior_components(ref.rotmat_to_aa(R64[:, 1:]).reshape(B, 69), means, d64(Pm), nlw)
        comp = selected(ll, pb)
        sel = ll.gather(1, comp[:, None]).squeeze(1)
        # a near-tie is a choice, not an error: the fp64 minimum lies within fp32 rounding of the chosen component
        tie = finite(float(((sel - ll.min(1)[0]) / sel.abs()).detach().max()))
        (sel.sum() * scale).backward()
        assert bool((drot[:, 0] == 0).all()), 'root joint'
        errs['prior_value'] = max(errs['prior_value'], rel_each(pb, sel), tie)
        errs['prior_dR'] = max(errs['prior_dR'], rel(drot, R64.grad))
    report(f'pose prior B={B}', errs)


@pytest.mark.parametrize('B', [1, 9, 64])
def test_gmm_prior(env, B):
    from oracle import loss_head_ref as ref
    gen = torch.Generator().manual_seed(400 + B)
    pose = (torch.randn(B, 69, generator=gen) * 0.4).cuda()
    means, _, nlw = env.consts64
    errs = {'gmm_value': 0.0, 'gmm_dpose': 0.0}
    for Pm in (env.prior.precisions, asymmetric(env.prior.precisions, gen)):
        pb, dpose = nan(B), nan(B, 69)
        call('dboa_gmm_prior', P(pose), P(env.prior.means), P(Pm), P(env.prior.neg_log_weights), P(pb), P(dpose), 0.7, B)
        torch.cuda.synchronize()
        x64 = d64(pose, True)
        ll = ref.prior_components(x64, means, d64(Pm), nlw)
        sel = ll.gather(1, selected(ll, pb)[:, None]).squeeze(1)
        tie = finite(float(((sel - ll.min(1)[0]) / sel.abs()).detach().max()))
        (sel.sum() * 0.7).backward()
        errs['gmm_value'] = max(errs['gmm_value'], rel_each(pb, sel), tie)
        errs['gmm_dpose'] = max(errs['gmm_dpose'], rel(dpose, x64.grad))
    report(f'gmm prior B={B}', errs)


# ------------------------------------------------------------------ 4. the multi-term head as fused._loss_head issues it
FRAME_W = [10.0, 2e-6, 1e-4, 0, 0, 0, 0, 0]                    # s2dloss, shape prior, pose prior weights
TEACHER_W = FRAME_W[:3] + [0.5, 0.5, 1e-4, 0.1, 0]            # + 5 tw, 5 tw, 0.001 tw, tw with tw = 0.1
LABEL_W = [0.5, 0, 0, 0, 0, 1e-4, 0.1, 0.5]                   # fused.py labelled exemplar head, lw = 0.1
HEADS = {'frame': (FRAME_W, (25, 24)), 'teacher': (TEACHER_W, (25, 24)), 'labelled': (LABEL_W, (25, 24)), 'webcam': (FRAME_W, (0, 25))}
SHAPES = [(G, b) for G in (1, 2, 8) for b in (1, 2, 8, 9)] + [(64, 1)]


def head_inputs(head, B, gen):
    """Network-side tensors (p2d, j3d, R, beta) and the head's keypoints and targets for B rows."""
    t = {'p2d': torch.randn(B, 49, 2, generator=gen) * 0.3, 'j3d': torch.randn(B, 49, 3, generator=gen) * 0.3,
         'beta': torch.randn(B, 10, generator=gen),
         'kp': torch.cat([torch.randn(B, 49, 2, generator=gen) * 0.3, (torch.rand(B, 49, 1, generator=gen) > 0.2).float()], -1)}
    t = {k: v.cuda() for k, v in t.items()}
    t['R'] = rot6d(B * 24, gen).view(B, 24, 3, 3)
    if head == 'teacher':
        t.update(t_p2d=(torch.randn(B, 49, 2, generator=gen) * 0.3).cuda(), t_j3d=(torch.randn(B, 49, 3, generator=gen) * 0.3).cuda(),
                 t_beta=torch.randn(B, 10, generator=gen).cuda(), t_R=rot6d(B * 24, gen).view(B, 24, 3, 3))
    if head == 'labelled':
        t.update(t_beta=torch.randn(B, 10, generator=gen).cuda(), t_R=rodrigues(torch.randn(B * 24, 3, generator=gen) * 0.4).view(B, 24, 3, 3),
                 gt_s3d=torch.cat([torch.randn(B, 24, 3, generator=gen) * 0.3, torch.ones(B, 24, 1)], -1).cuda())
    return t


TARGETS = ('t_p2d', 't_j3d', 't_beta', 't_R', 'gt_s3d')


def run_head(env, head, t, G, nb, rows=None):
    """fused._loss_head on a prediction of ``rows`` rows (default nb) whose first nb are scored, into NaN-filled gradient
    buffers whose rows [nb:] hold a sentinel.  Returns (terms, (dp2d, dj3d, dR, dbeta), sentinels)."""
    from dynaboa_b200 import fused
    w, kp_range = HEADS[head]
    rows = nb if rows is None else rows
    p = SimpleNamespace(p2d=t['p2d'], joints=t['j3d'], rot=t['R'], shape=t['beta'], B=rows, groups=G)
    ad = SimpleNamespace(gmm_f=env.prior, kp_range=kp_range)
    grads = [nan(rows, 49, 2), nan(rows, 49, 3), nan(rows, 24, 3, 3), nan(rows, 10)]
    sentinel = []
    for g in grads:
        g[nb:] = torch.arange(g[nb:].numel(), device='cuda', dtype=torch.float32).view(g[nb:].shape) * 0.25 - 7.0
        sentinel.append(g[nb:].clone())
    kw = {k: t[k][:nb] for k in TARGETS if k in t}
    terms, *out = fused._loss_head(ad, p, w, kp=t['kp'][:nb], grads=grads, nb=nb, **kw)
    torch.cuda.synchronize()
    return terms, out, sentinel


def head_reference(env, head, t, G, nb, pb):
    """fp64 terms (G, 9) and gradients w.r.t. (p2d, j3d, R, beta) of the first nb rows; the pose prior at the GPU's
    components (``pb``: the GPU's per-body prior values)."""
    from oracle import loss_head_ref as ref
    w, kp_range = HEADS[head]
    x = {k: d64(t[k][:nb], True) for k in ('p2d', 'j3d', 'R', 'beta')}
    prior = None
    if w[2] != 0:
        ll = ref.prior_components(ref.rotmat_to_aa(x['R'][:, 1:]).reshape(nb, 69), *env.consts64)
        prior = ll.gather(1, selected(ll, pb)[:, None]).squeeze(1)
    terms = ref.head_terms(G, x['p2d'], x['j3d'], x['R'], x['beta'], w, kp=d64(t['kp'][:nb]), prior=prior, kp_range=kp_range,
                           **{k: d64(t[k][:nb]) for k in TARGETS if k in t})
    terms[:, 8].sum().backward()
    return terms.detach(), [torch.zeros_like(x[k]) if x[k].grad is None else x[k].grad for k in ('p2d', 'j3d', 'R', 'beta')]


@pytest.mark.parametrize('G,b', SHAPES, ids=[f'G{G}-b{b}' for G, b in SHAPES])
@pytest.mark.parametrize('head', list(HEADS))
def test_loss_head(env, head, G, b):
    gen = torch.Generator().manual_seed(500 + 17 * G + b + 1000 * list(HEADS).index(head))
    nb = G * b
    rows = 2 * nb if G == 1 else nb                  # one video: the motion pair's 2 nb-row buffers, the head on rows [:nb]
    t = head_inputs(head, rows, gen)
    terms, grads, sentinel = run_head(env, head, t, G, nb, rows)
    for g, s in zip(grads, sentinel):
        assert torch.equal(g[nb:], s), 'rows [nb:] of the gradient buffers'
    pb = gpu_prior(env, t['R'][:nb].contiguous()) if HEADS[head][0][2] != 0 else None
    ref_terms, ref_grads = head_reference(env, head, t, G, nb, pb)
    term_err = max(rel_each(terms[g, k], ref_terms[g, k]) for g in range(G) for k in range(9))
    errs = {'head_terms': term_err}
    for name, gpu, r in zip(('head_dp2d', 'head_dj3d', 'head_dR', 'head_dbeta'), grads, ref_grads):
        errs[name] = per_video(gpu[:nb], r, G)
    report(f'{head} G={G} b={b}', errs)


@pytest.mark.parametrize('G,b', [(2, 1), (8, 2), (8, 9), (64, 1)], ids=['G2-b1', 'G8-b2', 'G8-b9', 'G64-b1'])
@pytest.mark.parametrize('head', list(HEADS))
def test_loss_head_isolation(env, head, G, b):
    """Video g of a grouped call is bit-identical to a groups = 1 call on its rows alone, with NaN in every other video's
    inputs and with finite ones."""
    gen = torch.Generator().manual_seed(600 + G + b)
    nb = G * b
    t = head_inputs(head, nb, gen)
    terms, grads, _ = run_head(env, head, t, G, nb)
    for g in sorted({0, G // 2, G - 1}):
        s = slice(g * b, (g + 1) * b)
        alone = {k: v[s].contiguous() for k, v in t.items()}
        t1, g1, _ = run_head(env, head, alone, 1, b)
        poisoned = {k: torch.full_like(v, float('nan')) for k, v in t.items()}
        for k in poisoned:
            poisoned[k][s] = t[k][s]
        tn, gn, _ = run_head(env, head, poisoned, G, nb)
        assert torch.equal(terms[g], t1[0]) and torch.equal(tn[g], t1[0]), (g, terms[g], t1[0], tn[g])
        for a, one, pz in zip(grads, g1, gn):
            assert torch.equal(a[s], one) and torch.equal(pz[s], one), g


# ------------------------------------------------------------------ 5. motion term
def motion_inputs(B, gen):
    pa, ph = (torch.randn(B, 49, 2, generator=gen) * 0.3).cuda(), (torch.randn(B, 49, 2, generator=gen) * 0.3).cuda()
    ka = torch.cat([torch.randn(B, 49, 2, generator=gen) * 0.3, (torch.rand(B, 49, 1, generator=gen) > 0.3).float()], -1).cuda()
    kh = torch.cat([torch.randn(B, 49, 2, generator=gen) * 0.3, (torch.rand(B, 49, 1, generator=gen) > 0.3).float()], -1).cuda()
    return pa, ph, ka, kh


@pytest.mark.parametrize('G', [1, 8, 64])
def test_motion(env, G):
    from oracle import loss_head_ref as ref
    b, w = 2, 0.8
    B = G * b
    gen = torch.Generator().manual_seed(700 + G)
    pa, ph, ka, kh = motion_inputs(B, gen)
    base = torch.randn(B, 49, 2, generator=gen).cuda()
    active = {1: 1, 8: 0b10110010, 64: 0x9C3E00F0A5A50F61}[G]
    errs = {'motion_term': 0.0, 'motion_grad': 0.0}
    for first, count in ((25, 24), (0, 25)):
        a64, h64 = d64(pa, True), d64(ph, True)
        m64 = ref.motion_terms(G, a64, h64, d64(ka), d64(kh), first, count)
        (w * m64.sum()).backward()
        runs = {}
        for kind in ('groups', 'active', 'joints'):
            if kind == 'joints' and G != 1:
                continue
            for acc in (0, 1):
                term, dpa, dph = nan(G), base.clone(), torch.full_like(pa, 7.0)
                args = (P(pa), P(ph), P(ka), P(kh), w, P(term), P(dpa), P(dph), B, acc, first, count)
                if kind == 'groups':
                    call('dboa_loss_motion_groups', *args, G)
                elif kind == 'active':
                    call('dboa_loss_motion_active', *args, G, active)
                else:
                    call('dboa_loss_motion_joints', *args)
                runs[kind, acc] = (term, dpa, dph)
        torch.cuda.synchronize()
        t0, a0, h0 = runs['groups', 0]
        errs['motion_term'] = max(errs['motion_term'], rel_each(t0, m64))
        errs['motion_grad'] = max(errs['motion_grad'], per_video(a0, a64.grad, G), per_video(h0, h64.grad, G))
        for (kind, acc), (term, dpa, dph) in runs.items():
            for g in range(G):
                s = slice(g * b, (g + 1) * b)
                if kind == 'active' and not (active >> g) & 1:
                    assert float(term[g]) == 0.0 and torch.equal(dpa[s], base[s]) and bool((dph[s] == 7.0).all()), (kind, acc, g)
                    continue
                assert torch.equal(term[g], t0[g]), (kind, acc, g)
                assert torch.equal(dpa[s], base[s] + a0[s] if acc else a0[s]) and torch.equal(dph[s], h0[s]), (kind, acc, g)
    report(f'motion G={G}', errs)


# ------------------------------------------------------------------ 6. the production composition
def make_pred(env, B, G, gen, active=None):
    """A fused._Pred from random network outputs (GPU rot6d rotations, shapes, cameras), through fused._smpl_fwd and
    dboa_project_fwd as fused.forward_graph runs them, without the network."""
    from dynaboa_b200 import fused
    p = fused._Pred()
    p.rot = rot6d(B * 24, gen).view(B, 24, 3, 3)
    p.shape = (torch.randn(B, 10, generator=gen) * 0.5).cuda()
    p.cam = torch.stack([torch.rand(B, generator=gen) * 0.5 + 0.7, torch.randn(B, generator=gen) * 0.1,
                         torch.randn(B, generator=gen) * 0.1], 1).cuda()
    p.B, p.groups, p.active, p.masked, p.tape, p.image = B, G, active, False, None, None
    p.verts, p.joints, p.smpl_tape = fused._smpl_fwd(env.smpl, p.shape, p.rot)
    p.p2d = nan(B, 49, 2)
    call('dboa_project_fwd', P(p.cam), P(p.joints), P(p.p2d), B, 49)
    return p


def capture_backward(monkeypatch):
    """Replaces the network backward with a recorder of the (dR, dbeta, dcam) fused.backward_graph hands it."""
    from dynaboa_b200 import fused
    got = []

    def raw_backward(arena, tape, B, masked, dR, dbeta, dcam, grad_arena, groups=1, active=None):
        got.append((dR.clone(), dbeta.clone(), dcam.clone()))
    monkeypatch.setattr(fused.hmr_mod, 'raw_backward', raw_backward)
    return got


def level_reference(env, preds, G, nb, kp, hist_kp, targets, w, wm, live, pb):
    """fp64 autograd of the level loss sum_g [head_g + wm * motion_g (g live)] w.r.t. (R, beta, cam) of every prediction;
    ``preds``: [main] with the history frame in rows [nb:] of main, or [main, hist]."""
    from oracle import loss_head_ref as ref
    xs = [{k: d64(getattr(p, k), True) for k in ('rot', 'shape', 'cam')} for p in preds]
    p2d, j3d = [], []
    for x in xs:
        _, j = ref.smpl(*env.smpl64, x['shape'], x['rot'])
        j3d.append(j)
        p2d.append(ref.project(x['cam'], j))
    m = xs[0]
    ll = ref.prior_components(ref.rotmat_to_aa(m['rot'][:nb, 1:]).reshape(nb, 69), *env.consts64)
    prior = ll.gather(1, selected(ll, pb)[:, None]).squeeze(1)
    terms = ref.head_terms(G, p2d[0][:nb], j3d[0][:nb], m['rot'][:nb], m['shape'][:nb], w, kp=d64(kp), prior=prior,
                           **{k: d64(v) for k, v in targets.items()})
    hist_p2d = p2d[0][nb:] if len(preds) == 1 else p2d[1]
    motion = ref.motion_terms(G, p2d[0][:nb], hist_p2d, d64(kp), d64(hist_kp)) * torch.tensor([float((live >> g) & 1) for g in range(G)],
                                                                                                dtype=torch.float64)
    (terms[:, 8].sum() + wm * motion.sum()).backward()
    return terms.detach(), motion.detach(), [[x['rot'].grad, x['shape'].grad, x['cam'].grad] for x in xs]




E2E = ('e2e_dR', 'e2e_dbeta', 'e2e_dcam')


def level_errors(terms, mterm, ref_terms, ref_motion, pairs):
    """Errors of a level: its terms and motion terms element-wise, and per video the (dR, dbeta, dcam) handed to each
    network backward.  ``pairs``: (captured gradients, fp64 gradients, rows compared (None: all), videos among them)."""
    errs = {'e2e_terms': max(rel_each(terms, ref_terms), rel_each(mterm, ref_motion))}
    errs.update(dict.fromkeys(E2E, 0.0))
    for gpu, ref, rows, n in pairs:
        for name, a, r in zip(E2E, gpu, ref):
            if rows is not None:
                a, r = a[rows.cuda()], r[rows]
            errs[name] = max(errs[name], per_video(a, r, n))
    return errs


def live_rows(live, G, b):
    """Rows of the videos whose motion term is live (an idle video's history rows are never read by the network)."""
    on = [g for g in range(G) if (live >> g) & 1]
    return torch.tensor([g * b + i for g in on for i in range(b)]), len(on)


@pytest.mark.parametrize('nb', [1, 9])
def test_level_one_video_motion_pair(env, nb, monkeypatch):
    """One video: frame + teacher head on rows [:nb] of a 2 nb-row prediction whose rows [nb:] are the history frame, the
    motion term between them, one backward_graph over all 2 nb rows.  This restates fused.level_backward's batched
    sequence call by call; test_level_backward runs level_backward itself."""
    from dynaboa_b200 import fused
    gen = torch.Generator().manual_seed(800 + nb)
    B2, wm = 2 * nb, 0.8
    main = make_pred(env, B2, 1, gen)
    kp = head_inputs('frame', nb, gen)['kp']
    hist_kp = head_inputs('frame', nb, gen)['kp']
    tg = head_inputs('teacher', nb, gen)
    targets = {k: tg[k] for k in ('t_p2d', 't_j3d', 't_beta', 't_R')}
    ad = SimpleNamespace(smpl_neutral=env.smpl, gmm_f=env.prior, kp_range=(25, 24))
    grads = (torch.zeros(B2, 49, 2, device='cuda'), torch.zeros(B2, 49, 3, device='cuda'), torch.zeros(B2, 24, 3, 3, device='cuda'),
             torch.zeros(B2, 10, device='cuda'))
    terms, dp2d, dj3d, dR, dbeta = fused._loss_head(ad, main, TEACHER_W, kp=kp, grads=grads, nb=nb, **targets)
    mterm = nan(1)
    call('dboa_loss_motion_groups', P(main.p2d), P(main.p2d[nb:]), P(kp), P(hist_kp), wm, P(mterm), P(dp2d), P(dp2d[nb:]), nb, 1, 25, 24, 1)
    got = capture_backward(monkeypatch)
    fused.backward_graph(ad, None, main, dp2d, dj3d, dR, dbeta, None)
    torch.cuda.synchronize()
    assert len(got) == 1
    pb = gpu_prior(env, main.rot[:nb].contiguous())
    ref_terms, ref_motion, refs = level_reference(env, [main], 1, nb, kp, hist_kp, targets, TEACHER_W, wm, 1, pb)
    report(f'level pair nb={nb}', level_errors(terms, mterm, ref_terms, ref_motion, [(got[0], refs[0], None, 1)]))


def test_level_grouped_partial_live(env, monkeypatch):
    """Eight videos of two rows: frame + teacher head, the motion term of the live videos only against a separate history
    forward (dboa_loss_motion_active), the history backward and the main backward.  This restates fused.level_backward's
    grouped sequence call by call; test_level_backward runs level_backward itself."""
    from dynaboa_b200 import fused
    G, b, wm, live = 8, 2, 0.8, 0b01101001
    nb = G * b
    gen = torch.Generator().manual_seed(900)
    main = make_pred(env, nb, G, gen)
    hist = make_pred(env, nb, G, gen, active=live)
    kp = head_inputs('frame', nb, gen)['kp']
    hist_kp = head_inputs('frame', nb, gen)['kp']
    tg = head_inputs('teacher', nb, gen)
    targets = {k: tg[k] for k in ('t_p2d', 't_j3d', 't_beta', 't_R')}
    ad = SimpleNamespace(smpl_neutral=env.smpl, gmm_f=env.prior, kp_range=(25, 24))
    terms, dp2d, dj3d, dR, dbeta = fused._loss_head(ad, main, TEACHER_W, kp=kp, **targets)
    mterm, dph = nan(G), nan(nb, 49, 2)
    call('dboa_loss_motion_active', P(main.p2d), P(hist.p2d), P(kp), P(hist_kp), wm, P(mterm), P(dp2d), P(dph), nb, 1, 25, 24, G, live)
    got = capture_backward(monkeypatch)
    fused.backward_graph(ad, None, hist, dph, torch.zeros_like(hist.joints), torch.zeros_like(hist.rot), torch.zeros_like(hist.shape), None)
    fused.backward_graph(ad, None, main, dp2d, dj3d, dR, dbeta, None)
    torch.cuda.synchronize()
    assert len(got) == 2                                            # [history, main]
    pb = gpu_prior(env, main.rot)
    ref_terms, ref_motion, refs = level_reference(env, [main, hist], G, nb, kp, hist_kp, targets, TEACHER_W, wm, live, pb)
    rows, n_live = live_rows(live, G, b)
    report('level grouped G=8 b=2', level_errors(terms, mterm, ref_terms, ref_motion,
                                                 [(got[1], refs[0], None, G), (got[0], refs[1], rows, n_live)]))


class _Teacher:
    """The mean teacher as fused.level_backward reads it: weights and buffers (used only as keys here), no dropout."""

    def __init__(self, arena):
        self.arena, self._buffers = arena, None

    def _masks(self, B, device):
        return None


def fake_network(monkeypatch, outputs):
    """Replaces the network forward: ``outputs[arena.data_ptr()][key]`` is the (rot, shape, cam) of the image row whose
    pixel [0, 0, 0] holds ``key``, so a row keeps its outputs wherever level_backward stages it (the motion pair included)."""
    from dynaboa_b200 import fused

    def raw_forward(arena, buffers, image, masks=None, tape=None, groups=1, active=None):
        table = outputs[arena.data_ptr()]
        rows = [table[int(k)] for k in image[:, 0, 0, 0].tolist()]
        rot, shape, cam = (torch.stack([r[i] for r in rows]).contiguous() for i in range(3))
        return rot, shape, cam, None, torch.zeros(1, device=image.device)
    monkeypatch.setattr(fused.hmr_mod, 'raw_forward', raw_forward)


@pytest.mark.parametrize('G,b,live', [(1, 1, 1), (1, 9, 1), (8, 2, 0b01101001)], ids=['pair-b1', 'pair-b9', 'G8-b2-partial'])
def test_level_backward(env, G, b, live, monkeypatch):
    """fused.level_backward itself (upper level: frame + teacher + motion, no retrieval) with only the network replaced:
    its staging of the one-video motion pair or the grouped history forward, its motion call (accumulation, history
    gradient, live mask) and its backward calls, against fp64 autograd of the level loss w.r.t. every network output."""
    from dynaboa_b200 import fused
    from oracle import adaptor_ref
    gen = torch.Generator().manual_seed(1000 + 10 * G + b)
    nb = G * b
    arena = torch.zeros((G, 1) if G > 1 else (1,), device='cuda')
    t_arena = torch.zeros_like(arena)
    cur, hist, teach = (make_pred(env, nb, G, gen) for _ in range(3))
    outputs = {arena.data_ptr(): {}, t_arena.data_ptr(): {}}
    image, hist_image = torch.zeros(nb, 3, 224, 224, device='cuda'), torch.zeros(nb, 3, 224, 224, device='cuda')
    for i in range(nb):
        image[i, 0, 0, 0], hist_image[i, 0, 0, 0] = i, 100 + i
        outputs[arena.data_ptr()][i] = (cur.rot[i], cur.shape[i], cur.cam[i])
        outputs[arena.data_ptr()][100 + i] = (hist.rot[i], hist.shape[i], hist.cam[i])
        outputs[t_arena.data_ptr()][i] = (teach.rot[i], teach.shape[i], teach.cam[i])
    kp = head_inputs('frame', nb, gen)['kp']
    hist_kp = head_inputs('frame', nb, gen)['kp']
    o = adaptor_ref.default_options(retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0)
    ad = SimpleNamespace(options=o, smpl_neutral=env.smpl, gmm_f=env.prior, kp_range=(25, 24), teacher=_Teacher(t_arena),
                         global_step=o.interval + 1, motion_active=live if G > 1 else None, fit_losses={}, kp2dlosses_lower=[],
                         kp2dlosses_upper={}, get_hist=lambda: (hist_image, hist_kp))
    fake_network(monkeypatch, outputs)
    got = capture_backward(monkeypatch)
    total, _ = fused.level_backward(ad, arena, None, image, kp, False, None)
    torch.cuda.synchronize()
    # the teacher's targets are its forward through the same (deterministic) SMPL and projection kernels
    targets = dict(t_p2d=teach.p2d, t_j3d=teach.joints, t_beta=teach.shape, t_R=teach.rot)
    pb = gpu_prior(env, cur.rot)
    wm = o.motionloss_weight
    if G == 1:
        assert len(got) == 1                                        # one backward over the 2 nb-row pair
        pair = SimpleNamespace(**{k: torch.cat([getattr(cur, k), getattr(hist, k)]) for k in ('rot', 'shape', 'cam')})
        ref_terms, ref_motion, refs = level_reference(env, [pair], 1, nb, kp, hist_kp, targets, TEACHER_W, wm, live, pb)
        pairs = [(got[0], refs[0], None, 1)]
    else:
        assert len(got) == 2                                        # [history, main]
        ref_terms, ref_motion, refs = level_reference(env, [cur, hist], G, nb, kp, hist_kp, targets, TEACHER_W, wm, live, pb)
        rows, n_live = live_rows(live, G, b)
        pairs = [(got[1], refs[0], None, G), (got[0], refs[1], rows, n_live)]
    errs = level_errors(total, ad.fit_losses['ul/motion_loss'], ref_terms[:, 8] + wm * ref_motion, ref_motion, pairs)
    report(f'level_backward G={G} b={b}', errs)


def test_error_measures_keep_nan():
    """A NaN output fails its bound however the errors are combined: an unwritten gradient, or one video of several."""
    ref = torch.randn(2, 24, 3, 3, dtype=torch.float64)
    drot = ref.clone()
    drot[:, 1:] = float('nan')
    drot[:, 0] = 0.0
    assert rel(drot, ref) == math.inf and max(0.0, rel(drot, ref)) == math.inf
    video1 = ref.clone()
    video1[1] = float('nan')
    assert per_video(video1, ref, 2) == math.inf and rel_each(video1, ref) == math.inf
    with pytest.raises(AssertionError):
        report('nan', {'prior_dR': max(0.0, rel(drot, ref)), 'head_dR': per_video(video1, ref, 2)})
