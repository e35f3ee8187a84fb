"""Per-kernel parity of libdynaboa_b200 (through the C ABI) against the CPU oracle on seeded inputs.
Tolerances are relative to the largest reference magnitude; fp32 kernels with a different summation
order than torch's CPU kernels are expected to agree to ~1e-5, the bar of the north star is 1e-3."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    _lib.load()
    return _lib


def dev(t):
    return t.cuda().contiguous()


def ohwi(w, pitch=None):
    """(O,I,kh,kw) -> [O][kh*kw*I] rows with optional zero-padded pitch."""
    O, I, kh, kw = w.shape
    m = w.permute(0, 2, 3, 1).reshape(O, kh * kw * I)
    K = m.shape[1]
    pitch = pitch or (K + 15) // 16 * 16
    out = torch.zeros(O, pitch)
    out[:, :K] = m
    return out, pitch


CONV_CASES = [  # B, H, Cin, Cout, k, stride, pad
    (1, 224, 3, 64, 7, 2, 3),      # stem (scalar gather path, padded pitch; row-per-CTA weight gradient)
    (3, 224, 3, 64, 7, 2, 3),      # stem, several output rows per CTA
    (2, 56, 64, 64, 1, 1, 0),
    (1, 56, 64, 64, 3, 1, 1),
    (2, 28, 128, 128, 3, 2, 1),    # stride-2 3x3
    (1, 56, 256, 512, 1, 2, 0),    # stride-2 downsample
    (1, 7, 512, 512, 3, 1, 1),     # small M, long K -> split-K
    (3, 7, 2048, 512, 1, 1, 0),
    (1, 14, 256, 1024, 1, 1, 0),
]


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_fwd_dgrad_wgrad(L, case):
    B, H, Cin, Cout, k, s, p = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x = torch.randn(B, Cin, H, H, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (k * k * Cin) ** 0.5
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = F.conv2d(xr, wr, stride=s, padding=p)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    Ho = y.shape[2]
    wm, pitch = ohwi(w)
    xd, wd = dev(x.permute(0, 2, 3, 1)), dev(wm)
    ws = torch.empty(8 << 20, device='cuda')
    yd = torch.empty(B, Ho, Ho, Cout, device='cuda')
    L.call('dboa_conv2d_fwd', L.ptr(xd), L.ptr(wd), L.ptr(yd), B, H, H, Cin, Cout, k, s, p, pitch, L.ptr(ws), ws.numel(), L.stream())
    assert rel_err(yd.permute(0, 3, 1, 2), y.detach()) < 2e-5
    dyd = dev(dy.permute(0, 2, 3, 1))
    # weight gradient accumulates into an existing buffer
    base = torch.randn(Cout, pitch, generator=g) * 0.1
    base[:, k * k * Cin:] = 0
    dwd = dev(base)
    L.call('dboa_conv2d_wgrad', L.ptr(dyd), L.ptr(xd), L.ptr(dwd), B, H, H, Cin, Cout, k, s, p, pitch, L.ptr(ws), ws.numel(), L.stream())
    ref_dw, _ = ohwi(wr.grad, pitch)
    assert rel_err(dwd.cpu() - base, ref_dw) < 5e-5
    if Cin % 64 == 0:
        for acc in (0, 1):
            basex = torch.randn(B, H, H, Cin, generator=g)
            dxd = dev(basex)
            L.call('dboa_conv2d_dgrad', L.ptr(dyd), L.ptr(wd), L.ptr(dxd), B, H, H, Cin, Cout, k, s, p, pitch, acc, L.ptr(ws), ws.numel(),
                   L.stream())
            got = dxd.cpu() - (basex if acc else 0)
            assert rel_err(got.permute(0, 3, 1, 2), xr.grad) < 5e-5


@pytest.mark.parametrize('shape', [(2, 112, 64), (1, 56, 256), (3, 14, 1024), (2, 7, 2048), (1, 28, 128), (1, 56, 64), (1, 14, 256), (1, 7, 512)])
@pytest.mark.parametrize('with_res', [False, True])
def test_groupnorm_fwd_bwd(L, shape, with_res):
    B, H, Cc = shape
    g = torch.Generator().manual_seed(B * 1000 + H + Cc)
    y = torch.randn(B, Cc, H, H, generator=g) * 1.7 + 0.6
    gamma, beta = torch.randn(Cc, generator=g) * 0.3 + 1, torch.randn(Cc, generator=g) * 0.2
    res = torch.randn(B, Cc, H, H, generator=g) if with_res else None
    yr, gr, br = y.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    z = F.group_norm(yr, 4, gr, br, 1e-5)
    out = F.relu(z + res) if with_res else F.relu(z)
    dout = torch.randn(out.shape, generator=g)
    out.backward(dout)
    HW = H * H
    yd = dev(y.permute(0, 2, 3, 1))
    resd = dev(res.permute(0, 2, 3, 1)) if with_res else None
    gammad, betad, doutd = dev(gamma), dev(beta), dev(dout.permute(0, 2, 3, 1))
    outd = torch.empty_like(yd)
    stats = torch.empty(B * 8, device='cuda')
    part = torch.empty(L.load().dboa_gn_partial_floats(B, HW, Cc), device='cuda')
    L.call('dboa_groupnorm_fwd', L.ptr(yd), L.ptr(gammad), L.ptr(betad), L.ptr(resd), L.ptr(outd), L.ptr(stats), L.ptr(part),
           B, HW, Cc, 1, L.stream())
    assert rel_err(outd.permute(0, 3, 1, 2), out.detach()) < 2e-5
    dyd = torch.empty_like(yd)
    dgam, dbet = torch.ones(Cc, device='cuda'), torch.ones(Cc, device='cuda')       # accumulate semantics
    bpart = torch.empty(L.load().dboa_gn_bwd_partial_floats(B, HW, Cc), device='cuda')
    L.call('dboa_groupnorm_bwd', L.ptr(doutd), L.ptr(outd), L.ptr(yd), L.ptr(stats), L.ptr(gammad),
           L.ptr(dyd), L.ptr(dgam), L.ptr(dbet), L.ptr(bpart), B, HW, Cc, L.stream())
    assert rel_err(dyd.permute(0, 3, 1, 2), yr.grad) < 1e-4
    assert rel_err(dgam.cpu() - 1, gr.grad) < 1e-4 and rel_err(dbet.cpu() - 1, br.grad) < 1e-4


def test_maxpool(L):
    g = torch.Generator().manual_seed(7)
    x = F.relu(torch.randn(2, 64, 112, 112, generator=g))
    xr = x.clone().requires_grad_(True)
    y = F.max_pool2d(xr, 3, 2, 1)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    xd = dev(x.permute(0, 2, 3, 1))
    yd = torch.empty(2, 56, 56, 64, device='cuda')
    idx = torch.empty(2 * 56 * 56 * 64, dtype=torch.uint8, device='cuda')
    L.call('dboa_maxpool_fwd', L.ptr(xd), L.ptr(yd), L.ptr(idx), 2, 112, 112, 64, L.stream())
    assert torch.equal(yd.permute(0, 3, 1, 2).cpu(), y.detach())
    dxd = torch.empty_like(xd)
    dyd = dev(dy.permute(0, 2, 3, 1))
    L.call('dboa_maxpool_bwd', L.ptr(dyd), L.ptr(idx), L.ptr(dxd), 2, 112, 112, 64, L.stream())
    # ties only occur between zeros, whose gradient the preceding ReLU discards: compare where x > 0
    m = (x > 0)
    assert rel_err(dxd.permute(0, 3, 1, 2).cpu() * m, xr.grad * m) < 1e-6


def test_rotations_against_golden(L, golden):
    gd = golden('geometry')
    x6 = torch.from_numpy(gd['rot6d_in'])
    x6d = dev(x6)
    R = torch.empty(x6.shape[0], 3, 3, device='cuda')
    L.call('dboa_rot6d_fwd', L.ptr(x6d), L.ptr(R), x6.shape[0], L.stream())
    assert rel_err(R, gd['rot6d_out']) < 1e-6
    aa = torch.from_numpy(gd['rodrigues_in'])
    R = torch.empty(aa.shape[0], 3, 3, device='cuda')
    aad = dev(aa)
    L.call('dboa_rodrigues', L.ptr(aad), L.ptr(R), aa.shape[0], 0, L.stream())
    assert rel_err(R, gd['rodrigues_out']) < 2e-6
    Rin = torch.from_numpy(gd['r2aa_in'])
    out = torch.empty(Rin.shape[0], 3, device='cuda')
    Rind, wd = dev(Rin), dev(torch.from_numpy(gd['r2aa_w']))
    L.call('dboa_rotmat_to_aa_fwd', L.ptr(Rind), L.ptr(out), Rin.shape[0], L.stream())
    assert rel_err(out, gd['r2aa_out']) < 2e-6
    dR = torch.empty(Rin.shape[0], 3, 3, device='cuda')
    L.call('dboa_rotmat_to_aa_bwd', L.ptr(Rind), L.ptr(wd), L.ptr(dR), Rin.shape[0], L.stream())
    assert rel_err(dR, gd['r2aa_grad']) < 1e-5
    p = torch.empty(4, 49, 2, device='cuda')
    camd, ptsd = dev(torch.from_numpy(gd['proj_cam'])), dev(torch.from_numpy(gd['proj_pts']))
    L.call('dboa_project_fwd', L.ptr(camd), L.ptr(ptsd), L.ptr(p), 4, 49, L.stream())
    assert rel_err(p, gd['proj_out']) < 1e-6


def test_python_geometry_functions_autograd(L):
    from dynaboa_b200 import geometry
    from oracle import geometry_ref as G
    g = torch.Generator().manual_seed(11)
    x = torch.randn(48, 6, generator=g)
    w = torch.randn(48, 3, 3, generator=g)
    xc = x.clone().requires_grad_(True)
    (G.rot6d_to_rotmat(xc) * w).sum().backward()
    xg = x.cuda().requires_grad_(True)
    (geometry.rot6d_to_rotmat(xg) * w.cuda()).sum().backward()
    assert rel_err(xg.grad, xc.grad) < 1e-5
    R = G.batch_rodrigues(torch.randn(46, 3, generator=g))
    wa = torch.randn(46, 3, generator=g)
    Rc = R.clone().requires_grad_(True)
    (G.rotation_matrix_to_angle_axis(Rc) * wa).sum().backward()
    Rg = R.cuda().requires_grad_(True)
    (geometry.rotation_matrix_to_angle_axis(Rg) * wa.cuda()).sum().backward()
    assert rel_err(Rg.grad, Rc.grad) < 1e-5
    assert rel_err(geometry.batch_rodrigues(wa.cuda()), G.batch_rodrigues(wa)) < 2e-6


def test_gmm_prior_against_golden(L, golden):
    from dynaboa_b200.prior import MaxMixturePrior
    gd = golden('prior')
    prior = MaxMixturePrior().cuda()
    assert rel_err(prior.neg_log_weights[1:], gd['neg_log_w'].reshape(-1)[1:]) < 1e-6
    pose = torch.from_numpy(gd['pose']).cuda().requires_grad_(True)
    out = prior(pose, None)
    out.sum().backward()
    assert rel_err(out, gd['nll']) < 1e-5
    assert rel_err(pose.grad, gd['grad']) < 1e-4


def _smpl_models():
    from dynaboa_b200 import constants as K, synthetic
    from dynaboa_b200.smpl import SMPL
    body, ex = synthetic.make_smpl_model('neutral'), synthetic.make_extra_regressors()
    ours = SMPL(data=body, extra_regressor=ex['J_regressor_extra']).cuda()
    m = {k: (torch.as_tensor(v, dtype=torch.long) if k == 'parents' else torch.as_tensor(v)) for k, v in body.items() if k != 'faces'}
    return ours, m, torch.as_tensor(ex['J_regressor_extra']), torch.tensor(K.JOINT_MAP_49), torch.tensor(K.SMPL_EXTRA_VERTEX_IDS)


def test_smpl_forward_backward(L, golden):
    from oracle import smplx_ref
    ours, m, Jx, jm, vid = _smpl_models()
    gd = golden('smpl')
    betas, R = torch.from_numpy(gd['betas']), torch.from_numpy(gd['rotmat'])
    out = ours(betas=betas.cuda(), body_pose=R[:, 1:].cuda(), global_orient=R[:, :1].cuda(), pose2rot=False)
    assert rel_err(out.vertices, gd['vertices']) < 1e-5 and rel_err(out.joints, gd['joints']) < 1e-5
    aa = torch.from_numpy(gd['aa'])
    out_aa = ours(betas=betas.cuda(), body_pose=aa[:, 3:].cuda(), global_orient=aa[:, :3].cuda(), pose2rot=True)
    assert rel_err(out_aa.vertices, gd['vertices_aa']) < 1e-5 and rel_err(out_aa.joints, gd['joints_aa']) < 1e-5
    # gradients of a random functional of the joints w.r.t. betas and rotations
    g = torch.Generator().manual_seed(9)
    wj = torch.randn(3, 49, 3, generator=g)
    bc, Rc = betas.clone().requires_grad_(True), R.clone().requires_grad_(True)
    ref = smplx_ref.smpl_forward(m, Jx, jm, vid, bc, Rc[:, 1:], Rc[:, :1], pose2rot=False)
    (ref.joints * wj).sum().backward()
    bg, Rg = betas.cuda().requires_grad_(True), R.cuda().requires_grad_(True)
    o = ours(betas=bg, body_pose=Rg[:, 1:], global_orient=Rg[:, :1], pose2rot=False)
    (o.joints * wj.cuda()).sum().backward()
    assert rel_err(bg.grad, bc.grad) < 1e-4 and rel_err(Rg.grad, Rc.grad) < 1e-4


def test_loss_heads(L):
    from dynaboa_b200 import losses
    from dynaboa_b200.prior import MaxMixturePrior
    from oracle import adaptor_ref, geometry_ref as G, prior_ref
    import os
    B = 3
    g = torch.Generator().manual_seed(21)
    p2d = torch.randn(B, 49, 2, generator=g) * 0.3
    j3d = torch.randn(B, 49, 3, generator=g) * 0.3
    R = G.batch_rodrigues(torch.randn(B * 24, 3, generator=g) * 0.4).view(B, 24, 3, 3)
    beta = torch.randn(B, 10, generator=g)
    kp = torch.cat([torch.randn(B, 49, 2, generator=g) * 0.3, (torch.rand(B, 49, 1, generator=g) > 0.2).float()], -1)
    t_p2d, t_j3d = torch.randn(B, 49, 2, generator=g) * 0.3, torch.randn(B, 49, 3, generator=g) * 0.3
    t_beta, t_R = torch.randn(B, 10, generator=g), G.batch_rodrigues(torch.randn(B * 24, 3, generator=g) * 0.4).view(B, 24, 3, 3)
    gt_s3d = torch.cat([torch.randn(B, 24, 3, generator=g) * 0.3, torch.ones(B, 24, 1)], -1)
    w = [10.0, 2e-3, 1e-2, 5.0, 5.0, 0.001, 1.0, 5.0]
    from dynaboa_b200 import config
    consts = prior_ref.gmm_constants(dict(np.load(config.GMM_PRIOR)))

    def ref_total(p2d, j3d, R, beta):
        conf = kp[:, 25:, -1:].clone()
        s2d = (((p2d[:, 25:] - kp[:, 25:, :2]) ** 2) * conf).mean()
        aa = G.rotation_matrix_to_angle_axis(R[:, 1:].reshape(-1, 3, 3)).view(-1, 69)
        terms = [s2d, (beta ** 2).sum(-1).mean(), prior_ref.merged_nll(aa, consts).mean(), F.mse_loss(p2d, t_p2d), F.mse_loss(j3d, t_j3d),
                 F.mse_loss(beta, t_beta), F.mse_loss(R, t_R), adaptor_ref.OracleAdaptor.s3d_loss(j3d[:, 25:], gt_s3d[:, :, :3], conf)]
        return sum(wi * t for wi, t in zip(w, terms)), terms
    cpu = [t.clone().requires_grad_(True) for t in (p2d, j3d, R, beta)]
    tot, terms = ref_total(*cpu)
    tot.backward()
    gpu = [t.cuda().requires_grad_(True) for t in (p2d, j3d, R, beta)]
    prior = MaxMixturePrior().cuda()
    total, parts = losses.loss_multi(*gpu, w, prior=prior, kp=kp.cuda(), t_p2d=t_p2d.cuda(), t_j3d=t_j3d.cuda(), t_beta=t_beta.cuda(),
                                     t_R=t_R.cuda(), gt_s3d=gt_s3d.cuda())
    (total * 0.7).backward()
    assert rel_err(total, tot.detach()) < 1e-5
    for a, b in zip(parts.cpu(), terms):
        assert abs(a.item() - b.item()) <= 2e-5 * max(1.0, abs(b.item()))
    for a, b in zip(gpu, cpu):
        assert rel_err(a.grad, b.grad * 0.7) < 1e-4
    # motion loss
    kh = torch.cat([torch.randn(B, 49, 2, generator=g) * 0.3, (torch.rand(B, 49, 1, generator=g) > 0.2).float()], -1)
    pa, ph = p2d.clone().requires_grad_(True), t_p2d.clone().requires_grad_(True)
    conf = ((kp[:, 25:, -1] + kh[:, 25:, -1]) == 2).float().unsqueeze(-1)
    ref = ((((pa[:, 25:] - ph[:, 25:]) - (kp[:, 25:, :2] - kh[:, 25:, :2])) ** 2) * conf).mean()
    ref.backward()
    ga, gh = p2d.cuda().requires_grad_(True), t_p2d.cuda().requires_grad_(True)
    ml = losses.loss_motion(ga, gh, kp.cuda(), kh.cuda())
    ml.backward()
    assert rel_err(ml, ref.detach()) < 1e-5 and rel_err(ga.grad, pa.grad) < 1e-5 and rel_err(gh.grad, ph.grad) < 1e-5


def test_projection_autograd(L):
    from dynaboa_b200.geometry import project_normalized
    from oracle import geometry_ref as G
    g = torch.Generator().manual_seed(31)
    cam = torch.tensor([[0.9, 0.01, -0.02], [1.1, 0.1, 0.05]])
    X = torch.randn(2, 49, 3, generator=g) * 0.4
    w = torch.randn(2, 49, 2, generator=g)
    cc, Xc = cam.clone().requires_grad_(True), X.clone().requires_grad_(True)
    (G.weak_perspective_project(cc, Xc)[1] * w).sum().backward()
    cg, Xg = cam.cuda().requires_grad_(True), X.cuda().requires_grad_(True)
    (project_normalized(cg, Xg) * w.cuda()).sum().backward()
    assert rel_err(cg.grad, cc.grad) < 1e-5 and rel_err(Xg.grad, Xc.grad) < 1e-5


def test_sweeps_match_torch_optimisers(L):
    n = 1 << 20
    g = torch.Generator().manual_seed(41)
    p0, grad = torch.randn(n, generator=g), torch.randn(n, generator=g) * 1e-3
    grad[:1000] = 0
    # inner SGD step: p + (-lr * g)
    out = torch.empty(n, device='cuda')
    p0d, gradd = dev(p0), dev(grad)
    L.call('dboa_sgd_update', L.ptr(p0d), L.ptr(gradd), L.ptr(out), 8e-6, n, L.stream())
    assert torch.equal(out.cpu(), p0 + (-8e-6 * grad))
    # Adam(lr 3e-6, betas (0.5, 0.9)) x 3 steps + EMA teacher, against torch.optim.Adam on CPU, element by element in units
    # of the fp32 roundoff u: torch's vectorised lerp_ / addcmul_ / addcdiv_ may fuse, the sweep rounds every operation
    # (tests/test_gpu_step_kernels.py holds it to the bit); p and the teacher carry their own earlier differences.  Worst
    # measured (the bit-exact fp32 restatement against torch): p 2.0 u (|p| + 1e-5), m 0, v 2.0 u |v|, teacher 3.7 u (|t| + 1e-5).
    u = 2.0 ** -24
    pc = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pc], lr=3e-6, betas=(0.5, 0.9), foreach=False)
    teacher_c = p0.clone()
    pd, m, v, td = dev(p0), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda'), dev(p0)
    for step in range(1, 4):
        gstep = grad * step
        pc.grad = gstep.clone()
        opt.step()
        teacher_c = teacher_c * 0.1 + pc.data * 0.9
        gstepd = dev(gstep)
        L.call('dboa_adam_ema', L.ptr(pd), L.ptr(gstepd), L.ptr(m), L.ptr(v), L.ptr(td), n, 3e-6, 0.5, 0.9, 1e-8, step, 0.1, L.stream())
        st = opt.state[pc]
        assert ((pd.cpu() - pc.data).abs() <= 4 * u * (pc.data.abs() + 1e-5)).all()
        assert ((m.cpu() - st['exp_avg']).abs() <= 4 * u * (st['exp_avg'].abs() + gstep.abs())).all()
        assert ((v.cpu() - st['exp_avg_sq']).abs() <= 4 * u * st['exp_avg_sq']).all()
        assert ((td.cpu() - teacher_c).abs() <= 8 * u * (teacher_c.abs() + 1e-5)).all()
    t2 = dev(p0)
    L.call('dboa_ema_update', L.ptr(t2), L.ptr(pd), n, 0.1, L.stream())
    assert torch.equal(t2.cpu(), p0 * 0.1 + pd.cpu() * 0.9)


def test_cosine_and_retrieval(L):
    g = torch.Generator().manual_seed(51)
    sizes = [802816, 100352, 2048, 1024, 7]
    A = [torch.randn(s, generator=g) for s in sizes]
    Bt = [a + 0.05 * torch.randn(a.shape, generator=g) for a in A]
    Ad, Bd = [dev(a) for a in A], [dev(b) for b in Bt]
    n = len(sizes)
    pa = (C.c_void_p * n)(*[t.data_ptr() for t in Ad])
    pb = (C.c_void_p * n)(*[t.data_ptr() for t in Bd])
    ln = (C.c_longlong * n)(*sizes)
    part = torch.empty(3 * 4096, device='cuda')
    out = torch.empty(n, device='cuda')
    L.call('dboa_cosine_pairs', pa, pb, ln, n, L.ptr(part), part.numel(), L.ptr(out), 1e-12, L.stream())
    ref = torch.stack([F.cosine_similarity(a.double(), b.double(), dim=0) for a, b in zip(A, Bt)])
    assert (out.cpu().double() - ref).abs().max().item() < 2e-6
    feat = torch.rand(2048, generator=g)
    centers = torch.rand(10, 2048, generator=g)
    centers[6] = feat * 1.3 + 0.01 * torch.rand(2048, generator=g)
    best = torch.zeros(1, dtype=torch.int32, device='cuda')
    d = torch.zeros(10, device='cuda')
    featd, centersd = dev(feat), dev(centers)
    L.call('dboa_retrieval_nearest', L.ptr(featd), L.ptr(centersd), 10, 2048, L.ptr(best), L.ptr(d), L.stream())
    refd = 1 - F.cosine_similarity(feat.unsqueeze(0), centers)
    assert int(best.item()) == int(torch.argsort(refd)[0]) == 6
    assert rel_err(d, refd) < 1e-5


def test_eval_metrics_on_device(L, golden):
    """dboa_eval_metrics (H36M joints, MPJPE, 3x3-SVD Procrustes, PVE) against the reference's numpy path (golden) and,
    on fresh random meshes with the real 6890-vertex size, against the oracle restatement."""
    from oracle import eval_ref
    gd = golden('eval_metrics')

    def run(pred, gt, gtn, J, jmap):
        B, NV, NJ = pred.shape[0], pred.shape[1], J.shape[0]
        pd, gd_, gn, Jd = dev(torch.from_numpy(pred)), dev(torch.from_numpy(gt)), dev(torch.from_numpy(gtn)), dev(torch.from_numpy(J))
        jm = torch.from_numpy(jmap.astype(np.int32)).cuda()
        scratch = torch.empty(L.load().dboa_eval_scratch_floats(B, NJ), device='cuda')
        out = torch.empty(B, 3, device='cuda')
        L.call('dboa_eval_metrics', L.ptr(pd), L.ptr(gd_), L.ptr(gn), L.ptr(Jd), NJ, NV, L.ptr(jm), jm.numel(), L.ptr(scratch), L.ptr(out), B,
               L.stream())
        return out.cpu().numpy()

    out = run(gd['pred'], gd['gt'], gd['gt_neutral'], gd['J'], gd['joint_map'])
    scale = gd['mpjpe'].max()
    assert np.abs(out[:, 0] - gd['mpjpe']).max() <= 2e-5 * scale
    assert np.abs(out[:, 1] - gd['pampjpe']).max() <= 5e-5 * scale          # includes the mirrored and the exact-similarity sample
    assert abs(out[:, 2].mean() - gd['pve']) <= 2e-5 * gd['pve']
    rng = np.random.RandomState(11)
    B, NV, NJ = 3, 6890, 17
    J = (rng.rand(NJ, NV) ** 12).astype(np.float32)
    J /= J.sum(1, keepdims=True)
    gt = (rng.randn(B, NV, 3) * 0.5).astype(np.float32)
    pred = (gt * 1.1 + rng.randn(B, NV, 3) * 0.08).astype(np.float32)
    gtn = (gt + 0.02).astype(np.float32)
    m, p, v = eval_ref.eval_metrics(pred, gt, gtn, J, gd['joint_map'])
    out = run(pred, gt, gtn, J, gd['joint_map'])
    assert np.abs(out[:, 0] - m).max() <= 5e-5 * m.max() and np.abs(out[:, 1] - p).max() <= 1e-4 * m.max()
    assert abs(out[:, 2].mean() - v) <= 5e-5 * v
