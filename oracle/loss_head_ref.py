"""fp64 restatement of the loss head that follows the HMR network in every forward graph (test infrastructure only).

SMPL (smplx_ref), the weak-perspective projection (geometry_ref), the merged GMM pose prior on rotation matrices
(prior_ref), the multi-term head of ``dboa_loss_multi`` and the motion term, all written per video: the rows of video g
are ``[g * b, (g + 1) * b)`` and every mean is that video's own, as ``fused._loss_head`` asks of the kernels.  The loss
formulas are those of adaptor_ref (``frame_losses``, ``teacher_loss``, ``labelled_loss``, ``motion_loss``, ``s3d_loss``).

Every function is plain torch and works in the dtype it is given; the GPU tests call it in float64 on the GPU's own fp32
inputs.  Two choices make it the exact derivative of what the kernels compute rather than a neighbour of it:

* the axis-angle branch test ``r22 < eps`` uses the kernel's float constant ``1e-6f`` (``R2AA_EPS``);
* the pose prior can be evaluated at a given mixture component (the one the GPU selected) instead of the minimum.
"""
import numpy as np
import torch

from . import geometry_ref as G
from . import smplx_ref
from .adaptor_ref import OracleAdaptor

R2AA_EPS = float(np.float32(1e-6))          # rotmath.cuh r2aa_quat: r22 < 1e-6f
TERMS = 9                                   # 8 weighted terms and their weighted sum (include/dynaboa_b200.h)


def rotmat_to_aa(R):
    """(N, 3, 3) -> (N, 3): geometry_ref.rotation_matrix_to_angle_axis with the kernel's branch constant."""
    aa = G.quaternion_to_angle_axis(G.rotation_matrix_to_quaternion(R.reshape(-1, 3, 3), R2AA_EPS))
    return torch.where(torch.isnan(aa), torch.zeros_like(aa), aa)


def r2aa_branch(R):
    """(N, 3, 3) -> (N,) the quaternion branch (0..3) that rotmath.cuh r2aa_quat takes."""
    R = R.reshape(-1, 3, 3)
    d2, d0_d1, d0_nd1 = R[:, 2, 2] < R2AA_EPS, R[:, 0, 0] > R[:, 1, 1], R[:, 0, 0] < -R[:, 1, 1]
    return torch.where(d2, torch.where(d0_d1, 0, 1), torch.where(d0_nd1, 2, 3))


def prior_components(pose69, means, precisions, neg_log_w):
    """(B, 69) -> (B, 8): 0.5 (x - mu_m)^T P_m (x - mu_m) + neg_log_w[m] of every component (prior_ref.merged_nll before
    its minimum).  ``neg_log_w`` is -log(nll_weights); an entry of +inf is a component that is never selected."""
    diff = pose69.unsqueeze(1) - means
    quad = (torch.einsum('mij,bmj->bmi', precisions, diff) * diff).sum(-1)
    return 0.5 * quad + neg_log_w


def pose_prior(R, consts, comp=None):
    """(B, 24, 3, 3) -> (B,) the prior of the 23 body joints (the root carries none), at component ``comp`` (B,) when it is
    given, else at the minimum (base_adaptor.py:405-409)."""
    B = R.shape[0]
    ll = prior_components(rotmat_to_aa(R[:, 1:]).reshape(B, 69), *consts)
    return ll.min(1)[0] if comp is None else ll.gather(1, comp.view(B, 1)).squeeze(1)


def smpl(model, J_extra, joint_map, vertex_ids, betas, R):
    """(vertices (B, 6890, 3), joints (B, 49, 3)) of rotation-matrix input (B, 24, 3, 3)."""
    out = smplx_ref.smpl_forward(model, J_extra, joint_map, vertex_ids, betas, R[:, 1:], R[:, :1], pose2rot=False)
    return out.vertices, out.joints


def project(cam, j3d):
    """Normalised 2D keypoints (B, NJ, 2), base_adaptor.py:160-170."""
    return G.weak_perspective_project(cam, j3d)[1]


def _per_video(x, G_):
    return x.reshape(G_, -1)


def head_terms(G_, p2d, j3d, R, beta, w, kp=None, prior=None, t_p2d=None, t_j3d=None, t_beta=None, t_R=None, gt_s3d=None,
               kp_range=(25, 24)):
    """(G, 9) terms of the multi-term head for G videos of equal batch: 0 masked 2D keypoints on joints ``kp_range``
    (first, count), 1 shape prior, 2 pose prior (``prior``: the (B,) per-body values), 3..6 MSE to the targets, 7 the
    hip-centred 3D loss on joints 25..48, 8 the weighted sum.  An absent input gives a zero term, as in the kernel."""
    dt = p2d.dtype
    zero = torch.zeros(G_, dtype=dt)
    t = [zero] * 8
    if kp is not None:
        f, n = kp_range
        conf = kp[:, f:f + n, 2:]
        t[0] = _per_video((p2d[:, f:f + n] - kp[:, f:f + n, :2]) ** 2 * conf, G_).mean(1)
    t[1] = _per_video(beta ** 2, G_).sum(1) / (beta.shape[0] // G_)
    if prior is not None:
        t[2] = _per_video(prior, G_).mean(1)
    for i, (x, y) in zip((3, 4, 5, 6), ((p2d, t_p2d), (j3d, t_j3d), (beta, t_beta), (R, t_R))):
        if y is not None:
            t[i] = _per_video((x - y) ** 2, G_).mean(1)
    if gt_s3d is not None:
        b = j3d.shape[0] // G_
        t[7] = torch.stack([OracleAdaptor.s3d_loss(j3d[g * b:(g + 1) * b, 25:], gt_s3d[g * b:(g + 1) * b, :, :3],
                                                   kp[g * b:(g + 1) * b, 25:, 2:]) for g in range(G_)])
    total = sum(float(w[i]) * t[i] for i in range(8))
    return torch.stack(t + [total], 1)


def motion_terms(G_, pa, ph, ka, kh, first=25, count=24):
    """(G,) motion term of each video, base_adaptor.py:387-396: the mean over (b, count, 2) of [both visible] *
    ((pa - ph) - (ka - kh))^2 on joints [first, first + count)."""
    s = slice(first, first + count)
    conf = ((ka[:, s, 2:] + kh[:, s, 2:]) == 2).to(pa.dtype)
    d = (pa[:, s] - ph[:, s]) - (ka[:, s, :2] - kh[:, s, :2])
    return _per_video(conf * d ** 2, G_).mean(1)
