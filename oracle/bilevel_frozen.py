"""One level of the bilevel problem in fp64 on a given kink pattern (test infrastructure only).

The loss of one video's lower or upper level (reference base_adaptor.py:222-317, restated in adaptor_ref ``_level``), written
so that every network forward goes through ``hmr_frozen.forward``: with the ReLU, max-pool and dropout pattern of the GPU
forward that served the level, the autograd gradient is the exact derivative of what the GPU computed, and the GPU's
gradient arena must equal it to rounding.  With ``pattern=None`` everywhere (and the prior at its minimum) this is
adaptor_ref's level itself (tests/test_bilevel_frozen.py checks it against ``OracleAdaptor(dtype=torch.float64)``).

The terms are those of ``fused.level_backward`` and of the per-video loss head (loss_head_ref):

- frame terms (``use_frame_losses_*``): the 2D reprojection on joints ``kp_range``, the shape prior and the pose prior at a
  given GMM component (None: the minimum);
- teacher consistency (``use_temporal_losses_*`` with ``use_meanteacher``): MSE to given teacher outputs (``teacher``);
- the motion term against the history frame (``hist``), when the caller says it is live;
- the labelled term of an exemplar minibatch (``exemplars``), when mixtrain is on for the level.

Everything is plain torch in the dtype of the inputs (the GPU tests run it in float64 on the device).
"""
from types import SimpleNamespace

import torch

from . import geometry_ref, hmr_frozen
from . import loss_head_ref as L


class Model(SimpleNamespace):
    """What a level reads besides the weights: ``buffers`` (init_pose / init_shape / init_cam), ``smpl`` (the neutral SMPL
    arrays, J_regressor_extra, joint map, extra vertex ids, as ``loss_head_ref.smpl`` takes them), ``gmm`` (means,
    precisions, -log weights of the pose prior) and ``kp_range`` (first, count) of the 2D and motion terms."""


def network(model, params, image, pattern=None, drop=None):
    """The forward graph of ``fused.forward_graph``: HMR on ``pattern`` (None: its own, with ``drop``), neutral SMPL and the
    weak-perspective projection.  Returns rot, shape, cam, j3d, p2d, feats (15) and the pattern."""
    rot, shape, cam, pattern, feats = hmr_frozen.forward(image, dict(params, **model.buffers), pattern, drop, need_feature=True)
    _, j3d = L.smpl(*model.smpl, shape, rot)
    return SimpleNamespace(rot=rot, shape=shape, cam=cam, j3d=j3d, p2d=L.project(cam, j3d), feats=feats, pattern=pattern)


def teacher_outputs(model, params, image, pattern=None, drop=None):
    """The mean teacher's targets (p2d, j3d, shape, rot) of ``image``, without gradient."""
    with torch.no_grad():
        t = network(model, params, image, pattern, drop)
    return dict(t_p2d=t.p2d, t_j3d=t.j3d, t_beta=t.shape, t_R=t.rot)


def prior_components(model, rot):
    """(B, 8): the pose prior of each body at each mixture component (the prior is their minimum)."""
    B = rot.shape[0]
    return L.prior_components(L.rotmat_to_aa(rot[:, 1:]).reshape(B, 69), *model.gmm)


def level(o, model, params, lower, image, kp, pattern=None, comp=None, teacher=None, hist=None, exemplars=None):
    """One video's level loss on weights ``params`` ({name: tensor}, the 169 parameters) and its gradient.

    ``o``: the adaptation options; ``image`` (b, 3, 224, 224) and ``kp`` (b, 49, 3) the frame; ``pattern`` the kink pattern of
    its forward (None: its own); ``comp`` (b,) the pose prior's component (None: the minimum); ``teacher`` the targets of
    ``teacher_outputs`` (None: no teacher term); ``hist`` {image, kp, pattern} of the history frame (None: the motion term
    is not live); ``exemplars`` the exemplar minibatch {img, keypoints, pose, betas, pose_3d, pattern} (None: no labelled
    term).  Returns ``terms`` (the records of ``fused.level_backward`` under its names, as 0-d tensors), ``total``,
    ``grads`` ({name: d total / d param}), the main forward's ``feats`` and its prior components ``ll``."""
    tag = 'll' if lower else 'ul'
    use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
    p = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    main = network(model, p, image, pattern)
    w = [0.0] * 8
    if use_frame:
        w[0], w[1], w[2] = o.s2dloss_weight, o.shape_prior_weight, o.pose_prior_weight
    ll = prior_components(model, main.rot)
    prior = ll.min(1)[0] if comp is None else ll.gather(1, comp.view(-1, 1).to(ll.device)).squeeze(1)
    targets = {}
    if teacher is not None:
        tw = o.teacherloss_weight
        w[3], w[4], w[5], w[6] = 5 * tw, 5 * tw, 0.001 * tw, 1 * tw
        targets = teacher
    t = L.head_terms(1, main.p2d, main.j3d, main.rot, main.shape, w, kp=kp if use_frame else None, prior=prior if use_frame else None,
                     kp_range=model.kp_range, **targets)[0]
    terms, total = {}, t[8]
    if use_frame:
        terms[f'{tag}/s2dloss'], terms[f'{tag}/shape_prior'], terms[f'{tag}/pose_prior'] = t[0], t[1], t[2]
    if hist is not None:
        h = network(model, p, hist['image'], hist.get('pattern'))
        m = L.motion_terms(1, main.p2d, h.p2d, kp, hist['kp'], *model.kp_range)[0]
        terms['ul/motion_loss'] = m
        total = total + m * o.motionloss_weight
    if exemplars is not None:
        ex = exemplars
        e = network(model, p, ex['img'], ex.get('pattern'))
        n = ex['img'].shape[0]
        gt_R = geometry_ref.batch_rodrigues(ex['pose'].reshape(-1, 3)).view(n, 24, 3, 3)
        lw = o.labelloss_weight
        et = L.head_terms(1, e.p2d, e.j3d, e.rot, e.shape, [5 * lw, 0, 0, 0, 0, 0.001 * lw, 1 * lw, 5 * lw], kp=ex['keypoints'],
                          t_beta=ex['betas'], t_R=gt_R, gt_s3d=ex['pose_3d'], kp_range=model.kp_range)[0]
        terms[f'{tag}/labled_loss'] = et[8]
        total = total + et[8]
    total.backward()
    return SimpleNamespace(terms={k: v.detach() for k, v in terms.items()}, total=total.detach(), grads={k: v.grad for k, v in p.items()},
                           feats=[f.detach() for f in main.feats], ll=ll.detach())


def cosines(fa, fb):
    """The dynamic loop's 15 feature cosines (reference base_adaptor.py:211-219) of two lists of features."""
    return [float((a.flatten() * b.flatten()).sum() / (a.flatten().norm() * b.flatten().norm())) for a, b in zip(fa, fb)]
