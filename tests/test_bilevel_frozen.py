"""oracle/bilevel_frozen.py is adaptor_ref's level: on its own kink pattern (``pattern=None``) and with the pose prior at its
minimum, its loss and its gradient in all 169 parameters equal ``OracleAdaptor(dtype=torch.float64)``'s lower and upper
levels to rounding (CPU, fp64, batch 1).  The golden trajectories pin OracleAdaptor to the reference's own code; this pins
the oracle that tests/test_gpu_bilevel_step.py evaluates on the GPU's kink pattern to OracleAdaptor."""
import random

import numpy as np
import pytest
import torch

from dynaboa_b200 import config, constants as C, synthetic
from oracle import adaptor_ref, bilevel_frozen, hmr_frozen, hmr_ref, prior_ref

TOL = 1e-12
T = 6                      # the frame of the motion cases: with interval 5 the history frame is frame 1


def oracle64(**over):
    opts = adaptor_ref.default_options(**over)
    return adaptor_ref.OracleAdaptor(
        opts, synthetic.make_basemodel(), {g: synthetic.make_smpl_model(g) for g in ('neutral', 'male', 'female')},
        synthetic.make_extra_regressors(), dict(np.load(config.GMM_PRIOR)), bank=synthetic.make_exemplar_bank(),
        clusters=synthetic.make_clusters(), dtype=torch.float64, joint_map=C.JOINT_MAP_49, vertex_ids=C.SMPL_EXTRA_VERTEX_IDS,
        h36m_to_j14=C.H36M_TO_J14)


def model_of(ora):
    gmm = prior_ref.gmm_constants(dict(np.load(config.GMM_PRIOR)), torch.float64)
    smpl = (ora.smpl['neutral'], ora.J_extra, ora.joint_map, ora.vertex_ids)
    return bilevel_frozen.Model(buffers=ora.buffers, smpl=smpl, gmm=(gmm['means'], gmm['precisions'], -torch.log(gmm['nll_weights']).reshape(-1)),
                                kp_range=(25, 24))


# (name, options, motion live, teacher dropout)
CASES = [
    ('frame', dict(use_temporal_losses_upper=0, retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0), False, False),
    ('teacher', dict(retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0, use_motion=0), False, True),
    ('motion', dict(retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0), True, True),
    ('exemplars', dict(sample_num=8), True, True),
]


@pytest.mark.parametrize('name,over,motion,masked', CASES, ids=[c[0] for c in CASES])
def test_level_is_the_adaptor_oracle(name, over, motion, masked):
    ora = oracle64(**over)
    o, model = ora.o, model_of(ora)
    stream = synthetic.SyntheticStream(length=T + 1, batch_size=1)
    frame = stream[T]
    image, kp = frame['image'].double(), frame['smpl_j2d'].double()
    g = torch.Generator().manual_seed(31)
    drop = (torch.rand(3, 2, 1, 1024, generator=g) >= 0.5).double() * 2 if masked else None
    ora.teacher_masks = lambda B: None if drop is None else [(drop[i, 0], drop[i, 1]) for i in range(3)]
    h = stream[T - o.interval]
    ora.history[T - o.interval] = {'image': h['image'].double(), 's2d': h['smpl_j2d'].double()}
    ora.global_step = T if motion else 1
    theta = {k: v.detach() for k, v in ora.theta.items()}
    for lower in (True, False):
        use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
        mix = o.retrieval and (o.lower_level_mixtrain if lower else o.upper_level_mixtrain)
        params = {k: v.detach().clone().requires_grad_(True) for k, v in theta.items()}
        random.seed(7)
        ora.fit_losses = {}
        loss, _ = ora._level(image, kp, params, lower)
        loss.backward()
        teacher = None
        if use_temporal and o.use_meanteacher:
            teacher = bilevel_frozen.teacher_outputs(model, ora.teacher, image, drop=drop)
        hist = None
        if use_temporal and o.use_motion and motion:
            hist = {'image': h['image'].double(), 'kp': h['smpl_j2d'].double()}
        ex = None
        if mix:
            picks = ora.last_retrieval[1]
            assert len(picks) == o.sample_num
            ex = {k: v[torch.as_tensor(picks)] for k, v in ora.bank.items()}
        r = bilevel_frozen.level(o, model, theta, lower, image, kp, teacher=teacher, hist=hist, exemplars=ex)
        tag = 'll' if lower else 'ul'
        what = f'{name} {tag}'
        assert abs(float(r.total) - float(loss.detach())) <= TOL * abs(float(loss)), what
        for k, v in r.terms.items():
            ref = float(ora.fit_losses[k]) * (o.labelloss_weight if k.endswith('labled_loss') else 1.0)    # fused records it weighted
            assert abs(float(v) - ref) <= TOL * abs(ref), (what, k)
        expect = {f'{tag}/s2dloss', f'{tag}/shape_prior', f'{tag}/pose_prior'}
        expect |= {'ul/motion_loss'} if hist is not None else set()
        expect |= {f'{tag}/labled_loss'} if ex is not None else set()
        assert set(r.terms) == expect, what
        assert len(r.grads) == 169 and set(r.grads) == set(params)
        for k, p in params.items():
            ref = p.grad
            assert ref.abs().max() > 0, (what, k)
            assert (r.grads[k] - ref).abs().max() <= TOL * ref.abs().max(), (what, k)
        if mix:                                    # retrieval reads the frozen forward's pooled feature as the oracle's
            f = bilevel_frozen.network(model, theta, image)
            d = 1 - torch.nn.functional.cosine_similarity(f.feats[5], ora.centers)
            assert int(d.argmin()) == ora.last_retrieval[0], what


def test_frozen_features_are_the_reference_features():
    """hmr_frozen's 15 features on its own pattern are hmr_ref's (fp64, with dropout masks)."""
    sd = {k: v.double() for k, v in hmr_ref.strip_prefix(synthetic.make_basemodel()['model']).items()}
    g = torch.Generator().manual_seed(12)
    x = torch.randn(1, 3, 224, 224, generator=g, dtype=torch.float64)
    drop = (torch.rand(3, 2, 1, 1024, generator=g) >= 0.5).double() * 2
    with torch.no_grad():
        *out_f, _, feats_f = hmr_frozen.forward(x, sd, drop=drop, need_feature=True)
        *out_r, feats_r = hmr_ref.forward(x, sd, need_feature=True, masks=[(drop[i, 0], drop[i, 1]) for i in range(3)])
    assert len(feats_f) == 15
    for a, b in zip(out_f + feats_f, out_r + feats_r):
        assert a.shape == b.shape and (a - b).abs().max() <= TOL * b.abs().max()
