"""MultiVideoAdaptor: G = 4 videos (SyntheticStream(rank=g)) adapted in lockstep, 8 frames at C2 and 2 at C3.  Video 0
(rank 0, the golden stream) is held to tests/golden/adapt_{c2,c3}.npz directly; videos 1..3 to their own single-video
``Adaptor.adapt`` runs given the same teacher masks and retrieval picks.  Criteria of test_gpu_adapt.run_and_compare: upper
loss within 1e-3 (2e-4 on the first frame against the golden), outputs within 1e-3, theta within 4 * lr * n_outer.  Two
grouped runs give bit-identical theta, and one video takes the single-video schedule bit for bit."""
import ast
import random

import pytest
import torch

from conftest import rel_err
from test_gpu_adapt import make_options

pytestmark = pytest.mark.gpu
G = 4


def masks_for(g, t, call, gd):
    """Teacher keep-masks of video g, frame t, teacher forward `call`: the golden's for video 0, seeded for the others."""
    if g == 0:
        m = torch.from_numpy(gd['teacher_masks']).float()
        return m[t, min(call, m.shape[1] - 1)]
    gen = torch.Generator().manual_seed(100000 * g + 100 * t + call)
    return (torch.rand(3, 2, 1, 1024, generator=gen) >= 0.5).float() * 2.0


def seed_for(g, t):
    return 1000 + t if g == 0 else 1000 * (g + 1) + t


def grouped(opts, gd, n_videos=G):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = MultiVideoAdaptor(opts, n_videos)
    calls = [0] * n_videos

    def provider(g, B, dev):
        m = masks_for(g, mv.global_step, calls[g], gd)
        calls[g] += 1
        return m.to(dev)
    mv.mask_provider = provider

    def step(batches):
        for g in range(n_videos):
            calls[g] = 0
            mv.rngs[g].seed(seed_for(g, mv.global_step))
        mv.adapt(batches)
    return mv, step


def frame(streams, t):
    return [{k: v.cuda() if torch.is_tensor(v) else v for k, v in s[t].items()} for s in streams]


@pytest.mark.parametrize('tag,n_frames', [('c2', 8), ('c3', 2)])
def test_every_video_follows_its_own_trajectory(asset_dir, tmp_path, golden, tag, n_frames):
    from dynaboa_b200 import config, synthetic
    from dynaboa_b200.adaptor import Adaptor
    from oracle.make_golden import sample_indices
    gd = golden(f'adapt_{tag}')
    opts = make_options(tmp_path, str(gd['options']), model_file=config.BASE_MODEL)
    assert not opts.dynamic_boa
    streams = [synthetic.SyntheticStream(length=n_frames, batch_size=1, rank=g) for g in range(G)]
    mv, step = grouped(opts, gd)
    singles = {}
    for g in range(1, G):
        o = make_options(tmp_path / f'v{g}', str(gd['options']), model_file=config.BASE_MODEL)
        singles[g] = Adaptor(o)
        singles[g].fused_eval = 'none'
    names = [str(s) for s in gd['param_names']]
    lay_names = mv.base.model.module._lay.names
    for t in range(n_frames):
        batches = frame(streams, t)
        step(batches)
        n_outer = t + 1
        bound = 4 * opts.lr * n_outer
        preds = mv.predict(torch.cat([b['image'] for b in batches]))
        up = mv.last_upper_loss.cpu()
        # video 0 against the golden trajectory
        tol = 2e-4 if t == 0 else 1e-3
        assert abs(float(up[0]) - gd['upper_loss'][t]) <= tol * abs(gd['upper_loss'][t]), (tag, t)
        p = preds[0]
        assert rel_err(p['rotmat'], gd['rotmat'][t]) < 1e-3 and rel_err(p['betas'], gd['betas'][t]) < 1e-3, (tag, t)
        assert rel_err(p['cam'], gd['cam'][t]) < 1e-3 and rel_err(p['joints'], gd['joints'][t]) < 1e-3, (tag, t)
        assert rel_err(p['vertices'][:, ::10], gd['verts_sub'][t]) < 1e-3, (tag, t)
        views = dict(zip(lay_names, mv.base.model.module._lay.views(mv.theta(0).clone())))
        for i, name in enumerate(names):
            idx = sample_indices(name, views[name].numel())
            th = views[name].contiguous().flatten()[idx].double().cpu().numpy()
            assert abs(th - gd['theta_samples'][t][i]).max() <= bound, (tag, t, name)
        # videos 1..3 against their own single-video runs
        for g, ad in singles.items():
            calls = {'i': 0}

            def provider(B, dev, g=g, t=t, calls=calls):
                m = masks_for(g, t, calls['i'], gd)
                calls['i'] += 1
                return m.to(dev)
            ad.teacher.mask_provider = provider
            random.seed(seed_for(g, t))
            ad.global_step, ad.fit_losses = t, {}
            ad.model.eval()
            ad.adapt(batches[g])
            ref_up = float(ad.last_upper_loss)
            assert abs(float(up[g]) - ref_up) <= 1e-3 * abs(ref_up), (tag, t, g, float(up[g]), ref_up)
            ref = ad.predict(batches[g]['image'])
            for k in ('rotmat', 'betas', 'cam', 'joints', 'vertices'):
                assert rel_err(preds[g][k], ref[k].cpu().numpy()) < 1e-3, (tag, t, g, k)
            d = float((mv.theta(g) - ad.model.module.arena).abs().max())
            assert d <= bound, (tag, t, g, d, bound)
            if opts.retrieval:
                assert mv.last_retrieval[g] == ad.last_retrieval, (tag, t, g)
        print(f'[{tag}] frame {t}: upper ' + ' '.join(f'{float(u):.6f}' for u in up) + f' (golden v0 {gd["upper_loss"][t]:.6f})')


def test_grouped_adaptation_is_bit_reproducible(asset_dir, tmp_path, golden):
    from dynaboa_b200 import config, synthetic
    gd = golden('adapt_c2')
    thetas = []
    for run in range(2):
        opts = make_options(tmp_path / f'r{run}', str(gd['options']), model_file=config.BASE_MODEL)
        streams = [synthetic.SyntheticStream(length=3, batch_size=1, rank=g) for g in range(G)]
        mv, step = grouped(opts, gd)
        for t in range(3):
            step(frame(streams, t))
        torch.cuda.synchronize()
        thetas.append(mv.thetas.clone())
        del mv
    assert torch.equal(thetas[0], thetas[1])


def test_one_video_is_bit_identical_to_the_single_video_step(asset_dir, tmp_path, golden):
    """With one video the grouped adaptor runs ``Adaptor.adapt``'s schedule (history frame paired with the current frame,
    teacher forward on the side stream): given the same teacher masks, theta, teacher and upper loss are bit-identical after
    8 frames at C2."""
    from dynaboa_b200 import config, synthetic
    from dynaboa_b200.adaptor import Adaptor
    gd = golden('adapt_c2')
    mv, step = grouped(make_options(tmp_path / 'mv', str(gd['options']), model_file=config.BASE_MODEL), gd, n_videos=1)
    ad = Adaptor(make_options(tmp_path / 'ad', str(gd['options']), model_file=config.BASE_MODEL))
    ad.fused_eval = 'none'
    stream = synthetic.SyntheticStream(length=8, batch_size=1)
    for t in range(8):
        batches = frame([stream], t)
        step(batches)
        calls = {'i': 0}

        def provider(B, dev, t=t, calls=calls):
            m = masks_for(0, t, calls['i'], gd)
            calls['i'] += 1
            return m.to(dev)
        ad.teacher.mask_provider = provider
        random.seed(seed_for(0, t))
        ad.global_step, ad.fit_losses = t, {}
        ad.model.eval()
        ad.adapt(batches[0])
        assert torch.equal(mv.last_upper_loss[0], ad.last_upper_loss), t
    assert torch.equal(mv.theta(0), ad.model.module.arena)
    assert torch.equal(mv.teachers[0], ad.teacher.arena)
