"""MultiVideoAdaptor: G = 4 videos (SyntheticStream(rank=g)) adapted in lockstep, 8 frames at C2 and 2 at C3.  Video 0
(rank 0, the golden stream) is held to tests/golden/adapt_{c2,c3}.npz directly; videos 1..3 to their own single-video
``Adaptor.adapt`` runs given the same teacher masks and retrieval picks.  Criteria of test_gpu_adapt.run_and_compare: upper
loss within 1e-3 (2e-4 on the first frame against the golden), outputs within 1e-3, theta within 4 * lr * n_outer.  Two
grouped runs give bit-identical theta, and one video takes the single-video schedule bit for bit."""
import pytest
import torch

from conftest import rel_err
from harness import PoolRun, SingleRun, adapt_options, masks_for, seed_for, stream

pytestmark = pytest.mark.gpu
G = 4


def grouped(opts, gd, n_frames, n_videos=G):
    """A pool of `n_videos` slots, video g in slot g from the first frame, with the golden's masks for video 0."""
    p = PoolRun(opts, n_videos, masks=lambda vid, t, call: masks_for(vid, t, call, gd), seed=seed_for)
    for g in range(n_videos):
        p.start(g, g, stream(g, n_frames))
    return p


def single(opts, gd, g):
    return SingleRun(opts, g, masks=lambda vid, t, call: masks_for(vid, t, call, gd), seed=seed_for)


@pytest.mark.parametrize('tag,n_frames', [('c2', 8), ('c3', 2)])
def test_every_video_follows_its_own_trajectory(asset_dir, tmp_path, golden, tag, n_frames):
    from oracle.make_golden import sample_indices
    gd = golden(f'adapt_{tag}')
    opts = adapt_options(tmp_path, gd)
    assert not opts.dynamic_boa
    pool = grouped(opts, gd, n_frames)
    mv = pool.mv
    singles = {g: single(adapt_options(tmp_path / f'v{g}', gd), gd, g) for g in range(1, G)}
    names = [str(s) for s in gd['param_names']]
    lay_names = mv.base.model.module._lay.names
    for t in range(n_frames):
        done = pool.step(range(G))
        batches = [done[g][2] for g in range(G)]
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
        for g, s in singles.items():
            s.step(t, batches[g])
            ad = s.ad
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
    gd = golden('adapt_c2')
    thetas = []
    for run in range(2):
        p = grouped(adapt_options(tmp_path / f'r{run}', gd), gd, 3)
        for t in range(3):
            p.step(range(G))
        torch.cuda.synchronize()
        thetas.append(p.mv.thetas.clone())
        del p
    assert torch.equal(thetas[0], thetas[1])


def test_one_video_is_bit_identical_to_the_single_video_step(asset_dir, tmp_path, golden):
    """With one video the grouped adaptor runs ``Adaptor.adapt``'s schedule (history frame paired with the current frame,
    teacher forward on the side stream): given the same teacher masks, theta, teacher and upper loss are bit-identical after
    8 frames at C2."""
    gd = golden('adapt_c2')
    p = grouped(adapt_options(tmp_path / 'mv', gd), gd, 8, n_videos=1)
    mv = p.mv
    s = single(adapt_options(tmp_path / 'ad', gd), gd, 0)
    ad = s.ad
    for t in range(8):
        s.step(t, p.step([0])[0][2])
        assert torch.equal(mv.last_upper_loss[0], ad.last_upper_loss), t
    assert torch.equal(mv.theta(0), ad.model.module.arena)
    assert torch.equal(mv.teachers[0], ad.teacher.arena)
