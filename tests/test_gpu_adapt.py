"""End-to-end bilevel adaptation on the GPU against trajectories recorded from the reference's own
``BaseAdaptor`` / ``Adaptor`` code (tests/golden/adapt_*.npz, see oracle/make_golden.py): configs C2
(1 inner step), C3 (3 inner steps + retrieval minibatch) and C5 (dynamic re-adaptation loop)."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import adapt_options, fetch

pytestmark = pytest.mark.gpu


def build_adaptor(asset_dir, tmp, gd):
    from dynaboa_b200.adaptor import Adaptor
    opts = adapt_options(tmp, gd)
    return Adaptor(opts), opts


def run_and_compare(asset_dir, tmp_path, golden, tag, fused):
    from dynaboa_b200 import synthetic
    from oracle.make_golden import sample_indices
    gd = golden(f'adapt_{tag}')
    ad, opts = build_adaptor(asset_dir, tmp_path, gd)
    n_frames = gd['upper_loss'].shape[0]
    stream = synthetic.SyntheticStream(length=n_frames, batch_size=opts.batch_size)
    names = [str(s) for s in gd['param_names']]
    masks_all = torch.from_numpy(gd['teacher_masks']).float()
    n_outer = 0
    for t in range(n_frames):
        batch = fetch(stream[t])
        random.seed(1000 + t)
        calls = {'i': 0}

        def provider(B, dev, t=t, calls=calls):
            m = masks_all[t, min(calls['i'], masks_all.shape[1] - 1)]
            calls['i'] += 1
            return m.to(dev)
        ad.teacher.mask_provider = provider
        ad.global_step, ad.fit_losses = t, {}
        ad.model.eval()
        mpjpe, pampjpe, pve = ad.adapt(batch) if fused else ad.adaptation(batch)
        dyn = int(gd['dyn_steps'][t])
        n_outer += 1 + min(dyn, opts.optim_steps)
        tol = 2e-4 if t == 0 else 1e-3
        assert abs(float(ad.last_upper_loss) - gd['upper_loss'][t]) <= tol * abs(gd['upper_loss'][t]) , (tag, t)
        pred = ad.predict(batch['image'])
        assert rel_err(pred['rotmat'], gd['rotmat'][t]) < 1e-3, (tag, t)
        assert rel_err(pred['betas'], gd['betas'][t]) < 1e-3 and rel_err(pred['cam'], gd['cam'][t]) < 1e-3, (tag, t)
        assert rel_err(pred['joints'], gd['joints'][t]) < 1e-3, (tag, t)
        assert rel_err(pred['vertices'][:, ::10], gd['verts_sub'][t]) < 1e-3, (tag, t)
        assert abs(np.mean(mpjpe) - gd['metrics'][t][0].mean()) <= 1e-3 * gd['metrics'][t][0].mean(), (tag, t)
        assert abs(np.mean(pampjpe) - gd['metrics'][t][1].mean()) <= 2e-3 * gd['metrics'][t][1].mean(), (tag, t)
        if 'cos12' in gd and opts.dynamic_boa:
            assert ad.optim_step_record[-1] == dyn, (tag, t)
        params = dict(ad.model.module.named_parameters())
        bound = 4 * opts.lr * n_outer
        gnorm = gd['grad_norms'][t]
        bad = 0
        for i, name in enumerate(names):
            p = params[name]
            idx = sample_indices(name, p.numel())
            th = p.detach().contiguous().flatten()[idx].double().cpu().numpy()
            assert np.abs(th - gd['theta_samples'][t][i]).max() <= bound, (tag, t, name)
            if t == 0 and not opts.dynamic_boa:     # one outer step from identical weights: the sensitive gradient check
                gr = p.grad.contiguous().flatten()[idx].double().cpu().numpy()
                scale = max(gnorm[i] / p.numel() ** 0.5, 1e-12)
                err = np.abs(gr - gd['grad_samples'][t][i]).max()
                if err > 2e-2 * max(scale, np.abs(gd['grad_samples'][t][i]).max()):   # gradient kinks: DESIGN.md section 6
                    bad += 1
                    print(f'  grad off: {name} err {err:.3e} rms {scale:.3e} golden-max {np.abs(gd["grad_samples"][t][i]).max():.3e}')
        assert bad <= 2, (tag, t, f'{bad} tensors with outer-gradient samples off')
        print(f'[{tag}{"/fused" if fused else ""}] frame {t}: upper {float(ad.last_upper_loss):.6f} (golden {gd["upper_loss"][t]:.6f})')
    return ad


@pytest.mark.parametrize('tag', ['c2', 'c3', 'c5'])
def test_autograd_path_follows_reference_trajectory(asset_dir, tmp_path, golden, tag):
    run_and_compare(asset_dir, tmp_path, golden, tag, fused=False)


@pytest.mark.parametrize('tag', ['c2', 'c3', 'c5'])
def test_fused_path_follows_reference_trajectory(asset_dir, tmp_path, golden, tag):
    run_and_compare(asset_dir, tmp_path, golden, tag, fused=True)


def test_excute_loop_runs(asset_dir, tmp_path, golden):
    gd = golden('adapt_c2')
    ad, _ = build_adaptor(asset_dir, tmp_path, gd)
    ad.teacher.eval()
    ad.options.cache_results = 1          # Pred_<step>.pt as the reference always writes them
    out = ad.excute(max_frames=3)
    assert np.isfinite(out['mpjpe']) and np.isfinite(out['pampjpe'])
    # the eight result files of the reference driver (dynaboa_benchmark.py:111-123): same names, joblib pickles, same keys
    import joblib
    keys = {'lowerlevel_kp2dloss.pt': ['kp2dloss'], 'upperlevel_kp2dloss.pt': ['kp2dloss'], 'res.pt': ['mpjpe', 'pampjpe', 'pve'],
            'lower_res.pt': ['mpjpe', 'pampjpe'], 'steps_statistic_res.pt': ['mpjpe', 'pampjpe'], 'feat_sims.pt': ['feat'],
            'optim_step_record.pt': ['step']}
    for name, ks in keys.items():
        d = joblib.load(os.path.join(ad.exppath, name))
        assert sorted(d) == sorted(ks), name
    res = joblib.load(os.path.join(ad.exppath, 'res.pt'))
    assert len(res['mpjpe']) == 3 and abs(np.mean(res['mpjpe']) - out['mpjpe']) < 1e-6
    assert len(joblib.load(os.path.join(ad.exppath, 'lowerlevel_kp2dloss.pt'))['kp2dloss']) == 3
    lines = open(os.path.join(ad.exppath, 'res.txt')).read().splitlines()
    assert lines[0].startswith('Step:2: MPJPE:') and lines[1].startswith('Lower-level  Step:0 MPJPE:')
    assert sorted(joblib.load(os.path.join(ad.exppath, 'result', 'Pred_2.pt'))) == ['beta', 'cam', 'rotmat', 'verts']


def test_output_forward_on_side_stream_is_equivalent(asset_dir, tmp_path, golden):
    """``predict_async`` (output forward of frame t overlapped with the adaptation of frame t+1) must give the same
    outputs and leave the adaptation trajectory bit-identical to the serial ``predict``: the optimiser step waits for the
    side-stream read of the weights before it overwrites them."""
    from dynaboa_b200 import synthetic
    gd = golden('adapt_c2')
    runs = []
    for overlap in (False, True):
        ad, opts = build_adaptor(asset_dir, tmp_path / f'o{int(overlap)}', gd)
        ad.teacher.eval()                                  # deterministic teacher (no dropout masks)
        ad.fused_eval = 'none'
        stream = synthetic.SyntheticStream(length=6, batch_size=opts.batch_size)
        outs = []
        for t in range(6):
            batch = fetch(stream[t])
            ad.global_step, ad.fit_losses = t, {}
            ad.adapt(batch)
            if overlap:
                pred, ev = ad.predict_async(batch['image'])
                outs.append((pred, ev))
            else:
                outs.append((ad.predict(batch['image']), None))
        torch.cuda.synchronize()
        runs.append((ad.model.module.arena.clone(), [{k: v.clone() for k, v in p.items()} for p, _ in outs]))
    (theta_s, out_s), (theta_a, out_a) = runs
    assert torch.equal(theta_s, theta_a)
    for a, b in zip(out_s, out_a):
        for k in a:
            assert torch.equal(a[k], b[k]), k
