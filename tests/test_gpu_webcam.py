"""Third client of the hot path (N3): ``WebcamAdaptor`` (the role of reference dynaboa_webcam.py ``Adaptor``) against
tests/golden/adapt_webcam.npz -- the trajectory of the reference class itself, executed unmodified on CPU by
oracle/make_golden.py ``golden_webcam`` (OpenPose joints 0..24 in the 2D / motion terms, teacher in eval mode, dynamic loop) --
and its GPU input side (bounding box from the detections, confidence threshold, crop) against the CPU restatement."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import cam_options

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    _lib.load()
    return _lib


def make_adaptor(tmp, gd, **extra):
    from dynaboa_b200.webcam import WebcamAdaptor
    return WebcamAdaptor(cam_options(tmp, gd, **extra))


def test_webcam_adaptor_follows_the_reference_class(asset_dir, tmp_path, golden):
    from dynaboa_b200 import synthetic
    from oracle.make_golden import sample_indices
    gd = golden('adapt_webcam')
    ad = make_adaptor(tmp_path, gd)
    o = ad.options
    n_frames = gd['kp25'].shape[0]
    stream = synthetic.SyntheticStream(length=n_frames, batch_size=1)
    names = [str(s) for s in gd['param_names']]
    n_outer = 0
    for t in range(n_frames):
        image = stream[t]['image'].cuda()
        kp = torch.zeros(1, 49, 3, device='cuda')
        kp[:, :25] = torch.from_numpy(gd['kp25'][t]).cuda()
        res = ad.adapt_processed(image, kp)
        assert ad.global_step == t + 1                          # save_hist advances the step (reference :105-108)
        dyn = int(gd['dyn_steps'][t])
        assert min(ad.optim_step_record[-1], o.optim_steps) == dyn, t
        n_outer += 1 + dyn
        assert rel_err(res['vts'][:, ::10], gd['verts_sub'][t]) < 1e-3, t
        assert rel_err(res['cam'], gd['cam'][t]) < 1e-3, t
        params = dict(ad.model.module.named_parameters())
        bound = 4 * o.lr * n_outer
        for i, name in enumerate(names):
            p = params[name]
            th = p.detach().contiguous().flatten()[sample_indices(name, p.numel())].double().cpu().numpy()
            assert np.abs(th - gd['theta_samples'][t][i]).max() <= bound, (t, name)


def test_keypoint_range_selects_the_joints_of_the_2d_terms(L):
    """dboa_loss_multi / dboa_loss_motion_joints with (first, count) = (0, 25) against torch on the reference formulas
    (dynaboa_webcam.py:236 and :161-181); (0, 0) keeps the benchmark's joints 25..48."""
    import ctypes as C
    from dynaboa_b200._lib import LossArgsStruct, ptr, stream
    lib = L.load()
    g = torch.Generator().manual_seed(5)
    B = 2
    p2d, j3d = torch.randn(B, 49, 2, generator=g).cuda(), torch.randn(B, 49, 3, generator=g).cuda()
    R, beta = torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda()
    kp = torch.randn(B, 49, 3, generator=g).cuda()
    kp[:, :, 2] = (torch.rand(B, 49, generator=g) > 0.3).float().cuda()
    for first, count in ((0, 25), (0, 0), (25, 24)):
        terms, dp2d = torch.empty(9, device='cuda'), torch.empty_like(p2d)
        a = LossArgsStruct()
        a.B = B
        for n, t in (('p2d', p2d), ('j3d', j3d), ('R', R), ('beta', beta), ('kp', kp), ('terms', terms), ('dp2d', dp2d)):
            setattr(a, n, t.data_ptr())
        a.w[0] = 3.0
        a.kp_first, a.kp_count = first, count
        L.call('dboa_loss_multi', C.byref(a), stream())
        f, n = (25, 24) if count == 0 else (first, count)
        x = p2d.double().clone().requires_grad_(True)
        ref = (((x[:, f:f + n] - kp[:, f:f + n, :2].double()) ** 2) * kp[:, f:f + n, 2:].double()).mean()
        (3.0 * ref).backward()
        assert abs(terms[0].item() - ref.item()) <= 1e-5 * abs(ref.item()), (first, count)
        assert rel_err(dp2d, x.grad) < 1e-5, (first, count)
    ph, kh = torch.randn(B, 49, 2, generator=g).cuda(), kp.roll(1, 1).contiguous()
    term, da, dh = torch.empty(1, device='cuda'), torch.empty_like(p2d), torch.empty_like(p2d)
    L.call('dboa_loss_motion_joints', ptr(p2d), ptr(ph), ptr(kp), ptr(kh), 0.8, ptr(term), ptr(da), ptr(dh), B, 0, 0, 25, stream())
    x, y = p2d.double().clone().requires_grad_(True), ph.double().clone().requires_grad_(True)
    conf = ((kp[:, :25, 2] + kh[:, :25, 2]) == 2).double().unsqueeze(-1)
    ref = ((((x[:, :25] - y[:, :25]) - (kp[:, :25, :2] - kh[:, :25, :2]).double()) ** 2) * conf).mean()
    (0.8 * ref).backward()
    assert abs(term.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-9
    assert rel_err(da, x.grad) < 1e-5 and rel_err(dh, y.grad) < 1e-5


def test_webcam_input_side_and_result_dictionary(asset_dir, tmp_path, golden):
    """``dataprocess`` (reference :197-218) on the GPU against the CPU restatement (oracle/dataprocess_ref.py), then one
    ``online_adaptation`` on the raw frame: result keys and shapes of the reference, base-model outputs side by side."""
    from oracle import dataprocess_ref as R
    gd = golden('adapt_webcam')
    ad = make_adaptor(tmp_path, gd, test_basemodel=1, dynamic_boa=0)
    rng = np.random.default_rng(3)
    frame = rng.uniform(0, 255, size=(240, 320, 3)).astype(np.uint8)
    det = np.concatenate([np.array([160.0, 120.0]) + rng.uniform(-60, 60, size=(25, 2)), rng.uniform(0, 1, size=(25, 1))], 1)
    image, kp, bbox = ad.dataprocess(frame, det, scaleFactor=1.2)
    x0, y0, x1, y1 = det[:, 0].min(), det[:, 1].min(), det[:, 0].max(), det[:, 1].max()
    center, scale = [(x1 + x0) / 2, (y1 + y0) / 2], 1.2 * max(x1 - x0, y1 - y0) / 200
    assert np.allclose(bbox, [[center[0], center[1], scale * 200]])
    ref_kp = det.copy()
    ref_kp[:, 2] = ref_kp[:, 2] > 0.3
    ref_kp = R.j2d_processing(ref_kp, center, scale)
    assert np.array_equal(kp[0, :25].cpu().numpy(), ref_kp.astype(np.float32)) and float(kp[0, 25:].abs().sum()) == 0.0
    ref_img = R.rgb_processing(frame.astype(np.float32), center, scale)
    assert rel_err(image[0], ref_img) < 1e-5
    res = ad.online_adaptation(frame, det[None])
    assert res['vts'].shape == (1, 6890, 3) and res['cam'].shape == (1, 3) and res['bbox'].shape == (1, 3)
    assert res['vts_base'].shape == (1, 6890, 3) and res['cam_base'].shape == (1, 3)
    assert torch.isfinite(res['vts']).all() and not torch.equal(res['vts'], res['vts_base'])      # one step moved the adapted model
    ad.reload()                                                                                   # key `r`: back to the base model
    with torch.no_grad():
        rot, shape, cam = ad.model(image)
    assert rel_err(cam, res['cam_base']) < 1e-5
