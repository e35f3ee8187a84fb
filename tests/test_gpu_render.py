"""Mesh overlay on the GPU (csrc/render.cu) against the numpy rasteriser of the same contract (oracle/render_ref.py): analytic
scenes, a closed tessellated sphere and the synthetic SMPL mesh posed by an HMR forward, 1x and 4x sampled.  The winning
face of every sample must be identical, the bytes within 1 wherever the faces agree, and uncovered pixels untouched.
Then determinism, the numpy / CUDA paths of ``Renderer.render``, the webcam ``render`` and the UNCHANGED
``dynaboa_internet.py`` with ``--save_res 1``."""
import os
import runpy
import sys

import numpy as np
import pytest
import torch

from harness import (CAM, COLOR, DRIVER, FLAGS, N, SHADOWED, check_against_oracle, frame, gpu_draw, make_video, posed_smpl_mesh, px_verts,
                     quad, sphere)
from oracle import render_ref

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def analytic_scenes():
    a, fa = quad(5, 5, 40, 30, 0.5)
    b, fb = quad(20.5, 15.5, 60, 45, -0.2, first=4)
    c, fc = quad(10, 10, 30, 20, 0.0, first=8, flip=True)                       # back-facing: culled
    d, fd = quad(2, 35, 30, 46, 1.5, first=12)                                   # beyond the far plane
    big = [(-100, -100, 0.9), (-100, 300, 0.9), (300, -100, 0.9)]                # covers the whole viewport, behind everything
    pts = a + b + c + d + big
    return px_verts(pts, 64, 48), np.array(fa + fb + fc + fd + [[16, 17, 18]])


@pytest.fixture(scope='module')
def posed_smpl(asset_dir):
    """harness.posed_smpl_mesh with the vertices on the host."""
    verts, faces, cam4 = posed_smpl_mesh()
    return verts.cpu().numpy(), faces, cam4


@pytest.mark.parametrize('samples', [1, 4])
def test_analytic_scenes_match_oracle(samples):
    verts, faces = analytic_scenes()
    img = frame(48, 64)
    _, ids = check_against_oracle(img, verts, faces, CAM, samples=samples, min_covered=48 * 64)
    assert set(np.unique(ids)) == {0, 1, 2, 3, 8}                               # quads a, b and the big face


@pytest.mark.parametrize('samples', [1, 4])
def test_sphere_matches_oracle(samples):
    from dynaboa_b200 import render
    v, f = sphere()
    img = frame(480, 640, 1)
    check_against_oracle(img, v, f, np.array([1.2, 1.6, 0.1, -0.05]), samples=samples, min_covered=20000)
    check_against_oracle(img, v, f, np.array([1.2, 1.6, 0.1, -0.05]), rot=render.rotation_matrix(30, [0, 1, 0]), samples=samples,
                         min_covered=20000)


@pytest.mark.parametrize('samples', [1, 4])
def test_posed_smpl_at_1080p_matches_oracle(posed_smpl, samples):
    verts, faces, cam4 = posed_smpl
    check_against_oracle(frame(1080, 1920, 2), verts, faces, cam4, samples=samples, min_covered=10000)


def test_two_calls_are_bit_identical(posed_smpl):
    verts, faces, cam4 = posed_smpl
    img = frame(1080, 1920, 3)
    o1, i1 = gpu_draw(img, verts, faces, cam4)
    o2, i2 = gpu_draw(img, verts, faces, cam4)
    assert np.array_equal(o1, o2) and np.array_equal(i1, i2)


def test_renderer_numpy_and_cuda_paths_agree(posed_smpl):
    from dynaboa_b200 import render
    verts, faces, _ = posed_smpl
    cam4 = render.convert_crop_cam_to_orig_img(np.array([[0.9, 0.0, 0.1]]), np.array([[320.0, 240.0, 300.0]]), 640, 480)[0]
    img = frame(480, 640, 4)
    r = render.Renderer(resolution=(640, 480), orig_img=True, wireframe=False)
    host = r.render(img, verts, cam4, color=COLOR)
    dev = r.render(torch.from_numpy(img).cuda(), torch.from_numpy(verts).cuda(), torch.tensor(cam4).cuda(), color=COLOR)
    assert isinstance(host, np.ndarray) and torch.is_tensor(dev) and dev.is_cuda
    assert np.array_equal(host, dev.cpu().numpy())
    assert not np.array_equal(host, img)


def test_webcam_render_returns_bgr_of_the_rgb_frame(posed_smpl):
    from dynaboa_b200 import render
    verts, faces, _ = posed_smpl
    rgb = frame(480, 640, 5)
    cam, bbox = torch.tensor([[0.9, 0.02, 0.08]]).cuda(), np.array([[330.0, 250.0, 320.0]])
    out = render.render(torch.from_numpy(verts)[None].cuda(), cam, torch.from_numpy(rgb).cuda(), bbox)
    assert torch.is_tensor(out) and out.is_cuda
    cam4 = render.convert_crop_cam_to_orig_img(cam.cpu().numpy(), bbox, 640, 480)[0]
    _, ids = gpu_draw(rgb, verts, faces, cam4, color=np.array([205, 129, 98]) / 255)
    ref, ref_ids = render_ref.render(rgb, verts, faces, cam4, color=np.array([205, 129, 98]) / 255, samples=4)
    assert np.array_equal(ids, ref_ids)
    assert np.abs(out.cpu().numpy().astype(int) - ref[:, :, ::-1].astype(int)).max() <= 1


@pytest.mark.skipif(not os.path.exists(DRIVER), reason='reference files not staged (oracle/_ref/, built from a reference checkout)')
def test_unchanged_internet_driver_with_save_res(asset_dir, tmp_path, monkeypatch):
    import cv2
    import joblib
    from dynaboa_b200 import base_adaptor, config, render
    root = tmp_path / 'video'
    make_video(str(root))
    drawn, saved = [], []
    render_fn, save_fn = render.Renderer.render, base_adaptor.BaseAdaptor.save_results

    def spy_render(self, img, verts, cam, *a, **k):
        drawn.append((img.cpu().numpy(), verts.detach().cpu().numpy(), np.array(cam, dtype=np.float64), np.array(k['color'])))
        return render_fn(self, img, verts, cam, *a, **k)

    def spy_save(self, vts, cam_trans, images, name, bbox, prefix=None):
        saved.append((cam_trans.detach().cpu().numpy(), np.asarray(bbox.cpu() if torch.is_tensor(bbox) else bbox), self.global_step))
        return save_fn(self, vts, cam_trans, images, name, bbox, prefix=prefix)
    monkeypatch.setattr(render.Renderer, 'render', spy_render)
    monkeypatch.setattr(base_adaptor.BaseAdaptor, 'save_results', spy_save)
    monkeypatch.setenv('DYNABOA_INTERNET_ROOT', str(root))
    monkeypatch.chdir(tmp_path)
    dropin = os.path.join(REPO, 'dynaboa_b200', 'dropin')
    stash = {m: sys.modules.pop(m) for m in list(sys.modules) if m.split('.')[0] in SHADOWED + ('render_demo',)}
    monkeypatch.setattr(sys, 'path', [dropin, REPO] + sys.path)
    argv = [DRIVER, '--expdir', str(tmp_path / 'exps'), '--expname', 'net', '--dataset', 'internet', '--model_file', config.BASE_MODEL,
            '--save_res', '1']
    for k, v in FLAGS.items():
        argv += [f'--{k}', str(v)]
    monkeypatch.setattr(sys, 'argv', argv)
    try:
        runpy.run_path(DRIVER, run_name='__main__')
    finally:
        for m in list(sys.modules):
            if m.split('.')[0] in SHADOWED + ('render_demo',):
                del sys.modules[m]
        sys.modules.update(stash)
    assert len(drawn) == N and len(saved) == N
    faces = render.get_smpl_faces()
    for t in range(N):
        png = cv2.imread(str(tmp_path / 'exps' / 'net' / 'image' / f'Pred_{t}.png'))
        assert png is not None and png.shape == (240, 320, 3), t
        img, verts, cam4, color = drawn[t]
        cam_trans, bbox, step = saved[t]
        assert step == t
        pred = joblib.load(tmp_path / 'exps' / 'net' / 'result' / f'Pred_{t}.pt')
        assert np.array_equal(verts, pred['verts'][0]), t
        cam_t = np.stack([cam_trans[:, 1], cam_trans[:, 2], 2 * 5000. / (224 * cam_trans[:, 0] + 1e-9)], -1)
        assert np.allclose(cam_t, pred['cam'], rtol=1e-6, atol=1e-6), t
        assert np.array_equal(cam4, render.convert_crop_cam_to_orig_img(cam_trans, bbox, 320, 240)[0]), t
        assert np.allclose(color, np.array([205, 129, 98]) / 255)
        assert np.array_equal(img, cv2.imread(str(root / 'images' / f'f{t:03d}.png')))
        out, ids = gpu_draw(img, verts, faces, cam4, color=color)
        assert np.array_equal(out, png), t
        ref, ref_ids = render_ref.render(img, verts, faces, cam4, color=color, samples=4)
        assert np.array_equal(ids, ref_ids), t
        covered = (ids >= 0).any(2)
        assert covered.any() and np.array_equal(png[~covered], img[~covered])
        assert np.abs(png.astype(int) - ref.astype(int))[covered].max() <= 1, t
    lines = open(tmp_path / 'demo.obj').read().splitlines()
    assert sum(1 for s in lines if s.startswith('v ')) == 6890 and sum(1 for s in lines if s.startswith('f ')) == 13776
