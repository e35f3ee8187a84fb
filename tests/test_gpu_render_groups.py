"""Grouped mesh overlay (dboa_render_overlay_groups) on the GPU.

- Each mesh equals itself drawn alone: M = 1 .. 64 meshes over frames of mixed sizes up to 1920 x 1080, 1x and 4x sampled,
  with their own cameras, rotations and colours, a mesh wholly off the frame, a mesh beyond the far plane and two entries
  reading one frame; every entry's out and face_ids are bit-identical to dboa_render_overlay on that entry alone and the
  input frames are left unchanged.
- Two grouped entries against the numpy rasteriser of the contract (oracle/render_ref.py).
- Determinism and the launch count (6 kernels whatever M).
- MultiWebcamAdaptor.render on a four-stream pool against render.render per stream."""
import ctypes

import numpy as np
import pytest
import torch

from harness import SIZES, check_against_oracle, frame, posed_smpl_mesh, sphere, webcam_pool
from oracle import render_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def posed_smpl(asset_dir):
    """harness.posed_smpl_mesh with the vertices on the host."""
    verts, faces, cam4 = posed_smpl_mesh()
    return verts.cpu().numpy(), faces, cam4


def entries(verts, M, seed):
    """M (frame, verts, cam4, rot, colour) entries over frames of SIZES.  Entry 1 reads entry 0's frame, entry 3 lies wholly off
    its frame, entry 4 beyond the far plane; the others differ in crop camera, rotation (every other one) and colour."""
    from dynaboa_b200 import render
    rng = np.random.default_rng(seed)
    frames, out = {}, []
    for k in range(M):
        H, W = SIZES[k % len(SIZES)]
        src = 0 if k == 1 else k
        if src not in frames:
            frames[src] = torch.from_numpy(frame(H, W, seed * 100 + k)).cuda()
        img = frames[src]
        H, W = img.shape[:2]
        box = np.array([[rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H, rng.uniform(0.4, 0.9) * min(H, W)]])
        cam = np.array([[rng.uniform(0.7, 1.1), rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.2)]])
        cam4 = render.convert_crop_cam_to_orig_img(cam, box, W, H)[0]
        v = verts + torch.from_numpy(rng.normal(0, 0.003, size=verts.shape).astype(np.float32)).cuda()
        if k == 3:
            cam4 = cam4 + np.array([0, 0, 40.0, 0])                        # 20 frame widths to the right
        if k == 4:
            v = v + torch.tensor([0.0, 0.0, 3.0], device='cuda')          # ndc_z > 1 everywhere
        rot = render.rotation_matrix(rng.uniform(-40, 40), rng.normal(size=3)) if k % 2 else None
        out.append((img, v, cam4, rot, rng.uniform(0.2, 1.0, size=3)))
    return out


def single(e, faces, samples):
    """dboa_render_overlay on one entry, through its own scratch."""
    from dynaboa_b200 import _lib, render
    img, v, cam4, rot, col = e
    lib = _lib.load()
    H, W = img.shape[:2]
    f_dev, vf_off, vf_faces = render._device_faces(faces, v.shape[0], img.device)
    need = lib.dboa_render_scratch_bytes(W, H, v.shape[0], f_dev.shape[0], samples)
    scratch = torch.empty(need, dtype=torch.uint8, device='cuda')
    out = torch.empty_like(img)
    ids = torch.empty(H, W, samples, dtype=torch.int32, device='cuda')
    F = ctypes.c_float
    R = None if rot is None else (F * 9)(*np.asarray(rot, dtype=np.float64).reshape(9))
    _lib.call('dboa_render_overlay', _lib.ptr(v.contiguous()), _lib.ptr(f_dev), _lib.ptr(vf_off), _lib.ptr(vf_faces), v.shape[0],
              f_dev.shape[0], (F * 4)(*cam4), R, (F * 3)(*col), _lib.ptr(img), W, H, samples, _lib.ptr(scratch), need, _lib.ptr(out),
              _lib.ptr(ids), _lib.stream())
    return out, ids


def grouped(es, faces, samples):
    from dynaboa_b200 import render
    return render.draw_groups([e[0] for e in es], [e[1] for e in es], faces, [e[2] for e in es], [e[4] for e in es],
                              rots=[e[3] for e in es], samples=samples, face_ids=True)


@pytest.mark.parametrize('samples', [1, 4])
@pytest.mark.parametrize('M', [1, 2, 5, 16, 64])
def test_each_mesh_is_itself_drawn_alone(posed_smpl, M, samples):
    verts, faces, _ = posed_smpl
    es = entries(torch.from_numpy(verts).cuda(), M, M * 10 + samples)
    before = {id(e[0]): e[0].clone() for e in es}
    outs, ids = grouped(es, faces, samples)
    torch.cuda.synchronize()
    for e in es:
        assert torch.equal(e[0], before[id(e[0])])
    for k, e in enumerate(es):
        ref_out, ref_ids = single(e, faces, samples)
        assert outs[k].shape == e[0].shape and ids[k].shape == (*e[0].shape[:2], samples), k
        assert torch.equal(ids[k], ref_ids), k
        assert torch.equal(outs[k], ref_out), k
        covered = int((ids[k] >= 0).any(2).sum())
        if k in (3, 4):
            assert covered == 0 and torch.equal(outs[k], e[0]), k                  # off the frame / beyond the far plane
        elif e[3] is None:
            assert covered > 0, k
    if M >= 2:
        assert outs[0].data_ptr() != outs[1].data_ptr() and not torch.equal(ids[0], ids[1])   # one frame, two results


def test_sphere_entries_are_themselves_drawn_alone():
    v, f = sphere()
    es = entries(torch.from_numpy(v).cuda(), 6, 5)
    for samples in (1, 4):
        outs, ids = grouped(es, f, samples)
        for k, e in enumerate(es):
            ref_out, ref_ids = single(e, f, samples)
            assert torch.equal(ids[k], ref_ids) and torch.equal(outs[k], ref_out), (samples, k)


@pytest.mark.parametrize('samples', [1, 4])
def test_two_grouped_entries_match_the_oracle(samples):
    from dynaboa_b200 import render
    v, f = sphere()
    imgs = [frame(120, 160, 11), frame(150, 200, 12)]
    cams = [np.array([1.2, 1.6, 0.1, -0.05]), np.array([1.0, 1.3, -0.2, 0.1])]
    rots = [None, render.rotation_matrix(30, [0, 1, 0])]
    cols = [np.array([205, 129, 98]) / 255, np.array([100, 100, 200]) / 255]
    outs, ids = render.draw_groups([torch.from_numpy(i).cuda() for i in imgs], [torch.from_numpy(v).cuda()] * 2, f, cams, cols, rots=rots,
                                   samples=samples, face_ids=True)
    for k in range(2):
        out, fid = outs[k].cpu().numpy(), ids[k].cpu().numpy()
        ref_out, ref_ids = render_ref.render(imgs[k], v, f, cams[k], rot=rots[k], color=cols[k], samples=samples)
        assert np.array_equal(fid, ref_ids), k
        covered = (fid >= 0).any(2)
        assert covered.sum() > 2000, k
        assert np.array_equal(out[~covered], imgs[k][~covered]), k
        assert np.abs(out.astype(int) - ref_out.astype(int))[covered].max() <= 1, k
    check_against_oracle(imgs[1], v, f, cams[1], rot=rots[1], color=cols[1], samples=samples, min_covered=2000)   # the M = 1 path too


@pytest.mark.parametrize('M', [1, 64])
def test_deterministic_and_six_launches(posed_smpl, M):
    from dynaboa_b200 import _lib
    verts, faces, _ = posed_smpl
    es = entries(torch.from_numpy(verts).cuda(), M, 3)
    lib = _lib.load()
    first = grouped(es, faces, 4)
    torch.cuda.synchronize()
    n0 = lib.dboa_launch_count()
    second = grouped(es, faces, 4)
    torch.cuda.synchronize()
    assert lib.dboa_launch_count() - n0 == 6
    for a, b in zip(first[0] + first[1], second[0] + second[1]):
        assert torch.equal(a, b)


def webcam_ticks(seed):
    """One tick of four cameras: numpy 720p, CUDA 320x240, numpy 640x480 (this one sees nobody), CUDA 1080p; uint8 RGB."""
    rng = np.random.default_rng(seed)
    frames, dets = [], []
    for g, (H, W) in enumerate([(720, 1280), (240, 320), (480, 640), (1080, 1920)]):
        img = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
        frames.append(img if g % 2 == 0 else torch.from_numpy(img).cuda())
        c = np.array([W / 2, H / 2]) + rng.uniform(-W / 8, W / 8, size=2)
        d = np.concatenate([c + rng.uniform(-H / 4, H / 4, size=(25, 2)), rng.uniform(0, 1, size=(25, 1))], 1)
        dets.append(None if g == 2 else d[None])
    return frames, dets


@pytest.mark.parametrize('test_basemodel', [1, 0])
def test_pool_render_is_render_per_stream(asset_dir, tmp_path, golden, test_basemodel):
    from dynaboa_b200 import render
    gd = golden('adapt_webcam')
    mv = webcam_pool(tmp_path, gd, 4, 'mv', test_basemodel=test_basemodel, dynamic_boa=0)
    frames, dets = webcam_ticks(4)
    res = mv.online_adaptation(frames, dets)
    assert res[2] is None
    before = [f.clone() if torch.is_tensor(f) else f.copy() for f in frames]
    drawn = mv.render(frames, res)
    assert drawn[2] is None
    for g in (0, 1, 3):
        f, r = frames[g], res[g]
        img, base = drawn[g]
        ref = render.render(r['vts'], r['cam'], f, r['bbox'])
        assert type(img) is type(ref) and (not torch.is_tensor(img) or img.is_cuda), g
        to_np = (lambda x: x.cpu().numpy()) if torch.is_tensor(ref) else np.asarray
        assert np.array_equal(to_np(img), to_np(ref)), g
        if test_basemodel:
            ref_b = render.render(r['vts_base'], r['cam_base'], f, r['bbox'], color=[100, 100, 200])
            assert type(base) is type(ref_b) and np.array_equal(to_np(base), to_np(ref_b)), g
        else:
            assert base is None
        assert np.array_equal(to_np(f), to_np(before[g])), g
