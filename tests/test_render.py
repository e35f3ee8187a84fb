"""Mesh overlay on the CPU: the numpy rasteriser of the contract (oracle/render_ref.py) on analytic scenes, the camera
conversion against the reference's own function, and the C-ABI argument checks (no GPU needed)."""
import ctypes
import os

import numpy as np
import pytest

from harness import CAM, px_verts, quad
from oracle import render_ref

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def raster(pts, faces, W, H, samples):
    p, X, Y, z, ok = render_ref.transform(px_verts(pts, W, H), CAM, None, W, H)
    return render_ref.rasterise(np.array(faces), X, Y, z, ok, W, H, samples)


scenes_geom = [(s, e) for s in (1, 4) for e in (10.0, 10.5)]


@pytest.mark.parametrize('samples,edge', scenes_geom)
def test_shared_edge_covered_once(samples, edge):
    W = H = 64
    pts, faces = quad(edge, edge, edge + 32, edge + 32, 0.0)
    both = raster(pts, faces, W, H, samples)
    single = [raster(pts, [f], W, H, samples) >= 0 for f in faces]
    assert not (single[0] & single[1]).any(), 'a sample on the shared diagonal was covered twice'
    assert ((single[0] | single[1]) == (both >= 0)).all()
    # the diagonal runs through sample points; the square's area in samples is exact under the top-left rule
    assert (both >= 0).sum() == 32 * 32 * samples
    assert (both == 0).sum() > 0 and (both == 1).sum() > 0


def test_nearer_quad_wins():
    W, H = 64, 48
    a, fa = quad(5, 5, 40, 30, 0.5)
    b, fb = quad(20, 15, 60, 45, -0.2, first=4)
    fid = raster(a + b, fa + fb, W, H, 1)
    assert set(np.unique(fid[20:30, 25:40])) <= {2, 3}                     # overlap: quad b (ndc_z -0.2) is nearer
    assert set(np.unique(fid[6:14, 6:18])) <= {0, 1}
    # equal depth: the lower face id wins
    fid = raster(a + [(x, y, 0.5) for x, y, _ in b], fa + fb, W, H, 1)
    assert set(np.unique(fid[20:30, 25:40])) <= {0, 1}


def test_back_facing_quad_is_culled():
    pts, faces = quad(5, 5, 40, 30, 0.0, flip=True)
    assert (raster(pts, faces, 48, 40, 4) == -1).all()
    pts, faces = quad(5, 5, 40, 30, 0.0)
    assert (raster(pts, faces, 48, 40, 4) >= 0).sum() == 35 * 25 * 4


@pytest.mark.parametrize('d', [1.5, -1.25])
def test_outside_depth_range_is_discarded(d):
    pts, faces = quad(5, 5, 40, 30, d)
    assert (raster(pts, faces, 48, 40, 1) == -1).all()
    # a face crossing the far plane keeps exactly its fragments with ndc_z <= 1
    pts = [(0, 0, 0.0), (48, 0, 2.0), (48, 40, 2.0), (0, 40, 0.0)]           # ndc_z = column / 24
    fid = raster(pts, [[0, 3, 2], [0, 2, 1]], 48, 40, 1)
    assert (fid[:, :24] >= 0).all() and (fid[:, 24:] == -1).all()


def test_one_face_covers_the_viewport():
    W, H = 40, 30
    pts = [(-100, -100, 0.0), (-100, 300, 0.0), (300, -100, 0.0)]
    for s in (1, 4):
        assert (raster(pts, [[0, 1, 2]], W, H, s) == 0).all()


def test_half_covered_pixel_with_4_samples():
    W, H = 16, 16
    pts, faces = quad(7.5, 2, 14, 14, 0.0)                   # left edge through the centres of column 7
    v = px_verts(pts, W, H)
    img = np.full((H, W, 3), 77, np.uint8)
    out4, fid4 = render_ref.render(img, v, faces, CAM, samples=4)
    out1, fid1 = render_ref.render(img, v, faces, CAM, samples=1)
    col = fid4[5, 7]
    assert (col >= 0).sum() == 2                                  # coverage 2/4: the samples right of the centre
    assert fid1[5, 7, 0] >= 0                                    # the centre is on a left edge: covered
    b = out1[5, 7].astype(int)                                   # the face's byte, shaded at the same centre
    assert (out4[5, 7].astype(int) == (2 * b + 2) // 4).all()   # darkened towards black
    assert (out4[5, 5] == 77).all() and (out4[5, 9] == out1[5, 9]).all()


def test_convert_crop_cam_matches_reference(golden):
    from dynaboa_b200 import render
    g = golden('render_cam')
    for (w, h), ref in zip(g['sizes'], g['orig_cam']):
        got = render.convert_crop_cam_to_orig_img(g['cam'], g['bbox'], int(w), int(h))
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


def test_wireframe_is_rejected():
    from dynaboa_b200 import render
    with pytest.raises(NotImplementedError):
        render.Renderer(resolution=(64, 48), wireframe=True)


def test_abi_argument_errors_without_gpu():
    from dynaboa_b200 import _lib, build
    build.build()
    lib = _lib.load()
    assert lib.dboa_render_scratch_bytes(9000, 10, 6890, 13776, 4) == -2
    assert lib.dboa_render_scratch_bytes(640, 480, -1, 10, 4) == -2
    assert lib.dboa_render_scratch_bytes(640, 480, 10, 10, 2) == -1
    assert lib.dboa_render_scratch_bytes(640, 480, 6890, 13776, 4) >= 640 * 480 * 4 * 8
    cam = (ctypes.c_float * 4)(1, 1, 0, 0)
    col = (ctypes.c_float * 3)(1, 1, 1)
    fake = ctypes.c_void_p(16)
    args = [fake] * 4 + [3, 1, cam, None, col, fake]
    assert lib.dboa_render_overlay(None, *args[1:], 64, 48, 4, fake, 1 << 30, fake, None, None) == -1
    assert lib.dboa_render_overlay(*args, 9000, 48, 4, fake, 1 << 30, fake, None, None) == -2
    assert lib.dboa_render_overlay(*args, 64, 48, 3, fake, 1 << 30, fake, None, None) == -1
    assert lib.dboa_render_overlay(*args, 64, 48, 4, fake, 16, fake, None, None) == -1      # scratch too small
    assert lib.dboa_render_overlay(*args[:6], None, None, col, fake, 64, 48, 4, fake, 1 << 30, fake, None, None) == -1
