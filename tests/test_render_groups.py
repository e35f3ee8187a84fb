"""Grouped mesh overlay without a GPU: the error codes of dboa_render_overlay_groups and its size query (fake device pointers,
every check happens before any device access), the scratch size against the one-mesh query, and the Python argument checks of
render.draw_groups and MultiWebcamAdaptor.render."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from harness import built_lib, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def ints(*v):
    return (ctypes.c_int * len(v))(*v)


def descs(n, W=64, H=48, fake=16):
    from dynaboa_b200 import _lib
    d = (_lib.RenderDescStruct * n)()
    for k in range(n):
        d[k].verts = d[k].img = d[k].out = fake
        d[k].cam4[:] = [1, 1, 0, 0]
        d[k].color3[:] = [1, 1, 1]
        d[k].W, d[k].H = W, H
    return d


def test_scratch_of_one_entry_is_the_one_mesh_scratch(lib):
    for W, H, nv, nf, s in [(640, 480, 6890, 13776, 4), (1920, 1080, 6890, 13776, 1), (7, 3, 0, 0, 4), (8192, 8192, 10, 5, 1)]:
        assert lib.dboa_render_scratch_bytes_groups(ints(W), ints(H), 1, nv, nf, s) == lib.dboa_render_scratch_bytes(W, H, nv, nf, s)
    one = [lib.dboa_render_scratch_bytes(w, h, 6890, 13776, 4) for w, h in [(640, 480), (1280, 720), (320, 240)]]
    both = lib.dboa_render_scratch_bytes_groups(ints(640, 1280, 320), ints(480, 720, 240), 3, 6890, 13776, 4)
    assert both == sum(one)                                   # every array on 256 bytes: the layouts add up


def test_scratch_query_errors(lib):
    q = lib.dboa_render_scratch_bytes_groups
    assert q(None, ints(48), 1, 10, 10, 4) == -1
    assert q(ints(64), None, 1, 10, 10, 4) == -1
    assert q(ints(64), ints(48), 0, 10, 10, 4) == -2
    assert q(ints(*[64] * 65), ints(*[48] * 65), 65, 10, 10, 4) == -2
    assert q(ints(64, 9000), ints(48, 48), 2, 10, 10, 4) == -2
    assert q(ints(64, 64), ints(48, 0), 2, 10, 10, 4) == -2
    assert q(ints(64), ints(48), 1, -1, 10, 4) == -2
    assert q(ints(64), ints(48), 1, 10, -1, 4) == -2
    assert q(ints(64), ints(48), 1, 10, 10, 2) == -1
    assert q(ints(*[64] * 64), ints(*[48] * 64), 64, 10, 10, 1) > 0


def test_abi_argument_errors_without_gpu(lib):
    fake = ctypes.c_void_p(16)
    call = lib.dboa_render_overlay_groups
    big = 1 << 40

    def run(d, M=None, faces=fake, vo=fake, vf=fake, nv=3, nf=1, s=4, scratch=fake, nbytes=big):
        return call(d, len(d) if M is None else M, faces, vo, vf, nv, nf, s, scratch, nbytes, None)
    assert call(None, 1, fake, fake, fake, 3, 1, 4, fake, big, None) == -1
    assert run(descs(1), faces=None) == -1
    assert run(descs(1), vo=None) == -1
    assert run(descs(1), vf=None) == -1
    assert run(descs(1), scratch=None) == -1
    assert run(descs(1), M=0) == -2
    assert run(descs(65)) == -2
    assert run(descs(2), nv=-1) == -2
    assert run(descs(2), nf=-1) == -2
    for field, v in (('W', 0), ('W', 8193), ('H', 0), ('H', 8193)):
        d = descs(3)
        setattr(d[2], field, v)
        assert run(d) == -2, (field, v)
    assert run(descs(2), s=2) == -1
    for field in ('verts', 'img', 'out'):
        d = descs(3)
        setattr(d[1], field, None)
        assert run(d) == -1, field
    d = descs(2)
    need = lib.dboa_render_scratch_bytes_groups(ints(64, 64), ints(48, 48), 2, 3, 1, 4)
    assert run(d, nbytes=need - 1) == -1
    d[0].face_ids = None                                    # optional: still only the scratch size is wrong
    assert run(d, nbytes=16) == -1


FACES = np.array([[0, 1, 2]])


def test_draw_groups_argument_checks():
    from dynaboa_b200 import render
    img = torch.zeros(4, 5, 3, dtype=torch.uint8)
    v = torch.zeros(3, 3)
    cam, col = np.array([1.0, 1, 0, 0]), np.array([1.0, 1, 1])
    with pytest.raises(ValueError, match='1 to 64'):
        render.draw_groups([], [], FACES, [], [])
    with pytest.raises(ValueError, match='1 to 64'):
        render.draw_groups([img] * 65, [v] * 65, FACES, [cam] * 65, [col] * 65)
    with pytest.raises(ValueError, match='one per frame'):
        render.draw_groups([img] * 2, [v], FACES, [cam] * 2, [col] * 2)
    with pytest.raises(ValueError, match='one per frame'):
        render.draw_groups([img] * 2, [v] * 2, FACES, [cam], [col] * 2)
    with pytest.raises(ValueError, match='one per frame'):
        render.draw_groups([img] * 2, [v] * 2, FACES, [cam] * 2, [col] * 2, rots=[None])
    with pytest.raises(ValueError, match='samples'):
        render.draw_groups([img], [v], FACES, [cam], [col], samples=2)
    with pytest.raises(ValueError, match='entry 1: img must be an'):
        render.draw_groups([img, img.float()], [v] * 2, FACES, [cam] * 2, [col] * 2)
    with pytest.raises(ValueError, match='entry 0: img must be an'):
        render.draw_groups([torch.zeros(4, 5, 4, dtype=torch.uint8)], [v], FACES, [cam], [col])
    with pytest.raises(RuntimeError, match='CUDA'):
        render.draw_groups([img], [v], FACES, [cam], [col])       # host tensors: there is no CPU path


def test_render_groups_argument_checks():
    from dynaboa_b200 import render
    assert render.render_groups([], [], [], [], []) == []
    with pytest.raises(ValueError, match='one per image'):
        render.render_groups([None], [None, None], [None], [None], [None])


def test_pool_render_argument_checks():
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    mv = idle_pool(MultiWebcamAdaptor, 3, options=SimpleNamespace(test_basemodel=1))
    frame = np.zeros((48, 64, 3), np.uint8)
    res = {'vts': None, 'cam': None, 'bbox': None, 'vts_base': None, 'cam_base': None}
    with pytest.raises(ValueError, match='3 frames and 3 results'):
        mv.render([frame] * 2, [res] * 3)
    with pytest.raises(ValueError, match='3 frames and 3 results'):
        mv.render([frame] * 3, [res] * 4)
    with pytest.raises(ValueError, match='stream 1: expected the'):
        mv.render([frame, frame.astype(np.float32), frame], [res] * 3)
    with pytest.raises(ValueError, match='stream 2: expected the'):
        mv.render([frame, frame, np.zeros((48, 64), np.uint8)], [res] * 3)
    with pytest.raises(ValueError, match='stream 0: expected the'):
        mv.render([None, frame, frame], [res] * 3)
    assert mv.render([None, None, frame.astype(np.float32)], [None] * 3) == [None] * 3   # no result: the frame is not looked at
