"""Webcam pool without a device: the bindings of dboa_crop_resize_normalize_groups / dboa_keypoint_transform_groups and their
argument errors (returned on the host before any device access), the ctypes mirror of dboa_crop_desc against the compiled
header, and the argument checks of MultiWebcamAdaptor.online_adaptation / adapt_processed."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from dynaboa_b200 import _lib, build

DBOA_ERR_ARG, DBOA_ERR_SHAPE = -1, -2
FAKE = 0x1000            # stand-in device pointers: every case below is rejected before one is dereferenced
P, I, L, U = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_ulonglong


@pytest.fixture(scope='module')
def lib():
    build.build()
    return _lib.load()


def descs(groups, **over):
    """`groups` valid descriptors of a 480 x 640 frame cropped to 300 rows; over: field -> value for descriptor 0."""
    a = (_lib.CropDescStruct * max(groups, 1))()
    for d in a:
        d.img = d.wx = d.sx = d.wy = d.sy = FAKE
        d.is_u8, d.H, d.W, d.ul_x, d.ul_y, d.Hc, d.Tx, d.Ty = 1, 480, 640, -10, 20, 300, 4, 4
    for k, v in over.items():
        setattr(a[0], k, v)
    return a


def crop(lib, groups=2, active=0b11, res=224, tmp_floats=10 ** 9, frames=None, null=None):
    frames = descs(groups) if frames is None else frames
    p = [frames, (ctypes.c_float * 3)(), (ctypes.c_float * 3)(), P(FAKE), P(FAKE)]
    if null is not None:
        p[null] = None
    return lib.dboa_crop_resize_normalize_groups(p[0], groups, active, res, p[1], p[2], p[3], tmp_floats, p[4], None)


def keypoints(lib, n=25, groups=2, active=0b11, res=224, null=None):
    p = [P(FAKE), (ctypes.c_double * (4 * max(groups, 1)))(), P(FAKE)]
    if null is not None:
        p[null] = None
    return lib.dboa_keypoint_transform_groups(p[0], n, p[1], res, p[2], groups, active, None)


def test_bindings():
    sig = _lib.SIGNATURES
    assert sig['dboa_crop_resize_normalize_groups'] == (I, [ctypes.POINTER(_lib.CropDescStruct), I, U, I, P, P, P, L, P, P])
    assert sig['dboa_keypoint_transform_groups'] == (I, [P, I, ctypes.POINTER(ctypes.c_double), I, P, I, U, P])
    # the per-frame fields of the one-frame call, in its order
    one = sig['dboa_crop_resize_normalize'][1]
    assert one[:7] == [P, I, I, I, I, I, I] and [f[0] for f in _lib.CropDescStruct._fields_][5:] == ['is_u8', 'H', 'W', 'ul_x', 'ul_y',
                                                                                                   'Hc', 'Tx', 'Ty']


def test_descriptor_layout_matches_the_header(tmp_path):
    """offsetof / sizeof of dboa_crop_desc compiled from the header against the ctypes mirror."""
    fields = [f[0] for f in _lib.CropDescStruct._fields_]
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "dynaboa_b200.h"\nint main(void) {\n'
                   + ''.join(f'  printf("%zu\\n", offsetof(dboa_crop_desc, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(dboa_crop_desc));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(repo, 'include'), str(src), '-o', str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = [getattr(_lib.CropDescStruct, f).offset for f in fields] + [ctypes.sizeof(_lib.CropDescStruct)]
    assert got == want
    assert 64 * got[-1] < 32 * 1024                          # 64 descriptors fit the kernel parameter space


@pytest.mark.parametrize('null', range(5))
def test_crop_null_pointers(lib, null):
    assert crop(lib, null=null) == DBOA_ERR_ARG


@pytest.mark.parametrize('field', ['img', 'wx', 'sx', 'wy', 'sy'])
def test_crop_null_descriptor_pointers(lib, field):
    assert crop(lib, frames=descs(2, **{field: None})) == DBOA_ERR_ARG
    assert crop(lib, active=0b10, frames=descs(2, **{field: None}), tmp_floats=0) == DBOA_ERR_ARG       # idle: not read; tmp


@pytest.mark.parametrize('kw', [dict(groups=0), dict(groups=65), dict(groups=-1), dict(res=0), dict(res=-224)])
def test_crop_shape_errors(lib, kw):
    assert crop(lib, **kw) == DBOA_ERR_SHAPE
    assert crop(lib, active=0, **kw) == DBOA_ERR_SHAPE          # the shape is checked before the mask


@pytest.mark.parametrize('field', ['H', 'W', 'Hc', 'Tx', 'Ty'])
@pytest.mark.parametrize('value', [0, -3])
def test_crop_descriptor_shape_errors(lib, field, value):
    assert crop(lib, frames=descs(2, **{field: value})) == DBOA_ERR_SHAPE
    # an idle stream's descriptor is not looked at: the error left is the scratch size, which counts the active frame only
    assert crop(lib, active=0b10, frames=descs(2, **{field: value}), tmp_floats=300 * 224 * 3 - 1) == DBOA_ERR_ARG


@pytest.mark.parametrize('groups,active', [(2, 0), (2, 0b100), (4, 0b10000), (4, 1 << 63), (1, 0b10), (1, 0), (8, 1 << 8)])
def test_crop_mask_errors(lib, groups, active):
    assert crop(lib, groups=groups, active=active) == DBOA_ERR_ARG


def test_crop_scratch_size(lib):
    need = 300 * 224 * 3
    assert crop(lib, groups=3, active=0b101, tmp_floats=2 * need - 1) == DBOA_ERR_ARG
    assert crop(lib, groups=1, active=1, tmp_floats=need - 1) == DBOA_ERR_ARG
    assert crop(lib, groups=64, active=~0 & (2 ** 64 - 1), tmp_floats=64 * need - 1) == DBOA_ERR_ARG


@pytest.mark.parametrize('null', range(3))
def test_keypoint_null_pointers(lib, null):
    assert keypoints(lib, null=null) == DBOA_ERR_ARG


@pytest.mark.parametrize('kw', [dict(groups=0), dict(groups=65), dict(n=-1), dict(n=50), dict(res=0)])
def test_keypoint_shape_errors(lib, kw):
    assert keypoints(lib, **kw) == DBOA_ERR_SHAPE
    assert keypoints(lib, active=0, **kw) == DBOA_ERR_SHAPE


@pytest.mark.parametrize('groups,active', [(2, 0), (2, 0b100), (1, 0b10), (8, 1 << 8), (63, 1 << 63)])
def test_keypoint_mask_errors(lib, groups, active):
    assert keypoints(lib, groups=groups, active=active) == DBOA_ERR_ARG


# ------------------------------------------------------------------ the pool's checks
def pool(G=3):
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    mv = MultiWebcamAdaptor.__new__(MultiWebcamAdaptor)        # no device: only the checks before any device work run
    mv.G = G
    return mv


def frame():
    return np.zeros((48, 64, 3), np.uint8)


def det(shape=(1, 25, 3)):
    return np.random.default_rng(0).uniform(5, 40, size=shape)


def test_online_adaptation_checks():
    mv = pool(3)
    with pytest.raises(ValueError, match='3 frames'):
        mv.online_adaptation([frame()] * 2, [det()] * 3)
    with pytest.raises(ValueError, match='3 frames'):
        mv.online_adaptation([frame()] * 3, [det()] * 4)
    for bad in ((25, 2), (2, 25, 3), (24, 3), (25,)):
        with pytest.raises(ValueError, match=r'stream 1: detections'):
            mv.online_adaptation([None, frame(), frame()], [det(), det(bad), det()])
    for f in (np.zeros((48, 64), np.uint8), np.zeros((48, 64, 4), np.uint8), np.zeros((48, 64, 3), np.float64)):
        with pytest.raises(ValueError, match='stream 2: expected'):
            mv.online_adaptation([None, None, f], [None, None, det((25, 3))])
    assert mv.online_adaptation([None] * 3, [None] * 3) == [None] * 3      # nobody in view: nothing advances
    assert mv.online_adaptation([frame(), None, None], [None, det(), None]) == [None] * 3


def test_adapt_processed_checks():
    import torch
    mv = pool(2)
    img, kp = torch.zeros(1, 3, 224, 224), torch.zeros(1, 49, 3)
    with pytest.raises(ValueError, match='2 images'):
        mv.adapt_processed([img], [kp, kp])
    with pytest.raises(ValueError, match='both'):
        mv.adapt_processed([img, img], torch.zeros(2, 49, 3))
    with pytest.raises(ValueError, match='stream 1'):
        mv.adapt_processed([img, img], [kp, torch.zeros(1, 25, 3)])
    with pytest.raises(ValueError, match=r'\(2, 3, 224, 224\)'):
        mv.adapt_processed(torch.zeros(3, 3, 224, 224), torch.zeros(3, 49, 3))
    assert mv.adapt_processed([None, img], [kp, None]) == [None, None]
    assert mv.adapt_processed(torch.zeros(2, 3, 224, 224), torch.zeros(2, 49, 3), active=0) == [None, None]


def webcam_opts(**extra):
    from dynaboa_b200.webcam import webcam_options
    o = dict(lr=3e-6, beta1=0.5, beta2=0.9, fastlr=8e-6, s2dloss_weight=10.0, shape_prior_weight=2e-6, pose_prior_weight=1e-4,
             use_boa=1, model_file='unused', expdir='/nonexistent')
    o.update(extra)
    return webcam_options(SimpleNamespace(**o))


def test_pool_options(lib):
    from dynaboa_b200.multivideo import check_options
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    assert MultiWebcamAdaptor.kp_range == (0, 25) and MultiWebcamAdaptor.motion_lead == 1
    o = webcam_opts(dynamic_boa=1)
    assert o.retrieval == 0 and o.teacher_dropout == 0 and o.batch_size == 1
    with pytest.raises(ValueError, match='dynamic_loop'):
        check_options(o, 2)
    check_options(o, 64, dynamic_loop=True)
    with pytest.raises(ValueError, match='exceed'):
        check_options(o, 65, dynamic_loop=True)
    prev = lib.dboa_get_fused_forward()
    lib.dboa_set_fused_forward(1)
    try:
        with pytest.raises(ValueError, match='fused'):
            check_options(webcam_opts(), 2)
    finally:
        lib.dboa_set_fused_forward(prev)
