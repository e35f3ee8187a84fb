"""Grouped HMR plan (several videos, one launch sequence): the argument errors of dboa_hmr_forward_groups /
dboa_hmr_backward_groups are returned on the host before any device access, and header and bindings agree."""
import ctypes

import pytest

from dynaboa_b200 import _lib, build

DBOA_ERR_SHAPE, DBOA_ERR_UNSUPPORTED = -2, -4
# stand-in device pointers: every case below is rejected before a pointer is dereferenced or a device is touched
FAKE = ctypes.c_void_p(0x1000)


@pytest.fixture(scope='module')
def lib():
    build.build()
    return _lib.load()


def forward(lib, B, groups):
    return lib.dboa_hmr_forward_groups(FAKE, FAKE, FAKE, FAKE, FAKE, B, None, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, groups)


def backward(lib, B, groups):
    return lib.dboa_hmr_backward_groups(FAKE, FAKE, B, 0, FAKE, None, None, FAKE, FAKE, None, groups)


@pytest.mark.parametrize('B,groups', [(4, 0), (4, -1), (6, 4), (9, 2), (65, 1), (65, 5), (0, 1), (128, 2)])
def test_shape_errors(lib, B, groups):
    assert forward(lib, B, groups) == DBOA_ERR_SHAPE
    assert backward(lib, B, groups) == DBOA_ERR_SHAPE


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_fused_plans_are_not_grouped(lib, setter):
    prev = getattr(lib, setter.replace('set', 'get'))()
    getattr(lib, setter)(1)
    try:
        assert forward(lib, 8, 2) == DBOA_ERR_UNSUPPORTED
        assert backward(lib, 8, 4) == DBOA_ERR_UNSUPPORTED
        assert forward(lib, 9, 2) == DBOA_ERR_SHAPE              # the shape is checked first
    finally:
        getattr(lib, setter)(prev)


def test_gradient_buckets_are_not_grouped(lib):
    """Armed data-parallel buckets make a grouped backward fail; a grouped call consumes the request whatever it returns,
    so the stand-in events armed here never reach a later backward."""
    prev = lib.dboa_get_fused_forward(), lib.dboa_get_fused_backward()
    lib.dboa_set_fused_forward(0)
    lib.dboa_set_fused_backward(0)
    try:
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 8, 2) == DBOA_ERR_UNSUPPORTED
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 9, 2) == DBOA_ERR_SHAPE             # consumes the second request
    finally:
        lib.dboa_set_fused_forward(prev[0])
        lib.dboa_set_fused_backward(prev[1])


def test_bindings(lib):
    P, I = ctypes.c_void_p, ctypes.c_int
    assert _lib.SIGNATURES['dboa_hmr_forward_groups'] == (I, [P, P, P, P, P, I, P, P, P, P, P, P, P, P, I])
    assert _lib.SIGNATURES['dboa_hmr_backward_groups'] == (I, [P, P, I, I, P, P, P, P, P, P, I])
    fwd, bwd = _lib.SIGNATURES['dboa_hmr_forward'][1], _lib.SIGNATURES['dboa_hmr_backward'][1]
    assert _lib.SIGNATURES['dboa_hmr_forward_groups'][1] == fwd + [I]
    assert _lib.SIGNATURES['dboa_hmr_backward_groups'][1] == bwd + [I]


def test_python_rejects_bad_groups():
    import torch
    from dynaboa_b200.hmr import _check_groups, layout
    P = layout().floats
    with pytest.raises(ValueError):
        _check_groups(torch.empty(0), 6, 4)
    with pytest.raises(ValueError):
        _check_groups(torch.empty(P), 4, 2)                      # one arena for two videos
    _check_groups(torch.empty(2, P), 4, 2)


def c2_options(**extra):
    from bench import WORKLOADS, default_options
    o = default_options(expdir='/nonexistent', expname='x', model_file='unused', synthetic_frames=2, **WORKLOADS['c2'])
    for k, v in extra.items():
        setattr(o, k, v)
    return o


@pytest.mark.parametrize('extra,G,why', [({'dynamic_boa': 1}, 2, 'dynamic_boa'), ({'use_boa': 0}, 2, 'use_boa'), ({}, 65, 'exceed'),
                                         ({}, 0, 'at least'),
                                         ({'retrieval': 1, 'upper_level_mixtrain': 1, 'lower_level_mixtrain': 0, 'sample_num': 8}, 9, 'exceed')])
def test_multivideo_rejects_unsupported_options(lib, extra, G, why):
    from dynaboa_b200.multivideo import check_options
    with pytest.raises(ValueError, match=why):
        check_options(c2_options(**extra), G)
    check_options(c2_options(retrieval=1, upper_level_mixtrain=1, lower_level_mixtrain=0, sample_num=8), 8)
    check_options(c2_options(), 64)


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_multivideo_rejects_fused_plans(lib, setter):
    from dynaboa_b200.multivideo import check_options
    getter = setter.replace('set', 'get')
    prev = getattr(lib, getter)()
    getattr(lib, setter)(1)
    try:
        assert getattr(lib, getter)() == 1
        with pytest.raises(ValueError, match='fused'):
            check_options(c2_options(), 2)
    finally:
        getattr(lib, setter)(prev)


def test_multivideo_rejects_a_data_parallel_optimizer(lib):
    from types import SimpleNamespace
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = MultiVideoAdaptor.__new__(MultiVideoAdaptor)           # no device: only the run-time check is exercised
    mv.options, mv.G = c2_options(), 2
    mv.base = SimpleNamespace(optimizer=SimpleNamespace(grad_sync=None, pre_step_hook=lambda g: None))
    with pytest.raises(ValueError, match='data-parallel'):
        mv._check_runtime()
    mv.base.optimizer.pre_step_hook = None
    mv._check_runtime()


def test_loss_struct_layout_matches_the_header(tmp_path):
    """offsetof / sizeof of dboa_loss_args compiled from the header against the ctypes mirror, new `groups` field included."""
    import os
    import subprocess
    fields = [f[0] for f in _lib.LossArgsStruct._fields_]
    assert fields[-1] == 'groups'
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / 'layout.c'
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "dynaboa_b200.h"\nint main(void) {\n'
                   + ''.join(f'  printf("%zu\\n", offsetof(dboa_loss_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(dboa_loss_args));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(repo, 'include'), str(src), '-o', str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = [getattr(_lib.LossArgsStruct, f).offset for f in fields] + [ctypes.sizeof(_lib.LossArgsStruct)]
    assert got == want


def test_loss_bindings(lib):
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    assert _lib.SIGNATURES['dboa_loss_motion_groups'] == (I, [P, P, P, P, F, P, P, P, I, I, I, I, I, P])
    assert _lib.SIGNATURES['dboa_loss_motion_groups'][1][:12] == _lib.SIGNATURES['dboa_loss_motion_joints'][1][:12]
