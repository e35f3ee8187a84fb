"""Grouped HMR plan (several videos, one launch sequence): the argument errors of dboa_hmr_forward_groups /
dboa_hmr_backward_groups are returned on the host before any device access."""
import pytest

from harness import ERR_SHAPE, ERR_UNSUPPORTED, FAKE, built_lib, cpu_options, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def forward(lib, B, groups):
    return lib.dboa_hmr_forward_groups(FAKE, FAKE, FAKE, FAKE, FAKE, B, None, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, groups)


def backward(lib, B, groups):
    return lib.dboa_hmr_backward_groups(FAKE, FAKE, B, 0, FAKE, None, None, FAKE, FAKE, None, groups)


@pytest.mark.parametrize('B,groups', [(4, 0), (4, -1), (6, 4), (9, 2), (65, 1), (65, 5), (0, 1), (128, 2)])
def test_shape_errors(lib, B, groups):
    assert forward(lib, B, groups) == ERR_SHAPE
    assert backward(lib, B, groups) == ERR_SHAPE


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_fused_plans_are_not_grouped(lib, setter):
    prev = getattr(lib, setter.replace('set', 'get'))()
    getattr(lib, setter)(1)
    try:
        assert forward(lib, 8, 2) == ERR_UNSUPPORTED
        assert backward(lib, 8, 4) == ERR_UNSUPPORTED
        assert forward(lib, 9, 2) == ERR_SHAPE              # the shape is checked first
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
        assert backward(lib, 8, 2) == ERR_UNSUPPORTED
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 9, 2) == ERR_SHAPE             # consumes the second request
    finally:
        lib.dboa_set_fused_forward(prev[0])
        lib.dboa_set_fused_backward(prev[1])


def test_python_rejects_bad_groups():
    import torch
    from dynaboa_b200.hmr import _check_groups, layout
    P = layout().floats
    with pytest.raises(ValueError):
        _check_groups(torch.empty(0), 6, 4)
    with pytest.raises(ValueError):
        _check_groups(torch.empty(P), 4, 2)                      # one arena for two videos
    _check_groups(torch.empty(2, P), 4, 2)


@pytest.mark.parametrize('extra,G,why', [({'dynamic_boa': 1}, 2, 'dynamic_boa'), ({'use_boa': 0}, 2, 'use_boa'), ({}, 65, 'exceed'),
                                         ({}, 0, 'at least'),
                                         ({'retrieval': 1, 'upper_level_mixtrain': 1, 'lower_level_mixtrain': 0, 'sample_num': 8}, 9, 'exceed')])
def test_multivideo_rejects_unsupported_options(lib, extra, G, why):
    from dynaboa_b200.multivideo import check_options
    with pytest.raises(ValueError, match=why):
        check_options(cpu_options('c2', **extra), G)
    check_options(cpu_options('c2', retrieval=1, upper_level_mixtrain=1, lower_level_mixtrain=0, sample_num=8), 8)
    check_options(cpu_options('c2'), 64)


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_multivideo_rejects_fused_plans(lib, setter):
    from dynaboa_b200.multivideo import check_options
    getter = setter.replace('set', 'get')
    prev = getattr(lib, getter)()
    getattr(lib, setter)(1)
    try:
        assert getattr(lib, getter)() == 1
        with pytest.raises(ValueError, match='fused'):
            check_options(cpu_options('c2'), 2)
    finally:
        getattr(lib, setter)(prev)


def test_multivideo_rejects_a_data_parallel_optimizer(lib):
    from types import SimpleNamespace
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = idle_pool(MultiVideoAdaptor, 2, options=cpu_options('c2'),
                   base=SimpleNamespace(optimizer=SimpleNamespace(grad_sync=None, pre_step_hook=lambda g: None)))
    with pytest.raises(ValueError, match='data-parallel'):
        mv._check_runtime()
    mv.base.optimizer.pre_step_hook = None
    mv._check_runtime()
