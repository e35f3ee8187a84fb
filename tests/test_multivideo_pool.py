"""Slots of MultiVideoAdaptor and the active-video mask of the grouped plan, without a device: the argument errors of
dboa_hmr_forward_active / dboa_hmr_backward_active / dboa_loss_motion_active (returned on the host before any device access), and
the Python-side checks of adapt(batches) and start(g)."""
import pytest

from dynaboa_b200.multivideo import MultiVideoAdaptor
from harness import ERR_ARG, ERR_SHAPE, ERR_UNSUPPORTED, FAKE, built_lib, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def forward(lib, B, groups, active):
    return lib.dboa_hmr_forward_active(FAKE, FAKE, FAKE, FAKE, FAKE, B, None, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, groups, active)


def backward(lib, B, groups, active):
    return lib.dboa_hmr_backward_active(FAKE, FAKE, B, 0, FAKE, None, None, FAKE, FAKE, None, groups, active)


def motion(lib, B, groups, active):
    return lib.dboa_loss_motion_active(FAKE, FAKE, FAKE, FAKE, 1.0, FAKE, FAKE, FAKE, B, 1, 25, 24, groups, active, None)


@pytest.mark.parametrize('B,groups,active', [(4, 2, 0), (4, 2, 0b100), (8, 4, 0b10000), (8, 4, 1 << 63), (1, 1, 0b10), (2, 1, 0),
                                             (64, 8, 1 << 8)])
def test_mask_errors(lib, B, groups, active):
    assert forward(lib, B, groups, active) == ERR_ARG
    assert backward(lib, B, groups, active) == ERR_ARG
    assert motion(lib, B, groups, active) == ERR_ARG


@pytest.mark.parametrize('B,groups,active', [(4, 0, 1), (6, 4, 1), (65, 1, 1), (0, 1, 1), (128, 2, 3)])
def test_shape_errors_come_first(lib, B, groups, active):
    assert forward(lib, B, groups, active) == ERR_SHAPE
    assert backward(lib, B, groups, active) == ERR_SHAPE
    assert forward(lib, B, groups, 0) == ERR_SHAPE


def test_motion_shape_errors(lib):
    assert motion(lib, 130, 65, 1) == ERR_SHAPE
    assert motion(lib, 9, 2, 1) == ERR_SHAPE


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_fused_plans_are_not_masked(lib, setter):
    prev = getattr(lib, setter.replace('set', 'get'))()
    getattr(lib, setter)(1)
    try:
        assert forward(lib, 8, 2, 0b01) == ERR_UNSUPPORTED
        assert backward(lib, 8, 4, 0b0110) == ERR_UNSUPPORTED
        assert forward(lib, 8, 2, 0) == ERR_ARG              # the mask is checked before the plan
    finally:
        getattr(lib, setter)(prev)


def test_masked_backward_consumes_an_armed_bucket_request(lib):
    prev = lib.dboa_get_fused_forward(), lib.dboa_get_fused_backward()
    lib.dboa_set_fused_forward(0)
    lib.dboa_set_fused_backward(0)
    try:
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 8, 2, 0b01) == ERR_UNSUPPORTED
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 8, 2, 0) == ERR_ARG             # consumes the second request
        assert lib.dboa_hmr_backward_buckets(FAKE, FAKE, FAKE) == 0
        assert backward(lib, 9, 2, 1) == ERR_SHAPE           # and the third
    finally:
        lib.dboa_set_fused_forward(prev[0])
        lib.dboa_set_fused_backward(prev[1])


def test_adapt_rejects_wrong_entries(lib):
    mv = idle_pool(MultiVideoAdaptor, 3)
    with pytest.raises(ValueError, match='expected 3'):
        mv.adapt([None, None])
    with pytest.raises(ValueError, match='expected 3'):
        mv.adapt([None] * 4)
    with pytest.raises(ValueError, match='at least one'):
        mv.adapt([None] * 3)


@pytest.mark.parametrize('g', [-1, 3, 7, 1.0, None])
def test_start_rejects_a_slot_out_of_range(lib, g):
    mv = idle_pool(MultiVideoAdaptor, 3)
    with pytest.raises(ValueError, match='slot'):
        mv.start(g)


def test_runs():
    from dynaboa_b200.fused import runs
    assert runs(0b1111, 4) == [[0, 4]]
    assert runs(0b1011, 4) == [[0, 2], [3, 4]]
    assert runs(0b0100, 4) == [[2, 3]]
    steps = [3, 3, 1, 1, 1, 5]
    assert runs(0b111111, 6, key=lambda g: steps[g]) == [[0, 2], [2, 5], [5, 6]]
    assert runs(0b110111, 6, key=lambda g: steps[g]) == [[0, 2], [2, 3], [4, 5], [5, 6]]
