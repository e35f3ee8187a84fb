"""The entry points of the single-video CUDA graph (include/dynaboa_b200.h): the Adam scalar block, the Adam sweep that reads
it, the external event wait and the launch credit refuse bad arguments before any device access, and the scalar block holds
what torch's Adam derives from its hyperparameters."""
import ctypes

import numpy as np
import pytest

from harness import ERR_ARG, FAKE, built_lib


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def test_adam_scalars_follow_torchs_derivation(lib):
    out = (ctypes.c_float * 9)()
    lr, b1, b2, eps, step, alpha, gscale = 3e-6, 0.5, 0.9, 1e-8, 7, 0.1, 0.5
    assert lib.dboa_adam_scalars(ctypes.cast(out, ctypes.c_void_p), lr, b1, b2, eps, step, alpha, gscale) == 0
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    want = np.array([1.0 - b1, b2, 1.0 - b2, bc2 ** 0.5, eps, -(lr / bc1), alpha, 1.0 - alpha, gscale], np.float64).astype(np.float32)
    assert np.array(out[:], np.float32).tobytes() == want.tobytes()


def test_graph_entries_check_their_arguments(lib):
    out = ctypes.cast((ctypes.c_float * 9)(), ctypes.c_void_p)
    assert lib.dboa_adam_scalars(None, 3e-6, 0.5, 0.9, 1e-8, 1, 0.1, 1.0) == ERR_ARG
    assert lib.dboa_adam_scalars(out, 3e-6, 0.5, 0.9, 1e-8, 0, 0.1, 1.0) == ERR_ARG          # steps count from 1
    assert lib.dboa_adam_ema_dev(FAKE, FAKE, FAKE, FAKE, None, 8, None, None) == ERR_ARG     # no scalar block
    assert lib.dboa_adam_ema_dev(None, FAKE, FAKE, FAKE, None, 8, FAKE, None) == ERR_ARG
    assert lib.dboa_adam_ema_dev(FAKE, FAKE, FAKE, FAKE, None, -4, FAKE, None) == ERR_ARG
    assert lib.dboa_stream_wait_external(None, None) == ERR_ARG
    assert lib.dboa_launch_credit(-1) == ERR_ARG


def test_launch_credit_adds_to_the_count(lib):
    n0 = lib.dboa_launch_count()
    assert lib.dboa_launch_credit(0) == 0 and lib.dboa_launch_count() == n0
    assert lib.dboa_launch_credit(806) == 0 and lib.dboa_launch_count() == n0 + 806
