"""The shapes the fp32 convolution gradients and the max-pool refuse with DBOA_ERR_SHAPE: a weight row pitch the float4 row
accesses cannot take, and max-pool extents or channel counts the kernels would compute with a row, a column or channels
missing.  Only refusals are called, with stand-in pointers.  Every problem is empty, so a call let through by mistake fails on
its empty grid (or, without a device, at its launch) instead of running on the stand-ins: B = 0 empties the grids of the
max-pool, the forward and the data gradient, and Cout = 0 empties all three convolution grids, the weight gradient's included
(its grid is sized by Cout and K, not by B).  The pitch rule reads K = k * k * Cin, which Cout = 0 leaves as it is."""
import pytest

from harness import ERR_SHAPE, FAKE, built_lib


@pytest.fixture(scope='module')
def lib():
    return built_lib()


# B, Hi, Wi, Cin, Cout, k, stride, pad.  Each shape passes every other check of the entry points it is used with.
DGRAD = (0, 14, 14, 64, 0, 3, 1, 1)             # K = 576: the data gradient takes Cin % 64 == 0 and Cout % 16 == 0
STEM = (0, 224, 224, 3, 0, 7, 2, 3)             # the stem's frame and filter, K = 147, roundup16(K) = 160
BAD_PITCH = {                                   # shape -> refused pitches: not a multiple of 4, or shorter than roundup16(K)
    DGRAD: (578, 574, 560, 4),
    STEM: (147, 148, 150, 156, 144),
}


def dgrad(lib, s, pitch):
    return lib.dboa_conv2d_dgrad(FAKE, FAKE, FAKE, *s, pitch, 0, None, 0, None)


def wgrad(lib, s, pitch):
    # no workspace (and Cout = 0): the stem shape goes to the general weight gradient, not to the stem kernel
    return lib.dboa_conv2d_wgrad(FAKE, FAKE, FAKE, *s, pitch, None, 0, None)


@pytest.mark.parametrize('shape', [DGRAD, STEM], ids=['3x3', 'stem'])
def test_conv_wgrad_refuses_pitch(lib, shape):
    for pitch in BAD_PITCH[shape]:
        assert wgrad(lib, shape, pitch) == ERR_SHAPE, pitch


def test_conv_dgrad_refuses_pitch(lib):
    for pitch in BAD_PITCH[DGRAD]:
        assert dgrad(lib, DGRAD, pitch) == ERR_SHAPE, pitch


def test_conv_fwd_refuses_the_same_pitches(lib):
    """The rule the gradients now share with the forward."""
    for shape in (DGRAD, STEM):
        for pitch in BAD_PITCH[shape]:
            assert lib.dboa_conv2d_fwd(FAKE, FAKE, FAKE, *shape, pitch, None, 0, None) == ERR_SHAPE, (shape, pitch)


MAXPOOL_REFUSED = {  # (H, W, C)
    'odd H': (7, 8, 64), 'odd W': (8, 7, 64), 'odd H and W': (113, 113, 64), 'H = 1': (1, 8, 64),
    'C % 4 = 2': (8, 8, 6), 'C % 4 = 1': (112, 112, 65), 'C % 4 = 3': (112, 112, 3),
}


@pytest.mark.parametrize('why', sorted(MAXPOOL_REFUSED))
def test_maxpool_refuses(lib, why):
    H, W, C = MAXPOOL_REFUSED[why]
    assert lib.dboa_maxpool_fwd(FAKE, FAKE, FAKE, 0, H, W, C, None) == ERR_SHAPE
    assert lib.dboa_maxpool_bwd(FAKE, FAKE, FAKE, 0, H, W, C, None) == ERR_SHAPE
