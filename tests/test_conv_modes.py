"""The stand-alone tensor-core convolution entry points under each tensor-core mode (dboa_set_tensor_core_conv): which modes
refuse each of them with DBOA_ERR_UNSUPPORTED, and the shapes refused under every mode.  Only refusals are called, with stand-in
pointers.  Without a GPU a tensor-core launch is refused as well, so only a run on a machine with a device tells a refusal from a
launch; there, a call let through by mistake fails on the empty grid of these problems instead of running on the stand-ins."""
import pytest

from harness import ERR_UNSUPPORTED, FAKE, built_lib

MODES = (0, 1, 2, 3)
# B, Hi, Wi, Cin, Cout, k, stride, pad, Kpitch.  Every problem is empty: B = 0, and Cin = 0 or Cout = 0.
TAKEN = (0, 14, 14, 256, 0, 3, 1, 1, 3 * 3 * 256)           # passes every shape check
REFUSED = {  # shapes no mode runs on the tensor cores
    'Cin % 64': (0, 14, 14, 96, 0, 3, 1, 1, 3 * 3 * 96),
    'Cout % 64': (0, 14, 14, 0, 96, 3, 1, 1, 0),
    'Kpitch': (0, 14, 14, 256, 0, 3, 1, 1, 3 * 3 * 256 + 16),
}
ODD_STRIDE2 = (0, 15, 15, 128, 0, 3, 2, 1, 3 * 3 * 128)     # refused by the data gradient only (its parity classes need even extents)


def conv2d(name, *extra):
    return lambda lib, s: getattr(lib, name)(FAKE, FAKE, FAKE, *s, *extra, None)


def conv1x1(lib, s):
    B, Hi, Wi, Cin, Cout = s[:5]
    return lib.dboa_conv1x1_tc_fwd(FAKE, FAKE, FAKE, B * Hi * Wi, Cin, Cout, None, 0, None)


ENTRIES = {  # entry point -> (call, the modes that let it run)
    'dboa_conv2d_tc_fwd': (conv2d('dboa_conv2d_tc_fwd'), {1, 2, 3}),
    'dboa_conv1x1_tc_fwd': (conv1x1, {1, 2, 3}),
    'dboa_conv2d_tc_dgrad': (conv2d('dboa_conv2d_tc_dgrad', 0), {2, 3}),
    'dboa_conv2d_tc_wgrad': (conv2d('dboa_conv2d_tc_wgrad'), {2, 3}),
    'dboa_conv2d_wgrad_tma': (conv2d('dboa_conv2d_wgrad_tma'), set(MODES)),
}


@pytest.fixture(scope='module')
def lib():
    lib = built_lib()
    yield lib
    lib.dboa_set_tensor_core_conv(3)          # the library default: later test modules must not inherit this module's mode


@pytest.mark.parametrize('entry,mode', [(e, m) for e, (_, runs) in ENTRIES.items() for m in MODES if m not in runs])
def test_mode_refusals(lib, entry, mode):
    """A mode that does not select the product refuses a shape the kernel takes."""
    lib.dboa_set_tensor_core_conv(mode)
    assert ENTRIES[entry][0](lib, TAKEN) == ERR_UNSUPPORTED


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('entry', sorted(ENTRIES))
def test_shape_refusals(lib, entry, mode):
    call = ENTRIES[entry][0]
    lib.dboa_set_tensor_core_conv(mode)
    for why, shape in REFUSED.items():
        if entry == 'dboa_conv1x1_tc_fwd' and why == 'Kpitch':
            continue                          # the 1x1 entry point takes no Kpitch: it is Cin
        assert call(lib, shape) == ERR_UNSUPPORTED, why
    if entry == 'dboa_conv2d_tc_dgrad':
        assert call(lib, ODD_STRIDE2) == ERR_UNSUPPORTED, 'stride 2, odd extents'
