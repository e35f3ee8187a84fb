"""The C-ABI library loads on a CPU-only machine and exports every symbol the public header declares; the
layout table it reports matches the Python-side statement of the reference's state_dict contract."""
import ctypes
import os
import re

import pytest

from dynaboa_b200 import _lib, build, layout

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    build.build()
    return _lib.load()


def header_symbols():
    src = open(os.path.join(REPO, 'include', 'dynaboa_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(dboa_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported(lib):
    syms = header_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/dynaboa_b200.h but not exported'
    assert set(syms) == set(_lib.SIGNATURES), 'ctypes signature table out of sync with the header'


def test_version_and_counters(lib):
    assert b'sm_90a' in lib.dboa_version()
    assert lib.dboa_launch_count() >= 0


def test_layout_matches_reference_contract(lib):
    from dynaboa_b200.hmr import ArenaLayout
    lay = ArenaLayout()
    ref = layout.param_shapes()
    assert lay.n == 169 and lay.names == list(ref.keys())
    assert [tuple(s) for s in lay.shapes] == [tuple(v) for v in ref.values()]
    assert sum(int(__import__('numpy').prod(s)) for s in lay.shapes) == layout.num_params() == 26977501
    # views must not overlap and must stay inside the arena
    spans = sorted((o, o + 1 + sum((s - 1) * st for s, st in zip(sh, stv))) for o, sh, stv in zip(lay.offsets, lay.shapes, lay.strides))
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 <= b0
    assert spans[-1][1] <= lay.floats


def test_size_queries(lib):
    assert lib.dboa_hmr_tape_floats(1) > 20_000_000 and lib.dboa_hmr_tape_floats(0) < 0
    assert lib.dboa_hmr_scratch_floats(2) > 0
    assert lib.dboa_smpl_tape_floats(2) == 2 * (8 * 20670 + 648)      # 7 blend-shape row splits + posed vertices, chain state


@pytest.mark.parametrize('B', [1, 2, 9, 22, 64])
def test_tape_offsets_cover_disjoint_regions_of_the_layer_shapes(lib, B):
    """dboa_hmr_tape_offset: every region lies inside dboa_hmr_tape_floats(B), no two overlap, and each is as large as
    the layer it holds (shapes from the parameter table); the convolution output sizes agree with dboa_hmr_feature_info."""
    from dynaboa_b200 import hmr
    geo = hmr.conv_geometry()
    assert len(geo) == 53 and sum('downsample' in g[0] for g in geo) == 4
    regions = []
    for i, (name, cin, cout, k, stride, h) in enumerate(geo):
        n = B * h * h * cout
        regions += [(lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y, i), n, ('y', name)),
                    (lib.dboa_hmr_tape_offset(B, hmr.TAPE_STATS, i), B * 8, ('stats', name))]
        if 'downsample' in name:
            assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_A, i) == -1, name
        else:
            regions.append((lib.dboa_hmr_tape_offset(B, hmr.TAPE_A, i), n, ('a', name)))
    # consecutive convolutions chain: Cin of each conv is the channel count of its input, Hin = Hout * stride
    for (n0, _, c0, _, _, h0), (n1, cin1, _, _, s1, h1) in zip(geo, geo[1:]):
        if n1.endswith('conv2') or n1.endswith('conv3'):
            assert cin1 == c0 and h0 == h1 * s1, (n0, n1)
    sizes = {'x0': B * 224 * 224 * 3, 'p0': B * 56 * 56 * 64, 'p0_idx': (B * 56 * 56 * 64 + 3) // 4, 'xc': 3 * B * 2208,
             'h1pre': 3 * B * 1024, 'h1post': 3 * B * 1024, 'h2pre': 3 * B * 1024, 'h2post': 3 * B * 1024, 'params': 4 * B * 160,
             'masks': 6 * B * 1024}
    for kind, n in sizes.items():
        regions.append((lib.dboa_hmr_tape_offset(B, hmr.TAPE_WHOLE[kind], 0), n, (kind,)))
    assert all(o >= 0 for o, _, _ in regions), [r for r in regions if r[0] < 0]
    regions.sort()
    for (o0, n0, w0), (o1, _, w1) in zip(regions, regions[1:]):
        assert o0 + n0 <= o1, (w0, w1)
    assert regions[-1][0] + regions[-1][1] <= lib.dboa_hmr_tape_floats(B)
    off, nd = ctypes.c_longlong(), ctypes.c_int()
    shp, st = (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
    firsts = [0] + [i for i, g in enumerate(geo) if g[0].endswith('.conv3') and g[0].split('.')[1] == {1: '2', 2: '3', 3: '5', 4: '2'}[int(g[0][5])]]
    for feat, ci in enumerate(firsts):
        assert lib.dboa_hmr_feature_info(B, feat, ctypes.byref(off), ctypes.byref(nd), shp, st) == 0
        assert (shp[1], shp[2]) == (geo[ci][2], geo[ci][5]), feat
        assert off.value == lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y if feat == 0 else hmr.TAPE_A, ci), feat


def test_tape_offset_errors(lib):
    from dynaboa_b200 import hmr
    for B in (0, -1, 65):
        assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y, 0) == -2
        assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_WHOLE['x0'], 0) == -2
    for kind in (-1, 13, 99):
        assert lib.dboa_hmr_tape_offset(1, kind, 0) == -1
    for conv in (-1, 53, 1000):
        for kind in (hmr.TAPE_Y, hmr.TAPE_STATS, hmr.TAPE_A):
            assert lib.dboa_hmr_tape_offset(1, kind, conv) == -1
    assert lib.dboa_hmr_tape_offset(1, hmr.TAPE_A, 4) == -1            # layer1.0.downsample.0
    assert lib.dboa_hmr_tape_offset(1, hmr.TAPE_Y, 4) >= 0


def test_argument_errors_do_not_need_a_gpu(lib):
    assert lib.dboa_rot6d_fwd(None, None, 4, None) == -1
    assert lib.dboa_sgd_update(None, None, None, 0.1, 8, None) == -1
    off, nd = ctypes.c_longlong(), ctypes.c_int()
    shp, st = (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
    assert lib.dboa_hmr_param_info(999, None, 0, ctypes.byref(off), ctypes.byref(nd), shp, st) == -1

