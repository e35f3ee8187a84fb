"""The per-video dynamic loop of MultiVideoAdaptor without a device: the bindings of dboa_cosine_terms_active /
dboa_cosine_partial_floats_groups, their argument errors (returned on the host before any device access), and the opt-in of
check_options(..., dynamic_loop=True)."""
import ctypes

import pytest

from dynaboa_b200 import _lib, build

DBOA_ERR_ARG, DBOA_ERR_SHAPE = -1, -2
FAKE = ctypes.c_void_p(0x1000)        # stand-in device pointers: every case below is rejected before one is dereferenced
COS_CHUNK = 256 * 16


@pytest.fixture(scope='module')
def lib():
    build.build()
    return _lib.load()


def lengths(*n):
    return (ctypes.c_longlong * len(n))(*n)


def ptrs(k):
    return (ctypes.c_void_p * k)(*([0x1000] * k))


def terms_active(lib, n, groups, active, partial_floats=1 << 30, a=True, b=True, partial=FAKE, terms=FAKE, npairs=None):
    k = 1 if n is None else len(n)
    return lib.dboa_cosine_terms_active(ptrs(k) if a else None, ptrs(k) if b else None, None if n is None else lengths(*n),
                                        k if npairs is None else npairs, partial, partial_floats, terms, None, groups, active)


def test_bindings():
    P, I, L, U = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_ulonglong
    sig = _lib.SIGNATURES
    assert sig['dboa_cosine_terms_active'] == (I, sig['dboa_cosine_terms'][1] + [I, U])
    assert sig['dboa_cosine_partial_floats_groups'] == (L, [ctypes.POINTER(L), I, I])
    assert sig['dboa_cosine_partial_floats_groups'][1][:2] == sig['dboa_cosine_partial_floats'][1]


def test_partial_floats_groups(lib):
    n = [64 * 2048, 3 * COS_CHUNK + 5, 1024, 7]
    assert lib.dboa_cosine_partial_floats_groups(lengths(*n), len(n), 1) == lib.dboa_cosine_partial_floats(lengths(*n), len(n))
    for G, part in ((2, [32 * 2048, 6 * COS_CHUNK + 10, 512, 14]), (4, [16 * 2048, 12 * COS_CHUNK + 20, 256, 28])):
        whole = [G * p for p in part]
        one = lib.dboa_cosine_partial_floats(lengths(*part), len(part))
        assert lib.dboa_cosine_partial_floats_groups(lengths(*whole), len(whole), G) == G * one
    assert lib.dboa_cosine_partial_floats_groups(lengths(64 * COS_CHUNK), 1, 64) == 3 * 64


@pytest.mark.parametrize('n,npairs,groups,err', [(None, 1, 1, DBOA_ERR_ARG), ([8], 0, 1, DBOA_ERR_ARG), ([8] * 17, 17, 1, DBOA_ERR_ARG),
                                                  ([8], 1, 0, DBOA_ERR_SHAPE), ([130], 1, 65, DBOA_ERR_SHAPE), ([8], 1, -2, DBOA_ERR_SHAPE),
                                                  ([8, 9], 2, 2, DBOA_ERR_SHAPE), ([12, 16], 2, 8, DBOA_ERR_SHAPE)])
def test_partial_floats_groups_errors(lib, n, npairs, groups, err):
    assert lib.dboa_cosine_partial_floats_groups(None if n is None else lengths(*n), npairs, groups) == err


@pytest.mark.parametrize('kw', [dict(a=False), dict(b=False), dict(n=None), dict(partial=None), dict(terms=None)])
def test_null_pointers(lib, kw):
    args = dict(n=[16], groups=2, active=0b11)
    args.update(kw)
    assert terms_active(lib, **args) == DBOA_ERR_ARG


@pytest.mark.parametrize('npairs', [0, -1, 17])
def test_pair_count(lib, npairs):
    assert terms_active(lib, [16] * 17, 2, 0b11, npairs=npairs) == DBOA_ERR_ARG


@pytest.mark.parametrize('groups,active', [(2, 0), (2, 0b100), (4, 0b10000), (4, 1 << 63), (1, 0b10), (1, 0), (8, 1 << 8)])
def test_mask_errors(lib, groups, active):
    assert terms_active(lib, [64, 128], groups, active) == DBOA_ERR_ARG


def test_a_full_mask_of_64_videos_is_accepted_up_to_the_scratch_check(lib):
    assert terms_active(lib, [64 * 16], 64, (1 << 64) - 1, partial_floats=3 * 64 - 1) == DBOA_ERR_ARG


@pytest.mark.parametrize('n,groups', [([16], 0), ([130], 65), ([16], -1), ([16, 18], 4), ([9], 2)])
def test_shape_errors(lib, n, groups):
    assert terms_active(lib, n, groups, 1) == DBOA_ERR_SHAPE
    assert terms_active(lib, n, groups, 0) == DBOA_ERR_SHAPE              # the shape is checked before the mask


@pytest.mark.parametrize('n,groups', [([2 * COS_CHUNK + 2, 64], 2), ([4 * 2048] * 15, 4), ([8], 8), ([1], 1)])
def test_too_small_a_partial(lib, n, groups):
    need = lib.dboa_cosine_partial_floats_groups(lengths(*n), len(n), groups)
    assert need > 0
    assert terms_active(lib, n, groups, 1, partial_floats=need - 1) == DBOA_ERR_ARG
    assert terms_active(lib, n, groups, 1, partial_floats=0) == DBOA_ERR_ARG


def test_the_one_video_call_keeps_its_errors(lib):
    k = 2
    assert lib.dboa_cosine_terms(ptrs(k), ptrs(k), lengths(8, 8), 0, FAKE, 100, FAKE, None) == DBOA_ERR_ARG
    assert lib.dboa_cosine_terms(ptrs(k), ptrs(k), lengths(8, 8), k, FAKE, 5, FAKE, None) == DBOA_ERR_ARG
    assert lib.dboa_cosine_terms(ptrs(k), ptrs(k), lengths(8, 8), k, FAKE, 100, None, None) == DBOA_ERR_ARG


# ------------------------------------------------------------------ opting in
def c5_options(**extra):
    from bench import WORKLOADS, default_options
    o = default_options(expdir='/nonexistent', expname='x', model_file='unused', synthetic_frames=2, **WORKLOADS['c5'])
    for k, v in extra.items():
        setattr(o, k, v)
    return o


def test_c5_is_the_dynamic_workload():
    o = c5_options()
    assert o.dynamic_boa and o.use_boa and o.retrieval and o.sample_num == 8


@pytest.mark.parametrize('G', [1, 2, 8])
def test_dynamic_boa_needs_the_keyword(lib, G):
    from dynaboa_b200.multivideo import check_options
    with pytest.raises(ValueError, match='dynamic_boa') as e:
        check_options(c5_options(), G)
    assert 'dynamic_loop' in str(e.value)
    with pytest.raises(ValueError, match='dynamic_loop'):
        check_options(c5_options(), G, dynamic_loop=False)
    check_options(c5_options(), G, dynamic_loop=True)
    check_options(c5_options(dynamic_boa=0), G, dynamic_loop=True)
    check_options(c5_options(dynamic_boa=0), G)


@pytest.mark.parametrize('extra,G,why', [({'use_boa': 0}, 2, 'use_boa'), ({}, 9, 'exceed'), ({}, 0, 'at least'),
                                         ({'upper_level_mixtrain': 0, 'lower_level_mixtrain': 0}, 65, 'exceed'),
                                         ({'sample_num': 16}, 5, 'exceed')])
def test_every_other_rejection_still_applies(lib, extra, G, why):
    from dynaboa_b200.multivideo import check_options
    with pytest.raises(ValueError, match=why):
        check_options(c5_options(**extra), G, dynamic_loop=True)


@pytest.mark.parametrize('setter', ['dboa_set_fused_forward', 'dboa_set_fused_backward'])
def test_fused_plans_are_still_rejected(lib, setter):
    from dynaboa_b200.multivideo import check_options
    prev = getattr(lib, setter.replace('set', 'get'))()
    getattr(lib, setter)(1)
    try:
        with pytest.raises(ValueError, match='fused'):
            check_options(c5_options(), 2, dynamic_loop=True)
    finally:
        getattr(lib, setter)(prev)


def test_runtime_check_passes_the_keyword_through(lib):
    from types import SimpleNamespace
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = MultiVideoAdaptor.__new__(MultiVideoAdaptor)           # no device: only the run-time check is exercised
    mv.options, mv.G = c5_options(), 2
    mv.base = SimpleNamespace(optimizer=SimpleNamespace(grad_sync=None, pre_step_hook=None))
    mv.dynamic_loop = True
    mv._check_runtime()
    mv.dynamic_loop = False
    with pytest.raises(ValueError, match='dynamic_boa'):
        mv._check_runtime()
