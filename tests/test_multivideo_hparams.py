"""Per-video hyperparameters of a pool without a device: every rule of multivideo.check_hparams, the checks of start(g, hparams=)
that run before any device work, and the argument errors of the per-video entry points (returned on the host before any
device access)."""
import ctypes
import math
from types import SimpleNamespace

import pytest

from dynaboa_b200.multivideo import PER_VIDEO, MultiVideoAdaptor, check_hparams, own_values
from harness import ERR_ARG, ERR_SHAPE, FAKE, built_lib, cpu_options, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


@pytest.fixture
def opts():
    return cpu_options('c2')


def test_per_video_keys():
    assert PER_VIDEO == {'lr', 'beta1', 'beta2', 'fastlr', 'alpha', 's2dloss_weight', 'shape_prior_weight', 'pose_prior_weight',
                         'teacherloss_weight', 'motionloss_weight', 'labelloss_weight', 'cos_sim_threshold', 'optim_steps'}


def test_accepted_values_are_normalised(opts):
    hp = check_hparams(opts, {'lr': 1e-5, 'beta1': 0, 'beta2': 0.999, 'alpha': 1, 'fastlr': 0.0, 'optim_steps': 0,
                              'cos_sim_threshold': -1.0, 'pose_prior_weight': 2 * opts.pose_prior_weight})
    assert hp['optim_steps'] == 0 and type(hp['optim_steps']) is int
    assert all(type(v) is float for k, v in hp.items() if k != 'optim_steps')
    assert check_hparams(opts, {}) == {}
    assert own_values(opts, {'lr': opts.lr, 'fastlr': 2 * opts.fastlr}) == {'fastlr': 2 * opts.fastlr}


def test_numpy_numbers_are_accepted(opts):
    import numpy as np
    hp = check_hparams(opts, {'lr': np.float32(1e-5), 'fastlr': np.float64(2e-5), 'optim_steps': np.int64(4), 'beta1': np.float16(0.25)})
    assert hp == {'lr': float(np.float32(1e-5)), 'fastlr': 2e-5, 'optim_steps': 4, 'beta1': 0.25}
    assert type(hp['optim_steps']) is int and type(hp['lr']) is float
    for bad in ({'optim_steps': np.int32(-1)}, {'optim_steps': np.bool_(True)}, {'lr': np.bool_(True)}, {'alpha': np.float32('nan')}):
        with pytest.raises(ValueError, match=next(iter(bad))):
            check_hparams(opts, bad)


@pytest.mark.parametrize('key', ['inner_step', 'retrieval', 'batch_size', 'dynamic_boa', 'eps', 'no_such_option'])
def test_a_key_outside_per_video_is_named(opts, key):
    with pytest.raises(ValueError, match=key):
        check_hparams(opts, {'lr': 1e-6, key: 1})


@pytest.mark.parametrize('key', sorted(PER_VIDEO - {'optim_steps'}))
@pytest.mark.parametrize('value', [math.nan, math.inf, -math.inf, '1e-5', None, True])
def test_non_finite_or_non_numeric_values(opts, key, value):
    with pytest.raises(ValueError, match=key):
        check_hparams(opts, {key: value})


@pytest.mark.parametrize('key,value', [('lr', -1e-9), ('fastlr', -1.0), ('beta1', 1.0), ('beta1', -0.1), ('beta2', 1.0), ('beta2', 1.5),
                                       ('beta2', -1e-3), ('alpha', -0.01), ('alpha', 1.01)])
def test_out_of_range_values(opts, key, value):
    with pytest.raises(ValueError, match=key):
        check_hparams(opts, {key: value})


@pytest.mark.parametrize('value', [-1, 2.0, 1.5, True, '3', None])
def test_optim_steps_is_a_non_negative_int(opts, value):
    with pytest.raises(ValueError, match='optim_steps'):
        check_hparams(opts, {'optim_steps': value})


def test_pose_prior_weight_keeps_the_pools_zero_ness(opts):
    assert opts.pose_prior_weight != 0
    with pytest.raises(ValueError, match='pose_prior_weight'):
        check_hparams(opts, {'pose_prior_weight': 0.0})
    zero = SimpleNamespace(**{**vars(opts), 'pose_prior_weight': 0.0})
    with pytest.raises(ValueError, match='pose_prior_weight'):
        check_hparams(zero, {'pose_prior_weight': 1e-4})
    assert check_hparams(zero, {'pose_prior_weight': 0}) == {'pose_prior_weight': 0.0}


def test_one_dict_or_none_per_video(opts):
    assert check_hparams(opts, None, 3) == [{}, {}, {}]
    assert check_hparams(opts, [None, {'lr': 1e-5}], 2) == [{}, {'lr': 1e-5}]
    for bad in ([{}], [{}, {}, {}], []):
        with pytest.raises(ValueError, match='2 videos'):
            check_hparams(opts, bad, 2)
    with pytest.raises(ValueError, match='alpha'):
        check_hparams(opts, [{}, {'alpha': 2.0}], 2)
    with pytest.raises(ValueError, match='dict'):
        check_hparams(opts, [[('lr', 1e-5)]], 1)


def test_start_checks_hparams_before_device_work(opts):
    mv = idle_pool(MultiVideoAdaptor, 3, options=opts)
    with pytest.raises(ValueError, match='inner_step'):
        mv.start(1, hparams={'inner_step': 2})
    with pytest.raises(ValueError, match='beta1'):
        mv.start(0, hparams={'beta1': 1.0})
    with pytest.raises(ValueError, match='slot'):
        mv.start(3, hparams={'lr': 1e-5})


def test_run_checks_the_hparams_list_before_device_work(opts):
    mv = idle_pool(MultiVideoAdaptor, 2, options=opts)
    with pytest.raises(ValueError, match='3 videos'):
        mv.run([[], [], []], hparams=[{}, {}])
    with pytest.raises(ValueError, match='cos_sim_threshold'):
        mv.run([[]], hparams=[{'cos_sim_threshold': math.nan}])


# ------------------------------------------------------------------ the per-video entry points' argument errors
def floats(*v):
    return (ctypes.c_float * max(1, len(v)))(*v)


TABLE = floats(*([0.5] * 64 * 9))


def sgd(lib, n=8, groups=2, active=0b11, table=TABLE, p=FAKE):
    return lib.dboa_sgd_update_groups(p, FAKE, FAKE, table, n, groups, active, None)


def adam(lib, n=8, groups=2, active=0b11, table=TABLE, p=FAKE):
    return lib.dboa_adam_ema_groups(p, FAKE, FAKE, FAKE, None, n, table, groups, active, None)


def motion(lib, B=4, groups=2, active=0b11, table=TABLE, p=FAKE):
    return lib.dboa_loss_motion_weights(p, FAKE, FAKE, FAKE, table, FAKE, FAKE, FAKE, B, 1, 25, 24, groups, active, None)


def prior(lib, B=4, groups=2, table=TABLE, p=FAKE):
    return lib.dboa_pose_prior_groups(p, FAKE, FAKE, FAKE, FAKE, FAKE, table, B, groups, None)


def head(lib, B=4, groups=2, table=TABLE, p=FAKE):
    from dynaboa_b200 import _lib
    a = _lib.LossArgsStruct()
    a.B, a.groups = B, groups
    for name in ('p2d', 'j3d', 'R', 'beta', 'terms'):
        setattr(a, name, p.value if p is not None else None)
    return lib.dboa_loss_multi_weights(ctypes.byref(a), table, None)


MASKED = {'sgd': sgd, 'adam': adam, 'motion': motion}
ALL = {**MASKED, 'prior': prior, 'head': head}


@pytest.mark.parametrize('entry', sorted(ALL))
def test_null_pointer_or_table(lib, entry):
    assert ALL[entry](lib, table=None) == ERR_ARG
    assert ALL[entry](lib, p=None) == ERR_ARG


@pytest.mark.parametrize('entry', sorted(MASKED))
@pytest.mark.parametrize('groups,active', [(2, 0), (2, 0b100), (4, 0b10000), (8, 1 << 63), (1, 0b10), (63, 1 << 63)])
def test_mask_errors(lib, entry, groups, active):
    kw = dict(B=2 * groups) if entry == 'motion' else {}
    assert MASKED[entry](lib, groups=groups, active=active, **kw) == ERR_ARG


@pytest.mark.parametrize('entry', sorted(MASKED))
@pytest.mark.parametrize('groups', [0, -1, 65])
def test_groups_out_of_range(lib, entry, groups):
    assert MASKED[entry](lib, groups=groups, active=1, **(dict(B=130) if entry == 'motion' else {})) == ERR_SHAPE
    assert MASKED[entry](lib, groups=groups, active=0, **(dict(B=130) if entry == 'motion' else {})) == ERR_SHAPE   # shape first


@pytest.mark.parametrize('entry', ['sgd', 'adam'])
@pytest.mark.parametrize('n', [1, 6, 4097])
def test_sweep_length_not_a_multiple_of_four(lib, entry, n):
    assert MASKED[entry](lib, n=n) == ERR_SHAPE


@pytest.mark.parametrize('entry', ['motion', 'prior', 'head'])
@pytest.mark.parametrize('B,groups', [(5, 2), (9, 4), (130, 65)])
def test_rows_not_split_into_groups(lib, entry, B, groups):
    assert ALL[entry](lib, B=B, groups=groups) == ERR_SHAPE


def test_rows_out_of_range(lib):
    assert prior(lib, B=4, groups=0) == ERR_SHAPE
    assert motion(lib, B=4, groups=0) == ERR_SHAPE
    assert prior(lib, B=0, groups=1) == ERR_SHAPE
    assert head(lib, B=0, groups=1) == ERR_SHAPE
    assert motion(lib, B=0, groups=1) == ERR_ARG         # as dboa_loss_motion_active
