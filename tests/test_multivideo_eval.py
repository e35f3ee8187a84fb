"""Evaluation of a MultiVideoAdaptor pool without a device: the binding of dboa_eval_metrics_active and its argument errors
(returned on the host before any device access), the ground-truth checks of ``adapt``, and the shared result writer."""
import ctypes
import os
from types import SimpleNamespace

import joblib
import numpy as np
import pytest

from dynaboa_b200 import _lib, build

DBOA_ERR_ARG, DBOA_ERR_SHAPE = -1, -2
FAKE = ctypes.c_void_p(0x1000)        # stand-in device pointers: every case below is rejected before one is dereferenced


@pytest.fixture(scope='module')
def lib():
    build.build()
    return _lib.load()


def metrics_active(lib, NJ=17, n_map=14, B=4, groups=2, active=0b11, null=None):
    p = [FAKE] * 7
    if null is not None:
        p[null] = None
    return lib.dboa_eval_metrics_active(p[0], p[1], p[2], p[3], NJ, 6890, p[4], n_map, p[5], p[6], B, groups, active, None)


def test_binding():
    P, I, U = ctypes.c_void_p, ctypes.c_int, ctypes.c_ulonglong
    sig = _lib.SIGNATURES
    one = sig['dboa_eval_metrics'][1]
    assert sig['dboa_eval_metrics_active'] == (I, one[:-1] + [I, U, P])


@pytest.mark.parametrize('null', range(7))
def test_null_pointers(lib, null):
    assert metrics_active(lib, null=null) == DBOA_ERR_ARG


@pytest.mark.parametrize('kw', [dict(NJ=0), dict(NJ=33), dict(n_map=0), dict(n_map=33), dict(B=0), dict(B=-1), dict(groups=0), dict(groups=65),
                                dict(groups=-1), dict(B=6, groups=4), dict(B=1, groups=2), dict(B=64, groups=128)])
def test_shape_errors(lib, kw):
    assert metrics_active(lib, **kw) == DBOA_ERR_SHAPE
    assert metrics_active(lib, active=0, **kw) == DBOA_ERR_SHAPE             # the shape is checked before the mask


@pytest.mark.parametrize('groups,active', [(2, 0), (2, 0b100), (4, 0b10000), (4, 1 << 63), (1, 0b10), (1, 0), (8, 1 << 8)])
def test_mask_errors(lib, groups, active):
    assert metrics_active(lib, B=8, groups=groups, active=active) == DBOA_ERR_ARG


def test_the_one_video_call_keeps_its_errors(lib):
    p = [FAKE] * 7
    call = lambda NJ=17, n_map=14, B=2, null=None: lib.dboa_eval_metrics(*[None if i == null else p[i] for i in range(4)], NJ, 6890,
                                                                          None if null == 4 else p[4], n_map, None if null == 5 else p[5],
                                                                          None if null == 6 else p[6], B, None)
    for i in range(7):
        assert call(null=i) == DBOA_ERR_ARG
    assert call(NJ=33) == call(n_map=0) == call(B=0) == DBOA_ERR_SHAPE


# ------------------------------------------------------------------ adapt's checks
def pool(fused_eval, G=2):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = MultiVideoAdaptor.__new__(MultiVideoAdaptor)          # no device: only the checks before any device work run
    mv.G, mv.fused_eval = G, fused_eval
    return mv


@pytest.mark.parametrize('mode', ['final', 'all'])
@pytest.mark.parametrize('key', ['pose', 'betas', 'gender'])
def test_evaluation_needs_the_ground_truth(mode, key):
    full = dict(image=None, smpl_j2d=None, pose=None, betas=None, gender=None)
    part = {k: v for k, v in full.items() if k != key}
    with pytest.raises(ValueError, match=f'slot 1: .*{key}'):
        pool(mode).adapt([full, part])
    with pytest.raises(ValueError, match=key):
        pool(mode).adapt([None, part])


def test_an_unknown_mode_is_refused():
    with pytest.raises(ValueError, match='fused_eval'):
        pool('every').adapt([dict(image=None), None])


# ------------------------------------------------------------------ the shared writer
def fixed_records(inner=3, frames=4, dynamic=True):
    rng = np.random.RandomState(5)
    arr = lambda: (rng.rand(1) * 100).astype(np.float32)
    return dict(mpjpe=[arr() for _ in range(frames)], pampjpe=[arr() for _ in range(frames)], pve=[float(rng.rand()) for _ in range(frames)],
                mpjpe_all_lower=[[arr() for _ in range(frames)] for _ in range(inner)] if dynamic else [[] for _ in range(inner)],
                pampjpe_all_lower=[[arr() for _ in range(frames)] for _ in range(inner)] if dynamic else [[] for _ in range(inner)],
                mpjpe_statistics=[[arr(), arr()] for _ in range(frames)], pampjpe_statistics=[[arr(), arr()] for _ in range(frames)],
                feat_sims={t: [{i: {'cos': 0.5} for i in range(15)}] for t in range(frames)} if dynamic else {},
                optim_step_record=[2] * frames if dynamic else [], kp2dlosses_lower=[np.float32(0.25)] * (inner * frames),
                kp2dlosses_upper={t: np.float32(0.5 + t) for t in range(frames)})


def test_writer_files_and_keys(tmp_path):
    from dynaboa_b200.adaptor import RESULT_FILES, write_records
    rec = fixed_records()
    write_records(str(tmp_path), 3, rec)
    assert sorted(os.listdir(tmp_path)) == sorted(RESULT_FILES) and len(RESULT_FILES) == 8
    keys = {'lowerlevel_kp2dloss.pt': ['kp2dloss'], 'upperlevel_kp2dloss.pt': ['kp2dloss'], 'res.pt': ['mpjpe', 'pampjpe', 'pve'],
            'lower_res.pt': ['mpjpe', 'pampjpe'], 'steps_statistic_res.pt': ['mpjpe', 'pampjpe'], 'feat_sims.pt': ['feat'],
            'optim_step_record.pt': ['step']}
    loaded = {name: joblib.load(tmp_path / name) for name in keys}
    for name, k in keys.items():
        assert list(loaded[name]) == k, name
    assert loaded['lowerlevel_kp2dloss.pt']['kp2dloss'] == [0.25] * 12
    assert loaded['upperlevel_kp2dloss.pt']['kp2dloss'] == {t: 0.5 + t for t in range(4)}
    assert all(type(x) is float for x in loaded['lowerlevel_kp2dloss.pt']['kp2dloss'])
    for k in ('mpjpe', 'pampjpe', 'pve'):
        assert len(loaded['res.pt'][k]) == 4
        assert all(np.array_equal(a, b) for a, b in zip(loaded['res.pt'][k], rec[k]))
    assert loaded['steps_statistic_res.pt']['mpjpe'][2][1] == rec['mpjpe_statistics'][2][1]
    assert loaded['optim_step_record.pt']['step'] == [2] * 4 and loaded['feat_sims.pt']['feat'] == rec['feat_sims']
    lines = (tmp_path / 'res.txt').read_text().splitlines()
    assert lines[0] == f"Step:3: MPJPE:{np.mean(rec['mpjpe'])}, PAMPJPE:{np.mean(rec['pampjpe'])}, PVE:{np.mean(rec['pve'])}"
    assert len(lines) == 4
    for i in range(3):
        assert lines[1 + i] == (f"Lower-level  Step:{i} MPJPE:{np.mean(rec['mpjpe_all_lower'][i])}, "
                                f"PAMPJPE:{np.mean(rec['pampjpe_all_lower'][i])}")


def test_adaptor_save_records_writes_what_it_wrote_before(tmp_path):
    """Adaptor.save_records through the shared writer, against the files its own body wrote before (restated here)."""
    from dynaboa_b200.adaptor import Adaptor
    rec = fixed_records(dynamic=False)
    ad = SimpleNamespace(exppath=str(tmp_path), global_step=3, options=SimpleNamespace(inner_step=3), mpjpe_all_lower=rec['mpjpe_all_lower'],
                         pampjpe_all_lower=rec['pampjpe_all_lower'], mpjpe_statistics=rec['mpjpe_statistics'],
                         pampjpe_statistics=rec['pampjpe_statistics'], feat_sims=rec['feat_sims'], optim_step_record=rec['optim_step_record'],
                         kp2dlosses_lower=rec['kp2dlosses_lower'], kp2dlosses_upper=rec['kp2dlosses_upper'])
    Adaptor.save_records(ad, rec['mpjpe'], rec['pampjpe'], rec['pve'])
    expect = {'lowerlevel_kp2dloss.pt': {'kp2dloss': [float(x) for x in rec['kp2dlosses_lower']]},
              'upperlevel_kp2dloss.pt': {'kp2dloss': {k: float(v) for k, v in rec['kp2dlosses_upper'].items()}},
              'lower_res.pt': {'mpjpe': rec['mpjpe_all_lower'], 'pampjpe': rec['pampjpe_all_lower']},
              'feat_sims.pt': {'feat': {}}, 'optim_step_record.pt': {'step': []}}
    for name, v in expect.items():
        assert joblib.load(tmp_path / name) == v, name
    res = joblib.load(tmp_path / 'res.pt')
    assert all(np.array_equal(a, b) for k in ('mpjpe', 'pampjpe', 'pve') for a, b in zip(res[k], rec[k]))
    text = f"Step:3: MPJPE:{np.mean(rec['mpjpe'])}, PAMPJPE:{np.mean(rec['pampjpe'])}, PVE:{np.mean(rec['pve'])}\n"
    text += ''.join(f'Lower-level  Step:{i} MPJPE:nan, PAMPJPE:nan\n' for i in range(3))
    assert (tmp_path / 'res.txt').read_text() == text
