"""The saved-state format (dynaboa_b200/state.py) without a device: a video state round-trips, every refusal is a ValueError
raised before any device work, weights-only loading refuses pickled objects, a pool checkpoint without a manifest is passed
over, and the exported model maps the flat arena to the reference's state_dict."""
import os
import pickle
import random

import numpy as np
import pytest
import torch

from harness import built_lib, cpu_options


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def arenas(P, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(P, generator=gen) for _ in range(4)]


def make_state(options, seed=5):
    from dynaboa_b200 import layout, state
    P = layout.arena_layout().floats
    theta, teacher, m, v = arenas(P, seed)
    gen = torch.Generator().manual_seed(seed + 1)
    hist = [(k, torch.randn(1, 3, 224, 224, generator=gen), torch.randn(1, 49, 3, generator=gen)) for k in range(3, 9)]
    rng = random.Random(seed)
    rng.random()
    records = dict(mpjpe_all=[np.float32([1.5]), np.float32([2.25])], pve_all=[3.0, 4.5], feat_sims={0: [{12: {'cos': 0.9}}]},
                   optim_step_record=[0, 3], mpjpe_statistics={1: [np.float32([7.0])]}, kp2dloss_upper_all={4: 0.125},
                   last_retrieval=(2, [5, 9]), optimized_step=None, last_upper_loss=torch.tensor([0.5]))
    st = state.video_state(options, 'slot', 4, theta, teacher, m, v, 7, 9, hist, dict(random=rng.getstate()), records)
    return st, (theta, teacher, m, v, hist, rng, records)


def test_round_trip(lib, tmp_path):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    st, (theta, teacher, m, v, hist, rng, records) = make_state(o)
    path = str(tmp_path / 'slot.pt')
    state.write(path, st)
    back = state.read_video(path, o, 'slot', G=4)
    for k, t in zip(('theta', 'teacher', 'm', 'v'), (theta, teacher, m, v)):
        assert torch.equal(back[k].view(torch.int32), t.view(torch.int32)), k
    assert back['step_count'] == 7 and back['frames'] == 9
    assert sorted(back['history']) == [k for k, _, _ in hist]
    for k, a, b in hist:
        assert torch.equal(back['history'][k][0], a) and torch.equal(back['history'][k][1], b)
    r = random.Random()
    r.setstate(back['rng']['random'])
    assert r.random() == rng.random()
    rec = back['records']
    assert [type(x) for x in rec['mpjpe_all']] == [np.ndarray] * 2 and rec['mpjpe_all'][1].dtype == np.float32
    assert pickle.dumps(rec['mpjpe_all']) == pickle.dumps(records['mpjpe_all'])          # the record files come out byte-identical
    assert pickle.dumps(rec['mpjpe_statistics']) == pickle.dumps(records['mpjpe_statistics'])
    assert rec['feat_sims'] == records['feat_sims'] and rec['kp2dloss_upper_all'] == records['kp2dloss_upper_all']
    assert rec['last_retrieval'] == (2, [5, 9]) and rec['optim_step_record'] == [0, 3] and rec['optimized_step'] is None
    with pytest.raises(ValueError, match='kind'):
        state.read_video(path, o, 'adaptor')
    with pytest.raises(ValueError, match='8'):
        state.read_video(path, o, 'slot', G=8)


def rewrite(path, **fields):
    obj = torch.load(path, weights_only=True)
    obj.update(fields)
    torch.save(obj, path)


@pytest.mark.parametrize('field,value,match', [('version', 2, 'version'), ('P', 1234, 'arena of 1234'),
                                               ('layout', '0' * 64, 'parameter table'), ('format', 'something.else', 'unknown format')])
def test_refusals_of_the_header(lib, tmp_path, field, value, match):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    path = str(tmp_path / 's.pt')
    state.write(path, make_state(o)[0])
    rewrite(path, **{field: value})
    with pytest.raises(ValueError, match=match):
        state.read_video(path, o, 'slot', G=4)


def test_truncated_file(lib, tmp_path):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    path = str(tmp_path / 's.pt')
    state.write(path, make_state(o)[0])
    size = os.path.getsize(path)
    with open(path, 'r+b') as f:
        f.truncate(size // 2)
    with pytest.raises(ValueError, match='truncated or malformed'):
        state.read_video(path, o, 'slot', G=4)


def test_options_rule(lib, tmp_path):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    path = str(tmp_path / 's.pt')
    state.write(path, make_state(o)[0])
    allowed = cpu_options('c2')
    vars(allowed).update(expdir='/elsewhere', expname='other', tensorboard=1, save_res=1, model_file='exported.pt', synthetic_frames=99,
                         cache_results=1)
    state.read_video(path, allowed, 'slot', G=4)
    with pytest.raises(ValueError) as e:
        state.read_video(path, cpu_options('c2', lr=1e-5, interval=4), 'slot', G=4)
    assert 'lr' in str(e.value) and 'interval' in str(e.value) and 'expdir' not in str(e.value)
    with pytest.raises(ValueError, match='retrieval'):
        state.read_video(path, cpu_options('c3'), 'slot', G=4)
    extra = cpu_options('c2', new_flag=1)
    with pytest.raises(ValueError, match='new_flag'):
        state.read_video(path, extra, 'slot', G=4)


class _Payload:
    ran = []

    def __reduce__(self):
        return (_Payload.ran.append, ('executed',))


def test_weights_only_refuses_pickled_objects(lib, tmp_path):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    st = make_state(o)[0]
    st['records'] = {'evil': _Payload()}
    path = str(tmp_path / 's.pt')
    torch.save(st, path)
    with pytest.raises(ValueError, match='truncated or malformed'):
        state.read_video(path, o, 'slot', G=4)
    assert _Payload.ran == []


def test_atomic_write_keeps_the_previous_file(lib, tmp_path):
    from dynaboa_b200 import state
    path = str(tmp_path / 'x.pt')
    state.write(path, {'a': torch.ones(3)})

    class Boom:
        def __reduce__(self):
            raise RuntimeError('cut short')
    with pytest.raises(RuntimeError, match='cut short'):
        state.write(path, {'a': Boom()})
    assert torch.equal(torch.load(path, weights_only=True)['a'], torch.ones(3))
    assert os.listdir(tmp_path) == ['x.pt']                                # no temporary file left behind


def test_a_checkpoint_without_manifest_is_ignored(lib, tmp_path):
    from dynaboa_b200 import state
    root = str(tmp_path / 'ck')
    assert state.latest(root) is None
    first = state.new_checkpoint(root)
    state.write(os.path.join(first, 'pool.pt'), {'n': 1})
    state.commit(root, first, {0: 'slot0.pt'})
    second = state.new_checkpoint(root)                   # a checkpoint cut short before its manifest
    state.write(os.path.join(second, 'pool.pt'), {'n': 2})
    path, man = state.latest(root)
    assert path == first and man['slots'] == {0: 'slot0.pt'}
    with open(os.path.join(second, state.MANIFEST_FILE), 'wb') as f:
        f.write(b'\x80\x02garbage')                       # a torn manifest counts as none
    assert state.latest(root)[0] == first
    third = state.new_checkpoint(root)
    state.commit(root, third, {})
    assert state.latest(root)[0] == third
    assert sorted(os.listdir(root)) == [os.path.basename(third)]          # older checkpoints are removed once a newer one is complete


def test_export_mapping_loads_into_the_reference_hmr(lib, tmp_path):
    from dynaboa_b200 import layout, synthetic
    from oracle import hmr_ref
    lay = layout.arena_layout()
    arena = torch.randn(lay.floats, generator=torch.Generator().manual_seed(3))
    mean = synthetic.make_mean_params()
    buffers = {k: torch.as_tensor(np.asarray(mean[k.split('_')[1]]), dtype=torch.float32).reshape(shape)
               for k, shape in layout.buffer_shapes().items()}
    sd = layout.state_dict(arena, buffers, prefix='module.')
    want = list(layout.param_shapes().items()) + list(layout.buffer_shapes().items())
    assert [(k[len('module.'):], tuple(v.shape)) for k, v in sd.items()] == [(k, tuple(s)) for k, s in want]
    for (name, view) in zip(lay.names, lay.views(arena)):
        t = sd['module.' + name]
        assert t.is_contiguous() and torch.equal(t, view), name
        assert t.untyped_storage().nbytes() == t.numel() * 4, name          # its own storage, not the arena's
    ref_hmr = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'model', 'hmr.py')
    if not os.path.exists(ref_hmr):
        pytest.skip('the reference model/hmr.py is not staged under oracle/_ref')
    import importlib.util
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(ref_hmr)))
    try:
        spec = importlib.util.spec_from_file_location('staged_ref_hmr', ref_hmr)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.pop(0)
    np.savez(tmp_path / 'mean.npz', **mean)
    model = mod.hmr(str(tmp_path / 'mean.npz'))
    model.load_state_dict(hmr_ref.strip_prefix(sd), strict=True)
    for name, t in model.state_dict().items():
        assert torch.equal(t, sd['module.' + name]), name
