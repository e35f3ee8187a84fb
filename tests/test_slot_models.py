"""Per-slot checkpoints without a device: every refusal of layout.read_checkpoint, the digest as a model's identity,
arena_from_state_dict as the inverse of state_dict, the argument checks of start(g, model=) and run(..., models=) that run
before any file or device work, and the model entry of a slot state."""
import os
import random
from collections import OrderedDict
from types import SimpleNamespace

import pytest
import torch

from harness import built_lib, cpu_options, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def buffers(seed=22):
    """The pool's init_* buffers: those every synthetic checkpoint carries."""
    from dynaboa_b200 import synthetic
    sd = synthetic.make_basemodel(seed)['model']
    return {k: sd['module.' + k] for k in ('init_pose', 'init_shape', 'init_cam')}


def write(tmp_path, name, obj):
    path = str(tmp_path / name)
    torch.save(obj, path)
    return path


def checkpoint(seed=3):
    from dynaboa_b200 import synthetic
    return synthetic.make_basemodel(seed)


def test_checkpoint_reads_into_the_state_dict_arena(lib, tmp_path):
    from dynaboa_b200 import layout
    ck = checkpoint()
    arena, digest = layout.read_checkpoint(write(tmp_path, 'x.pt', ck), buffers())
    lay = layout.arena_layout()
    assert arena.shape == (lay.floats,) and arena.dtype == torch.float32 and len(digest) == 64
    sd = layout.state_dict(arena, buffers(), prefix='module.')
    assert list(sd) == list(ck['model'])
    for k, v in ck['model'].items():
        assert torch.equal(sd[k].view(torch.int32), v.view(torch.int32)), k
    covered = torch.zeros(lay.floats, dtype=torch.bool)
    for v in lay.views(covered):
        v.fill_(True)
    assert not arena[~covered].any()                        # the padding stays zero, as in a model loaded with load_state_dict


def test_the_digest_is_the_weights(lib, tmp_path):
    """Key order, container type and file name do not change the digest; one changed bit does."""
    from dynaboa_b200 import layout
    ck = checkpoint()
    _, d = layout.read_checkpoint(write(tmp_path, 'a.pt', ck), buffers())
    shuffled = list(ck['model'].items())
    random.Random(1).shuffle(shuffled)
    _, d2 = layout.read_checkpoint(write(tmp_path, 'b.pt', {'model': dict(shuffled), 'epoch': 3}), buffers())
    assert d2 == d
    _, d3 = layout.read_checkpoint(write(tmp_path, 'c.pt', checkpoint(4)), buffers())
    assert d3 != d
    flipped = OrderedDict(ck['model'])
    w = flipped['module.deccam.bias'].clone()
    w.view(torch.int32)[0] ^= 1
    flipped['module.deccam.bias'] = w
    _, d4 = layout.read_checkpoint(write(tmp_path, 'd.pt', {'model': flipped}), buffers())
    assert d4 != d


def test_float64_and_float16_values_are_cast_as_load_state_dict_casts_them(lib, tmp_path):
    from dynaboa_b200 import layout
    ck = checkpoint()
    a, _ = layout.read_checkpoint(write(tmp_path, 'a.pt', ck), buffers())
    sd = OrderedDict((k, v.double() if k.endswith('fc2.weight') else v) for k, v in ck['model'].items())
    b, _ = layout.read_checkpoint(write(tmp_path, 'b.pt', {'model': sd}), buffers())
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def edited(edit):
    sd = OrderedDict(checkpoint()['model'])
    edit(sd)
    return {'model': sd}


def _nan(sd):
    w = sd['module.layer2.0.conv2.weight'].clone()
    w[0, 0, 1, 1] = float('nan')
    sd['module.layer2.0.conv2.weight'] = w


def _inf(sd):
    sd['module.fc1.bias'] = sd['module.fc1.bias'].clone().fill_(float('inf'))


BAD = {
    'missing': (lambda sd: sd.pop('module.layer3.4.bn2.bias'), 'missing key .*layer3.4.bn2.bias'),
    'missing buffer': (lambda sd: sd.pop('module.init_cam'), 'missing key .*init_cam'),
    'unprefixed': (lambda sd: sd.update({k[len('module.'):]: sd.pop(k) for k in list(sd)}), 'missing key .*module.conv1.weight'),
    'extra': (lambda sd: sd.update({'module.fc3.weight': torch.zeros(3)}), 'unexpected key .*fc3.weight'),
    'extra buffer': (lambda sd: sd.update({'module.init_scale': torch.zeros(1)}), 'unexpected key .*init_scale'),
    'shape': (lambda sd: sd.update({'module.conv1.weight': sd['module.conv1.weight'].reshape(64, 3, 49)}), 'conv1.weight has shape'),
    'transposed': (lambda sd: sd.update({'module.fc2.weight': sd['module.fc2.weight'][:, :1000]}), 'fc2.weight has shape'),
    'buffer shape': (lambda sd: sd.update({'module.init_shape': torch.zeros(10)}), 'init_shape has shape'),
    'integer': (lambda sd: sd.update({'module.decshape.bias': torch.zeros(10, dtype=torch.int32)}), 'decshape.bias is not float'),
    'not a tensor': (lambda sd: sd.update({'module.deccam.bias': [0.0, 0.0, 0.0]}), 'deccam.bias is not float'),
    'nan': (_nan, 'layer2.0.conv2.weight holds values that are not finite'),
    'inf': (_inf, 'fc1.bias holds values that are not finite'),
    'foreign init_cam': (lambda sd: sd.update({'module.init_cam': sd['module.init_cam'] + 0.5}), 'init_cam differs'),
    'init_pose one bit off': (lambda sd: sd['module.init_pose'].view(torch.int32)[0, 3].__ixor__(1), 'init_pose differs'),
}


@pytest.mark.parametrize('case', sorted(BAD))
def test_refusals_name_the_file_and_the_key(lib, tmp_path, case):
    from dynaboa_b200 import layout
    edit, match = BAD[case]
    path = write(tmp_path, 'bad.pt', edited(edit))
    with pytest.raises(ValueError, match=match) as e:
        layout.read_checkpoint(path, buffers())
    assert path in str(e.value)


@pytest.mark.parametrize('case', ['missing file', 'garbage', 'truncated', 'pickled object', 'list', 'no model', 'model not a dict'])
def test_a_file_that_is_no_checkpoint(lib, tmp_path, case):
    from dynaboa_b200 import layout
    path = str(tmp_path / 'x.pt')
    if case == 'garbage':
        with open(path, 'wb') as f:
            f.write(b'\x00not a torch file' * 10)
    elif case == 'truncated':
        torch.save(checkpoint(), path)
        with open(path, 'r+b') as f:
            f.truncate(os.path.getsize(path) // 2)
    elif case == 'pickled object':
        torch.save({'model': checkpoint()['model'], 'options': SimpleNamespace(lr=1)}, path)
    elif case != 'missing file':
        torch.save({'list': [torch.zeros(2)], 'no model': {'state_dict': checkpoint()['model']},
                    'model not a dict': {'model': torch.zeros(3)}}[case], path)
    with pytest.raises(ValueError, match='not a (readable )?checkpoint') as e:
        layout.read_checkpoint(path, buffers())
    assert path in str(e.value)


def test_arena_from_state_dict_inverts_state_dict(lib):
    from dynaboa_b200 import layout
    lay = layout.arena_layout()
    gen = torch.Generator().manual_seed(9)
    a = torch.zeros(lay.floats)
    for v in lay.views(a):
        v.copy_(torch.randn(v.shape, generator=gen))
    sd = layout.state_dict(a, buffers())
    back = layout.arena_from_state_dict(sd, torch.zeros(lay.floats))
    assert torch.equal(back.view(torch.int32), a.view(torch.int32))
    prefixed = layout.state_dict(a, buffers(), prefix='module.')
    assert torch.equal(layout.arena_from_state_dict(prefixed, torch.zeros(lay.floats), prefix='module.'), a)
    with pytest.raises(ValueError, match='flat fp32 arena'):
        layout.arena_from_state_dict(sd, torch.zeros(lay.floats + 4))
    with pytest.raises(ValueError, match='flat fp32 arena'):
        layout.arena_from_state_dict(sd, torch.zeros(lay.floats, dtype=torch.float64))


# ------------------------------------------------------------------ argument checks of the pools
def test_models_checks_in_run(lib):
    from dynaboa_b200.multivideo import MultiVideoAdaptor, check_models
    assert check_models(None, 2) == [None, None]
    import pathlib
    assert check_models([pathlib.Path('/a/b.pt'), None], 2) == ['/a/b.pt', None]
    mv = idle_pool(MultiVideoAdaptor, 2, options=cpu_options('c2'))
    with pytest.raises(ValueError, match='1 models for 2 videos'):
        mv.run([[], []], models=['x.pt'])
    with pytest.raises(ValueError, match='one path for all'):
        mv.run([[], []], models='x.pt')
    with pytest.raises(ValueError, match='video 1: model'):
        mv.run([[], []], models=[None, 3])
    with pytest.raises(ValueError, match='video 0: model'):
        mv.run([[]], models=[b'x.pt'])
    with pytest.raises(ValueError, match='video 0: model'):
        mv.run([[]], models=[''])


def test_models_checks_in_the_internet_run(lib, tmp_path):
    from dynaboa_b200.internet import MultiInternetAdaptor

    class Video:
        name = 'v'

        def __len__(self):
            return 1

        def frame(self, t):
            raise AssertionError('no frame is read before the checks')
    mv = idle_pool(MultiInternetAdaptor, 2, options=cpu_options('c2'))
    with pytest.raises(ValueError, match='1 models for 2 videos'):
        mv.run([Video(), Video()], str(tmp_path), names=['a', 'b'], models=[None])
    with pytest.raises(ValueError, match='video 0: model'):
        mv.run([Video()], str(tmp_path), models=[1.5])
    assert not os.listdir(tmp_path)


def test_start_checks_before_device_work(lib, tmp_path):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = idle_pool(MultiVideoAdaptor, 3, options=cpu_options('c2'), buffers=buffers())
    with pytest.raises(ValueError, match='slot 1: model'):
        mv.start(1, model=7)
    with pytest.raises(ValueError, match='slot'):
        mv.start(3, model=str(tmp_path / 'x.pt'))
    with pytest.raises(ValueError, match='not a readable checkpoint'):
        mv.start(0, model=str(tmp_path / 'missing.pt'))
    with pytest.raises(ValueError, match='init_cam differs'):
        mv.start(0, model=write(tmp_path, 'foreign.pt', edited(BAD['foreign init_cam'][0])))
    with pytest.raises(ValueError, match='beta1'):                    # hparams are checked before the file is read
        mv.start(0, hparams={'beta1': 2.0}, model=str(tmp_path / 'missing.pt'))


# ------------------------------------------------------------------ the model entry of a slot state
DIGEST = 'ab' * 32


def test_model_entry(lib):
    from dynaboa_b200 import state
    assert state.saved_model({}) is None and state.saved_model({'model': None}) is None
    assert state.saved_model({'model': {'path': '/m/x.pt', 'digest': DIGEST}}) == ('/m/x.pt', DIGEST)
    for bad in ({'path': '/m/x.pt'}, {'path': 3, 'digest': DIGEST}, {'path': 'x', 'digest': 'AB' * 32}, {'path': 'x', 'digest': 'ab'},
                {'path': 'x', 'digest': DIGEST, 'size': 1}, ('x', DIGEST), 'x'):
        with pytest.raises(ValueError, match='model entry'):
            state.saved_model({'model': bad}, 'slot.pt')


def make_state(options, model=None):
    from dynaboa_b200 import layout, state
    P = layout.arena_layout().floats
    z = torch.zeros(P)
    return state.video_state(options, 'slot', 2, z, z, z, z, 0, 0, [], dict(random=random.Random(1).getstate()),
                             dict(last_upper_loss=torch.zeros(1)), model=model)


def test_state_with_and_without_a_model_entry(lib, tmp_path):
    from dynaboa_b200 import state
    o = cpu_options('c2')
    assert 'model' not in make_state(o)                                 # a slot on the pool's checkpoint: the files of before
    path = str(tmp_path / 's.pt')
    state.write(path, make_state(o, model=('/m/x.pt', DIGEST)))
    st = state.read_video(path, o, 'slot', G=2)
    assert state.saved_model(st) == ('/m/x.pt', DIGEST) and st['version'] == 1
    obj = torch.load(path, weights_only=True)
    obj['model'] = {'path': '/m/x.pt', 'digest': 'not a digest'}
    torch.save(obj, path)
    with pytest.raises(ValueError, match=f'{path}: malformed video state: the model entry'):
        state.read_video(path, o, 'slot', G=2)
    del obj['model']
    torch.save(obj, path)
    assert state.saved_model(state.read_video(path, o, 'slot', G=2)) is None


def test_a_state_on_its_own_model_needs_it_again(lib, tmp_path):
    """start(g, state=) of a state whose model file is gone: ValueError before any device work (the pool has no device)."""
    from dynaboa_b200 import state
    from dynaboa_b200.multivideo import PER_VIDEO, MultiVideoAdaptor
    o = cpu_options('c2')
    path = str(tmp_path / 's.pt')
    gone = str(tmp_path / 'gone.pt')
    state.write(path, make_state(o, model=(gone, DIGEST)))
    mv = idle_pool(MultiVideoAdaptor, 2, options=o, buffers=buffers())
    with pytest.raises(ValueError, match='gone.pt: not a readable checkpoint'):
        mv.start(0, state=path)
    st = state.read_video(path, o, 'slot', G=2, own=PER_VIDEO)
    with pytest.raises(ValueError, match='missing.pt: not a readable checkpoint'):
        mv.start(1, state=st, model=str(tmp_path / 'missing.pt'))
