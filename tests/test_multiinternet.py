"""Internet pool without a device: ``datasets.internet_videos`` on empty and malformed folders, the argument checks of
MultiInternetAdaptor.run / input_side, the options the pool rejects, and the file layout ``write`` produces (a stub writer)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from dynaboa_b200.datasets import InternetVideo, internet_videos
from dynaboa_b200.internet import MultiInternetAdaptor, check_options, output_paths
from harness import built_lib, cpu_options, idle_pool


@pytest.fixture(scope='module')
def lib():
    return built_lib()


def npz(path, n=3, **over):
    d = dict(imgname=np.array([f'f{t:03d}.png' for t in range(n)]), center=np.full((n, 2), 100.0), scale=np.full(n, 0.9),
             part=np.ones((n, 49, 3)))
    d.update(over)
    np.savez(path, **{k: v for k, v in d.items() if v is not None})


def test_videos_sorted_by_name(tmp_path):
    for name, n in (('b', 3), ('a', 2), ('c', 0)):
        npz(tmp_path / f'{name}.npz', n)
    (tmp_path / 'notes.txt').write_text('not a sequence')
    vids = internet_videos(str(tmp_path))
    assert [v.name for v in vids] == ['a', 'b', 'c'] and [len(v) for v in vids] == [2, 3, 0]
    path, center, scale, kp, bbox = vids[1].frame(2)
    assert path == os.path.join(str(tmp_path), 'images', 'f002.png')
    assert center == [100.0, 100.0] and scale == 0.9 and kp.dtype == np.float32 and kp.shape == (49, 3)
    assert bbox.shape == (1, 3) and bbox.dtype == np.float64 and bbox[0, 2] == 0.9 * 200
    with pytest.raises(IndexError):
        vids[0].frame(2)


def test_empty_and_missing_folders(tmp_path):
    with pytest.raises(FileNotFoundError, match='no'):
        internet_videos(str(tmp_path))
    with pytest.raises(FileNotFoundError, match='not a directory'):
        internet_videos(str(tmp_path / 'absent'))


@pytest.mark.parametrize('over,match', [
    (dict(part=None), 'missing part'),
    (dict(center=None, scale=None), 'missing center, scale'),
    (dict(center=np.zeros((2, 2))), 'center of shape'),
    (dict(scale=np.zeros((3, 1))), 'scale of shape'),
    (dict(part=np.zeros((3, 25, 3))), 'part of shape'),
    (dict(imgname=np.array([['a', 'b', 'c']])), 'imgname of shape'),
])
def test_malformed_npz(tmp_path, over, match):
    npz(tmp_path / 'v.npz', **over)
    with pytest.raises(ValueError, match=match):
        internet_videos(str(tmp_path))


def test_unreadable_npz(tmp_path):
    (tmp_path / 'v.npz').write_bytes(b'not a zip archive')
    with pytest.raises(ValueError, match='not a readable npz'):
        InternetVideo(str(tmp_path / 'v.npz'), str(tmp_path / 'images'))


def videos(tmp_path, names=('a', 'b')):
    for n in names:
        npz(tmp_path / f'{n}.npz')
    return internet_videos(str(tmp_path))


def test_run_checks(tmp_path):
    mv = idle_pool(MultiInternetAdaptor, 2, options=SimpleNamespace(cache_results=1, save_res=0))
    vids = videos(tmp_path)
    with pytest.raises(ValueError, match='1 names for 2 videos'):
        mv.run(vids, str(tmp_path / 'out'), names=['x'])
    with pytest.raises(ValueError, match='3 names for 2 videos'):
        mv.run(vids, str(tmp_path / 'out'), names=['x', 'y', 'z'])
    with pytest.raises(ValueError, match='one directory'):
        mv.run(vids, str(tmp_path / 'out'), names=['x', 'x'])
    with pytest.raises(ValueError, match='one directory'):
        mv.run([vids[0], vids[0]], str(tmp_path / 'out'))
    with pytest.raises(ValueError, match='video 1 is a list'):
        mv.run([vids[0], [1, 2]], str(tmp_path / 'out'))
    assert not (tmp_path / 'out').exists()                   # nothing is written before the checks pass


def test_input_side_checks(tmp_path):
    mv = idle_pool(MultiInternetAdaptor, 2)
    vids = videos(tmp_path)
    with pytest.raises(ValueError, match='2 frames'):
        mv.input_side([(vids[0], 0)])
    with pytest.raises(ValueError, match='slot 1'):
        mv.input_side([None, vids[0]])
    with pytest.raises(IndexError):
        mv.input_side([(vids[0], 3), None])
    assert mv.input_side([None, None]) == (0, [None, None], [None, None])        # nothing to stage: no device work


def internet_opts(**extra):
    return cpu_options('c2', dataset='internet', save_res=1, **extra)


def test_pool_options(lib):
    assert MultiInternetAdaptor.kp_range == (25, 24) and MultiInternetAdaptor.motion_lead == 0
    check_options(internet_opts(dynamic_boa=1), 64, dynamic_loop=True)
    with pytest.raises(ValueError, match='dynamic_loop'):
        check_options(internet_opts(dynamic_boa=1), 2)
    with pytest.raises(ValueError, match='use_boa=0'):
        check_options(internet_opts(use_boa=0), 2, dynamic_loop=True)
    with pytest.raises(ValueError, match='batch_size=2'):
        check_options(internet_opts(batch_size=2), 2)
    with pytest.raises(ValueError, match='exceed'):
        check_options(internet_opts(), 65)
    with pytest.raises(ValueError, match='exceed'):
        check_options(internet_opts(retrieval=1, lower_level_mixtrain=1, sample_num=2), 33)
    with pytest.raises(ValueError, match='at least 1'):
        check_options(internet_opts(), 0)
    prev = lib.dboa_get_fused_backward()
    lib.dboa_set_fused_backward(1)
    try:
        with pytest.raises(ValueError, match='fused'):
            check_options(internet_opts(), 2)
    finally:
        lib.dboa_set_fused_backward(prev)
    with pytest.raises(ValueError, match='batch_size'):        # rejected before any device or file is touched
        MultiInternetAdaptor(internet_opts(batch_size=4), 2)


class Stub:
    def __init__(self):
        self.calls = []

    def pred(self, path, arrays):
        self.calls.append(('pred', path, sorted(arrays)))

    def image(self, path, bgr):
        self.calls.append(('image', path, bgr.shape))


@pytest.mark.parametrize('cache', [0, 1])
def test_file_layout(cache):
    mv = idle_pool(MultiInternetAdaptor, 3, options=SimpleNamespace(cache_results=cache), writer=Stub())
    pred = {k: np.zeros(1) for k in ('verts', 'cam', 'rotmat', 'beta')}
    for t in range(2):
        files = []
        for g, name in ((0, 'walk'), (2, 'run')):
            p, q = output_paths('/exp', name, t)
            files.append((g, p, pred, q if g == 2 else None, np.zeros((4, 6, 3), np.uint8) if g == 2 else None))
        mv.write(files)
    expect = []
    for t in range(2):
        if cache:
            expect.append(('pred', f'/exp/walk/result/Pred_{t}.pt', ['beta', 'cam', 'rotmat', 'verts']))
        if cache:
            expect.append(('pred', f'/exp/run/result/Pred_{t}.pt', ['beta', 'cam', 'rotmat', 'verts']))
        expect.append(('image', f'/exp/run/image/Pred_{t}.png', (4, 6, 3)))
    assert mv.writer.calls == expect
