"""Saving and resuming one video's adaptation (Adaptor.save_state / load_state / export_model, excute(checkpoint=...)).

N frames straight through must be bit-identical to `split` frames, save_state, a NEW Adaptor, load_state, then the rest: theta,
teacher, Adam m / v, step count, every per-frame upper loss and fit loss, every record, trip counts and cosines, the retrieval
picks and the predictions after each frame.  The teacher's dropout is drawn from torch's CUDA generator (nothing is injected),
so its state must travel with the file.  One case loads in a subprocess."""
import os
import subprocess
import sys

import pytest
import torch

from harness import bits, fetch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
# (id, workload, overrides, frames, split, path): C2 with the step graph live on both sides of the split (frames 6+ captured and
# replayed), C3 (retrieval, sample_num 8, 3 inner steps), C5 (dynamic loop), use_boa=0, the autograd path
CASES = [('c2-graph', 'c2', {}, 12, 9, 'adapt'), ('c3', 'c3', {}, 4, 2, 'adapt'), ('c5', 'c5', {}, 5, 3, 'adapt'),
         ('use_boa0', 'c2', dict(use_boa=0), 8, 4, 'adapt'), ('autograd', 'c2', {}, 8, 4, 'adaptation')]


def options(root, name, workload, n, **over):
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config
    return default_options(**{**dict(expdir=str(root), expname=name, model_file=config.BASE_MODEL, synthetic_frames=n),
                              **WORKLOADS[workload], **over})


def make(root, name, workload, n, **over):
    from dynaboa_b200.adaptor import Adaptor
    ad = Adaptor(options(root, name, workload, n, **over))
    ad.fused_eval = 'none'
    return ad


def frames(n):
    from dynaboa_b200 import synthetic
    s = synthetic.SyntheticStream(length=n, batch_size=1)
    return [fetch(s[t]) for t in range(n)]


def step(ad, t, batch, path):
    ad.global_step, ad.fit_losses = t, {}
    ad.model.eval()
    (ad.adapt if path == 'adapt' else ad.adaptation)(batch)
    pred = ad.predict(batch['image'])
    up = ad.last_upper_loss
    return dict(upper=up.detach().clone().reshape(-1).cpu() if torch.is_tensor(up) else torch.tensor([float(up)]),
                fit={k: torch.as_tensor(v).detach().clone().reshape(-1).cpu() for k, v in ad.fit_losses.items()},
                pred={k: v.clone() for k, v in pred.items()})


def final(ad):
    model = getattr(ad.model, 'module', ad.model)
    t = [model.arena, ad.optimizer.m, ad.optimizer.v] + ([ad.teacher.arena] if ad.options.use_meanteacher else [])
    fl = lambda xs: [float(x) for x in xs]
    return dict(arenas=[x.clone().cpu() for x in t], steps=ad.optimizer.step_count, lower=fl(ad.kp2dlosses_lower),
                upper={k: float(v) for k, v in ad.kp2dlosses_upper.items()}, trips=list(ad.optim_step_record),
                sims={k: v for k, v in ad.feat_sims.items()}, pick=getattr(ad, 'last_retrieval', None),
                rng=torch.cuda.get_rng_state())


def same(a, b):
    return torch.equal(bits(a), bits(b))


def compare(x, y, what):
    assert torch.equal(bits(x['upper']), bits(y['upper'])), what
    assert x['fit'].keys() == y['fit'].keys(), what
    for k in x['fit']:
        assert same(x['fit'][k], y['fit'][k]), (what, k)
    for k in x['pred']:
        assert same(x['pred'][k], y['pred'][k]), (what, k)


def compare_final(a, b):
    assert len(a['arenas']) == len(b['arenas'])
    for i, (x, y) in enumerate(zip(a['arenas'], b['arenas'])):
        assert same(x, y), ('theta', 'm', 'v', 'teacher')[i]
    for k in ('steps', 'lower', 'upper', 'trips', 'sims', 'pick'):
        assert a[k] == b[k], k
    assert torch.equal(a['rng'], b['rng'])


def child(root, assets, workload, over, n, split, path, ck, out):
    """The second half of a split run in a process of its own: a new Adaptor, load_state, the frames from `split` on."""
    from dynaboa_b200 import config
    config.set_data_root(assets)
    ad = make(root, 'child', workload, n, **over)
    ad.load_state(ck)
    fs = frames(n)
    recs = [step(ad, t, fs[t], path) for t in range(split, n)]
    torch.save(dict(recs=recs, final=final(ad)), out)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_save_load_continues_bit_for_bit(asset_dir, tmp_path, case):
    name, workload, over, n, split, path = case
    fs = frames(n)
    ad = make(tmp_path, 'straight', workload, n, **over)
    straight = [step(ad, t, fs[t], path) for t in range(n)]
    if name == 'c2-graph':
        assert ad._graph is not None, 'the step graph was not live'
    want = final(ad)
    del ad
    ad = make(tmp_path, 'first', workload, n, **over)
    first = [step(ad, t, fs[t], path) for t in range(split)]
    ck = str(tmp_path / 'state.pt')
    ad.save_state(ck)
    del ad
    for t in range(split):
        compare(straight[t], first[t], t)
    if name == 'c2-graph':                                    # a process of its own: no in-process state can leak
        out = str(tmp_path / 'child.pt')
        code = (f'import sys; sys.path[:0] = [{os.path.dirname(HERE)!r}, {HERE!r}]; import test_gpu_resume as m; '
                f'm.child({str(tmp_path)!r}, {str(asset_dir)!r}, {workload!r}, {over!r}, {n}, {split}, {path!r}, {ck!r}, {out!r})')
        subprocess.run([sys.executable, '-c', code], check=True, timeout=900)
        got = torch.load(out, weights_only=False)
        rest, end = got['recs'], got['final']
    else:
        ad = make(tmp_path, 'second', workload, n, **over)
        ad.load_state(ck)
        rest = [step(ad, t, fs[t], path) for t in range(split, n)]
        if name == 'c2-graph':
            assert ad._graph is not None
        end = final(ad)
    for t, r in zip(range(split, n), rest):
        compare(straight[t], r, t)
    compare_final(want, end)
    if workload == 'c5':
        assert any(want['trips']), 'the dynamic loop never ran'


def test_webcam_frame_count_round_trips(asset_dir, tmp_path, golden):
    from harness import cam_options
    from dynaboa_b200.webcam import WebcamAdaptor
    gd = golden('adapt_webcam')
    fs = frames(8)
    kps = fs
    a = WebcamAdaptor(cam_options(tmp_path / 'a', gd))
    for f in kps:
        a.adapt_processed(f['image'], f['smpl_j2d'])
    b = WebcamAdaptor(cam_options(tmp_path / 'b', gd))
    for f in kps[:5]:
        b.adapt_processed(f['image'], f['smpl_j2d'])
    ck = str(tmp_path / 'cam.pt')
    b.save_state(ck)
    c = WebcamAdaptor(cam_options(tmp_path / 'c', gd))
    c.load_state(ck)
    assert c.global_step == 5
    for f in kps[5:]:
        c.adapt_processed(f['image'], f['smpl_j2d'])
    assert c.global_step == a.global_step == 8
    assert same(c.model.module.arena, a.model.module.arena) and same(c.optimizer.m, a.optimizer.m)


def test_excute_resumes_to_identical_result_files(asset_dir, tmp_path):
    from dynaboa_b200.adaptor import RESULT_FILES, Adaptor
    n = 10
    Adaptor(options(tmp_path, 'straight', 'c2', n)).excute(fused=True)
    ck = str(tmp_path / 'excute.pt')
    Adaptor(options(tmp_path, 'cut', 'c2', n)).excute(max_frames=7, fused=True, checkpoint=ck, every=3)   # last checkpoint: frame 6
    resumed = Adaptor(options(tmp_path, 'resumed', 'c2', n))
    resumed.excute(fused=True, checkpoint=ck, every=3)
    for f in RESULT_FILES:
        with open(tmp_path / 'straight' / f, 'rb') as x, open(tmp_path / 'resumed' / f, 'rb') as y:
            assert x.read() == y.read(), f


def test_data_parallel_optimizer_is_refused(asset_dir, tmp_path):
    ad = make(tmp_path, 'dp', 'c2', 2)
    ad.optimizer.pre_step_hook = lambda g: None
    with pytest.raises(ValueError, match='data-parallel'):
        ad.save_state(str(tmp_path / 'x.pt'))
    with pytest.raises(ValueError, match='data-parallel'):
        ad.load_state(str(tmp_path / 'x.pt'))


@pytest.mark.parametrize('use_boa', [1, 0])
def test_exported_model_predicts_as_the_exporter(asset_dir, tmp_path, use_boa):
    from dynaboa_b200.adaptor import Adaptor
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    fs = frames(3)
    ad = make(tmp_path, 'exp', 'c2', 3, use_boa=use_boa)
    for t in range(3):
        step(ad, t, fs[t], 'adapt')
    path = str(tmp_path / 'basemodel.pt')
    ad.export_model(path)
    fresh = Adaptor(options(tmp_path, 'fresh', 'c2', 3, use_boa=use_boa, model_file=path))
    for f in fs:
        want, got = ad.predict(f['image']), fresh.predict(f['image'])
        assert all(same(want[k], got[k]) for k in want)
    if use_boa:                                            # a pool of the exported model: its slots start from the exporter's theta
        mv = MultiVideoAdaptor(options(tmp_path, 'pool', 'c2', 3, model_file=path), 2)
        assert same(mv.thetas[1], ad.model.module.arena)
        mv.export_model(1, str(tmp_path / 'again.pt'))
        again = torch.load(str(tmp_path / 'again.pt'), weights_only=True)['model']
        first = torch.load(path, weights_only=True)['model']
        assert list(again) == list(first) and all(torch.equal(again[k], first[k]) for k in first)
