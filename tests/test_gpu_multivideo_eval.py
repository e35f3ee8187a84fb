"""Evaluation of the videos of a MultiVideoAdaptor pool (``fused_eval`` 'final' / 'all', ``records``, ``run``).

- dboa_eval_metrics_active: every active row bit-identical to dboa_eval_metrics on that video's rows alone, idle rows' NaN
  inputs not read and their rows of out left with a sentinel, groups = 1 with every bit set is dboa_eval_metrics, and the
  eval_metrics.npz golden holds through the new entry.
- One video is Adaptor: every record of MultiVideoAdaptor(opts, 1) bit-identical to the captured ``Adaptor.inference`` values
  of the same frames, filed by the pool's rules, at C2 and at C5 with a loop whose trip counts vary, for 'all' and 'final'.
- Several videos: G = 4 at C2 and C5, each video's records with the entry counts of its own single-video run and values within
  1e-3 relative of it.
- Schedule invariance of a video's records, and no entry for a frame a slot sits out.
- ``run``: 6 videos through 4 slots, each video's summary and files bit-identical to that video alone through ``run``, and the
  files shaped like ``Adaptor.excute(fused=True)``'s.
- An all-active pool frame makes as many host synchronisations with 'final' as with 'none'."""
import os
import warnings

import joblib
import numpy as np
import pytest
import torch

from conftest import rel_err
from harness import MIXED_THRESHOLD, N_FRAMES, PoolRun, SingleRun, bits, fetch, pool_options, stream, video_masks

pytestmark = pytest.mark.gpu
SENTINEL = 0x7fc0dead                  # a NaN payload no kernel writes


# ------------------------------------------------------------------ kernel
def metrics(pred, gt, gtn, J, jmap, groups=None, active=None, out=None):
    """dboa_eval_metrics (groups None) or dboa_eval_metrics_active; ``out`` is written in place when given."""
    from dynaboa_b200 import _lib
    B, NV, NJ = pred.shape[0], pred.shape[1], J.shape[0]
    scratch = torch.full((_lib.load().dboa_eval_scratch_floats(B, NJ),), float('nan'), device='cuda')
    out = torch.empty(B, 3, device='cuda') if out is None else out
    args = (_lib.ptr(pred), _lib.ptr(gt), _lib.ptr(gtn), _lib.ptr(J), NJ, NV, _lib.ptr(jmap), jmap.numel(), _lib.ptr(scratch), _lib.ptr(out), B)
    if groups is None:
        _lib.call('dboa_eval_metrics', *args, _lib.stream())
    else:
        _lib.call('dboa_eval_metrics_active', *args, groups, active, _lib.stream())
    torch.cuda.synchronize()
    return out


def meshes(B, seed):
    rng = np.random.RandomState(seed)
    NV, NJ = 6890, 17
    J = (rng.rand(NJ, NV) ** 12).astype(np.float32)
    J /= J.sum(1, keepdims=True)
    gt = (rng.randn(B, NV, 3) * 0.5).astype(np.float32)
    pred = (gt * 1.1 + rng.randn(B, NV, 3) * 0.08).astype(np.float32)
    gtn = (gt + rng.randn(B, NV, 3) * 0.02).astype(np.float32)
    return [torch.from_numpy(t).cuda() for t in (pred, gt, gtn, J)]


@pytest.mark.parametrize('b', [1, 2])
@pytest.mark.parametrize('G', [1, 2, 4, 8])
def test_each_active_row_is_the_one_video_call(golden, G, b):
    jmap = torch.from_numpy(golden('eval_metrics')['joint_map'].astype(np.int32)).cuda()
    B = G * b
    pred, gt, gtn, J = meshes(B, 100 * G + b)
    every = (1 << G) - 1
    full = metrics(pred, gt, gtn, J, jmap, G, every)
    for g in range(G):
        s = slice(g * b, (g + 1) * b)
        one = metrics(pred[s].contiguous(), gt[s].contiguous(), gtn[s].contiguous(), J, jmap)
        assert torch.equal(bits(full[s]), bits(one)), g
    if G == 1:
        assert torch.equal(bits(full), bits(metrics(pred, gt, gtn, J, jmap)))
        return
    for mask in (1 << (G // 2), every & ~(1 << (G - 1))):        # one active video, and all but one
        ins = [t.clone() for t in (pred, gt, gtn)]
        for g in range(G):
            if not (mask >> g) & 1:
                for t in ins:
                    t[g * b:(g + 1) * b] = float('nan')
        out = torch.empty(B, 3, device='cuda')
        out.view(torch.int32).fill_(SENTINEL)
        metrics(*ins, J, jmap, G, mask, out=out)
        for g in range(G):
            s = slice(g * b, (g + 1) * b)
            if (mask >> g) & 1:
                assert torch.equal(bits(out[s]), bits(full[s])), (bin(mask), g)
            else:
                assert bool((bits(out[s]) == SENTINEL).all()), (bin(mask), g)


def test_golden_through_the_masked_entry(golden):
    """eval_metrics.npz (the reference's numpy path) through dboa_eval_metrics_active, to test_eval_metrics_on_device's bounds,
    as one video and as one video per sample, both bit-identical to dboa_eval_metrics."""
    gd = golden('eval_metrics')
    pred, gt, gtn, J = [torch.from_numpy(np.ascontiguousarray(gd[k], dtype=np.float32)).cuda() for k in ('pred', 'gt', 'gt_neutral', 'J')]
    jmap = torch.from_numpy(gd['joint_map'].astype(np.int32)).cuda()
    B = pred.shape[0]
    ref = metrics(pred, gt, gtn, J, jmap)
    for groups in (1, B):
        out = metrics(pred, gt, gtn, J, jmap, groups, (1 << groups) - 1)
        assert torch.equal(bits(out), bits(ref)), groups
        o = out.cpu().numpy()
        scale = gd['mpjpe'].max()
        assert np.abs(o[:, 0] - gd['mpjpe']).max() <= 2e-5 * scale
        assert np.abs(o[:, 1] - gd['pampjpe']).max() <= 5e-5 * scale
        assert abs(o[:, 2].mean() - gd['pve']) <= 2e-5 * gd['pve']


# ------------------------------------------------------------------ records
def capture(ad):
    """Wrap ``ad.inference``: every call's (is it theta, returned values), in order."""
    calls, orig = [], ad.inference

    def inference(batch, model, need_feature=False):
        r = orig(batch, model, need_feature)
        calls.append((model is ad.model, r))
        return r
    ad.inference = inference
    return calls


class Filed:
    """The captured single-video evaluations, filed frame by frame by the pool's rules (DESIGN.md section 10, "Evaluation")."""

    def __init__(self, inner, mode):
        self.mode = mode
        self.r = dict(mpjpe=[], pampjpe=[], pve=[], mpjpe_all_lower=[[] for _ in range(inner)], pampjpe_all_lower=[[] for _ in range(inner)],
                      mpjpe_statistics=[], pampjpe_statistics=[])

    def frame(self, calls):
        r = self.r
        theta = [v for is_theta, v in calls if is_theta]
        lower = [v for is_theta, v in calls if not is_theta]
        r['mpjpe'].append(theta[-1][0]); r['pampjpe'].append(theta[-1][1]); r['pve'].append(theta[-1][2])
        for i, v in enumerate(lower):
            r['mpjpe_all_lower'][i].append(v[0]); r['pampjpe_all_lower'][i].append(v[1])
        r['mpjpe_statistics'].append([v[0] for v in theta] if self.mode == 'all' else [])
        r['pampjpe_statistics'].append([v[1] for v in theta] if self.mode == 'all' else [])
        calls.clear()


def same(a, b):
    """Bit for bit, through nested lists / dicts of float32 arrays and floats."""
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return type(a) is type(b) and (a == b or (a != a and b != b))


def counts(x):
    """The entry counts of a nested record."""
    if isinstance(x, (list, tuple)):
        return [counts(v) for v in x]
    if isinstance(x, dict):
        return {k: counts(v) for k, v in x.items()}
    return None


def options_for(workload, tmp, golden, name):
    extra = {} if workload == 'c2' else {'cos_sim_threshold': MIXED_THRESHOLD}
    return pool_options(tmp, golden, workload, name, **extra)


def pool_for(workload, tmp, golden, name, G, mode):
    p = PoolRun(options_for(workload, tmp, golden, name), G, dynamic_loop=(workload == 'c5'))
    p.mv.fused_eval = mode
    return p


def single_for(workload, tmp, golden, name, vid, mode):
    s = SingleRun(options_for(workload, tmp, golden, name), vid)
    s.ad.fused_eval = mode
    return s


KEYS = ('mpjpe', 'pampjpe', 'pve', 'mpjpe_all_lower', 'pampjpe_all_lower', 'mpjpe_statistics', 'pampjpe_statistics')


@pytest.mark.parametrize('mode', ['all', 'final'])
@pytest.mark.parametrize('workload', ['c2', 'c5'])
def test_one_video_is_the_single_video_driver(asset_dir, tmp_path, golden, workload, mode):
    p = pool_for(workload, tmp_path, golden, 'mv', 1, mode)
    s = single_for(workload, tmp_path, golden, 'ad', 0, mode)
    calls = capture(s.ad)
    filed = Filed(p.mv.options.inner_step, mode)
    p.start(0, 0, stream(0, N_FRAMES))
    for t in range(N_FRAMES):
        batch = p.step([0])[0][2]
        s.step(t, batch)
        assert calls and all(is_theta for is_theta, _ in calls) == (mode == 'final'), t
        filed.frame(calls)
    rec = p.mv.records(0)
    assert rec['frames'] == N_FRAMES
    for k in KEYS:
        assert same(rec[k], filed.r[k]), k
    if mode == 'final':
        assert rec['mpjpe_all_lower'] == [[]] * p.mv.options.inner_step and rec['mpjpe_statistics'] == [[]] * N_FRAMES
    ad = s.ad
    assert rec['kp2dlosses_lower'] == [float(x) for x in ad.kp2dlosses_lower]
    assert rec['kp2dlosses_upper'] == {k: float(v) for k, v in ad.kp2dlosses_upper.items()}
    assert rec['feat_sims'] == ad.feat_sims and rec['optim_step_record'] == ad.optim_step_record


def close(a, b, what):
    if isinstance(a, (list, tuple)):
        for i, (x, y) in enumerate(zip(a, b)):
            close(x, y, what + (i,))
    elif isinstance(a, np.ndarray):
        assert rel_err(a, b) <= 1e-3, what
    else:
        assert abs(a - b) <= 1e-3 * abs(b), what


@pytest.mark.parametrize('workload', ['c2', 'c5'])
def test_every_video_follows_its_own_single_video_records(asset_dir, tmp_path, golden, workload):
    G = 4
    p = pool_for(workload, tmp_path, golden, 'mv', G, 'all')
    singles = [single_for(workload, tmp_path, golden, f'v{g}', g, 'all') for g in range(G)]
    calls = [capture(s.ad) for s in singles]
    filed = [Filed(p.mv.options.inner_step, 'all') for _ in range(G)]
    for g in range(G):
        p.start(g, g, stream(g, N_FRAMES))
    for t in range(N_FRAMES):
        done = p.step(range(G))
        for g in range(G):
            singles[g].step(t, done[g][2])
            filed[g].frame(calls[g])
    for g in range(G):
        rec = p.mv.records(g)
        for k in KEYS:
            assert counts(rec[k]) == counts(filed[g].r[k]), (g, k)
            close(rec[k], filed[g].r[k], (g, k))
        assert rec['optim_step_record'] == singles[g].ad.optim_step_record, g


def test_records_do_not_depend_on_the_slot_or_schedule(asset_dir, tmp_path, golden):
    """test_a_looping_video_does_not_depend_on_its_slot_or_schedule's two schedules with 'all': video X's records bit for bit,
    and every slot has exactly one entry per frame it advanced."""
    X = 5
    a = pool_for('c5', tmp_path, golden, 'a', 4, 'all')
    a.start(0, X, stream(X, N_FRAMES))
    for _ in range(N_FRAMES):
        a.step([0])
    rec_a = a.mv.records(0)
    del a
    b = pool_for('c5', tmp_path, golden, 'b', 4, 'all')
    total = N_FRAMES + 3
    b.start(0, 11, stream(11, total))
    b.start(1, 12, stream(12, total))
    b.start(2, 13, stream(13, 3))
    b.start(3, 14, stream(14, 2))
    advanced = [0] * 4
    for f in range(total):
        if f == 3:
            b.start(2, X, stream(X, N_FRAMES))
            advanced[2] = 0
        if f == 4:
            b.start(3, 15, stream(15, total))
            advanced[3] = 0
        run = [0, 2]
        if f not in (1, 4, 5):
            run.append(1)
        if f not in (2, 3):
            run.append(3)
        b.step(sorted(run))
        for g in run:
            advanced[g] += 1
    rec_b = b.mv.records(2)
    for k in KEYS + ('kp2dlosses_lower', 'kp2dlosses_upper', 'optim_step_record'):
        assert same(rec_b[k], rec_a[k]), k
    inner = b.mv.options.inner_step
    for g in range(4):
        rec = b.mv.records(g)
        n = advanced[g]
        assert rec['frames'] == n and len(rec['mpjpe']) == len(rec['pve']) == len(rec['mpjpe_statistics']) == n, g
        assert all(len(rec['mpjpe_all_lower'][i]) == n for i in range(inner)), g
        assert all(len(s) == 1 + min(k, b.mv.options.optim_steps) for s, k in zip(rec['mpjpe_statistics'], rec['optim_step_record'])), g
        assert sorted(rec['kp2dlosses_upper']) == list(range(n)) and len(rec['kp2dlosses_lower']) == inner * n, g


# ------------------------------------------------------------------ runner
LENGTHS = [3, 8, 2, 5, 6, 4]


def keyed_masks(mv):
    """mask_provider keyed by the video a slot holds and that video's own frame."""
    state = {}

    def provider(g, B, dev):
        key = (mv.slot_video[g], mv.video_steps[g])
        call = state[g][1] if g in state and state[g][0] == key else 0
        state[g] = (key, call + 1)
        return video_masks(key[0], key[1], call).to(dev)
    return provider


def runner(opts, G=4):
    from dynaboa_b200.multivideo import MultiVideoAdaptor
    mv = MultiVideoAdaptor(opts, G)
    mv.fused_eval = 'final'
    mv.mask_provider = keyed_masks(mv)
    return mv


def structure(x):
    """Names, keys, value types and entry counts of a loaded result."""
    if isinstance(x, (list, tuple)):
        return [type(x).__name__, [structure(v) for v in x]]
    if isinstance(x, dict):
        return ['dict', {k: structure(v) for k, v in x.items()}]
    if isinstance(x, np.ndarray):
        return ['ndarray', str(x.dtype), x.shape]
    return type(x).__name__


def test_run_gives_each_video_its_own_results(asset_dir, tmp_path, golden):
    from dynaboa_b200 import synthetic
    from dynaboa_b200.adaptor import RESULT_FILES, Adaptor
    videos = [synthetic.SyntheticStream(length=n, batch_size=1, rank=v) for v, n in enumerate(LENGTHS)]
    names = [f'video{v}' for v in range(len(LENGTHS))]
    mv = runner(pool_options(tmp_path, golden, 'c2', 'pool'))
    out = mv.run(videos, exppath=str(tmp_path / 'pool'), names=names)
    assert [s['name'] for s in out] == names and [s['frames'] for s in out] == LENGTHS
    assert mv.slot_video == [None] * 4
    alone = runner(pool_options(tmp_path, golden, 'c2', 'alone'))
    empty = synthetic.SyntheticStream(length=0, batch_size=1)
    for v, n in enumerate(LENGTHS):
        # video v at index v of the queue (so its seed and masks are those of the pool run), behind empty videos
        res = alone.run([empty] * v + [videos[v]], exppath=str(tmp_path / 'alone'), names=[f'e{i}' for i in range(v)] + [names[v]])
        assert res[v] == out[v], v
        assert all(r['frames'] == 0 for r in res[:v])
        for f in RESULT_FILES:
            with open(tmp_path / 'pool' / names[v] / f, 'rb') as x, open(tmp_path / 'alone' / names[v] / f, 'rb') as y:
                assert x.read() == y.read(), (v, f)
        assert not any((tmp_path / 'alone' / f'e{i}').exists() for i in range(v))
    for v in (1, 2):                                  # lengths 8 and 2: the single-video driver's files on a video that long
        o = pool_options(tmp_path, golden, 'c2', f'excute{v}')
        o.synthetic_frames = LENGTHS[v]
        ad = Adaptor(o)
        ad.fused_eval = 'final'
        ad.excute(fused=True)
        mine, theirs = tmp_path / 'pool' / names[v], ad.exppath
        assert sorted(os.listdir(mine)) == sorted(RESULT_FILES)
        for f in RESULT_FILES:
            assert os.path.exists(os.path.join(theirs, f)), f
            if f.endswith('.pt'):
                assert structure(joblib.load(mine / f)) == structure(joblib.load(os.path.join(theirs, f))), (v, f)
        a = (mine / 'res.txt').read_text().splitlines()
        b = open(os.path.join(theirs, 'res.txt')).read().splitlines()
        assert len(a) == len(b) and [x.split('MPJPE')[0] for x in a] == [x.split('MPJPE')[0] for x in b], v
    s = out[1]
    rec = joblib.load(tmp_path / 'pool' / names[1] / 'res.pt')
    assert s['mpjpe'] == float(np.mean(rec['mpjpe'])) and s['pve'] == float(np.mean(rec['pve']))


# ------------------------------------------------------------------ host synchronisations
def synchronising(fn):
    """The number of synchronising CUDA calls ``fn()`` makes (``torch.cuda.set_sync_debug_mode('warn')``)."""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum('synchroniz' in str(x.message) for x in w)


def test_evaluation_adds_no_host_synchronisation(asset_dir, tmp_path, golden):
    """All-active G = 4 pool frames at C2 with the motion term live, 'final' and 'none' alternating frame by frame on one pool,
    frames and teacher masks already on the device.  The first frame counted in a process takes one synchronisation in either
    mode (on an H100 it fell to whichever mode was counted first), so one priming frame is counted apart."""
    warm, timed = 7, 3
    n = warm + 1 + 2 * timed
    p = pool_for('c2', tmp_path, golden, 'sync', 4, 'final')
    masks = {(g, t): video_masks(g, t, 0).cuda() for g in range(4) for t in range(n)}
    p.mv.mask_provider = lambda g, B, dev: masks[(g, p.mv.video_steps[g])]
    for g in range(4):
        p.start(g, g, [fetch(f) for f in stream(g, n)])
    for _ in range(warm):
        p.step(range(4))
    torch.cuda.synchronize()
    assert synchronising(lambda: p.step(range(4))) <= 1
    count = {'none': 0, 'final': 0}
    for k in range(2 * timed):
        mode = ('final', 'none')[k % 2]
        p.mv.fused_eval = mode
        count[mode] += synchronising(lambda: p.step(range(4)))
    assert count['final'] == count['none'], count
    rec = {}
    assert synchronising(lambda: rec.update(p.mv.records(0))) >= 1      # the records are formed on the host when read
    assert rec['frames'] == n and len(rec['mpjpe']) == len(rec['pve']) == warm + 1 + timed   # no entry for a frame without evaluation
