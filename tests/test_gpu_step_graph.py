"""C2 frames of ``Adaptor.adapt`` replayed as one CUDA graph against the same frames run eagerly, from the same seeds: theta,
teacher, Adam moments, every record, the predictions, the teacher's dropout masks and the kernel count of every frame are
bit for bit the eager ones, also after a reset of the weights and optimiser in place (as bench.py does between its two
measurements); the frames the graph cannot serve run eagerly."""
import os

import pytest
import torch

from harness import bits, fetch

pytestmark = pytest.mark.gpu
N = 14           # frames 0..5 warm the history ring, 6 runs eagerly, 7 is captured, 8..13 are replays


@pytest.fixture
def assets(asset_dir, tmp_path):
    return tmp_path


def make_adaptor(root, name):
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config
    from dynaboa_b200.adaptor import Adaptor
    o = default_options(expdir=str(root), expname=name, model_file=config.BASE_MODEL, synthetic_frames=N, **WORKLOADS['c2'])
    ad = Adaptor(o)
    ad.fused_eval = 'none'
    return ad


def run(ad, graph, monkeypatch):
    """Two passes over the N frames with an in-place reset between them; per frame: records, kernels, teacher masks, outputs."""
    from dynaboa_b200 import _lib, adaptor, synthetic
    monkeypatch.setattr(adaptor, 'STEP_GRAPH', graph)
    lib = _lib.load()
    masks = []
    draw = ad.teacher._masks
    ad.teacher._masks = lambda B, device: masks.append(draw(B, device)) or masks[-1]
    stream = synthetic.SyntheticStream(length=N, batch_size=1)
    frames = [fetch(stream[t]) for t in range(N)]
    snap = (ad.model.module.arena.clone(), ad.teacher.arena.clone())
    recs, captured = [], None
    for rnd in range(2):
        if rnd:
            ad.model.module.arena.copy_(snap[0]); ad.teacher.arena.copy_(snap[1])
            ad.optimizer.m.zero_(); ad.optimizer.v.zero_(); ad.optimizer.step_count = 0
        ad.reset_records()
        for t in range(N):
            ad.global_step, ad.fit_losses = t, {}
            n0, drawn, had = lib.dboa_launch_count(), len(masks), ad._graph
            ad.adapt(frames[t])
            n = lib.dboa_launch_count() - n0
            if had is None and ad._graph is not None:
                captured = masks[-1]                      # a replay draws into the masks tensor of the capture
            mask = masks[-1] if len(masks) > drawn else captured
            pred, _ = ad.predict_async(frames[t]['image'])
            torch.cuda.synchronize()
            recs.append(dict(kernels=n, upper=ad.last_upper_loss.clone(), mask=mask.clone(),
                             fit={k: v.clone() for k, v in ad.fit_losses.items()}, pred={k: v.clone() for k, v in pred.items()}))
        recs[-1]['lower'] = [v.clone() for v in ad.kp2dlosses_lower]
    state = [ad.model.module.arena, ad.teacher.arena, ad.optimizer.m, ad.optimizer.v]
    return recs, [t.clone() for t in state], ad.optimizer.step_count, torch.cuda.get_rng_state()


def same(a, b):
    return torch.equal(bits(a), bits(b))


def test_graph_replay_is_bit_identical_to_eager(assets, monkeypatch):
    eager, e_state, e_steps, e_rng = run(make_adaptor(assets, 'eager'), False, monkeypatch)
    ad = make_adaptor(assets, 'graph')
    graph, g_state, g_steps, g_rng = run(ad, True, monkeypatch)
    assert ad._graph is not None and ad._graph.launches > 0, 'the graph path was not taken'
    for t, (e, g) in enumerate(zip(eager, graph)):
        assert e['kernels'] == g['kernels'], t
        assert same(e['upper'], g['upper']) and same(e['mask'], g['mask']), t
        assert e['fit'].keys() == g['fit'].keys() and all(same(e['fit'][k], g['fit'][k]) for k in e['fit']), t
        assert all(same(e['pred'][k], g['pred'][k]) for k in e['pred']), t
    assert len(eager[-1]['lower']) == len(graph[-1]['lower']) == N
    assert all(same(a, b) for a, b in zip(eager[-1]['lower'], graph[-1]['lower']))
    assert e_steps == g_steps == N
    assert all(same(a, b) for a, b in zip(e_state, g_state))               # theta, teacher, m, v
    assert torch.equal(e_rng, g_rng)                                        # the replays advanced torch's generator as eager frames do


def test_frames_the_graph_cannot_serve_run_eagerly(assets, monkeypatch):
    from dynaboa_b200 import adaptor, synthetic
    monkeypatch.setattr(adaptor, 'STEP_GRAPH', True)
    ad = make_adaptor(assets, 'fallback')
    stream = synthetic.SyntheticStream(length=N, batch_size=1)
    batch = fetch(stream[0])
    ad.global_step = N - 1
    assert ad._graph_key(batch) is not None
    ad.global_step = 0
    assert ad._graph_key(batch) is None                                     # motion term not live yet
    ad.global_step = N - 1
    for attr, value in (('fused_eval', 'final'), ('phase_events', []), ('step_graph', False)):
        old = getattr(ad, attr)
        setattr(ad, attr, value)
        assert ad._graph_key(batch) is None, attr
        setattr(ad, attr, old)
    for name in ('retrieval', 'dynamic_boa'):
        setattr(ad.options, name, 1)
        assert ad._graph_key(batch) is None, name
        setattr(ad.options, name, 0)
    ad.teacher.mask_provider = lambda B, device: torch.ones(3, 2, B, 1024, device=device)
    assert ad._graph_key(batch) is None
    ad.teacher.mask_provider = None
    ad.optimizer.pre_step_hook = lambda g: None                             # data parallel (dist.attach)
    assert ad._graph_key(batch) is None
    ad.optimizer.pre_step_hook = None
    # a run with evaluations never captures
    ad.fused_eval = 'final'
    for t in range(N):
        ad.global_step, ad.fit_losses = t, {}
        ad.adapt(fetch(stream[t]))
    assert ad._graph is None
