"""Data-parallel adaptation step for step against a rank-sum twin.  Every rank runs two adaptors on the same frames:

- ``dp``, set up by ``dist.attach`` as bench.py does: the outer gradient all-reduced bucket by bucket on a communication stream
  under the backward (or in one collective before the optimiser step), 1 / R folded into the Adam sweep, the feature test's sums
  all-reduced;
- ``solo``, plain data parallelism: no ``grad_sync``; its ``pre_step_hook`` gathers every rank's local gradient and sums them in
  rank order in fp32, its ``gscale`` is 1 / R.

After every outer step dp's reduced gradient must be the sum of the ranks' local gradients (bit for bit at R = 2, where the sum of
two fp32 values does not depend on the order; within the fp32 summation bound at R >= 3, after which solo takes dp's sum).  After
every frame theta, Adam's moments, the teacher, the step count and every record of the two must agree bit for bit, and theta must
be identical on every rank.  The dynamic loop's decisions must follow the fp64 cosine of the rank-summed sums.  The C3 and C5 runs
are repeated with the all-reduce unbucketed and with the weight gradients on the caller's stream, and the three orderings must end
bit-identical.  That compares orderings: it does not show that no race exists."""
import datetime
import json
import os
import pickle
import socket
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES = 8                     # interval 5: the motion term is live from frame 6 on
# C5 runs longer: its later frames stop after a few trips, close to the threshold, where one rank's terms can decide otherwise
FRAMES = {'c5': 12}
# dp's 1 - cos12 against the fp64 cosine of the summed (a.b, |a|^2, |b|^2): both come from the same fp64 sums, and dp rounds the
# cosine to fp32 (at most 2^-25 off below 1), so a decision is compared wherever the fp64 margin to the threshold exceeds 2^-24
DEC_TOL = 2.0 ** -24
TIMEOUT = datetime.timedelta(minutes=5)
# name -> (bench.py workload, option overrides, entry point)
CONFIGS = {
    'c2': ('c2', {}, 'adapt'),
    'c3': ('c3', {}, 'adapt'),
    'c5': ('c5', {}, 'adapt'),                                 # bench's threshold 2e-5, optim_steps 7, teacher dropout on
    'boa0': ('c2', {'use_boa': 0}, 'adapt'),                   # one level, lower=True, carries the sync
    'autograd': ('c2', {}, 'adaptation'),                      # Adaptor.adaptation: the all-reduce in pre_step_hook
}
ARMS = {'default': {}, 'unbucketed': {'DBOA_DP_BUCKETS': '0'},
        'serial': {'DBOA_DP_BUCKETS': '0', 'DBOA_ASYNC_WGRAD': '0'}}


# ------------------------------------------------------------------ helpers of the ranks
def _host(x):
    """``x`` with every tensor moved to a host numpy array (records of a frame, comparable across processes)."""
    if isinstance(x, dict):
        return {k: _host(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_host(v) for v in x)
    if torch.is_tensor(x):
        return x.detach().cpu().numpy()
    return x


def _same(a, b):
    """Bit-for-bit equality of two host records (NaN equals NaN, -0 differs from +0)."""
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, (np.ndarray, np.generic, float)):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return a == b


def _arena(ad):
    return getattr(ad.model, 'module', ad.model)


def _state(ad):
    opt = ad.optimizer
    return {'theta': _arena(ad).arena, 'm': opt.m, 'v': opt.v, 'teacher': ad.teacher.arena}


def _records(ad):
    return _host({'upper': ad.last_upper_loss, 'fit': dict(ad.fit_losses), 'lower': list(ad.kp2dlosses_lower),
                  'steps': list(ad.optim_step_record), 'retrieval': getattr(ad, 'last_retrieval', None)})


class _Checks:
    """Failed checks by name (first message kept).  A rank records a failure and runs on, so that every rank issues the same
    collectives; the parent asserts on what the ranks report."""

    def __init__(self):
        self.failed = {}

    def __call__(self, name, ok, msg):
        if not ok and name not in self.failed:
            self.failed[name] = msg


def _rank_main(rank, world, port, job, out_dir):
    import sys
    sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]
    os.environ.update(job['env'])                  # DBOA_ASYNC_WGRAD is read when the library loads: before any import of it
    import torch.distributed as dist
    nccl = job['backend'] == 'nccl'
    torch.cuda.set_device(rank if nccl else 0)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group(job['backend'], rank=rank, world_size=world, timeout=TIMEOUT)
    try:
        import gc
        from bench import N_EXEMPLARS
        from dynaboa_b200 import config, synthetic
        work = os.path.join(out_dir, f'work{rank}')
        synthetic.write_asset_dir(os.path.join(work, 'data'), n_exemplars=N_EXEMPLARS)
        config.set_data_root(os.path.join(work, 'data'))
        reports = {}
        for run in job['runs']:
            torch.cuda.reset_peak_memory_stats()
            reports[run['name']] = _run(rank, world, run, work, job.get('ref_dir'))
            gc.collect()                           # the adaptors of the run before (reference cycles through their step)
            torch.cuda.empty_cache()
        with open(os.path.join(out_dir, f'rank{rank}.pkl'), 'wb') as f:
            pickle.dump(reports, f)
    finally:
        dist.destroy_process_group()


def _run(rank, world, run, work, ref_dir):
    """One configuration: a fresh dp / solo pair over ``run['frames']`` frames of this rank's stream; returns the rank's report."""
    import random
    import torch.distributed as dist
    from bench import WORKLOADS, default_options
    from dynaboa_b200 import config, dist as ddist, synthetic
    from dynaboa_b200.adaptor import Adaptor
    from harness import bits
    t0 = time.perf_counter()
    workload, overrides, entry = CONFIGS[run['config']]
    flags = {**WORKLOADS[workload], **overrides}
    n_frames, control = run['frames'], run['control']
    opts = lambda name: default_options(expdir=work, expname=f'{run["name"]}_{name}', model_file=config.BASE_MODEL,
                                        synthetic_frames=n_frames, rank=rank, **flags)
    dp, solo = Adaptor(opts('dp')), Adaptor(opts('solo'))
    dp.fused_eval = solo.fused_eval = 'none'
    check = _Checks()

    # dp: the object under test, plus captures of its reduced gradient (as the Adam sweep reads it) and its local cosine sums
    sync = ddist.attach(dp, world)
    opt = dp.optimizer
    reduced, local_terms = [], []
    step, hook, reduce_terms = opt.step, opt.pre_step_hook, dp._reduce_terms

    def captured_step(*a, **k):
        if opt.reduced:
            torch.cuda.current_stream().wait_stream(opt.grad_sync.comm)
            reduced.append(_arena(dp).grad_arena().clone())
        return step(*a, **k)

    def captured_hook(g):
        hook(g)
        reduced.append(g.clone())

    def captured_terms(terms):
        local_terms.append(terms.detach().cpu().clone())
        reduce_terms(terms)
    opt.step, opt.pre_step_hook, dp._reduce_terms = captured_step, captured_hook, captured_terms
    if control == 'skip_bucket':                   # negative control (i): the smallest bucket stays local on every rank
        sizes = [hi - lo for lo, hi in sync.bounds]
        skip = sizes.index(min(sizes))

        def after_backward(flat_grad):
            for k, (ev, (lo, hi)) in enumerate(zip(sync.events, sync.bounds)):
                sync.comm.wait_event(ev)
                if k != skip:
                    with torch.cuda.stream(sync.comm):
                        dist.all_reduce(flat_grad[lo:hi], op=dist.ReduceOp.SUM)
            flat_grad.record_stream(sync.comm)
        sync.after_backward = after_backward

    # solo: the rank-sum reference
    stats = {'max_abs_vs_rank_sum': 0.0, 'max_err_over_bound': 0.0, 'outer_steps': 0}
    calls = []

    def rank_sum(g):
        i = len(calls)
        calls.append(i)
        parts = [torch.empty_like(g) for _ in range(world)]
        dist.all_gather(parts, g)
        total = parts[0].clone()
        for p in parts[1:]:
            total.add_(p)                          # rank order, fp32
        if i >= len(reduced):
            check('reduced gradient', False, f'outer step {i}: dp took {len(reduced)} outer steps')
            g.copy_(total)
            return
        red = reduced[i]
        stats['max_abs_vs_rank_sum'] = max(stats['max_abs_vs_rank_sum'], float((red - total).abs().max()))
        if world == 2:
            diff = int((bits(red) != bits(total)).sum())
            check('reduced gradient', diff == 0, f'outer step {i}: {diff} of {g.numel()} elements of the reduced gradient differ from '
                  f'g0 + g1, max |diff| {stats["max_abs_vs_rank_sum"]:.3e}')
            g.copy_(total)
        else:
            exact = sum(p.double() for p in parts)
            # R - 1 fp32 additions, each off by at most 2^-24 of its result, or by FLT_MIN where a backend flushes a subnormal sum
            u = (world - 1) * 2.0 ** -24
            bound = u / (1 - u) * sum(p.double().abs() for p in parts) + (world - 1) * 2.0 ** -126
            err = (red.double() - exact).abs()
            worst = float((err / bound.clamp_min(1e-300)).max())
            stats['max_err_over_bound'] = max(stats['max_err_over_bound'], worst)
            bad = int((err > bound).sum())
            check('reduced gradient', bad == 0, f'outer step {i}: {bad} elements of the reduced gradient outside '
                  f'(R - 1) 2^-24 sum |g_r| of the fp64 sum (worst {worst:.3f} of the bound)')
            g.copy_(red)                           # from here on solo follows dp's summation order
    solo.optimizer.pre_step_hook = rank_sum
    if control != 'gscale':                        # negative control (ii): solo's gradient stays R times too large in Adam
        solo.optimizer.gscale = 1.0 / world
    assert opt.gscale == 1.0 / world

    stream = synthetic.SyntheticStream(length=n_frames, batch_size=1, rank=rank)
    frames = []
    for t in range(n_frames):
        batch = {k: v.cuda() if torch.is_tensor(v) else v for k, v in stream[t].items()}
        rng = torch.cuda.get_rng_state(), random.getstate()
        ends = []
        del reduced[:], calls[:]
        for ad in (dp, solo):
            torch.cuda.set_rng_state(rng[0])
            random.setstate(rng[1])
            ad.global_step, ad.fit_losses = t, {}
            ad.model.eval()
            getattr(ad, entry)(batch)
            ends.append((torch.cuda.get_rng_state(), random.getstate()))
            check('cuda graph', ad._graph is None, f'frame {t}: an adaptor captured its frame as a CUDA graph')
        check('rng', torch.equal(ends[0][0], ends[1][0]) and ends[0][1] == ends[1][1],
              f'frame {t}: dp and solo leave the global generators in different states')
        check('reduced gradient', len(calls) == len(reduced), f'frame {t}: dp took {len(reduced)} outer steps, solo {len(calls)}')
        stats['outer_steps'] += len(reduced)
        # 2. state
        a, b = _state(dp), _state(solo)
        for k in a:
            diff = int((bits(a[k]) != bits(b[k])).sum())
            check('state', diff == 0, f'frame {t}: {diff} elements of {k} differ between dp and solo')
        check('state', dp.optimizer.step_count == solo.optimizer.step_count,
              f'frame {t}: step_count {dp.optimizer.step_count} != {solo.optimizer.step_count}')
        # 3. records
        rec = _records(dp)
        bad = [k for k, v in _records(solo).items() if not _same(rec[k], v)]
        check('records', not bad, f'frame {t}: records {bad} differ between dp and solo')
        frames.append(rec)
        # 4. replicas: every rank's whole theta
        theta = _arena(dp).arena
        parts = [torch.empty_like(theta) for _ in range(world)]
        dist.all_gather(parts, theta)
        diff = [int((bits(p) != bits(theta)).sum()) for p in parts]
        check('replicas', not any(diff), f'frame {t}: elements of theta differing from rank {rank}, by rank: {diff}')

    # 5. the dynamic loop's decisions against the fp64 cosine of the rank-summed sums
    decisions = None
    if flags['dynamic_boa']:
        every = [None] * world
        dist.all_gather_object(every, local_terms)
        thr = flags['cos_sim_threshold']
        values = [1.0 - s[12]['cos'] for t in range(n_frames) for s in dp.feat_sims[t]]
        made = [v > thr for v in values]
        check('decisions', all(len(x) == len(made) for x in every), f'{[len(x) for x in every]} feature tests for {len(made)} decisions')
        n = min([len(made)] + [len(x) for x in every])

        def one_minus_cos(terms):
            s = terms[0, 12].double()
            return 1.0 - float(s[0] / (s[1].sqrt() * s[2].sqrt()))
        summed = [one_minus_cos(sum(x[j] for x in every)) for j in range(n)]
        alone = [[one_minus_cos(x[j]) for j in range(n)] for x in every]
        worst = max([abs(v - w) for v, w in zip(values, summed)], default=0.0)
        check('decisions', worst <= DEC_TOL, f'1 - cos of dp\'s feature test differs by {worst:.3e} from the fp64 cosine of the summed terms')
        clear = [j for j in range(n) if abs(summed[j] - thr) > DEC_TOL]
        wrong = [j for j in clear if made[j] != (summed[j] > thr)]
        check('decisions', not wrong, f'feature tests {wrong}: dp decided against the fp64 cosine of the summed terms '
              f'(1 - cos {[summed[j] for j in wrong]}, threshold {thr})')
        trips = list(dp.optim_step_record)
        check('decisions', any(0 < k <= flags['optim_steps'] for k in trips) and len(set(trips)) > 1, f'trip counts {trips} are not mixed')
        # negative control (iii): the feature tests where the decision of one rank's sums alone differs from dp's, by rank
        decisions = {'trips': trips, 'made': made, 'clear': len(clear), 'max_abs_vs_fp64': worst, 'one_minus_cos': summed, 'one_rank': alone,
                     'one_rank_disagrees': [[j for j in clear if made[j] != (a[j] > thr) and abs(a[j] - thr) > DEC_TOL] for a in alone]}
    # the final state of an ordering of the all-reduce: rank 0 of the default ordering writes it, the others compare with it (the
    # replicas check holds it equal on every rank)
    arm_diff = None
    if run['save_state'] and rank == 0:
        final = torch.stack(list(_state(dp).values())).cpu().numpy()
        path = os.path.join(ref_dir or os.path.dirname(work), f'state_{run["config"]}.npy')
        if ref_dir is None:
            np.save(path, final)
        else:
            ref = np.load(path)
            arm_diff = {k: int((final[i].view(np.int32) != ref[i].view(np.int32)).sum()) for i, k in enumerate(_state(dp))}
    torch.cuda.synchronize()
    return {'failed': check.failed, 'frames': frames, 'stats': stats, 'decisions': decisions, 'arm_diff': arm_diff,
            'wall_s': time.perf_counter() - t0, 'peak_gb': torch.cuda.max_memory_reserved() / 2 ** 30}


# ------------------------------------------------------------------ the parent
def _runs(world, arm, backend):
    """The configurations one process group runs, in order: at R = 2 with gloo every configuration and the two negative controls
    (one frame of C2 each); at R = 3 the two ways the gradient is reduced (the autograd path's one collective, the fused path's
    buckets) and the dynamic loop; with the two other orderings only C3 and C5."""
    if arm != 'default':
        names = ['c3', 'c5']
    elif world == 2 and backend == 'gloo':
        names = list(CONFIGS) + ['skip_bucket', 'gscale']
    elif world == 3:
        names = ['autograd', 'c3', 'c5']
    else:
        names = list(CONFIGS)
    return [{'name': n, 'config': 'c2' if n in ('skip_bucket', 'gscale') else n, 'frames': 1 if n in ('skip_bucket', 'gscale') else FRAMES.get(n, N_FRAMES),
             'control': n if n in ('skip_bucket', 'gscale') else None, 'save_state': world == 2 and n in ('c3', 'c5')} for n in names]


def _spawn(out, world, arm, backend, ref_dir=None):
    """One process group of ``world`` ranks (all on cuda:0 with gloo, one GPU each with NCCL); returns each rank's reports by run."""
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    job = {'backend': backend, 'env': ARMS[arm], 'runs': _runs(world, arm, backend), 'ref_dir': ref_dir}
    t0 = time.perf_counter()
    mp.spawn(_rank_main, args=(world, port, job, str(out)), nprocs=world, join=True)
    reports = [pickle.load(open(out / f'rank{r}.pkl', 'rb')) for r in range(world)]
    for name, rep in reports[0].items():
        print(json.dumps({'group': f'{backend} R={world} {arm}', 'run': name, 'rank_wall_s': round(rep['wall_s'], 1),
                          'peak_reserved_gb': round(rep['peak_gb'], 2), **rep['stats'],
                          'trips': rep['decisions'] and rep['decisions']['trips'], 'failed': sorted(rep['failed'])}))
    print(json.dumps({'group': f'{backend} R={world} {arm}', 'wall_s': round(time.perf_counter() - t0, 1)}))
    return reports


@pytest.fixture(scope='module')
def group(tmp_path_factory):
    """group(world, arm='default', backend='gloo'): the reports of that process group, run once for the module."""
    done = {}

    def get(world, arm='default', backend='gloo'):
        key = (world, arm, backend)
        if key not in done:
            ref_dir = None if arm == 'default' else str(get(2)[1])
            out = tmp_path_factory.mktemp(f'{backend}{world}_{arm}')
            try:
                done[key] = (_spawn(out, world, arm, backend, ref_dir), out)
            except Exception as e:             # noqa: BLE001 -- every test of this group reports it, none runs it again
                done[key] = e
        if isinstance(done[key], Exception):
            raise done[key]
        return done[key]
    return lambda world, arm='default', backend='gloo': get(world, arm, backend)[0]


def _passes(reports, name):
    for r, rep in enumerate(reports):
        assert not rep[name]['failed'], f'rank {r}: {rep[name]["failed"]}'
    if reports[0][name]['decisions'] is not None:
        trips = [rep[name]['decisions']['trips'] for rep in reports]
        assert all(t == trips[0] for t in trips), trips


@pytest.mark.parametrize('world, config', [(2, c) for c in CONFIGS] + [(3, 'autograd'), (3, 'c3'), (3, 'c5')])
def test_dp_follows_the_rank_sum(group, world, config):
    _passes(group(world), config)


def test_the_loop_decides_on_the_sum_over_ranks(group):
    """Negative control (iii): in C5 at R = 2 the decisions of rank 0's sums alone differ from dp's in at least one feature test
    whose fp64 margin is clear, so the decision check would see a loop that decided on one rank's terms.  (The ranks' own values of
    1 - cos12 lie within a few per cent of the summed one, so only a test close to the threshold can tell them apart.)"""
    dec = group(2)[0]['c5']['decisions']
    print(json.dumps({'disagreeing tests by rank': dec['one_rank_disagrees'], 'one_minus_cos': dec['one_minus_cos'],
                      'one_rank': dec['one_rank'], 'max_abs_vs_fp64': dec['max_abs_vs_fp64']}))
    assert dec['one_rank_disagrees'][0], dec


@pytest.mark.parametrize('config', ['c3', 'c5'])
def test_orderings_of_the_all_reduce_end_bit_identical(group, config):
    """At R = 2 (the sum of two values does not depend on the order, in any backend) the bucketed, overlapped all-reduce, the
    single collective after the backward and the fully serial backward each follow the rank sum and end bit-identical: theta,
    Adam's moments, the teacher and every record of every frame."""
    ref = group(2)
    for arm in ('unbucketed', 'serial'):
        reports = group(2, arm)
        _passes(reports, config)
        assert reports[0][config]['arm_diff'] == dict.fromkeys(('theta', 'm', 'v', 'teacher'), 0), (arm, reports[0][config]['arm_diff'])
        for r in range(2):
            assert _same(reports[r][config]['frames'], ref[r][config]['frames']), (arm, r)


@pytest.mark.parametrize('world', [2, 4, 8])
def test_nccl_follows_the_rank_sum(group, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f'NCCL with one rank per GPU needs {world} GPUs, this box has {torch.cuda.device_count()}')
    reports = group(world, backend='nccl')
    for config in CONFIGS:
        _passes(reports, config)


@pytest.mark.parametrize('control, fails', [('skip_bucket', 'reduced gradient'), ('gscale', 'state')])
def test_negative_controls_fail_their_check(group, control, fails):
    """(i) The smallest bucket left un-reduced on every rank fails the reduced-gradient check; (ii) solo's Adam without 1 / R
    fails the state check.  Every rank issues the same collectives as in a passing run."""
    for rep in group(2):
        assert fails in rep[control]['failed'], rep[control]['failed']
        print(f'{control}: {fails}: {rep[control]["failed"][fails]}')
    if control == 'gscale':
        assert 'reduced gradient' not in group(2)[0][control]['failed']
