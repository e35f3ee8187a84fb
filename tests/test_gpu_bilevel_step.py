"""The fused bilevel step (fused.fused_adapt through Adaptor.adapt, unchanged) against fp64 on the GPU's own kink pattern.

``fused.forward_graph`` and ``fused.level_backward`` are wrapped to record each forward (arena, image, keep-masks, tape) and
each level (its forwards, its gradient arena, its records, retrieval's cluster).  A reference chain that derives its own
inputs follows every frame:

- lower level i on the reference's weights (theta, then sgd_ref of the previous inner gradient), the upper level on the
  reference's fast weights and each dynamic-loop level on the Adam-updated theta: the GPU's gradient arena equals
  oracle/bilevel_frozen.py evaluated in float64 on the kink pattern of the GPU forward that served the level (GRAD_TOL per
  tensor, GRAD_L2 over the arena), and its records equal the fp64 terms;
- the fast weights the GPU uses are sgd_ref of its own inputs, bit for bit;
- the pose prior's component and retrieval's cluster are the fp64 argmin (or within the measured near-tie margin), and the
  exemplars are what a copy of ``random``'s state taken before the frame draws from that cluster;
- theta, Adam's moments and the teacher after each frame are adam_ref / ema_ref of the GPU's outer gradients, bit for bit,
  so the chain is exact from frame to frame;
- the dynamic loop's cosines equal fp64 cosines of the frozen features, and its decisions and trip count follow fp64 wherever
  the margin exceeds the measured error.

Configurations: C2 (8 frames, the motion term live on the last two), C3 (3 inner steps, 8 exemplars on both levels), C5
(dynamic loop), C2 with the fused forward and backward plans, and a MultiVideoAdaptor pool of 4 videos at C2 that join on
different frames, with an idle slot and the motion term live for some videos only; each video of the pool follows its own
reference chain.

Negative controls show the bounds are sharp enough to see a composition mistake: the reference evaluated on theta instead of
the fast weights, without the motion term, with the frame and history rows swapped, or without the exemplar term must each
miss GRAD_L2 by at least 10x.  They run at the goldens' fastlr and lr: the smallest margin each test prints (CONTROLS lines)
is what shows those step sizes separate theta from the fast weights."""
import json
import random
from types import SimpleNamespace

import pytest
import torch

from harness import GRAD_L2, GRAD_TOL, adam_ref, adapt_options, bits, fetch, selected, sgd_ref, tape_pattern

pytestmark = pytest.mark.gpu

# Worst values measured over this file on an H100 80GB HBM3 (power limit 700 W) are given beside each bound.  The gradients use
# the layer tests' GRAD_TOL (worst here 1.9e-5 per tensor, C5 loop level) and GRAD_L2 (worst 6.5e-6, the pool).
TERM_TOL = 1.2e-5           # records (fit_losses terms, level totals) against fp64, element-wise relative: 3.8e-6 (the pool)
COS_TOL = 3e-7              # dynamic-loop cosines, absolute: 9.0e-8 (C5)
# Near-tie margins of the discrete choices: how far (relative) above the fp64 minimum the GPU's GMM component, and how far
# (absolute cosine distance) from the fp64 nearest centre its retrieval cluster, may lie.  Measured: 0 for both, every choice
# was the fp64 argmin; the prior's margin is test_gpu_loss_head.py's prior_value bound.
PRIOR_TIE = 7e-7
CLUSTER_TIE = 1e-6
# Each negative control must miss GRAD_L2 by this factor.  Measured (relative L2 / GRAD_L2, smallest over the frames): C2 theta
# 7546, no motion 50, swapped history 19812; C3 theta 73389, no exemplars 7410; the pool theta 3905, no motion 65, swapped
# history 12953.
CONTROL_MARGIN = 10


class Recorder:
    """Wraps fused.forward_graph / fused.level_backward; ``fwd`` every forward of the frame, ``levels`` every level."""

    def __init__(self, monkeypatch):
        from dynaboa_b200 import fused
        real_fwd, real_level = fused.forward_graph, fused.level_backward
        self.fwd, self.levels, self.depth = [], [], 0

        def forward_graph(s, arena, buffers, image, mask, masks=None):
            p = real_fwd(s, arena, buffers, image, mask, masks)
            # the one-video motion pair is staged in a buffer the step reuses: keep this pass's rows
            img = image.clone() if image is s._pair else image
            self.fwd.append(SimpleNamespace(arena=arena.data_ptr(), image=img, mask=mask, masks=masks, pred=p, tape=p.tape,
                                            in_level=self.depth > 0))
            return p

        def level_backward(s, out, arena, image, kp, lower, grad_arena, mask, live, main=None, sync=None):
            n0 = len(self.fwd)
            weights = arena.clone() if arena.data_ptr() != s.theta.data_ptr() else None      # the fast weights, before reuse
            self.depth += 1
            total, m = real_level(s, out, arena, image, kp, lower, grad_arena, mask, live, main=main, sync=sync)
            self.depth -= 1
            self.levels.append(SimpleNamespace(
                arena=arena.data_ptr(), weights=weights, lower=lower, main=m, given=main is not None, fwd=self.fwd[n0:],
                grad=grad_arena.clone(), fit={k: v.clone() for k, v in out.fit.items()}, total=total.clone(),
                best=None if s._best is None else s._best.clone()))
            return total, m
        monkeypatch.setattr(fused, 'forward_graph', forward_graph)
        monkeypatch.setattr(fused, 'level_backward', level_backward)

    def reset(self):
        self.fwd, self.levels = [], []


def reference_model(ad):
    """The constants of the reference levels.  SMPL and retrieval's exemplar bank (centres, clusters, exemplars) are built
    here from the synthetic assets, not read from the adaptor, so the exemplars the GPU forwards are checked against an
    independent copy.  The pose prior's fp32 means, precisions and -log weights are the adaptor's own, widened: the GPU's
    choice of component is judged on the values it computes with, and test_gpu_kernels.py::test_gmm_prior_against_golden
    holds those constants to the prior recorded from the reference's code."""
    from dynaboa_b200 import constants as K, synthetic
    from oracle import bilevel_frozen
    dev = torch.device('cuda')
    body, extra = synthetic.make_smpl_model('neutral'), synthetic.make_extra_regressors()['J_regressor_extra']
    smpl = ({k: torch.as_tensor(v, dtype=torch.long if k == 'parents' else torch.float64, device=dev) for k, v in body.items() if k != 'faces'},
            torch.as_tensor(extra, dtype=torch.float64, device=dev), torch.tensor(K.JOINT_MAP_49, device=dev),
            torch.tensor(K.SMPL_EXTRA_VERTEX_IDS, device=dev))
    g = ad.gmm_f
    m = ad.model.module
    cl = synthetic.make_clusters()
    bank = SimpleNamespace(centers=torch.as_tensor(cl['centers'], dtype=torch.float64, device=dev), index=cl['index'],
                           exemplars={k: v.float().to(dev) for k, v in synthetic.make_exemplar_bank().items()})
    return bilevel_frozen.Model(buffers={k: m._buffers[k].double() for k in ('init_pose', 'init_shape', 'init_cam')}, smpl=smpl,
                                gmm=(g.means.double(), g.precisions.double(), g.neg_log_weights.double()), kp_range=ad.kp_range, bank=bank)


def params64(arena):
    from dynaboa_b200.hmr import layout
    lay = layout()
    return {n: v.double() for n, v in zip(lay.names, lay.views(own(arena.cuda())))}


def own(t):
    """``t`` as a tensor of its own: layout().views() offsets are absolute in the storage, so a row of a (G, P) stack is copied."""
    return t.clone() if t.storage_offset() else t


def grad_errors(grad, ref):
    """(worst per-tensor max |g - ref| / max |ref|, its tensor, whole-arena relative L2) of a GPU arena against fp64."""
    from dynaboa_b200.hmr import layout
    lay = layout()
    worst, where, num, den = 0.0, '', 0.0, 0.0
    for n, gv in zip(lay.names, lay.views(own(grad))):
        r = ref[n]
        e = float((gv.double() - r).abs().max() / r.abs().max().clamp_min(1e-30))
        e = e if e == e else float('inf')
        if e > worst:
            worst, where = e, n
        num, den = num + float((gv.double() - r).pow(2).sum()), den + float(r.pow(2).sum())
    return worst, where, (num / den) ** 0.5


class Video:
    """Where one video lives in an adaptor: row ``g`` of its G-video (G, P) stacks and of every grouped batch (one row per
    video), and callables for what differs between ``Adaptor`` and ``MultiVideoAdaptor``: ``state()`` -> the video's (theta,
    Adam m, Adam v, teacher, Adam step count) on the host, ``masks(t, call)`` -> the (3, 2, 1, 1024) keep-masks its teacher
    forward ``call`` of its frame t must get, ``adam_args`` (lr, betas, eps), ``teacher_ptr`` (data pointer of the teacher
    arena), ``motion_lead``, and for the dynamic loop ``sims(t)`` / ``trips()`` (its cosines of frame t, its last
    trip count)."""

    def __init__(self, **kw):
        vars(self).update(kw)


class Chain:
    """The reference chain of one video: its own theta, teacher, Adam moments and step count (bit-equal to the GPU's as long as
    the chain holds), its inputs from its own stream and history, and every measured error."""

    def __init__(self, video, opts, stream, model):
        self.vid, self.o, self.stream, self.model = video, opts, stream, model
        self.g, self.G = video.g, video.G
        self.theta, self.m, self.v, self.teacher, self.step = video.state()
        self.worst = {'grad': 0.0, 'l2': 0.0, 'terms': 0.0, 'cos': 0.0, 'prior_tie': 0.0, 'cluster_tie': 0.0}
        self.controls = {}

    def note(self, k, v):
        self.worst[k] = max(self.worst[k], v)

    def level(self, L, weights, lower, t, rng, image, kp, controls=()):
        """Checks the recorded level ``L`` against fp64 on ``weights`` (fp32, the reference's); returns the level's picks."""
        from oracle import bilevel_frozen
        o, vid, dev, g, G = self.o, self.vid, torch.device('cuda'), self.g, self.G
        row = slice(g, g + 1)
        tag = 'll' if lower else 'ul'
        use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
        use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
        motion = bool(use_temporal and o.use_motion and t + vid.motion_lead - o.interval > 0)
        mix = bool(o.retrieval and (o.lower_level_mixtrain if lower else o.upper_level_mixtrain))
        tptr = vid.teacher_ptr
        teach = [f for f in L.fwd if f.arena == tptr]
        others = [f for f in L.fwd if f.arena != tptr and f.pred is not L.main]
        batched = L.main.B > G
        ex_f = others.pop() if mix else None
        hist_f = others.pop() if others else None       # the history pass, under the mask of the videos whose motion term is live
        assert not others and len(teach) == int(bool(use_temporal and o.use_meanteacher)), (t, tag, len(L.fwd))
        assert batched == (motion and not L.given and G == 1), (t, tag)
        assert (hist_f is not None and (hist_f.mask >> g) & 1) == (motion and not batched), (t, tag, g, 'history pass')
        image64, kp64 = image.double(), kp.double()
        with torch.device(dev):
            p = params64(weights)
            pattern = tape_pattern(L.main.tape, L.main.B, row)
            teacher = None
            if teach:
                f = teach[0]
                with torch.device('cpu'):                      # the masks come from seeded CPU generators
                    expect = vid.masks(t, self.calls)
                assert torch.equal(f.masks[:, :, row].cpu(), expect), (t, tag, g)
                self.calls += 1
                teacher = bilevel_frozen.teacher_outputs(self.model, params64(self.teacher), image64, tape_pattern(f.tape, G, row, f.masks))
            hist = None
            if motion:
                h = fetch(self.stream[t - o.interval])
                hist = {'image': h['image'].double(), 'kp': h['smpl_j2d'].double()}
                if batched:                                   # one video: rows [1:] of the pair are the history frame
                    pair = next(f.image for f in L.fwd if f.pred is L.main)
                    assert torch.equal(pair[1:], h['image']) and torch.equal(pair[:1], image), (t, tag)
                    hist['pattern'] = tape_pattern(L.main.tape, 2, slice(1, 2))
                else:                                         # its own (grouped) history pass: this video's row
                    assert torch.equal(hist_f.image[row], h['image']), (t, tag, g)
                    hist['pattern'] = tape_pattern(hist_f.tape, G, row)
            with torch.no_grad():
                main = bilevel_frozen.network(self.model, p, image64, pattern)
            comp = None
            if use_frame:
                ll = bilevel_frozen.prior_components(self.model, main.rot)
                comp = selected(ll.cpu(), L.fit[f'{tag}/pose_prior'][g:g + 1]).to(dev)
                lo = ll.min(1)[0]
                tie = float((ll.gather(1, comp.view(1, 1)).squeeze(1) - lo).abs().max() / lo.abs().max())
                self.note('prior_tie', tie)
                assert tie <= PRIOR_TIE, (t, tag, 'GMM component', tie)
            ex, picks = None, None
            if o.retrieval:
                d = 1 - torch.nn.functional.cosine_similarity(main.feats[5], self.model.bank.centers)
                c = int(L.best[g])
                self.note('cluster_tie', float(d[c] - d.min()))
                assert float(d[c] - d.min()) <= CLUSTER_TIE, (t, tag, 'cluster', c, int(d.argmin()))
                picks = rng.sample(self.model.bank.index[c], o.sample_num)
                if mix:
                    n = o.sample_num
                    idx = torch.as_tensor(picks, device=dev)
                    ex = {k: v.index_select(0, idx).double() for k, v in self.model.bank.exemplars.items()}
                    assert torch.equal(ex_f.image[g * n:(g + 1) * n], self.model.bank.exemplars['img'].index_select(0, idx)), (t, tag, g, 'exemplars')
                    ex['pattern'] = tape_pattern(ex_f.tape, G * n, slice(g * n, (g + 1) * n))
            r = bilevel_frozen.level(o, self.model, p, lower, image64, kp64, pattern, comp, teacher, hist, ex)
            worst, where, l2 = grad_errors(L.grad[g] if G > 1 else L.grad, r.grads)
            self.note('grad', worst)
            self.note('l2', l2)
            terms = max([abs(float(L.fit[k][g]) - float(v)) / abs(float(v)) for k, v in r.terms.items()]
                        + [abs(float(L.total[g]) - float(r.total)) / abs(float(r.total))])
            self.note('terms', terms)
            print(f'  {"" if G == 1 else f"video {g} "}t={t} {tag}: grad {worst:.2e} ({where}) L2 {l2:.2e} terms {terms:.2e}')
            assert worst <= GRAD_TOL and l2 <= GRAD_L2, (t, tag, worst, where, l2)
            assert terms <= TERM_TOL, (t, tag, terms)
            for name in controls:                          # the same level, evaluated wrongly on purpose
                q, x, kw = p, image64, dict(pattern=pattern, comp=comp, teacher=teacher, hist=hist, exemplars=ex)
                if name == 'theta':
                    q = params64(self.theta)
                elif name == 'no motion':
                    kw['hist'] = None
                elif name == 'swapped history':                # the frame's rows read the history frame and the other way round
                    x, kw['pattern'] = hist['image'], hist['pattern']
                    kw['hist'] = dict(hist, image=image64, pattern=pattern)
                elif name == 'no exemplars':
                    kw['exemplars'] = None
                rc = bilevel_frozen.level(o, self.model, q, lower, x, kp64, **kw)
                e = grad_errors(L.grad[g] if G > 1 else L.grad, rc.grads)
                self.controls[name] = min(self.controls.get(name, float('inf')), e[2] / GRAD_L2)
        return picks

    def row(self, t):
        """This video's row of a (G, P) stack, the arena itself for one video."""
        return t[self.g] if self.G > 1 else t

    def adam(self, grad):
        o = self.o
        lr, betas, eps = self.vid.adam_args
        self.step += 1
        teacher = adam_ref(self.theta, self.row(grad).cpu(), self.m, self.v, self.teacher if o.use_meanteacher else None, lr, betas, eps,
                           self.step, o.alpha)
        self.theta, self.m, self.v = teacher[:3]
        if o.use_meanteacher:
            self.teacher = teacher[3]

    def check_state(self, t):
        """The video's theta, Adam moments, teacher and step count on the GPU are the chain's, bit for bit."""
        theta, m, v, teacher, step = self.vid.state()
        assert step == self.step, (self.g, t, step, self.step)
        for name, gpu, ref in (('theta', theta, self.theta), ('m', m, self.m), ('v', v, self.v), ('teacher', teacher, self.teacher)):
            assert torch.equal(bits(gpu), bits(ref)), (self.g, t, name)

    def frame(self, rec, t, state, controls=()):
        """Follows the video's frame t through the levels recorded in ``rec``; ``state``: its retrieval generator's state
        before the frame."""
        from oracle import bilevel_frozen
        o, vid = self.o, self.vid
        batch = fetch(self.stream[t])
        image, kp = batch['image'], batch['smpl_j2d']
        rng = random.Random()
        rng.setstate(state)
        self.calls = 0
        levels = list(rec.levels)
        probe = [f for f in rec.fwd if not f.in_level]
        theta0 = self.theta
        fast = self.theta
        for i in range(o.inner_step):
            L = levels.pop(0)
            assert L.lower and (L.given == (i == 0)), (t, i)
            if i > 0:
                assert torch.equal(bits(self.row(L.weights).cpu()), bits(fast)), (self.g, t, i, 'fast weights')
            self.level(L, fast, True, t, rng, image, kp)
            fast = sgd_ref(fast, self.row(L.grad).cpu(), o.fastlr)
        L = levels.pop(0)
        assert not L.lower and not L.given
        assert torch.equal(bits(self.row(L.weights).cpu()), bits(fast)), (self.g, t, 'fast weights of the upper level')
        self.level(L, fast, False, t, rng, image, kp, controls)
        self.adam(L.grad)
        if o.dynamic_boa:
            sims = vid.sims(t)
            steps, before = 0, (theta0, probe.pop(0))
            for j, gpu in enumerate(sims):
                after = (self.theta, probe.pop(0))
                with torch.device('cuda'), torch.no_grad():
                    fa = bilevel_frozen.network(self.model, params64(before[0]), image.double(), tape_pattern(before[1].tape, 1)).feats
                    fb = bilevel_frozen.network(self.model, params64(after[0]), image.double(), tape_pattern(after[1].tape, 1)).feats
                cos = bilevel_frozen.cosines(fa, fb)
                err = max(abs(gpu[i]['cos'] - c) for i, c in enumerate(cos))
                self.note('cos', err)
                assert err <= COS_TOL, (t, j, err)
                go = 1 - cos[12] > o.cos_sim_threshold
                if abs(1 - cos[12] - o.cos_sim_threshold) > COS_TOL:
                    assert go == (1 - gpu[12]['cos'] > o.cos_sim_threshold), (t, j)
                if not go:
                    break
                steps += 1
                if steps > o.optim_steps:
                    break
                L = levels.pop(0)
                assert not L.lower and L.given and L.main is after[1].pred
                self.level(L, self.theta, False, t, rng, image, kp)
                self.adam(L.grad)
                before = after
            assert vid.trips() == steps, (t, steps)
        assert not levels, (t, len(levels))
        self.check_state(t)


def run_single(tmp_path, golden, monkeypatch, tag, frames, controls=None, fused_plans=False):
    from dynaboa_b200 import _lib, synthetic
    from dynaboa_b200.adaptor import Adaptor
    gd = golden(f'adapt_{tag}')
    opts = adapt_options(tmp_path, gd)
    ad = Adaptor(opts)
    ad.fused_eval = 'none'
    stream = synthetic.SyntheticStream(length=frames, batch_size=opts.batch_size)
    masks_all = torch.from_numpy(gd['teacher_masks']).float()
    rec = Recorder(monkeypatch)
    m = ad.model.module
    video = Video(g=0, G=1, state=lambda: (m.arena.cpu().clone(), ad.optimizer.m.cpu().clone(), ad.optimizer.v.cpu().clone(),
                                           ad.teacher.arena.cpu().clone(), ad.optimizer.step_count),
                  masks=lambda t, call: masks_all[t, min(call, masks_all.shape[1] - 1)], teacher_ptr=ad.teacher.arena.data_ptr(),
                  adam_args=(opts.lr, (opts.beta1, opts.beta2), ad.optimizer.param_groups[0]['eps']),
                  motion_lead=ad.motion_lead, sims=lambda t: ad.feat_sims[t], trips=lambda: ad.optim_step_record[-1])
    chain = Chain(video, opts, stream, reference_model(ad))
    lib = _lib.load()
    prev = lib.dboa_get_fused_forward(), lib.dboa_get_fused_backward()
    try:
        if fused_plans:
            lib.dboa_set_fused_forward(1)
            lib.dboa_set_fused_backward(1)
        for t in range(frames):
            batch = fetch(stream[t])
            calls = {'i': 0}

            def provider(B, dev, t=t, calls=calls):
                m = masks_all[t, min(calls['i'], masks_all.shape[1] - 1)]
                calls['i'] += 1
                return m.to(dev)
            ad.teacher.mask_provider = provider
            random.seed(1000 + t)
            state = random.getstate()
            ad.global_step, ad.fit_losses = t, {}
            ad.model.eval()
            rec.reset()
            ad.adapt(batch)
            torch.cuda.synchronize()
            chain.frame(rec, t, state, (controls or {}).get(t, ()))
    finally:
        lib.dboa_set_fused_forward(prev[0])
        lib.dboa_set_fused_backward(prev[1])
    print(f'\nBILEVEL {tag}{" fused plans" if fused_plans else ""} ' + json.dumps({k: f'{v:.2e}' for k, v in chain.worst.items()}))
    if controls:
        print(f'CONTROLS {tag} (rel L2 / GRAD_L2) ' + json.dumps({k: f'{v:.1f}' for k, v in chain.controls.items()}))
        for name, margin in chain.controls.items():
            assert margin >= CONTROL_MARGIN, (name, margin)
    return chain


# negative controls of the configurations, per frame: frames 6 and 7 of C2 carry the motion term
C2_CONTROLS = {t: ('theta', 'no motion', 'swapped history') if t >= 6 else ('theta',) for t in range(8)}
C3_CONTROLS = {t: ('theta', 'no exemplars') for t in range(2)}
CONFIGS = [('c2', 8, False, C2_CONTROLS), ('c3', 2, False, C3_CONTROLS), ('c5', 2, False, None), ('c2', 3, True, None)]


@pytest.mark.parametrize('tag,frames,fused_plans,controls', CONFIGS, ids=['c2', 'c3', 'c5', 'c2-fused-plans'])
def test_bilevel_step_against_fp64(asset_dir, tmp_path, golden, monkeypatch, tag, frames, fused_plans, controls):
    run_single(tmp_path, golden, monkeypatch, tag, frames, controls=controls, fused_plans=fused_plans)


# the pool: four videos (video g in slot g) that join on pool frames START[g]; slot 3 sits pool frame 4 out.  On the last two
# pool frames the motion term is live for some videos only (own frames 6 and 7 of videos 0, 1 and 3; video 2 never reaches it).
START, IDLE, POOL_FRAMES = (0, 1, 2, 0), {(4, 3)}, 8


def test_pool_of_four_videos_against_fp64(asset_dir, tmp_path, golden, monkeypatch):
    """A MultiVideoAdaptor of 4 videos at C2 (harness.PoolRun): every video follows its own reference chain through the grouped
    forwards and backwards (its row of each tape, of each gradient stack and of the fast weights), its own Adam step count and
    teacher, its own history frame and teacher masks; the slots outside a frame keep their state bit for bit."""
    from harness import PoolRun, pool_options, stream, video_masks, video_seed
    G = len(START)
    opts = pool_options(tmp_path, golden, 'c2', 'pool')
    pr = PoolRun(opts, G)
    mv = pr.mv
    rec = Recorder(monkeypatch)
    model = reference_model(mv.base)
    streams = [stream(g, POOL_FRAMES) for g in range(G)]
    chains = [None] * G

    def video(g):
        return Video(g=g, G=G, state=lambda: (mv.thetas[g].cpu().clone(), mv.m[g].cpu().clone(), mv.v[g].cpu().clone(),
                                              mv.teachers[g].cpu().clone(), mv.step_counts[g]),
                     masks=lambda t, call: video_masks(g, t, call), teacher_ptr=mv.teachers.data_ptr(),
                     adam_args=(opts.lr, (opts.beta1, opts.beta2), 1e-8), motion_lead=mv.motion_lead)
    live_mix = set()
    for f in range(POOL_FRAMES):
        for g in range(G):
            if f == START[g]:
                pr.start(g, g, streams[g])
                chains[g] = Chain(video(g), opts, streams[g], model)
        run = [g for g in range(G) if chains[g] is not None and (f, g) not in IDLE]
        rec.reset()
        done = pr.step(run)
        torch.cuda.synchronize()
        live_mix.add(tuple(done[g][1] - opts.interval > 0 for g in run))
        for g, c in enumerate(chains):
            if c is None:
                continue
            if g not in run:
                c.check_state(f)                                # a slot outside the frame is untouched
                continue
            _, t, _ = done[g]
            c.frame(rec, t, random.Random(video_seed(g, t)).getstate(),
                    ('theta', 'no motion', 'swapped history') if t - opts.interval > 0 else ('theta',))
    assert any(any(x) and not all(x) for x in live_mix), 'no frame with the motion term live for some videos only'
    worst = {k: max(c.worst[k] for c in chains) for k in chains[0].worst}
    controls = {k: min(c.controls[k] for c in chains if k in c.controls) for k in chains[0].controls}
    print(f'\nBILEVEL pool ' + json.dumps({k: f'{v:.2e}' for k, v in worst.items()}))
    print('CONTROLS pool (rel L2 / GRAD_L2) ' + json.dumps({k: f'{v:.1f}' for k, v in controls.items()}))
    for name, margin in controls.items():
        assert margin >= CONTROL_MARGIN, (name, margin)
