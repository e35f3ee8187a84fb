"""Autograd-free bilevel adaptation step: the arithmetic of reference dynaboa_benchmark.py:126-201
(``Adaptor.adaptation``) driven by direct C-ABI calls.

What changes relative to the autograd path (``Adaptor.adaptation``), none of it numerically:

* gradients of every forward graph of a level (frame, history frame, exemplar minibatch) are accumulated by
  ``dboa_hmr_backward`` straight into ONE flat arena -- no per-tensor ``.grad`` accumulation, no 169-way splits;
* inner step 0 reuses the no-grad probe forward (the fast weights equal theta before the first update), and
  each dynamic iteration reuses the feature-test forward as its upper-level forward (same weights, same image);
* the first-order MAML adjoint is the identity, so the outer gradient w.r.t. the fast weights IS the gradient
  applied to theta (SURVEY.md "facts": ``first_order=True``);
* Adam and the mean-teacher EMA run as one fused sweep; frame and teacher-consistency terms share one loss-head
  launch; the only host syncs are retrieval's cluster index and the ``dynamic_boa`` decision.

The step reads a ``Step``, built once by each adaptor: G videos' arenas (flat for ``adaptor.Adaptor``, (G, P) stacks for
``multivideo.MultiVideoAdaptor``; video g owns the rows [g * b, (g + 1) * b) of every batch, and every pass is one grouped
call) and callbacks for what stays with the adaptor.  A set of videos is an int whose bit g means video g takes part (all:
``(1 << G) - 1``); passes and sweeps skip the others.  ``fused_adapt`` returns the records (``Frame``).  DESIGN.md section 10.
"""
import collections
import ctypes as C

import torch

from . import _lib, hmr as hmr_mod
from ._lib import ptr, stream


_SIDE = {}

# retrieval's exemplars: cluster centres (K, 2048), each cluster's exemplars, their tensors by name, (K,) distance scratch
Bank = collections.namedtuple('Bank', 'centers index exemplars dists')


class Step:
    """What the bilevel step reads and owns.

    ``options``; ``G`` videos; ``theta``, ``grad``, ``buffers``: the weight and gradient arenas (flat for one video, (G, P)
    stacks) and the network's constant buffers; ``teacher``, ``teacher_buffers``: the mean teacher's (None without one);
    ``teacher_masks(B, device, mask)``: the keep-masks of the teacher forward (or None: no dropout); ``smpl_neutral``,
    ``gmm_f``: neutral SMPL and the pose prior; ``kp_range``: (first, count) joints of the 2D and motion terms; ``motion_lead``:
    video g's motion term is live while its frame count + ``motion_lead`` - ``interval`` > 0; ``bank``, ``rngs``: retrieval's ``Bank`` and
    per-video generators; ``save_hist(image, kp, mask)`` / ``get_hist(live)``: the history frames; ``adam(mask, teacher=None,
    alpha=0.0)``: Adam (+ EMA into ``teacher``) of the videos in ``mask``; ``evaluate(batch, arena, mask, inner)``: one
    evaluation of ``arena`` (``inner``: the inner step of fast weights, None for theta); ``reduce_terms(terms)``: the
    data-parallel sum of the feature test's sums (None: one rank); ``video_options``: G option namespaces, video g's learning
    rates, loss weights and dynamic-loop test (``multivideo.PER_VIDEO``) read from the g-th (default: ``options`` for every
    video; a pool sets them per frame).  Set per frame: ``eval_mode`` ('none', 'final', 'all'), ``grad_sync`` (the
    data-parallel ``BucketedGradSync`` or None) and ``phase_events`` (a list: CUDA events per phase)."""

    def __init__(self, options, G, theta, grad, buffers, smpl_neutral, gmm_f, teacher=None, teacher_buffers=None, teacher_masks=None,
                 kp_range=(25, 24), motion_lead=0, bank=None, rngs=None, save_hist=None, get_hist=None, adam=None, evaluate=None,
                 reduce_terms=None, video_options=None):
        self.options, self.G, self.theta, self.grad, self.buffers, self.smpl_neutral, self.gmm_f = options, G, theta, grad, buffers, smpl_neutral, gmm_f
        self.teacher, self.teacher_buffers, self.teacher_masks = teacher, teacher_buffers, teacher_masks
        self.kp_range, self.motion_lead, self.bank, self.rngs = kp_range, motion_lead, bank, rngs
        self.save_hist, self.get_hist, self.adam, self.evaluate, self.reduce_terms = save_hist, get_hist, adam, evaluate, reduce_terms
        self.eval_mode, self.grad_sync, self.phase_events = 'none', None, None
        self.video_options = [options] * G if video_options is None else video_options
        self._motion_w = None                   # (values, device tensor) of _motion_weights
        # the step's scratch: motion pair images and gradients, cosine partial sums, fast weights, inner gradient, cluster index
        self._pair = self._bgrad_flat = self._cos_partial = self._fast = self._inner_grad = None
        self._best = None if bank is None else torch.zeros(G, dtype=torch.int32, device=bank.centers.device)


class Frame:
    """What ``fused_adapt`` returns for the videos in ``mask``, each loss (G,) (unspecified outside them): ``fit`` (the ``fit_losses`` terms; the last
    upper level's 2D loss is ``ul/s2dloss``), ``lower`` (each lower level's 2D loss), ``upper_loss``; per video ``steps``
    and ``sims`` (the dynamic loop's trip count and cosines; None without it), ``picks`` (its last retrieval, None where it
    drew none; None without retrieval); ``result``: the return of the last evaluation of theta."""

    def __init__(self, mask):
        self.mask, self.fit, self.lower, self.upper_loss = mask, {}, [], None
        self.steps = self.sims = self.picks = self.result = None


def pick(mask, G, a, b=None):
    """(G,) per video: ``a`` for the videos in ``mask``, ``b`` (None: NaN) for the others; ``a`` itself for every video."""
    if mask == (1 << G) - 1:
        return a
    keep = torch.tensor([bool((mask >> g) & 1) for g in range(G)], device=a.device)
    return torch.where(keep, a, torch.full_like(a, float('nan')) if b is None else b)


def merge(old, new, mask, G):
    """Records ``old`` updated with the (G,) entries of ``new`` from a level evaluated under ``mask``: an entry already in
    ``old`` keeps its value for the videos outside ``mask``, whose last evaluation of the frame came earlier."""
    out = dict(old)
    for k, v in new.items():
        out[k] = pick(mask, G, v, old[k]) if k in old else v
    return out


def _motion_weights(s, device):
    """Every video's ``motionloss_weight`` as a factor of the (G,) motion term: the one float all videos share, or else a (G,)
    fp32 device tensor of the fp32 values a float factor rounds to (the same products).  The tensor is uploaded again only when
    a video's value changes (``start``), so a frame makes no copy, and a captured single-video frame holds no host-written
    tensor."""
    key = tuple(float(q.motionloss_weight) for q in s.video_options)
    if len(set(key)) == 1:
        return key[0]
    if s._motion_w is None or s._motion_w[0] != key or s._motion_w[1].device != device:
        s._motion_w = (key, torch.tensor(key, dtype=torch.float32, device=device))
    return s._motion_w[1]


def _side_stream(device):
    if device.index not in _SIDE:
        _SIDE[device.index] = torch.cuda.Stream(device=device)
    return _SIDE[device.index]


def _mark(s, name):
    """Diagnostics (scripts/phase_times.py): when ``s.phase_events`` is a list, record a CUDA event on the caller's stream."""
    if s.phase_events is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        s.phase_events.append((name, ev))


def runs(mask, G, key=lambda g: 0):
    """[a, b) ranges of consecutive videos whose bit is set in ``mask`` and that share ``key(g)``."""
    out = []
    for g in range(G):
        if (mask >> g) & 1:
            if out and out[-1][1] == g and key(out[-1][0]) == key(g):
                out[-1][1] = g + 1
            else:
                out.append([g, g + 1])
    return out


def _active_rows(t, mask, G):
    """``t`` itself for every video, else views of the (G, P) stack ``t``'s runs of videos in ``mask`` (sweeps skip the others)."""
    return [t] if mask == (1 << G) - 1 else [t[a:b] for a, b in runs(mask, G)]


class _Pred:
    """Everything one forward graph produces (kept for its backward); ``active``: the videos of its backward."""
    __slots__ = ('image', 'rot', 'shape', 'cam', 'tape', 'verts', 'joints', 'smpl_tape', 'p2d', 'B', 'masked', 'groups', 'active')


def _smpl_fwd(smpl, betas, rot):
    B, dev = betas.shape[0], betas.device
    verts = torch.empty(B, 6890, 3, dtype=torch.float32, device=dev)
    joints = torch.empty(B, 49, 3, dtype=torch.float32, device=dev)
    tape = torch.empty(_lib.load().dboa_smpl_tape_floats(B), dtype=torch.float32, device=dev)
    _lib.call('dboa_smpl_forward', smpl._struct_ref(), ptr(betas), ptr(rot), B, ptr(verts), ptr(joints), ptr(tape), stream())
    return verts, joints, tape


def forward_graph(s, arena, buffers, image, mask, masks=None):
    p = _Pred()
    p.image, p.B, p.masked, p.groups, p.active = image, image.shape[0], masks is not None, s.G, mask
    p.rot, p.shape, p.cam, _, p.tape = hmr_mod.raw_forward(arena, buffers, image, masks, groups=s.G, active=mask)
    p.verts, p.joints, p.smpl_tape = _smpl_fwd(s.smpl_neutral, p.shape, p.rot)
    p.p2d = torch.empty(p.B, 49, 2, dtype=torch.float32, device=image.device)
    _lib.call('dboa_project_fwd', ptr(p.cam), ptr(p.joints), ptr(p.p2d), p.B, 49, stream())
    return p


def _loss_head(s, p, w, kp=None, t_p2d=None, t_j3d=None, t_beta=None, t_R=None, gt_s3d=None, grads=None, nb=None):
    """Runs the (optional) pose prior and the multi-term head on the first ``nb`` samples of ``p``, each video's rows on their
    own (per-video means and gradient scaling); returns (terms (G, 9), dp2d, dj3d, dR, dbeta).  ``w``: one row of 8 weights
    per video, or one row of 8 for every video.  ``grads``: preallocated (possibly larger-batch) gradient buffers whose leading ``nb`` rows are written."""
    B, dev, G = (p.B if nb is None else nb), p.rot.device, p.groups
    if grads is None:
        dp2d, dj3d = torch.empty_like(p.p2d), torch.empty_like(p.joints)
        dR, dbeta = torch.empty_like(p.rot), torch.empty_like(p.shape)
    else:
        dp2d, dj3d, dR, dbeta = grads
    terms = torch.empty(G, 9, dtype=torch.float32, device=dev)
    if not isinstance(w[0], (list, tuple)):
        w = [w] * G
    prior_b = None
    if any(r[2] != 0.0 for r in w):
        prior_b = torch.empty(B, dtype=torch.float32, device=dev)
        g = s.gmm_f
        _lib.call('dboa_pose_prior_groups', ptr(p.rot), ptr(g.means), ptr(g.precisions), ptr(g.neg_log_weights), ptr(prior_b), ptr(dR),
                  (C.c_float * G)(*[float(r[2]) / (B // G) for r in w]), B, G, stream())     # per-video mean: scale w / b
    a = _lib.LossArgsStruct()
    a.B, a.groups = B, G
    keep = []
    for name, t in (('p2d', p.p2d), ('j3d', p.joints), ('R', p.rot), ('beta', p.shape), ('kp', kp), ('prior_b', prior_b), ('t_p2d', t_p2d),
                    ('t_j3d', t_j3d), ('t_beta', t_beta), ('t_R', t_R), ('gt_s3d', gt_s3d), ('terms', terms), ('dp2d', dp2d),
                    ('dj3d', dj3d), ('dR', dR), ('dbeta', dbeta)):
        if t is not None:
            t = t if (t.is_contiguous() and t.dtype == torch.float32) else t.contiguous().float()
            keep.append(t)
        setattr(a, name, None if t is None else t.data_ptr())
    a.dR_accumulate = 1 if prior_b is not None else 0
    a.kp_first, a.kp_count = s.kp_range                             # joints of the re-projection term (webcam client: (0, 25))
    _lib.call('dboa_loss_multi_weights', C.byref(a), (C.c_float * (8 * G))(*[float(x) for r in w for x in r]), stream())
    return terms, dp2d, dj3d, dR, dbeta


def _zero(t):
    """Stream-ordered memset (copy engine / driver memset node): no ATen fill kernel in the step."""
    _lib.call('dboa_fill_zero', ptr(t), t.numel() * t.element_size(), stream())


def backward_graph(s, arena, p, dp2d, dj3d, dR, dbeta, grad_arena, sync=None):
    """d(loss)/d(p2d, joints, R, beta) -> accumulate d(loss)/d(weights) of the videos ``p.active`` into ``grad_arena``.
    ``sync``: the data-parallel ``BucketedGradSync`` when this is the LAST graph accumulated into the outer gradient: its
    buckets are all-reduced on the communication stream while the rest of this backward runs."""
    B, dev = p.B, p.rot.device
    dcam = torch.empty(B, 3, dtype=torch.float32, device=dev)
    _lib.call('dboa_project_bwd', ptr(p.cam), ptr(p.joints), ptr(dp2d), ptr(dj3d), ptr(dcam), B, 49, 1, 0, stream())
    scratch = torch.empty(_lib.load().dboa_smpl_scratch_floats(B), dtype=torch.float32, device=dev)
    _lib.call('dboa_smpl_backward', s.smpl_neutral._struct_ref(), ptr(p.rot), B, ptr(p.smpl_tape), ptr(dj3d), ptr(scratch), ptr(dR),
              ptr(dbeta), 1, stream())
    if sync is not None:
        sync.arm()
    hmr_mod.raw_backward(arena, p.tape, B, p.masked, dR, dbeta, dcam, grad_arena, groups=p.groups, active=p.active)
    if sync is not None:
        sync.after_backward(grad_arena)


def retrieve(bank, rows, rngs, mask, best, n):
    """reference :82-96 for every video in ``mask``: the nearest cluster centre of video g's feature row ``rows[g]`` by cosine
    distance (into ``best[g]``; one host synchronisation for all videos), then ``rngs[g].sample`` of ``n`` exemplars inside
    that cluster.  Returns the (cluster, picks) of every video and the picked exemplar rows, video after video; a video
    outside ``mask`` draws nothing, gets None and placeholder rows (exemplar 0)."""
    on = [bool((mask >> g) & 1) for g in range(len(rows))]
    for g, f in enumerate(rows):
        if on[g]:
            _lib.call('dboa_retrieval_nearest', ptr(f.contiguous()), ptr(bank.centers), bank.centers.shape[0], 2048,
                      C.c_void_p(best.data_ptr() + 4 * g), ptr(bank.dists), stream())
    picked = [(c, rng.sample(bank.index[c], n)) if a else None for c, rng, a in zip(best.tolist(), rngs, on)]
    idx = torch.as_tensor([i for p in picked for i in (p[1] if p else [0] * n)], dtype=torch.long, device=rows.device)
    return picked, {k: v.index_select(0, idx) for k, v in bank.exemplars.items()}


def level_backward(s, out, arena, image, kp, lower, grad_arena, mask, live, main=None, sync=None):
    """One level of the bilevel problem (reference base_adaptor.py:222-317) for the videos in ``mask`` on weights ``arena``:
    evaluates the level's loss of every video and accumulates its gradient into ``grad_arena`` (``sync``: data-parallel
    bucketed all-reduce to attach to the last graph of the level).  ``live``: the videos whose motion term is live.
    ``main`` is an already computed forward of ``image`` with these weights (re-used when given).  The level's records go to
    the ``Frame`` ``out``, where a video of the frame outside ``mask`` keeps its earlier ones.  Returns (the (G,) loss, the
    forward whose first rows belong to ``image``).

    With one video, when the motion loss is live and no forward is supplied, the current and the history frame go through
    ONE batched forward / backward (same weights, independent samples), and the teacher forward runs on a side stream.
    With several, the history frame gets its own grouped pass and the teacher runs on the caller's stream."""
    o, G, vo = s.options, s.G, s.video_options
    tag = 'll' if lower else 'ul'
    nb = image.shape[0]
    use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
    use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
    live &= mask
    motion = bool(use_temporal and o.use_motion and live)
    fit = {}
    # the teacher forward is independent of the fast-weight forward: issue it on a side stream so that the two chains
    # of small, latency-bound kernels overlap on the GPU (each one alone leaves most SMs idle at batch 1)
    tpred, side = None, None
    if use_temporal and o.use_meanteacher:
        if G == 1:
            side = _side_stream(image.device)
            side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                           # None: the caller's stream
            tpred = forward_graph(s, s.teacher, s.teacher_buffers, image, mask, s.teacher_masks(nb, image.device, mask))
    if motion:
        hist_image, hist_kp = s.get_hist(live)
        if main is None and G == 1:
            if s._pair is None or s._pair.shape[0] != 2 * nb or s._pair.device != image.device:    # rows [nb:] = history frame
                s._pair = torch.empty(2 * nb, 3, 224, 224, dtype=torch.float32, device=image.device)
            pair, half = s._pair, image.numel() * 4
            _lib.call('dboa_copy_async', ptr(pair), ptr(image), half, stream())
            _lib.call('dboa_copy_async', C.c_void_p(pair.data_ptr() + half), ptr(hist_image.contiguous()), half, stream())
            main = forward_graph(s, arena, s.buffers, pair, mask)
    if main is None:
        main = forward_graph(s, arena, s.buffers, image, mask)
    batched = main.B > nb
    hist = forward_graph(s, arena, s.buffers, hist_image, live) if motion and not batched else None

    def head_weights(q):                                        # the head's 8 weights under the options q
        w = [0.0] * 8
        if use_frame:
            w[0], w[1], w[2] = q.s2dloss_weight, q.shape_prior_weight, q.pose_prior_weight
        if tpred is not None:
            tw = q.teacherloss_weight
            w[3], w[4], w[5], w[6] = 5 * tw, 5 * tw, 0.001 * tw, 1 * tw
        return w
    targets = {}
    if tpred is not None:
        t = tpred
        if side is not None:
            cur = torch.cuda.current_stream()
            cur.wait_stream(side)
            for ten in (t.p2d, t.joints, t.shape, t.rot, t.tape, t.verts, t.smpl_tape, t.cam):
                ten.record_stream(cur)
        targets = dict(t_p2d=t.p2d, t_j3d=t.joints, t_beta=t.shape, t_R=t.rot)
    _mark(s, f'{tag}: forward(s) issued')
    grads = None
    if batched:                                                 # gradients of the 2 nb rows in ONE zeroed buffer (rows [nb:] only get the motion term)
        Bm = main.B
        sizes = (Bm * 49 * 2, Bm * 49 * 3, Bm * 24 * 9, Bm * 10)
        if s._bgrad_flat is None or s._bgrad_flat.numel() != sum(sizes) or s._bgrad_flat.device != image.device:
            s._bgrad_flat = torch.empty(sum(sizes), dtype=torch.float32, device=image.device)
        flat = s._bgrad_flat
        _zero(flat)
        grads = tuple(t.view(Bm, *sh) for t, sh in zip(flat.split(sizes), ((49, 2), (49, 3), (24, 3, 3), (10,))))
    w = [head_weights(q) for q in vo]
    terms, dp2d, dj3d, dR, dbeta = _loss_head(s, main, w, kp=kp if use_frame else None, grads=grads, nb=nb, **targets)
    total = terms[:, 8]
    if use_frame:
        fit[f'{tag}/s2dloss'], fit[f'{tag}/shape_prior'], fit[f'{tag}/pose_prior'] = terms[:, 0], terms[:, 1], terms[:, 2]
        if lower:
            out.lower.append(terms[:, 0])
    if motion:
        mterm = torch.empty(G, dtype=torch.float32, device=image.device)
        p_hist = main.p2d[nb:] if batched else hist.p2d
        dph = dp2d[nb:] if batched else torch.empty_like(hist.p2d)
        kf, kn = s.kp_range
        _lib.call('dboa_loss_motion_weights', ptr(main.p2d), ptr(p_hist), ptr(kp), ptr(hist_kp.contiguous()),
                  (C.c_float * G)(*[q.motionloss_weight for q in vo]), ptr(mterm), ptr(dp2d), ptr(dph), nb, 1, kf, kn, G, live, stream())
        if not batched:
            backward_graph(s, arena, hist, dph, torch.zeros_like(hist.joints), torch.zeros_like(hist.rot), torch.zeros_like(hist.shape),
                           grad_arena)
        total = total + mterm * _motion_weights(s, image.device)
        fit['ul/motion_loss'] = mterm
    _mark(s, f'{tag}: loss head')
    mix = bool(o.retrieval and (o.lower_level_mixtrain if lower else o.upper_level_mixtrain))
    backward_graph(s, arena, main, dp2d, dj3d, dR, dbeta, grad_arena, sync=None if mix else sync)
    _mark(s, f'{tag}: backward')
    if o.retrieval:
        rows = hmr_mod._feature_views(main.tape, main.B)[5][:nb].reshape(G, -1, 2048)[:, 0]      # each video's first sample
        picked, ex = retrieve(s.bank, rows, s.rngs, mask, s._best, o.sample_num)
        out.picks = [p if p is not None else q for p, q in zip(picked, out.picks or picked)]
        if mix:
            e = forward_graph(s, arena, s.buffers, ex['img'], mask)
            n = e.B
            gt_R = torch.empty(n, 24, 3, 3, dtype=torch.float32, device=image.device)
            _lib.call('dboa_rodrigues', ptr(ex['pose'].reshape(-1, 3).contiguous()), ptr(gt_R), n * 24, 0, stream())
            label = lambda lw: [5 * lw, 0, 0, 0, 0, 0.001 * lw, 1 * lw, 5 * lw]
            ew = [label(q.labelloss_weight) for q in vo]
            eterms, a, b, c, d = _loss_head(s, e, ew, kp=ex['keypoints'], t_beta=ex['betas'], t_R=gt_R, gt_s3d=ex['pose_3d'])
            backward_graph(s, arena, e, a, b, c, d, grad_arena, sync=sync)
            total = total + eterms[:, 8]
            fit[f'{tag}/labled_loss'] = eterms[:, 8]
    out.fit = merge(out.fit, fit, mask | ~out.mask & ((1 << G) - 1), G)
    return total, main


def cosines(features_a, features_b, G, mask, partial, reduce_terms=None):
    """The cosines between the feature pairs (``features_a[i]``, ``features_b[i]``) of every video in ``mask``, each video's
    rows on their own: one ``dboa_cosine_terms_active`` call for the sums (a.b, |a|^2, |b|^2), summed over the data-parallel
    ranks by ``reduce_terms`` when given, and one copy to the host.  Returns ((G, n) float32 host cosines, unspecified outside
    ``mask``; the scratch ``partial`` (None: none yet) to pass next time)."""
    def dense(t):                      # one dense block of numel floats (permuted views qualify; xc, of row stride HEAD_LD, does not)
        t = t.detach()
        return t if t.dtype == torch.float32 and 1 + sum((a - 1) * b for a, b in zip(t.shape, t.stride())) == t.numel() else t.float().contiguous()
    n, fa, fb = len(features_a), [dense(t) for t in features_a], [dense(t) for t in features_b]
    pa = (C.c_void_p * n)(*[t.data_ptr() for t in fa])
    pb = (C.c_void_p * n)(*[t.data_ptr() for t in fb])
    ln = (C.c_longlong * n)(*[t.numel() for t in fa])
    need = _lib.load().dboa_cosine_partial_floats_groups(ln, n, G)
    _lib.check(0 if need > 0 else need, 'dboa_cosine_partial_floats_groups')
    dev = fa[0].device
    if partial is None or partial.numel() < need or partial.device != dev:
        partial = torch.empty(need, dtype=torch.float32, device=dev)
    terms = torch.empty(G, n, 3, dtype=torch.float64, device=dev)
    _lib.call('dboa_cosine_terms_active', pa, pb, ln, n, ptr(partial), partial.numel(), ptr(terms), stream(), G, mask)
    if reduce_terms is not None:
        reduce_terms(terms)
    t = terms.cpu()                                                   # the one host sync of the test, for every video
    return (t[..., 0] / (t[..., 1].sqrt().clamp_min(1e-12) * t[..., 2].sqrt().clamp_min(1e-12))).float(), partial


def feature_test(s, fit, a, b, mask):
    """The dynamic loop's feature test between the forwards ``a`` and ``b``: {video: {i: {'cos': c}}} of the videos in ``mask``,
    and their ``feat_sim/cos_sim`` in ``fit`` ((G,) host tensor; the others keep theirs, NaN at first), as ``cal_feature_diff``."""
    G = s.G
    cos, s._cos_partial = cosines(hmr_mod._feature_views(a.tape, a.B), hmr_mod._feature_views(b.tape, b.B), G, mask, s._cos_partial,
                                  s.reduce_terms)
    n = cos.shape[1]
    prev = fit.get('feat_sim/cos_sim')
    rec = torch.full((G,), float('nan')) if prev is None else prev.clone()
    out = {}
    for g in range(G):
        if (mask >> g) & 1:
            rec[g] = cos[g].sum() / (n - 1)                           # reference :218 divides by the last index
            out[g] = {i: {'cos': float(cos[g, i])} for i in range(n)}
    fit['feat_sim/cos_sim'] = rec
    return out


def _continuing(o, sims, steps, vo=None):
    """Bit mask of the videos of ``sims`` whose own test says 'continue' and whose trip count ``steps[g]`` (advanced here, as
    the reference's loop does before its cap test) is still within ``optim_steps``.  Video g's test uses the
    ``cos_sim_threshold`` and ``optim_steps`` of ``vo[g]`` (the step's ``video_options``; None: ``o`` for every video)."""
    mask = 0
    for g, s in sims.items():
        q = o if vo is None else vo[g]
        if 1 - s[12]['cos'] > q.cos_sim_threshold:
            steps[g] += 1
            if steps[g] <= q.optim_steps:
                mask |= 1 << g
    return mask


def fused_adapt(s, batch, mask, frames):
    """One adapted frame (reference dynaboa_benchmark.py:126-201) of the videos in ``mask``: probe forward, ``inner_step``
    SGD steps of the lower level, the upper level, one Adam + EMA teacher sweep, then the optional ``dynamic_boa`` loop.
    ``frames[g]``: the frames video g adapted before this one (its motion term's clock).  Returns the ``Frame``."""
    o, G, theta, buffers, grad = s.options, s.G, s.theta, s.buffers, s.grad
    out = Frame(mask)
    image, kp = batch['image'].contiguous().float(), batch['smpl_j2d'].contiguous().float()
    s.save_hist(image, kp, mask)
    live = sum(1 << g for g in range(G) if (mask >> g) & 1 and frames[g] + s.motion_lead - o.interval > 0)
    evaluate, sync = s.eval_mode, s.grad_sync
    with torch.no_grad():
        _mark(s, 'start')
        probe = forward_graph(s, theta, buffers, image, mask)             # init_features (reference :132-133)
        _mark(s, 'probe forward')
        if not o.use_boa:
            _zero(grad)
            out.upper_loss, _ = level_backward(s, out, theta, image, kp, True, grad, mask, live, main=probe, sync=sync)
            s.adam(mask)
            if evaluate != 'none':
                out.result = s.evaluate(batch, theta, mask, None)
            return out
        fast, cur = theta, probe
        if s._fast is None:
            s._fast, s._inner_grad = [torch.empty_like(theta), torch.empty_like(theta)], torch.empty_like(theta)
        for i in range(o.inner_step):
            for t in _active_rows(s._inner_grad, mask, G):
                _zero(t)
            level_backward(s, out, fast, image, kp, True, s._inner_grad, mask, live, main=cur if i == 0 else None)
            _mark(s, 'lower level (loss + backward)')
            nxt = s._fast[i % 2]
            lr = (C.c_float * G)(*[q.fastlr for q in s.video_options])
            _lib.call('dboa_sgd_update_groups', ptr(fast), ptr(s._inner_grad), ptr(nxt), lr, fast.numel() // G, G, mask, stream())
            fast = nxt
            _mark(s, 'inner SGD step')
            if evaluate == 'all':
                s.evaluate(batch, fast, mask, i)
        for t in _active_rows(grad, mask, G):
            _zero(t)
        out.upper_loss, _ = level_backward(s, out, fast, image, kp, False, grad, mask, live, sync=sync)
        _mark(s, 'upper level (forward + loss + backward)')
        s.adam(mask, s.teacher, o.alpha)                                  # Adam + EMA teacher, one sweep
        _mark(s, 'Adam + EMA')
        if evaluate == 'all' or (evaluate == 'final' and not o.dynamic_boa):
            out.result = s.evaluate(batch, theta, mask, None)
        if o.dynamic_boa:
            # every video runs the reference's loop (:161-192) on its own: the videos still in it (bit mask `loop`) make one
            # grouped pass per iteration, and the decisions of all of them share one host sync
            after = forward_graph(s, theta, buffers, image, mask)
            sims = feature_test(s, out.fit, probe, after, mask)
            out.sims, out.steps = {g: [x] for g, x in sims.items()}, dict.fromkeys(sims, 0)
            loop = _continuing(o, sims, out.steps, s.video_options)
            while loop:
                for t in _active_rows(grad, loop, G):
                    _zero(t)
                after.active = loop                         # its backward runs under the loop, not under its forward's wider mask
                level_backward(s, out, theta, image, kp, False, grad, loop, live, main=after, sync=sync)   # 'after' was computed with the current theta
                s.adam(loop, s.teacher, o.alpha)
                before, after = after, forward_graph(s, theta, buffers, image, loop)
                sims = feature_test(s, out.fit, before, after, loop)
                for g, x in sims.items():
                    out.sims[g].append(x)
                if evaluate == 'all':
                    out.result = s.evaluate(batch, theta, loop, None)
                loop = _continuing(o, sims, out.steps, s.video_options)
            if evaluate == 'final':
                out.result = s.evaluate(batch, theta, mask, None)
        return out


class _ArenaModel:
    """Minimal callable so ``inference`` can evaluate an arbitrary flat weight arena (fast weights)."""

    def __init__(self, model, arena):
        self.model, self.arena = model, arena

    def eval(self):
        return self

    def __call__(self, image, need_feature=False):
        rot, shape, cam, _, tape = hmr_mod.raw_forward(self.arena, self.model._buffers, image)
        if need_feature:
            return rot, shape, cam, hmr_mod._feature_views(tape, image.shape[0])
        return rot, shape, cam
