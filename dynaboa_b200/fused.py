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

The same step adapts G videos at once (``multivideo.MultiVideoAdaptor``): their weight, teacher and gradient arenas are
(G, P) stacks instead of flat arenas, video g owns the rows [g * b, (g + 1) * b) of every batch, and every network pass and
loss head is one grouped call.  When only some of the videos advance this frame (``ad.active``, an int whose bit g means video
g takes part; None: all), the network passes skip the others and the element-wise sweeps touch only the active videos' rows of
the stacks.  DESIGN.md section 10.
"""
import ctypes as C
import os
import random

import torch

from . import _lib, hmr as hmr_mod, losses
from ._lib import ptr, stream


_SIDE = {}
_TEACHER_OVERLAP = os.environ.get('DBOA_TEACHER_STREAM', '1') != '0'     # 0: teacher forward on the caller's stream


def _side_stream(device):
    if device.index not in _SIDE:
        _SIDE[device.index] = torch.cuda.Stream(device=device)
    return _SIDE[device.index]


def _mark(ad, name):
    """Diagnostics (scripts/phase_times.py): when ``ad.phase_events`` is a list, record a CUDA event on the caller's stream."""
    ev_list = getattr(ad, 'phase_events', None)
    if ev_list is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        ev_list.append((name, ev))


def _groups(arena):
    """Videos of a weight arena: one for a flat arena, G for a (G, P) stack."""
    return arena.shape[0] if arena.dim() == 2 else 1


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


def _active_rows(ad, t):
    """``t`` itself, or, for a (G, P) stack while only some videos take part, the views of its runs of active videos: element-wise
    sweeps over them leave the idle videos' rows untouched, and with every video active they are one sweep as before."""
    act = getattr(ad, 'active', None)
    return [t] if act is None else [t[a:b] for a, b in runs(act, t.shape[0])]


class _Pred:
    """Everything one forward graph produces (kept for its backward)."""
    __slots__ = ('image', 'rot', 'shape', 'cam', 'tape', 'verts', 'joints', 'smpl_tape', 'p2d', 'B', 'masked', 'groups', 'active')


def _smpl_fwd(smpl, betas, rot):
    B, dev = betas.shape[0], betas.device
    verts = torch.empty(B, 6890, 3, dtype=torch.float32, device=dev)
    joints = torch.empty(B, 49, 3, dtype=torch.float32, device=dev)
    tape = torch.empty(_lib.load().dboa_smpl_tape_floats(B), dtype=torch.float32, device=dev)
    _lib.call('dboa_smpl_forward', smpl._struct_ref(), ptr(betas), ptr(rot), B, ptr(verts), ptr(joints), ptr(tape), stream())
    return verts, joints, tape


def forward_graph(ad, arena, buffers, image, masks=None, active=None):
    p = _Pred()
    p.image, p.B, p.masked, p.groups, p.active = image, image.shape[0], masks is not None, _groups(arena), active
    p.rot, p.shape, p.cam, _, p.tape = hmr_mod.raw_forward(arena, buffers, image, masks, groups=p.groups, active=active)
    p.verts, p.joints, p.smpl_tape = _smpl_fwd(ad.smpl_neutral, p.shape, p.rot)
    p.p2d = torch.empty(p.B, 49, 2, dtype=torch.float32, device=image.device)
    _lib.call('dboa_project_fwd', ptr(p.cam), ptr(p.joints), ptr(p.p2d), p.B, 49, stream())
    return p


def _loss_head(ad, p, w, kp=None, t_p2d=None, t_j3d=None, t_beta=None, t_R=None, gt_s3d=None, grads=None, nb=None):
    """Runs the (optional) pose prior and the multi-term head on the first ``nb`` samples of ``p``, each video's rows on their
    own (per-video means and gradient scaling); returns (terms (G, 9), dp2d, dj3d, dR, dbeta).  ``grads``: preallocated
    (possibly larger-batch) gradient buffers whose leading ``nb`` rows are written."""
    B, dev, G = (p.B if nb is None else nb), p.rot.device, p.groups
    if grads is None:
        dp2d, dj3d = torch.empty_like(p.p2d), torch.empty_like(p.joints)
        dR, dbeta = torch.empty_like(p.rot), torch.empty_like(p.shape)
    else:
        dp2d, dj3d, dR, dbeta = grads
    terms = torch.empty(G, 9, dtype=torch.float32, device=dev)
    prior_b = None
    if w[2] != 0.0:
        prior_b = torch.empty(B, dtype=torch.float32, device=dev)
        g = ad.gmm_f
        _lib.call('dboa_pose_prior', ptr(p.rot), ptr(g.means), ptr(g.precisions), ptr(g.neg_log_weights), ptr(prior_b), ptr(dR),
                  float(w[2]) / (B // G), B, stream())                   # per-video mean: scale w / b
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
    for i in range(8):
        a.w[i] = float(w[i])
    a.dR_accumulate = 1 if prior_b is not None else 0
    a.kp_first, a.kp_count = getattr(ad, 'kp_range', (25, 24))      # joints of the re-projection term (webcam client: (0, 25))
    _lib.call('dboa_loss_multi', C.byref(a), stream())
    return terms, dp2d, dj3d, dR, dbeta


def _zero(t):
    """Stream-ordered memset (copy engine / driver memset node): no ATen fill kernel in the step."""
    _lib.call('dboa_fill_zero', ptr(t), t.numel() * t.element_size(), stream())


def backward_graph(ad, arena, p, dp2d, dj3d, dR, dbeta, grad_arena, sync=None):
    """d(loss)/d(p2d, joints, R, beta) -> accumulate d(loss)/d(weights) into ``grad_arena``.  ``sync``: the data-parallel
    ``BucketedGradSync`` when this is the LAST graph accumulated into the outer gradient: its buckets are all-reduced on the
    communication stream while the rest of this backward runs."""
    B, dev = p.B, p.rot.device
    dcam = torch.empty(B, 3, dtype=torch.float32, device=dev)
    _lib.call('dboa_project_bwd', ptr(p.cam), ptr(p.joints), ptr(dp2d), ptr(dj3d), ptr(dcam), B, 49, 1, 0, stream())
    scratch = torch.empty(_lib.load().dboa_smpl_scratch_floats(B), dtype=torch.float32, device=dev)
    _lib.call('dboa_smpl_backward', ad.smpl_neutral._struct_ref(), ptr(p.rot), B, ptr(p.smpl_tape), ptr(dj3d), ptr(scratch), ptr(dR),
              ptr(dbeta), 1, stream())
    if sync is not None:
        sync.arm()
    hmr_mod.raw_backward(arena, p.tape, B, p.masked, dR, dbeta, dcam, grad_arena, groups=p.groups, active=p.active)
    if sync is not None:
        sync.after_backward(grad_arena)
        ad.optimizer.reduced = True


def retrieve(ad, rows, rngs, active=None):
    """reference :82-96 for every video: the nearest cluster centre of video g's feature row ``rows[g]`` by cosine distance
    (one host synchronisation for all videos), then ``rngs[g].sample`` inside that cluster.  Returns the (cluster, picks) of
    every video and the picked exemplar rows, video after video.  ``active`` (bit mask, None: all): an idle video draws
    nothing, gets None and placeholder rows (exemplar 0)."""
    on = [active is None or bool((active >> g) & 1) for g in range(len(rows))]
    for g, f in enumerate(rows):
        if not on[g]:
            continue
        f = f.contiguous()
        _lib.call('dboa_retrieval_nearest', ptr(f), ptr(ad.centers), ad.centers.shape[0], 2048, C.c_void_p(ad._best.data_ptr() + 4 * g),
                  ptr(ad._dists), stream())
    picked = [(c, rng.sample(ad.index[c], ad.options.sample_num)) if a else None for c, rng, a in zip(ad._best.tolist(), rngs, on)]
    idx = torch.as_tensor([i for p in picked for i in (p[1] if p else [0] * ad.options.sample_num)], dtype=torch.long, device=rows.device)
    return picked, {k: v.index_select(0, idx) for k, v in ad.h36m_bank.items()}


def level_backward(ad, arena, buffers, image, kp, lower, grad_arena, main=None, sync=None):
    """One level of the bilevel problem (reference base_adaptor.py:222-317) on weights ``arena``, a flat arena or a (G, P)
    stack of G videos' arenas: evaluates the level's loss of every video and accumulates its gradient into ``grad_arena``
    (same layout; ``sync``: data-parallel bucketed all-reduce to attach to the last graph of the level).  ``main`` is an
    already computed forward of ``image`` with these weights (re-used when given).  Returns (the loss, a device scalar for
    a flat arena and (G,) for a stack; the forward whose first rows belong to ``image``).

    With one video, when the motion loss is live and no forward is supplied, the current and the history frame go through
    ONE batched forward / backward (same weights, independent samples), and the teacher forward runs on a side stream.
    With several, the history frame gets its own grouped pass and the teacher runs on the caller's stream."""
    o = ad.options
    tag = 'll' if lower else 'ul'
    nb = image.shape[0]
    G = _groups(arena)
    per_video = arena.shape[:-1]                                # shape of the losses recorded and returned: () or (G,)
    use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
    use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
    act = getattr(ad, 'active', None)                           # videos taking part (bit mask; None: all)
    # videos whose motion term is live (bit mask): all of them or none, by the frame count, unless the adaptor keeps one per video
    every = (1 << G) - 1
    live = getattr(ad, 'motion_active', None)
    if live is None:
        live = every if (ad.global_step - o.interval) > 0 else 0
    motion = bool(use_temporal and o.use_motion and live)
    live = None if live == every else live
    # the teacher forward is independent of the fast-weight forward: issue it on a side stream so that the two chains
    # of small, latency-bound kernels overlap on the GPU (each one alone leaves most SMs idle at batch 1)
    tpred, side = None, None
    if use_temporal and o.use_meanteacher:
        teacher = ad.teacher
        if _TEACHER_OVERLAP and G == 1:
            side = _side_stream(image.device)
            side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                           # None: the caller's stream
            tpred = forward_graph(ad, teacher.arena, teacher._buffers, image, teacher._masks(nb, image.device), act)
    if motion:
        hist_image, hist_kp = ad.get_hist()
        if main is None and G == 1:
            pair = getattr(ad, '_pair', None)                   # persistent (2 nb, 3, 224, 224) staging: rows [nb:] = history frame
            if pair is None or pair.shape[0] != 2 * nb or pair.device != image.device:
                pair = ad._pair = torch.empty(2 * nb, 3, 224, 224, dtype=torch.float32, device=image.device)
            half = image.numel() * 4
            _lib.call('dboa_copy_async', ptr(pair), ptr(image), half, stream())
            _lib.call('dboa_copy_async', C.c_void_p(pair.data_ptr() + half), ptr(hist_image.contiguous()), half, stream())
            main = forward_graph(ad, arena, buffers, pair)
    if main is None:
        main = forward_graph(ad, arena, buffers, image, active=act)
    batched = main.B > nb
    hist = forward_graph(ad, arena, buffers, hist_image, active=live) if motion and not batched else None
    w = [0.0] * 8
    targets = {}
    if use_frame:
        w[0], w[1], w[2] = o.s2dloss_weight, o.shape_prior_weight, o.pose_prior_weight
    if tpred is not None:
        t = tpred
        if side is not None:
            cur = torch.cuda.current_stream()
            cur.wait_stream(side)
            for ten in (t.p2d, t.joints, t.shape, t.rot, t.tape, t.verts, t.smpl_tape, t.cam):
                ten.record_stream(cur)
        tw = o.teacherloss_weight
        w[3], w[4], w[5], w[6] = 5 * tw, 5 * tw, 0.001 * tw, 1 * tw
        targets = dict(t_p2d=t.p2d, t_j3d=t.joints, t_beta=t.shape, t_R=t.rot)
    _mark(ad, f'{tag}: forward(s) issued')
    grads = None
    if batched:                                                 # gradients of the 2 nb rows in ONE zeroed buffer (rows [nb:] only get the motion term)
        Bm = main.B
        sizes = (Bm * 49 * 2, Bm * 49 * 3, Bm * 24 * 9, Bm * 10)
        flat = getattr(ad, '_bgrad_flat', None)
        if flat is None or flat.numel() != sum(sizes) or flat.device != image.device:
            flat = ad._bgrad_flat = torch.empty(sum(sizes), dtype=torch.float32, device=image.device)
        _zero(flat)
        e = [0, sizes[0], sizes[0] + sizes[1], sizes[0] + sizes[1] + sizes[2]]
        grads = (flat[e[0]:e[1]].view(Bm, 49, 2), flat[e[1]:e[2]].view(Bm, 49, 3), flat[e[2]:e[3]].view(Bm, 24, 3, 3), flat[e[3]:].view(Bm, 10))
    terms, dp2d, dj3d, dR, dbeta = _loss_head(ad, main, w, kp=kp if use_frame else None, grads=grads, nb=nb, **targets)
    terms = terms.view(*per_video, 9)
    total = terms[..., 8]
    if use_frame:
        ad.fit_losses[f'{tag}/s2dloss'], ad.fit_losses[f'{tag}/shape_prior'], ad.fit_losses[f'{tag}/pose_prior'] = terms[..., 0], terms[..., 1], terms[..., 2]
        (ad.kp2dlosses_lower.append(terms[..., 0]) if lower else ad.kp2dlosses_upper.__setitem__(ad.global_step, terms[..., 0]))
    if motion:
        mterm = torch.empty(per_video, dtype=torch.float32, device=image.device)
        p_hist = main.p2d[nb:] if batched else hist.p2d
        dph = dp2d[nb:] if batched else torch.empty_like(hist.p2d)
        kf, kn = getattr(ad, 'kp_range', (25, 24))
        margs = (ptr(main.p2d), ptr(p_hist), ptr(kp), ptr(hist_kp.contiguous()), float(o.motionloss_weight), ptr(mterm), ptr(dp2d), ptr(dph),
                 nb, 1, kf, kn, G)
        if live is None:
            _lib.call('dboa_loss_motion_groups', *margs, stream())
        else:
            _lib.call('dboa_loss_motion_active', *margs, live, stream())
        if not batched:
            backward_graph(ad, arena, hist, dph, torch.zeros_like(hist.joints), torch.zeros_like(hist.rot), torch.zeros_like(hist.shape),
                           grad_arena)
        total = total + mterm * o.motionloss_weight
        ad.fit_losses['ul/motion_loss'] = mterm
    _mark(ad, f'{tag}: loss head')
    mix = bool(o.retrieval and (o.lower_level_mixtrain if lower else o.upper_level_mixtrain))
    backward_graph(ad, arena, main, dp2d, dj3d, dR, dbeta, grad_arena, sync=None if mix else sync)
    _mark(ad, f'{tag}: backward')
    if o.retrieval:
        rows = hmr_mod._feature_views(main.tape, main.B)[5][:nb].reshape(G, -1, 2048)[:, 0]      # each video's first sample
        picked, ex = retrieve(ad, rows, getattr(ad, 'rngs', [random]), act)
        if per_video:
            ad.last_retrieval = [p if p is not None else q for p, q in zip(picked, ad.last_retrieval)]
        else:
            ad.last_retrieval = picked[0]
        if mix:
            e = forward_graph(ad, arena, buffers, ex['img'], active=act)
            n = e.B
            gt_R = torch.empty(n, 24, 3, 3, dtype=torch.float32, device=image.device)
            _lib.call('dboa_rodrigues', ptr(ex['pose'].reshape(-1, 3).contiguous()), ptr(gt_R), n * 24, 0, stream())
            lw = o.labelloss_weight
            eterms, a, b, c, d = _loss_head(ad, e, [5 * lw, 0, 0, 0, 0, 0.001 * lw, 1 * lw, 5 * lw], kp=ex['keypoints'], t_beta=ex['betas'],
                                            t_R=gt_R, gt_s3d=ex['pose_3d'])
            backward_graph(ad, arena, e, a, b, c, d, grad_arena, sync=sync)
            eterms = eterms.view(*per_video, 9)
            total = total + eterms[..., 8]
            ad.fit_losses[f'{tag}/labled_loss'] = eterms[..., 8]
    return total, main


def feature_cosines(ad, tape_a, tape_b, B):
    fa, fb = hmr_mod._feature_views(tape_a, B), hmr_mod._feature_views(tape_b, B)
    return ad.cal_feature_diff(fa, fb)


def feature_test(ad, a, b, stacked, mask):
    """The dynamic loop's feature test between the forwards ``a`` and ``b``: {video: {i: {'cos': c}}} of every video in ``mask``
    (a bit mask).  One arena: ``cal_feature_diff`` (it all-reduces under data parallelism).  A (G, P) stack: one
    ``dboa_cosine_terms_active`` call over the videos in ``mask`` and one copy to the host; each video's cosines and its
    ``fit_losses['feat_sim/cos_sim']`` entry are formed from its own sums exactly as ``cal_feature_diff`` forms them."""
    if not stacked:
        return {0: feature_cosines(ad, a.tape, b.tape, a.B)}
    from .base_adaptor import _dense_ptr_tensor
    G, n = a.groups, 15
    fa = [_dense_ptr_tensor(t) for t in hmr_mod._feature_views(a.tape, a.B)]      # xc (row stride HEAD_LD) is made dense
    fb = [_dense_ptr_tensor(t) for t in hmr_mod._feature_views(b.tape, b.B)]
    pa = (C.c_void_p * n)(*[t.data_ptr() for t in fa])
    pb = (C.c_void_p * n)(*[t.data_ptr() for t in fb])
    ln = (C.c_longlong * n)(*[t.numel() for t in fa])
    need = _lib.load().dboa_cosine_partial_floats_groups(ln, n, G)
    _lib.check(0 if need > 0 else need, 'dboa_cosine_partial_floats_groups')
    part = getattr(ad, '_cos_partial', None)
    if part is None or part.numel() < need or part.device != a.rot.device:
        part = ad._cos_partial = torch.empty(need, dtype=torch.float32, device=a.rot.device)
    terms = torch.empty(G, n, 3, dtype=torch.float64, device=a.rot.device)
    _lib.call('dboa_cosine_terms_active', pa, pb, ln, n, ptr(part), part.numel(), ptr(terms), stream(), G, mask)
    host = terms.cpu()                                                # the one host sync of this test, for every video
    prev = ad.fit_losses.get('feat_sim/cos_sim')
    rec = torch.full((G,), float('nan')) if prev is None else prev.clone()
    out = {}
    for g in range(G):
        if (mask >> g) & 1:
            t = host[g]
            cos = (t[:, 0] / (t[:, 1].sqrt().clamp_min(1e-12) * t[:, 2].sqrt().clamp_min(1e-12))).float()
            rec[g] = cos.sum() / (n - 1)
            out[g] = {i: {'cos': float(cos[i])} for i in range(n)}
    ad.fit_losses['feat_sim/cos_sim'] = rec
    return out


def _continuing(o, sims, steps):
    """Bit mask of the videos of ``sims`` whose own test says 'continue' and whose trip count ``steps[g]`` (advanced here, as
    the reference's loop does before its cap test) is still within ``optim_steps``."""
    mask = 0
    for g, s in sims.items():
        if 1 - s[12]['cos'] > o.cos_sim_threshold:
            steps[g] += 1
            if steps[g] <= o.optim_steps:
                mask |= 1 << g
    return mask


def _keep_records(ad, old, mask, G):
    """After a level evaluated under ``mask``: every ``fit_losses`` / ``kp2dlosses_upper`` entry of ``old`` (the records before
    that level) keeps its value for the videos outside ``mask``, whose last evaluation of the frame came earlier."""
    keep = torch.tensor([bool((mask >> g) & 1) for g in range(G)])
    for rec, prev in zip((ad.fit_losses, ad.kp2dlosses_upper), old):
        for k, v in prev.items():
            if rec[k] is not v:
                rec[k] = torch.where(keep.to(v.device), rec[k], v)


def fused_adapt(ad, batch):
    """One adapted frame (reference dynaboa_benchmark.py:126-201) of every video of ``ad``: probe forward, ``inner_step`` SGD
    steps of the lower level, the upper level, one Adam + EMA teacher sweep, then the optional ``dynamic_boa`` loop.

    Reads from ``ad``: ``model`` (``arena``, ``_buffers``, ``grad_arena()``), ``teacher`` (``arena``, ``_buffers``,
    ``_masks(B, device)``) and ``optimizer`` (``step(teacher=, alpha=)``, ``grad_sync``), whose arenas are flat for one video
    and (G, P) stacks for G videos; ``save_hist`` / ``get_hist``; ``global_step``; the records the level writes."""
    o = ad.options
    image, kp = batch['image'].contiguous().float(), batch['smpl_j2d'].contiguous().float()
    ad.save_hist(image, kp)
    model = getattr(ad.model, 'module', ad.model)
    theta, buffers = model.arena, model._buffers
    opt = ad.optimizer
    grad = model.grad_arena()
    teacher = ad.teacher if o.use_meanteacher else None
    evaluate = getattr(ad, 'fused_eval', 'final')
    with torch.no_grad():
        _mark(ad, 'start')
        probe = forward_graph(ad, theta, buffers, image, active=getattr(ad, 'active', None))       # init_features (reference :132-133)
        _mark(ad, 'probe forward')
        import torch.distributed as tdist
        sync = opt.grad_sync if (opt.grad_sync is not None and tdist.is_initialized() and tdist.get_world_size() > 1) else None
        if not o.use_boa:
            _zero(grad)
            ad.last_upper_loss, _ = level_backward(ad, theta, buffers, image, kp, True, grad, main=probe, sync=sync)
            opt.step()
            return ad.inference(batch, ad.model) if evaluate != 'none' else None
        fast, cur = theta, probe
        if not hasattr(ad, '_fast_bufs'):
            ad._fast_bufs = [torch.empty_like(theta), torch.empty_like(theta)]
            ad._inner_grad = torch.empty_like(theta)
        for i in range(o.inner_step):
            for t in _active_rows(ad, ad._inner_grad):
                _zero(t)
            level_backward(ad, fast, buffers, image, kp, True, ad._inner_grad, main=cur if i == 0 else None)
            _mark(ad, 'lower level (loss + backward)')
            nxt = ad._fast_bufs[i % 2]
            for f, g, n in zip(_active_rows(ad, fast), _active_rows(ad, ad._inner_grad), _active_rows(ad, nxt)):
                _lib.call('dboa_sgd_update', ptr(f), ptr(g), ptr(n), float(o.fastlr), f.numel(), stream())
            fast = nxt
            _mark(ad, 'inner SGD step')
            if evaluate == 'all':
                ad.inference(batch, _ArenaModel(model, fast))
        for t in _active_rows(ad, grad):
            _zero(t)
        ad.last_upper_loss, _ = level_backward(ad, fast, buffers, image, kp, False, grad, sync=sync)
        _mark(ad, 'upper level (forward + loss + backward)')
        opt.step(teacher=teacher, alpha=o.alpha)                    # Adam + EMA teacher, one sweep
        _mark(ad, 'Adam + EMA')
        result = None
        if evaluate == 'all' or (evaluate == 'final' and not o.dynamic_boa):
            result = ad.inference(batch, ad.model)
        if o.dynamic_boa:
            # every video runs the reference's loop (:161-192) on its own: the videos still in it (bit mask `loop`) make one
            # grouped pass per iteration, and the decisions of all of them share one host sync.  One arena: one bit.
            stacked, G = theta.dim() == 2, _groups(theta)
            every = (1 << G) - 1
            frame = getattr(ad, 'active', None)
            frame_bits = every if frame is None else frame
            after = forward_graph(ad, theta, buffers, image, active=frame)
            sims = feature_test(ad, probe, after, stacked, frame_bits)
            trace, steps = {g: [s] for g, s in sims.items()}, dict.fromkeys(sims, 0)
            if not stacked:
                ad.feat_sims[ad.global_step] = trace[0]
            loop = _continuing(o, sims, steps)
            while loop:
                act = None if loop == every else loop
                if stacked:
                    ad.active = act                         # the level, its draws, Adam and the motion mask follow the loop
                old = (dict(ad.fit_losses), dict(ad.kp2dlosses_upper)) if loop != frame_bits else None
                for t in _active_rows(ad, grad):
                    _zero(t)
                after.active = act                          # its backward runs under the loop, not under its forward's wider mask
                level_backward(ad, theta, buffers, image, kp, False, grad, main=after, sync=sync)   # 'after' was computed with the current theta
                if old is not None:
                    _keep_records(ad, old, loop, G)
                opt.step(teacher=teacher, alpha=o.alpha)
                before, after = after, forward_graph(ad, theta, buffers, image, active=act)
                sims = feature_test(ad, before, after, stacked, loop)
                for g, s in sims.items():
                    trace[g].append(s)
                if evaluate == 'all':
                    result = ad.inference(batch, ad.model)
                loop = _continuing(o, sims, steps)
            if stacked:
                ad.active = frame
                ad.optimized_step = [steps.get(g) for g in range(G)]
                ad.loop_feat_sims = [trace.get(g) for g in range(G)]
            else:
                ad.optimized_step = steps[0]
                ad.optim_step_record.append(steps[0])
            if evaluate == 'final':
                result = ad.inference(batch, ad.model)
        return result


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
