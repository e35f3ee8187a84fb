"""Several independent videos adapted in lockstep on one GPU: the bilevel step of ``fused.fused_adapt`` for G learners,
with every network forward and backward one grouped call (``dboa_hmr_forward_groups`` / ``dboa_hmr_backward_groups``).

Each video keeps the reference's semantics: its own theta, Adam moments, teacher, fast weights, gradient, history ring,
teacher dropout masks and retrieval picks.  The G weight arenas (and the teachers', the moments', the gradients') are one
contiguous (G, P) stack; video g owns the rows [g * b, (g + 1) * b) of every per-sample batch.  What the videos share is the
launch sequence and the step count of Adam (all videos advance together).  DESIGN.md section 10.
"""
import ctypes as C
import random

import torch

from . import _lib, hmr as hmr_mod
from ._lib import ptr, stream
from .fused import _smpl_fwd, _zero


def check_options(options, n_videos):
    """Raise ValueError for what the grouped path does not support (no device needed)."""
    G = int(n_videos)
    if G < 1:
        raise ValueError('n_videos must be at least 1')
    if getattr(options, 'dynamic_boa', 0):
        raise ValueError('dynamic_boa=1 is not supported with several videos: per-video trip counts diverge, which needs a masked '
                         'Adam and per-video cosine decisions')
    if not getattr(options, 'use_boa', 1):
        raise ValueError('use_boa=0 is not supported with several videos (only the bilevel step is grouped)')
    lib = _lib.load()
    if lib.dboa_get_fused_forward() or lib.dboa_get_fused_backward():
        raise ValueError('the fused plans are not grouped: dboa_set_fused_forward(0) / dboa_set_fused_backward(0)')
    rows = int(getattr(options, 'batch_size', 1))
    if getattr(options, 'retrieval', 0) and (options.lower_level_mixtrain or options.upper_level_mixtrain):
        rows = max(rows, int(options.sample_num))
    if G * rows > 64:
        raise ValueError(f'{G} videos x {rows} rows per grouped call exceed the 64 samples of the network tape')


class _Graph:
    __slots__ = ('rot', 'shape', 'cam', 'tape', 'joints', 'smpl_tape', 'p2d', 'B', 'masked')


class MultiVideoAdaptor:
    """``MultiVideoAdaptor(options, n_videos)``: every video starts from ``options.model_file`` as a fresh ``Adaptor`` does.

    ``adapt(batches)`` advances all videos by one frame (one batch dict per video, ``batch_size`` 1).  ``predict(images)``,
    ``theta(g)``, ``last_upper_loss`` ((G,) device tensor).  ``mask_provider(g, B, device)`` -> (3, 2, B, 1024) keep-masks of
    video g's teacher forward (None: drawn with torch's CUDA RNG, as ``HMR``).  ``rngs[g]``: the ``random.Random`` of video g's
    retrieval picks."""

    def __init__(self, options, n_videos):
        check_options(options, n_videos)
        from .adaptor import Adaptor
        self.G = G = int(n_videos)
        self.options = o = options
        self.base = Adaptor(options)               # checkpoint, SMPL, prior, exemplar bank; its weights are video 0's start
        model = self.base.model.module
        P = model.arena.numel()
        self.P = P
        self.thetas = model.arena.detach().repeat(G, 1)
        self.buffers = model._buffers
        self.teachers = self.base.teacher.arena.detach().repeat(G, 1) if o.use_meanteacher else None
        self.m, self.v = torch.zeros_like(self.thetas), torch.zeros_like(self.thetas)
        self.grad, self.inner_grad = torch.zeros_like(self.thetas), torch.zeros_like(self.thetas)
        self.fast_bufs = [torch.empty_like(self.thetas), torch.empty_like(self.thetas)]
        self.step_count = 0
        self.global_step = 0
        self.history = {}
        self.mask_provider = None
        self.rngs = [random.Random(o.seed * 1000 + g) for g in range(G)]
        self.last_upper_loss = torch.zeros(G, device=self.thetas.device)
        self.last_retrieval = [None] * G
        self.teacher_dropout = bool(getattr(o, 'teacher_dropout', 1))
        self.kp_range = (25, 24)
        if o.retrieval:
            self._best = torch.zeros(G, dtype=torch.int32, device=self.thetas.device)

    def theta(self, g):
        """View of video g's weights (flat arena layout)."""
        return self.thetas[g]

    def _check_runtime(self):
        opt = self.base.optimizer
        if opt.grad_sync is not None or opt.pre_step_hook is not None:
            raise ValueError('a data-parallel (dist.attach) optimizer is not supported with several videos: it all-reduces one arena '
                             'across ranks')
        check_options(self.options, self.G)

    # ------------------------------------------------------------------ graphs
    def _forward(self, arenas, image, masks=None):
        p = _Graph()
        p.B, p.masked = image.shape[0], masks is not None
        p.rot, p.shape, p.cam, _, p.tape = hmr_mod.raw_forward(arenas, self.buffers, image, masks, groups=self.G)
        _, p.joints, p.smpl_tape = _smpl_fwd(self.base.smpl_neutral, p.shape, p.rot)
        p.p2d = torch.empty(p.B, 49, 2, dtype=torch.float32, device=image.device)
        _lib.call('dboa_project_fwd', ptr(p.cam), ptr(p.joints), ptr(p.p2d), p.B, 49, stream())
        return p

    def _backward(self, arenas, p, dp2d, dj3d, dR, dbeta, grad):
        B, ad = p.B, self.base
        dcam = torch.empty(B, 3, dtype=torch.float32, device=p.rot.device)
        _lib.call('dboa_project_bwd', ptr(p.cam), ptr(p.joints), ptr(dp2d), ptr(dj3d), ptr(dcam), B, 49, 1, 0, stream())
        scratch = torch.empty(_lib.load().dboa_smpl_scratch_floats(B), dtype=torch.float32, device=p.rot.device)
        _lib.call('dboa_smpl_backward', ad.smpl_neutral._struct_ref(), ptr(p.rot), B, ptr(p.smpl_tape), ptr(dj3d), ptr(scratch), ptr(dR),
                  ptr(dbeta), 1, stream())
        hmr_mod.raw_backward(arenas, p.tape, B, p.masked, dR, dbeta, dcam, grad, groups=self.G)

    def _loss_head(self, p, w, kp=None, t_p2d=None, t_j3d=None, t_beta=None, t_R=None, gt_s3d=None):
        """Grouped ``fused._loss_head``: terms (G, 9), per-video means and gradient scaling."""
        B, dev, G = p.B, p.rot.device, self.G
        dp2d, dj3d, dR, dbeta = torch.empty_like(p.p2d), torch.empty_like(p.joints), torch.empty_like(p.rot), torch.empty_like(p.shape)
        terms = torch.empty(G, 9, dtype=torch.float32, device=dev)
        prior_b = None
        if w[2] != 0.0:
            prior_b = torch.empty(B, dtype=torch.float32, device=dev)
            g = self.base.gmm_f
            _lib.call('dboa_pose_prior', ptr(p.rot), ptr(g.means), ptr(g.precisions), ptr(g.neg_log_weights), ptr(prior_b), ptr(dR),
                      float(w[2]) / (B // G), B, stream())                # per-video mean: scale w / b
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
        a.kp_first, a.kp_count = self.kp_range
        _lib.call('dboa_loss_multi', C.byref(a), stream())
        return terms, dp2d, dj3d, dR, dbeta

    def _teacher_masks(self, nb, device):
        if not self.teacher_dropout:
            return None
        per = []
        for g in range(self.G):
            m = self.mask_provider(g, nb, device) if self.mask_provider is not None else None
            per.append(m if m is not None else (torch.rand(3, 2, nb, 1024, device=device) >= 0.5).float() * 2.0)
        return torch.cat(per, 2)

    def _retrieve(self, feature_rows):
        """Nearest cluster of every video's feature (one host synchronisation for all G), then ``random.sample`` from each
        video's own generator.  Returns the exemplar rows of the G videos, stacked video after video."""
        ad, G = self.base, self.G
        for g in range(G):
            f = feature_rows[g].contiguous()
            _lib.call('dboa_retrieval_nearest', ptr(f), ptr(ad.centers), ad.centers.shape[0], 2048, C.c_void_p(self._best.data_ptr() + 4 * g),
                      ptr(ad._dists), stream())
        clusters = self._best.tolist()
        picks = []
        for g in range(G):
            pk = self.rngs[g].sample(ad.index[clusters[g]], self.options.sample_num)
            self.last_retrieval[g] = (clusters[g], pk)
            picks += pk
        idx = torch.as_tensor(picks, dtype=torch.long, device=self.thetas.device)
        return {k: v.index_select(0, idx) for k, v in ad.h36m_bank.items()}

    def _level(self, arenas, image, kp, lower, grad, main=None):
        """Grouped ``fused.level_backward``: accumulates every video's level gradient into its row of ``grad``; returns the
        (G,) level losses.  The history frame goes through its own grouped forward / backward."""
        o, G = self.options, self.G
        nb = image.shape[0] // G
        use_frame = o.use_frame_losses_lower if lower else o.use_frame_losses_upper
        use_temporal = o.use_temporal_losses_lower if lower else o.use_temporal_losses_upper
        motion = bool(use_temporal and o.use_motion and (self.global_step - o.interval) > 0)
        tpred = None
        if use_temporal and o.use_meanteacher:
            tpred = self._forward(self.teachers, image, self._teacher_masks(nb, image.device))
        if main is None:
            main = self._forward(arenas, image)
        w = [0.0] * 8
        targets = {}
        if use_frame:
            w[0], w[1], w[2] = o.s2dloss_weight, o.shape_prior_weight, o.pose_prior_weight
        if tpred is not None:
            tw = o.teacherloss_weight
            w[3], w[4], w[5], w[6] = 5 * tw, 5 * tw, 0.001 * tw, 1 * tw
            targets = dict(t_p2d=tpred.p2d, t_j3d=tpred.joints, t_beta=tpred.shape, t_R=tpred.rot)
        terms, dp2d, dj3d, dR, dbeta = self._loss_head(main, w, kp=kp if use_frame else None, **targets)
        total = terms[:, 8].clone()
        if motion:
            h = self.history[self.global_step - o.interval]
            hist = self._forward(arenas, h['image'])
            mterm = torch.empty(G, dtype=torch.float32, device=image.device)
            dph = torch.empty_like(hist.p2d)
            kf, kn = self.kp_range
            _lib.call('dboa_loss_motion_groups', ptr(main.p2d), ptr(hist.p2d), ptr(kp), ptr(h['kp']), float(o.motionloss_weight), ptr(mterm),
                      ptr(dp2d), ptr(dph), main.B, 1, kf, kn, G, stream())
            self._backward(arenas, hist, dph, torch.zeros_like(hist.joints), torch.zeros_like(hist.rot), torch.zeros_like(hist.shape), grad)
            total += mterm * o.motionloss_weight
        self._backward(arenas, main, dp2d, dj3d, dR, dbeta, grad)
        if o.retrieval:
            feats = hmr_mod._feature_views(main.tape, main.B)[5].reshape(G, nb, 2048)[:, 0]
            ex = self._retrieve(feats)
            if o.lower_level_mixtrain if lower else o.upper_level_mixtrain:
                e = self._forward(arenas, ex['img'])
                gt_R = torch.empty(e.B, 24, 3, 3, dtype=torch.float32, device=image.device)
                _lib.call('dboa_rodrigues', ptr(ex['pose'].reshape(-1, 3).contiguous()), ptr(gt_R), e.B * 24, 0, stream())
                lw = o.labelloss_weight
                eterms, a, b, c, d = self._loss_head(e, [5 * lw, 0, 0, 0, 0, 0.001 * lw, 1 * lw, 5 * lw], kp=ex['keypoints'],
                                                     t_beta=ex['betas'], t_R=gt_R, gt_s3d=ex['pose_3d'])
                self._backward(arenas, e, a, b, c, d, grad)
                total += eterms[:, 8]
        return total, main

    # ------------------------------------------------------------------ public
    def adapt(self, batches):
        """One frame of every video (``batches[g]`` is video g's batch dict): probe forward, K inner SGD steps, the upper level
        with teacher and motion terms, retrieval with exemplar mix-training, then Adam + EMA teacher over all G arenas."""
        self._check_runtime()
        if len(batches) != self.G:
            raise ValueError(f'expected {self.G} batches, one per video, got {len(batches)}')
        o = self.options
        image = torch.cat([b['image'] for b in batches]).to(self.thetas.device).contiguous().float()
        kp = torch.cat([b['smpl_j2d'] for b in batches]).to(self.thetas.device).contiguous().float()
        self.history[self.global_step] = {'image': image.clone(), 'kp': kp.clone()}
        self.history.pop(self.global_step - o.interval - 1, None)
        n = self.thetas.numel()
        with torch.no_grad():
            probe = self._forward(self.thetas, image)
            fast = self.thetas
            for i in range(o.inner_step):
                _zero(self.inner_grad)
                self._level(fast, image, kp, True, self.inner_grad, main=probe if i == 0 else None)
                nxt = self.fast_bufs[i % 2]
                _lib.call('dboa_sgd_update', ptr(fast), ptr(self.inner_grad), ptr(nxt), float(o.fastlr), n, stream())
                fast = nxt
            _zero(self.grad)
            self.last_upper_loss, _ = self._level(fast, image, kp, False, self.grad)
            self.step_count += 1
            t = self.teachers if o.use_meanteacher else None
            _lib.call('dboa_adam_ema_scaled', ptr(self.thetas), ptr(self.grad), ptr(self.m), ptr(self.v), ptr(t), n, float(o.lr),
                      float(o.beta1), float(o.beta2), 1e-8, self.step_count, float(o.alpha), 1.0, stream())
        self.global_step += 1

    def predict(self, images):
        """Every video's prediction for its rows of ``images`` with its current weights: a list of G dicts with rotmat, betas,
        cam, joints (49) and vertices."""
        with torch.no_grad():
            image = images.to(self.thetas.device).contiguous().float()
            rot, shape, cam, _, _ = hmr_mod.raw_forward(self.thetas, self.buffers, image, groups=self.G)
            out = self.base.decode_smpl_params(rot, shape)
        b = image.shape[0] // self.G
        s = [slice(g * b, (g + 1) * b) for g in range(self.G)]
        return [dict(rotmat=rot[q], betas=shape[q], cam=cam[q], joints=out['s3d'][q], vertices=out['vts'][q]) for q in s]
