"""Several independent videos adapted in lockstep on one GPU: ``fused.fused_adapt`` over (G, P) stacks of weight arenas, with
every network forward and backward one grouped call (``dboa_hmr_forward_groups`` / ``dboa_hmr_backward_groups``).  This module
holds only the per-video state.

Each video keeps the reference's semantics: its own theta, Adam moments, teacher, fast weights, gradient, history ring,
teacher dropout masks and retrieval picks.  The G weight arenas (and the teachers', the moments', the gradients') are one
contiguous (G, P) stack; video g owns the rows [g * b, (g + 1) * b) of every per-sample batch.  What the videos share is the
launch sequence and the step count of Adam (all videos advance together).  DESIGN.md section 10.
"""
import random
from types import SimpleNamespace

import torch

from . import _lib, hmr as hmr_mod
from ._lib import ptr, stream
from .fused import fused_adapt


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


class MultiVideoAdaptor:
    """``MultiVideoAdaptor(options, n_videos)``: every video starts from ``options.model_file`` as a fresh ``Adaptor`` does.

    ``adapt(batches)`` advances all videos by one frame (one batch dict per video, ``batch_size`` 1).  ``predict(images)``,
    ``theta(g)``, ``last_upper_loss`` ((G,) device tensor).  ``mask_provider(g, B, device)`` -> (3, 2, B, 1024) keep-masks of
    video g's teacher forward (None: drawn with torch's CUDA RNG, as ``HMR``).  ``rngs[g]``: the ``random.Random`` of video g's
    retrieval picks; ``last_retrieval[g]``: video g's (cluster, picks)."""

    def __init__(self, options, n_videos):
        check_options(options, n_videos)
        from .adaptor import Adaptor
        self.G = G = int(n_videos)
        self.options = o = options
        self.base = base = Adaptor(options)        # checkpoint, SMPL, prior, exemplar bank; its weights are video 0's start
        self.smpl_neutral, self.gmm_f = base.smpl_neutral, base.gmm_f
        if o.retrieval:
            self.centers, self.index, self.h36m_bank, self._dists = base.centers, base.index, base.h36m_bank, base._dists
            self._best = torch.zeros(G, dtype=torch.int32, device=base.device)
        model = base.model.module
        self.thetas = model.arena.detach().repeat(G, 1)
        self.buffers = model._buffers
        self.teachers = base.teacher.arena.detach().repeat(G, 1) if o.use_meanteacher else None
        self.m, self.v, self.grad = torch.zeros_like(self.thetas), torch.zeros_like(self.thetas), torch.zeros_like(self.thetas)
        self.step_count = 0
        # what fused_adapt reads from a single-video adaptor's model, teacher and optimizer, over the (G, P) stacks
        self.model = SimpleNamespace(arena=self.thetas, _buffers=self.buffers, grad_arena=lambda: self.grad)
        self.teacher = SimpleNamespace(arena=self.teachers, _buffers=self.buffers, _masks=self._teacher_masks)
        self.optimizer = SimpleNamespace(step=self._adam_ema, grad_sync=None)
        self.fused_eval = 'none'
        self.global_step = 0
        self.history = {}
        self.mask_provider = None
        self.rngs = [random.Random(o.seed * 1000 + g) for g in range(G)]
        self.last_upper_loss = torch.zeros(G, device=self.thetas.device)
        self.last_retrieval = [None] * G
        self.teacher_dropout = bool(getattr(o, 'teacher_dropout', 1))

    def theta(self, g):
        """View of video g's weights (flat arena layout)."""
        return self.thetas[g]

    def _check_runtime(self):
        opt = self.base.optimizer
        if opt.grad_sync is not None or opt.pre_step_hook is not None:
            raise ValueError('a data-parallel (dist.attach) optimizer is not supported with several videos: it all-reduces one arena '
                             'across ranks')
        check_options(self.options, self.G)

    def save_hist(self, image, s2d):
        self.history[self.global_step] = (image.clone(), s2d.clone())
        self.history.pop(self.global_step - self.options.interval - 1, None)

    def get_hist(self):
        return self.history[self.global_step - self.options.interval]

    def _teacher_masks(self, B, device):
        if not self.teacher_dropout:
            return None
        b, per = B // self.G, []
        for g in range(self.G):
            m = self.mask_provider(g, b, device) if self.mask_provider is not None else None
            per.append(m if m is not None else (torch.rand(3, 2, b, 1024, device=device) >= 0.5).float() * 2.0)
        return torch.cat(per, 2)

    def _adam_ema(self, teacher=None, alpha=0.0):
        """Adam + EMA teacher over all G arenas in one sweep; the videos advance together and share the step count."""
        o = self.options
        self.step_count += 1
        t = None if teacher is None else teacher.arena
        _lib.call('dboa_adam_ema_scaled', ptr(self.thetas), ptr(self.grad), ptr(self.m), ptr(self.v), ptr(t), self.thetas.numel(),
                  float(o.lr), float(o.beta1), float(o.beta2), 1e-8, self.step_count, float(alpha), 1.0, stream())

    # ------------------------------------------------------------------ public
    def adapt(self, batches):
        """One frame of every video (``batches[g]`` is video g's batch dict): ``fused.fused_adapt`` over all G videos -- probe
        forward, K inner SGD steps, the upper level with teacher and motion terms, retrieval with exemplar mix-training, then
        Adam + EMA teacher.  ``fit_losses`` and ``kp2dlosses_lower`` / ``kp2dlosses_upper`` hold this frame's (G,) losses."""
        self._check_runtime()
        if len(batches) != self.G:
            raise ValueError(f'expected {self.G} batches, one per video, got {len(batches)}')
        batch = {k: torch.cat([b[k] for b in batches]).to(self.thetas.device) for k in ('image', 'smpl_j2d')}
        self.fit_losses, self.kp2dlosses_lower, self.kp2dlosses_upper = {}, [], {}
        fused_adapt(self, batch)
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
