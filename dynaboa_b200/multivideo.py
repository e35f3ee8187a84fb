"""Several independent videos adapted in lockstep on one GPU: ``fused.fused_adapt`` over (G, P) stacks of weight arenas, with
every network forward and backward one grouped call (``dboa_hmr_forward_groups`` / ``dboa_hmr_backward_groups``).  This module
holds only the per-video state.

Each video keeps the reference's semantics: its own theta, Adam moments and step count, teacher, fast weights, gradient,
history ring, motion warm-up, teacher dropout masks and retrieval picks.  The G weight arenas (and the teachers', the moments',
the gradients') are one contiguous (G, P) stack; video g owns the rows [g * b, (g + 1) * b) of every per-sample batch.  The
G slots are a pool: a slot whose batch is None sits the frame out (its CTAs return at once in every grouped call), and
``start(g)`` puts a new video into slot g.  DESIGN.md section 10.
"""
import ctypes as C
import random
from types import SimpleNamespace

import torch

from . import _lib, hmr as hmr_mod
from ._lib import ptr, stream
from .fused import fused_adapt, runs


def check_options(options, n_videos, dynamic_loop=False):
    """Raise ValueError for what the grouped path does not support (no device needed).  ``dynamic_loop=True`` accepts
    ``dynamic_boa=1``: every video then runs its own re-adaptation loop (DESIGN.md section 10, "Dynamic loop")."""
    G = int(n_videos)
    if G < 1:
        raise ValueError('n_videos must be at least 1')
    if getattr(options, 'dynamic_boa', 0) and not dynamic_loop:
        raise ValueError('dynamic_boa=1 with several videos runs a re-adaptation loop per video, whose trip counts differ: '
                         'opt in with dynamic_loop=True')
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
    """``MultiVideoAdaptor(options, n_videos)``: a pool of G slots, each holding one video that starts from
    ``options.model_file`` as a fresh ``Adaptor`` does.

    ``adapt(batches)`` advances every slot whose entry is a batch dict (``batch_size`` 1) by one frame; a None entry leaves that
    slot as it was.  ``start(g, seed=None)`` puts a new video into slot g.  ``predict(images)``, ``theta(g)``,
    ``last_upper_loss`` ((G,) device tensor).  ``video_steps[g]``: frames slot g adapted since its ``start``; ``global_step``:
    ``adapt`` calls.  ``mask_provider(g, B, device)`` -> (3, 2, B, 1024) keep-masks of video g's teacher forward (None: drawn
    with torch's CUDA RNG, as ``HMR``).  ``rngs[g]``: the ``random.Random`` of video g's retrieval picks; ``last_retrieval[g]``:
    video g's (cluster, picks).

    ``dynamic_loop=True`` runs the ``dynamic_boa`` loop: after its Adam + EMA step every video of the frame repeats the upper
    level until its own feature test passes or its own trip count exceeds ``optim_steps``.  Per slot, as ``Adaptor`` records
    them: ``optim_step_record[g]`` (one trip count per frame the slot advanced), ``feat_sims[g][frame]`` (the cosines of each
    test, ``frame`` counted from the slot's ``start``), and ``optimized_step`` ((G,), None for slots that sat the frame out)."""

    def __init__(self, options, n_videos, dynamic_loop=False):
        check_options(options, n_videos, dynamic_loop)
        from .adaptor import Adaptor
        self.dynamic_loop = bool(dynamic_loop)
        self.G = G = int(n_videos)
        self.options = o = options
        self.base = base = Adaptor(options)        # checkpoint, SMPL, prior, exemplar bank; never adapted, so it keeps the checkpoint
        self.smpl_neutral, self.gmm_f = base.smpl_neutral, base.gmm_f
        if o.retrieval:
            self.centers, self.index, self.h36m_bank, self._dists = base.centers, base.index, base.h36m_bank, base._dists
            self._best = torch.zeros(G, dtype=torch.int32, device=base.device)
        model = base.model.module
        self.thetas = torch.empty(G, model.arena.numel(), device=model.arena.device)
        self.buffers = model._buffers
        self.teachers = torch.empty_like(self.thetas) if o.use_meanteacher else None
        self.m, self.v, self.grad = torch.empty_like(self.thetas), torch.empty_like(self.thetas), torch.zeros_like(self.thetas)
        # what fused_adapt reads from a single-video adaptor's model, teacher and optimizer, over the (G, P) stacks
        self.model = SimpleNamespace(arena=self.thetas, _buffers=self.buffers, grad_arena=lambda: self.grad)
        self.teacher = SimpleNamespace(arena=self.teachers, _buffers=self.buffers, _masks=self._teacher_masks)
        self.optimizer = SimpleNamespace(step=self._adam_ema, grad_sync=None)
        self.fused_eval = 'none'
        self.global_step = 0
        self.mask_provider = None
        self.last_upper_loss = torch.zeros(G, device=self.thetas.device)
        self.last_retrieval = [None] * G
        self.teacher_dropout = bool(getattr(o, 'teacher_dropout', 1))
        self.step_counts, self.video_steps, self.histories, self.rngs = [0] * G, [0] * G, [{} for _ in range(G)], [None] * G
        self.optim_step_record, self.feat_sims, self.optimized_step = [[] for _ in range(G)], [{} for _ in range(G)], [None] * G
        self._on = (1 << G) - 1            # slots taking part now (bit mask): the frame's, narrowed by the dynamic loop
        self._live = 0                     # slots of the current frame whose motion term is live (bit mask)
        self._frames = self._hist = None   # persistent staging of the current frame's and the history frame's rows
        for g in range(G):
            self.start(g)

    def start(self, g, seed=None):
        """Put a new video into slot g: theta and teacher from the checkpoint, zero Adam moments, step and frame counts, an empty
        history, and ``rngs[g] = random.Random(seed)`` (default ``options.seed * 1000 + g``)."""
        if not isinstance(g, int) or not 0 <= g < self.G:
            raise ValueError(f'slot {g!r} is not one of the {self.G} slots')
        self.thetas[g].copy_(self.base.model.module.arena.detach())
        if self.teachers is not None:
            self.teachers[g].copy_(self.base.teacher.arena.detach())
        self.m[g].zero_()
        self.v[g].zero_()
        self.step_counts[g] = self.video_steps[g] = 0
        self.histories[g].clear()
        self.rngs[g] = random.Random(self.options.seed * 1000 + g if seed is None else seed)
        self.optim_step_record[g], self.feat_sims[g], self.optimized_step[g] = [], {}, None

    def theta(self, g):
        """View of video g's weights (flat arena layout)."""
        return self.thetas[g]

    @property
    def active(self):
        """What fused_adapt reads and narrows: None while every slot takes part, else the bit mask of the slots taking part."""
        return None if self._on == (1 << self.G) - 1 else self._on

    @active.setter
    def active(self, mask):
        self._on = (1 << self.G) - 1 if mask is None else mask

    @property
    def motion_active(self):
        """Slots taking part now whose motion term is live (bit mask)."""
        return self._on & self._live

    def _check_runtime(self):
        opt = self.base.optimizer
        if opt.grad_sync is not None or opt.pre_step_hook is not None:
            raise ValueError('a data-parallel (dist.attach) optimizer is not supported with several videos: it all-reduces one arena '
                             'across ranks')
        check_options(self.options, self.G, getattr(self, 'dynamic_loop', False))

    def _slots(self, mask):
        return [g for g in range(self.G) if (mask >> g) & 1]

    def save_hist(self, image, s2d):
        """One copy of the frame's staged rows, kept by every active slot under its own frame count."""
        frame = (image.clone(), s2d.clone())
        for g in self._slots(self._on):
            h, k = self.histories[g], self.video_steps[g]
            h[k] = frame
            h.pop(k - self.options.interval - 1, None)

    def get_hist(self):
        """The history rows of the slots whose motion term is live, each from its own frame ``interval`` frames back; the rows of
        the other slots are placeholders."""
        live = self._slots(self.motion_active)
        frames = [self.histories[g][self.video_steps[g] - self.options.interval] for g in live]
        if len(live) == self.G and all(f is frames[0] for f in frames):
            return frames[0]                                     # one pool frame holds every slot's history rows
        if self._hist is None:
            self._hist = tuple(torch.zeros_like(t) for t in frames[0])
        for g, frame in zip(live, frames):
            for dst, src in zip(self._hist, frame):
                n = src.numel() // self.G * src.element_size()
                _lib.call('dboa_copy_async', C.c_void_p(dst.data_ptr() + g * n), C.c_void_p(src.data_ptr() + g * n), n, stream())
        return self._hist

    def _teacher_masks(self, B, device):
        if not self.teacher_dropout:
            return None
        b, per = B // self.G, []
        for g in range(self.G):
            if not (self._on >> g) & 1:
                per.append(torch.ones(3, 2, b, 1024, device=device))       # placeholder rows: no draw for an idle slot
                continue
            m = self.mask_provider(g, b, device) if self.mask_provider is not None else None
            per.append(m if m is not None else (torch.rand(3, 2, b, 1024, device=device) >= 0.5).float() * 2.0)
        return torch.cat(per, 2)

    def _adam_ema(self, teacher=None, alpha=0.0):
        """Adam + EMA teacher of the active slots, each at its own step count: one sweep per run of consecutive active slots
        that share a step count (one sweep over the whole stack while every slot runs in step)."""
        o = self.options
        for g in self._slots(self._on):
            self.step_counts[g] += 1
        t = None if teacher is None else teacher.arena
        for a, b in runs(self._on, self.G, key=lambda g: self.step_counts[g]):
            _lib.call('dboa_adam_ema_scaled', ptr(self.thetas[a:b]), ptr(self.grad[a:b]), ptr(self.m[a:b]), ptr(self.v[a:b]),
                      ptr(None if t is None else t[a:b]), self.thetas[a:b].numel(), float(o.lr), float(o.beta1), float(o.beta2), 1e-8,
                      self.step_counts[a], float(alpha), 1.0, stream())

    def _stage(self, batches):
        """Copy the active slots' frames into the persistent (G b, ...) batch; the rows of idle slots keep what they held."""
        dev = self.thetas.device
        first = next(b for b in batches if b is not None)
        if self._frames is None:
            self._frames = {k: torch.zeros((self.G * first[k].shape[0],) + tuple(first[k].shape[1:]), dtype=torch.float32, device=dev)
                            for k in ('image', 'smpl_j2d')}
        for g, bt in enumerate(batches):
            if bt is None:
                continue
            for k, buf in self._frames.items():
                src = bt[k].to(dev).contiguous().float()
                rows = buf.shape[0] // self.G
                if tuple(src.shape) != (rows,) + tuple(buf.shape[1:]):
                    raise ValueError(f'slot {g}: {k} of shape {tuple(src.shape)}, expected {(rows,) + tuple(buf.shape[1:])}')
                n = src.numel() * 4
                _lib.call('dboa_copy_async', C.c_void_p(buf.data_ptr() + g * n), ptr(src), n, stream())
        return self._frames

    # ------------------------------------------------------------------ public
    def adapt(self, batches):
        """One frame of every slot whose entry is a batch (``batches[g]`` is slot g's batch dict, None: slot g sits this frame
        out): ``fused.fused_adapt`` over the active slots -- probe forward, K inner SGD steps, the upper level with teacher and
        motion terms, retrieval with exemplar mix-training, then Adam + EMA teacher.  ``fit_losses`` and ``kp2dlosses_lower`` /
        ``kp2dlosses_upper`` hold this frame's (G,) losses, NaN for idle slots; ``last_upper_loss[g]`` of an idle slot keeps its
        value.  With the dynamic loop, each slot's entries hold its own last level evaluation of the frame (its last loop
        iteration, or the upper level), ``fit_losses['feat_sim/cos_sim']`` is a (G,) host tensor, and ``last_upper_loss`` is the
        upper level's."""
        if len(batches) != self.G:
            raise ValueError(f'expected {self.G} batches, one per video, got {len(batches)}')
        on = sum(1 << g for g, b in enumerate(batches) if b is not None)
        if on == 0:
            raise ValueError('at least one slot needs a batch')
        self._check_runtime()
        o = self.options
        self._on = on
        self._live = sum(1 << g for g in self._slots(on) if self.video_steps[g] - o.interval > 0)
        batch = self._stage(batches)
        prev = self.last_upper_loss
        self.fit_losses, self.kp2dlosses_lower, self.kp2dlosses_upper = {}, [], {}
        fused_adapt(self, batch)
        if self.active is not None:
            keep = torch.tensor([bool((on >> g) & 1) for g in range(self.G)], device=prev.device)
            nan = lambda t: torch.where(keep.to(t.device), t, torch.full_like(t, float('nan')))
            self.last_upper_loss = torch.where(keep, self.last_upper_loss, prev)
            self.fit_losses = {k: nan(v) for k, v in self.fit_losses.items()}
            self.kp2dlosses_lower = [nan(v) for v in self.kp2dlosses_lower]
            self.kp2dlosses_upper = {k: nan(v) for k, v in self.kp2dlosses_upper.items()}
        if o.dynamic_boa:
            for g in self._slots(on):
                self.optim_step_record[g].append(self.optimized_step[g])
                self.feat_sims[g][self.video_steps[g]] = self.loop_feat_sims[g]
        for g in self._slots(on):
            self.video_steps[g] += 1
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
