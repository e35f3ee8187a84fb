"""Several independent videos adapted in lockstep on one GPU: ``fused.fused_adapt`` over (G, P) stacks of weight arenas, with
every network forward and backward one grouped call (``dboa_hmr_forward_active`` / ``dboa_hmr_backward_active``).  This module
holds the per-video state, hands the step a ``fused.Step`` over it and files the records the step returns per slot.

Each video keeps the reference's semantics: its own theta, Adam moments and step count, teacher, fast weights, gradient,
history ring, motion warm-up, teacher dropout masks and retrieval picks.  The G weight arenas (and the teachers', the moments',
the gradients') are one contiguous (G, P) stack; video g owns the rows [g * b, (g + 1) * b) of every per-sample batch.  The
G slots are a pool: a slot whose batch is None sits the frame out (its CTAs return at once in every grouped call), and
``start(g)`` puts a new video into slot g; ``run(videos)`` feeds a queue of videos through the slots.  With ``fused_eval``
'final' or 'all' every video gets the records and result files of the single-video driver.  DESIGN.md section 10.
"""
import ctypes as C
import itertools
import math
import numbers
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import torch

from . import _lib, hmr as hmr_mod, layout, state as state_mod
from ._lib import ptr, stream
from .fused import Step, fused_adapt, pick

EVAL_MODES = ('none', 'final', 'all')
GT_KEYS = ('pose', 'betas', 'gender')
PENDING_FRAMES = 256        # device records kept before adapt forms them on the host (one synchronisation)
# a slot's host records, one entry per slot, as a slot state holds them
SLOT_RECORDS = ('mpjpe_all', 'pampjpe_all', 'pve_all', 'mpjpe_all_lower', 'pampjpe_all_lower', 'mpjpe_statistics', 'pampjpe_statistics',
                'kp2dloss_lower_all', 'kp2dloss_upper_all', 'optim_step_record', 'feat_sims', 'optimized_step', 'last_retrieval')
# the options a slot may set for itself (start(g, hparams=...)): the learning rates, Adam's betas, the teacher rate, the loss
# weights and the dynamic loop's test.  Every other option changes which passes a step runs, or their rows, and is the pool's.
PER_VIDEO = frozenset({'lr', 'beta1', 'beta2', 'fastlr', 'alpha', 's2dloss_weight', 'shape_prior_weight', 'pose_prior_weight',
                       'teacherloss_weight', 'motionloss_weight', 'labelloss_weight', 'cos_sim_threshold', 'optim_steps'})


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


def check_hparams(options, hparams, n_videos=None):
    """Raise ValueError for per-video hyperparameters the pool of ``options`` cannot run (no device needed); return them checked.
    ``hparams``: a dict from keys of ``PER_VIDEO`` to values (one slot), or, given ``n_videos``, a list of such dicts or None, one
    per video (None for the list: none).  Returns the dict with float values (``optim_steps``: int), or the list of them ({} for
    None).  A slot's ``pose_prior_weight`` must be zero exactly when the pool's is: the prior pass runs for a non-zero weight
    only, so a mix would change the step's passes."""
    if n_videos is not None:
        if hparams is None:
            return [{} for _ in range(n_videos)]
        hparams = list(hparams)
        if len(hparams) != n_videos:
            raise ValueError(f'{len(hparams)} hparams for {n_videos} videos')
        return [{} if h is None else check_hparams(options, h) for h in hparams]
    if not isinstance(hparams, dict):
        raise ValueError(f'hparams must be a dict of options, got {type(hparams).__name__}')
    out = {}
    for k, v in hparams.items():
        if k not in PER_VIDEO:
            raise ValueError(f'{k!r} is not an option a slot may set: one of {", ".join(sorted(PER_VIDEO))}')
        if k == 'optim_steps':
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Integral) or v < 0:
                raise ValueError(f'optim_steps must be a non-negative int, got {v!r}')
            out[k] = int(v)
            continue
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Real) or not math.isfinite(v):
            raise ValueError(f'{k} must be a finite number, got {v!r}')
        v = float(v)
        if k in ('lr', 'fastlr') and v < 0:
            raise ValueError(f'{k} must not be negative, got {v!r}')
        if k in ('beta1', 'beta2') and not 0.0 <= v < 1.0:
            raise ValueError(f'{k} must lie in [0, 1), got {v!r}')
        if k == 'alpha' and not 0.0 <= v <= 1.0:
            raise ValueError(f'alpha must lie in [0, 1], got {v!r}')
        if k == 'pose_prior_weight' and (v == 0.0) != (getattr(options, 'pose_prior_weight', 0.0) == 0.0):
            raise ValueError(f'pose_prior_weight {v!r}: zero in some slots and non-zero in others would change the step '
                             f'(the pool\'s is {getattr(options, "pose_prior_weight", None)!r})')
        out[k] = v
    return out


def own_values(options, hparams):
    """The entries of ``hparams`` that differ from ``options``: what a slot runs with beyond the pool's options."""
    return {k: v for k, v in hparams.items() if v != getattr(options, k, None)}


def check_models(models, n_videos):
    """``run``'s ``models``: one checkpoint path (str or ``os.PathLike``) or None per video, None for the list: none.  Returns
    them as a list of str / None (no device or file needed)."""
    if models is None:
        return [None] * n_videos
    if isinstance(models, (str, bytes, os.PathLike)):
        raise ValueError(f'models must hold one checkpoint path or None per video, not one path for all: {models!r}')
    models = list(models)
    if len(models) != n_videos:
        raise ValueError(f'{len(models)} models for {n_videos} videos')
    return [check_model(m, f'video {i}') for i, m in enumerate(models)]


def check_model(model, who):
    """A checkpoint path (str or ``os.PathLike``) as str, or None.  The str is interned, as ``state.unplain`` interns the
    strings of a checkpoint's records: the summaries of a resumed run then pickle byte-identically to an uninterrupted run's."""
    if model is None:
        return None
    path = os.fspath(model) if isinstance(model, os.PathLike) else model
    if not isinstance(path, str) or not path:
        raise ValueError(f'{who}: model must be a checkpoint path or None, got {model!r}')
    return sys.intern(path)


def video_names(videos, names, default):
    """The directory names of ``videos`` for ``run``: ``names`` as strings (None: ``default``), one per video."""
    names = list(default) if names is None else [str(x) for x in names]
    if len(names) != len(videos):
        raise ValueError(f'{len(names)} names for {len(videos)} videos')
    return names


def slot_records(frame, G, prev_upper_loss):
    """A pool's (``fit_losses``, ``kp2dlosses_lower``, ``last_upper_loss``) of the ``fused.Frame`` ``frame``: NaN for the slots
    outside the frame, except in ``last_upper_loss``, where they keep ``prev_upper_loss``."""
    on = frame.mask
    return ({k: pick(on, G, v) for k, v in frame.fit.items()}, [pick(on, G, v) for v in frame.lower],
            pick(on, G, frame.upper_loss, prev_upper_loss))


def _items_from(video, k):
    """An iterator over ``video``'s items from item k on: by index for a video with ``len`` and indexing (nothing before k is
    read), with ``itertools.islice`` for any other iterable."""
    if k and hasattr(video, '__len__') and hasattr(video, '__getitem__'):
        return (video[t] for t in range(k, len(video)))
    return itertools.islice(iter(video), k, None)


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
    test, ``frame`` counted from the slot's ``start``), and ``optimized_step`` ((G,), None for slots that sat the frame out).

    ``start(g, model=path)`` starts slot g from a checkpoint of its own instead (``slot_model(g)``; DESIGN.md section 10,
    "Per-slot checkpoints"): the pool keeps one device arena per distinct model its slots hold.

    ``fused_eval`` ('none', 'final' or 'all', as ``Adaptor``'s): evaluate every advancing video against its ground truth
    (batches then need pose, betas and gender).  Each evaluation stays on the device; ``records(g)`` forms slot g's host
    records (``mpjpe_all[g]``, ``pampjpe_all[g]``, ``pve_all[g]``, with 'all' also ``mpjpe_all_lower[g]`` /
    ``pampjpe_all_lower[g]`` and ``mpjpe_statistics[g]`` / ``pampjpe_statistics[g]``, and the run's 2D keypoint losses), and
    ``start(g)`` forms them before it resets the slot.  ``run(videos, exppath=None, names=None)`` adapts a list of videos
    through the slots and returns one summary per video.

    ``motion_lead`` (class attribute, 0 here): slot g's motion term is live while ``video_steps[g] + motion_lead - interval > 0``
    and reads its frame ``video_steps[g] + motion_lead - interval``; ``feat_sims[g]`` and the upper-level 2D losses are keyed by
    ``video_steps[g] + motion_lead``.  The webcam client advances its step before the levels (1: webcam.MultiWebcamAdaptor)."""

    kp_range = (25, 24)
    motion_lead = 0

    def __init__(self, options, n_videos, dynamic_loop=False):
        check_options(options, n_videos, dynamic_loop)
        self.dynamic_loop = bool(dynamic_loop)
        self.G = G = int(n_videos)
        self.options = o = options
        self.base = base = self._make_base(options)    # checkpoint, SMPL, prior, exemplar bank; never adapted, so it keeps the checkpoint
        model = base.model.module
        self.thetas = torch.empty(G, model.arena.numel(), device=model.arena.device)
        self.buffers = model._buffers
        self.teachers = torch.empty_like(self.thetas) if o.use_meanteacher else None
        self.m, self.v, self.grad = torch.empty_like(self.thetas), torch.empty_like(self.thetas), torch.zeros_like(self.thetas)
        self.fused_eval = 'none'
        self.global_step = 0
        self.mask_provider = None
        self.last_upper_loss = torch.zeros(G, device=self.thetas.device)
        self.last_retrieval = [None] * G
        self.teacher_dropout = bool(getattr(o, 'teacher_dropout', 1))
        self.step_counts, self.video_steps, self.histories, self.rngs = [0] * G, [0] * G, [{} for _ in range(G)], [None] * G
        self.optim_step_record, self.feat_sims, self.optimized_step = [[] for _ in range(G)], [{} for _ in range(G)], [None] * G
        self._frames = self._hist = None   # persistent staging of the current frame's and the history frame's rows
        self._pending = []                 # device records of the frames adapted since the records were last formed
        self._gt = None                    # the current frame's ground-truth meshes (gender-selected, neutral)
        self.slot_video = [None] * G       # run(): index of the video slot g holds
        self.mpjpe_all, self.pampjpe_all, self.pve_all = [[] for _ in range(G)], [[] for _ in range(G)], [[] for _ in range(G)]
        self.mpjpe_all_lower, self.pampjpe_all_lower = [None] * G, [None] * G
        self.mpjpe_statistics, self.pampjpe_statistics = [{} for _ in range(G)], [{} for _ in range(G)]
        self.kp2dloss_lower_all, self.kp2dloss_upper_all = [[] for _ in range(G)], [{} for _ in range(G)]
        self._writer, self._pinned = state_mod.Writer(), state_mod.Pinned()     # checkpoints written in the background (save)
        self.hparams = [{} for _ in range(G)]   # per slot: the PER_VIDEO values it runs with where they differ from options
        self.slot_models = [None] * G           # per slot: (path, digest) of its own checkpoint, None: options.model_file
        self._store = {}                        # digest -> (P,) device arena of a model some slot holds
        self._pool_digest = None                # digest of the pool's checkpoint (computed when a slot is given a model)
        self._step = Step(o, G, self.thetas, self.grad, self.buffers, base.smpl_neutral, base.gmm_f, teacher=self.teachers,
                          teacher_buffers=self.buffers, teacher_masks=self._teacher_masks, kp_range=self.kp_range,
                          motion_lead=self.motion_lead, bank=base.bank if o.retrieval else None, rngs=self.rngs,
                          save_hist=self._save_hist, get_hist=self._get_hist, adam=self._adam_ema, evaluate=self._evaluate)
        for g in range(G):
            self.start(g)

    def _make_base(self, options):
        """The single-video adaptor whose checkpoint, SMPL models, prior and exemplar bank the pool shares."""
        from .adaptor import Adaptor
        return Adaptor(options)

    def start(self, g, seed=None, state=None, hparams=None, model=None):
        """Put a new video into slot g: theta and teacher from the checkpoint, zero Adam moments, step and frame counts, an empty
        history, empty records, and ``rngs[g] = random.Random(seed)`` (default ``options.seed * 1000 + g``).  The records of
        the frames adapted so far are formed on the host first (one synchronisation, if any are pending).

        ``hparams``: a dict from keys of ``PER_VIDEO`` to values (``check_hparams``): slot g runs with ``options`` plus these
        values until its next ``start`` (``slot_options(g)``).

        ``model``: a checkpoint path (``layout.read_checkpoint``; what ``export_model`` writes): slot g starts from it instead of
        ``options.model_file`` and keeps it until its next ``start`` (``slot_model(g)``; the webcam pool's ``reload`` and base
        outputs go back to it).  A checkpoint with the pool's weights is the pool's checkpoint.

        ``state``: a video state written by ``save_slot`` (its path, or the dict ``state.read_video`` returned) of a pool with
        the same G and compatible options, from any slot: slot g continues that video instead -- theta, teacher, moments, step
        count, ``video_steps[g]``, history ring, ``rngs[g]``, records and its hparams (``hparams`` that contradict them raise).
        A state of a slot on a checkpoint of its own needs that model again: ``model`` (default the path the state records)
        must hold the same weights.  Everything is checked before any device work (ValueError)."""
        self._start(g, seed, state, hparams, model)

    def _start(self, g, seed=None, state=None, hparams=None, model=None, expect=None):
        """``start``; ``expect``: the digest the checkpoint ``model`` had when ``run`` read it."""
        self._check_slot(g)
        model = check_model(model, f'slot {g}')
        if state is not None and not isinstance(state, dict):
            state = state_mod.read_video(state, self.options, 'slot', self.G, own=PER_VIDEO)
        hp = None if hparams is None else own_values(self.options, check_hparams(self.options, hparams))
        if state is not None:
            saved = own_values(self.options, check_hparams(self.options, state_mod.saved_options(state, PER_VIDEO)))
            if hp is not None and hp != saved:
                raise ValueError(f'slot {g}: hparams {hparams!r} contradict the state\'s {saved!r}')
            hp = saved
        want = None if state is None else state_mod.saved_model(state)
        if model is None and want is not None:
            model = want[0]                                  # the checkpoint the state was adapted from, where it was
        own = self._read_model(model, expect) if model is not None else None
        if state is not None and own is not None and own[1] != (want[1] if want is not None else self._pool_model_digest()):
            raise ValueError(f'slot {g}: model {model!r} (digest {own[1][:12]}...) is not the checkpoint the state was adapted from: '
                             + (f'{want[0]!r} (digest {want[1][:12]}...)' if want is not None else 'the pool\'s'))
        self._set_model(g, own)
        self._reset_weights(g)
        self._form_records()
        self.video_steps[g] = 0
        self.histories[g].clear()
        self.rngs[g] = random.Random(self.options.seed * 1000 + g if seed is None else seed)
        self.optim_step_record[g], self.feat_sims[g], self.optimized_step[g] = [], {}, None
        n = self.options.inner_step
        self.mpjpe_all[g], self.pampjpe_all[g], self.pve_all[g] = [], [], []
        self.mpjpe_all_lower[g], self.pampjpe_all_lower[g] = [[] for _ in range(n)], [[] for _ in range(n)]
        self.mpjpe_statistics[g], self.pampjpe_statistics[g] = {}, {}
        self.kp2dloss_lower_all[g], self.kp2dloss_upper_all[g] = [], {}
        self.hparams[g] = hp or {}
        if state is not None:
            self._restore_slot(g, state)

    def slot_model(self, g):
        """(path, digest) of slot g's own checkpoint (``start(g, model=...)``), or None when it is on the pool's."""
        self._check_slot(g)
        return self.slot_models[g]

    def _pool_model_digest(self):
        if self._pool_digest is None:
            self._pool_digest = layout.arena_digest(self.base.model.module.arena, self.buffers)
        return self._pool_digest

    def _read_model(self, path, expect=None):
        """(path, digest, host arena) of the checkpoint at ``path``, read and checked on the host; the arena is None when the
        checkpoint holds the pool's weights.  ``expect``: the digest the file must still have (ValueError otherwise)."""
        arena, digest = layout.read_checkpoint(path, self.buffers)
        if expect is not None and digest != expect:
            raise ValueError(f'{path}: the checkpoint changed since it was read (digest {digest[:12]}..., was {expect[:12]}...)')
        return path, digest, None if digest == self._pool_model_digest() else arena

    def _set_model(self, g, own):
        """Slot g on the model ``own`` (``_read_model``'s triple; None or a None arena: the pool's checkpoint): its arena
        uploaded unless a slot already holds it, and the arenas no slot refers to any more freed."""
        self.slot_models[g] = None if own is None or own[2] is None else (own[0], own[1])
        held = {m[1] for m in self.slot_models if m is not None}
        for d in [d for d in self._store if d not in held]:
            del self._store[d]
        if self.slot_models[g] is not None and own[1] not in self._store:
            self._store[own[1]] = own[2].to(self.thetas.device)
        self._slot_model_set(g)

    def _slot_model_set(self, g):
        """Called once slot g's model is set (the webcam pool keeps its base-output arenas here)."""

    def _model_arena(self, g):
        """The device arena slot g starts from: its own model's, or the pool's checkpoint."""
        m = self.slot_models[g]
        return self.base.model.module.arena if m is None else self._store[m[1]]

    def slot_options(self, g):
        """Slot g's effective options: the pool's ``options`` with the slot's hparams."""
        self._check_slot(g)
        return SimpleNamespace(**{**vars(self.options), **self.hparams[g]})

    def _check_slot(self, g):
        if not isinstance(g, int) or not 0 <= g < self.G:
            raise ValueError(f'slot {g!r} is not one of the {self.G} slots')

    def _reset_weights(self, g):
        """Slot g's theta and teacher back to its checkpoint (``slot_model(g)``, else the pool's) and a fresh Adam (zero
        moments, step count 0)."""
        self._check_slot(g)
        own = self.slot_models[g] is not None
        self.thetas[g].copy_(self._model_arena(g).detach())
        if self.teachers is not None:
            self.teachers[g].copy_(self._model_arena(g) if own else self.base.teacher.arena.detach())
        self.m[g].zero_()
        self.v[g].zero_()
        self.step_counts[g] = 0

    def theta(self, g):
        """View of video g's weights (flat arena layout)."""
        return self.thetas[g]

    def _check_runtime(self):
        opt = self.base.optimizer
        if opt.grad_sync is not None or opt.pre_step_hook is not None:
            raise ValueError('a data-parallel (dist.attach) optimizer is not supported with several videos: it all-reduces one arena '
                             'across ranks')
        check_options(self.options, self.G, getattr(self, 'dynamic_loop', False))

    def _slots(self, mask):
        return [g for g in range(self.G) if (mask >> g) & 1]

    def _save_hist(self, image, s2d, on):
        """One copy of the frame's staged rows, kept by every slot in ``on`` under its own frame count."""
        frame = (image.clone(), s2d.clone())
        for g in self._slots(on):
            h, k = self.histories[g], self.video_steps[g]
            h[k] = frame
            h.pop(k - self.options.interval - 1, None)

    def _get_hist(self, live):
        """The history rows of the slots in ``live``, each from its own frame ``interval - motion_lead`` frames back; the rows
        of the other slots are placeholders."""
        live = self._slots(live)
        frames = [self.histories[g][self.video_steps[g] + self.motion_lead - self.options.interval] for g in live]
        if len(live) == self.G and all(f is frames[0] for f in frames):
            return frames[0]                                     # one pool frame holds every slot's history rows
        if self._hist is None:
            self._hist = tuple(torch.zeros_like(t) for t in frames[0])
        for g, frame in zip(live, frames):
            for dst, src in zip(self._hist, frame):
                n = src.numel() // self.G * src.element_size()
                _lib.call('dboa_copy_async', C.c_void_p(dst.data_ptr() + g * n), C.c_void_p(src.data_ptr() + g * n), n, stream())
        return self._hist

    def _teacher_masks(self, B, device, on):
        if not self.teacher_dropout:
            return None
        b, per = B // self.G, []
        for g in range(self.G):
            if not (on >> g) & 1:
                per.append(torch.ones(3, 2, b, 1024, device=device))       # placeholder rows: no draw for an idle slot
                continue
            m = self.mask_provider(g, b, device) if self.mask_provider is not None else None
            per.append(m if m is not None else (torch.rand(3, 2, b, 1024, device=device) >= 0.5).float() * 2.0)
        return torch.cat(per, 2)

    def _adam_ema(self, on, teacher=None, alpha=0.0):
        """Adam + EMA into the teacher stack ``teacher`` of the slots in ``on``: one ``dboa_adam_ema_groups`` sweep in which each
        slot takes its own step count and the lr, betas and alpha of its options in the step (``alpha`` is not read)."""
        vo = self._step.video_options
        rows, one = (C.c_float * (self.G * _lib.ADAM_SCALARS))(), (C.c_float * _lib.ADAM_SCALARS)()
        for g in self._slots(on):
            self.step_counts[g] += 1
            q = vo[g]
            _lib.call('dboa_adam_scalars', one, float(q.lr), float(q.beta1), float(q.beta2), 1e-8, self.step_counts[g], float(q.alpha), 1.0)
            rows[g * _lib.ADAM_SCALARS:(g + 1) * _lib.ADAM_SCALARS] = one[:]
        _lib.call('dboa_adam_ema_groups', ptr(self.thetas), ptr(self.grad), ptr(self.m), ptr(self.v), ptr(teacher),
                  self.thetas.shape[1], rows, self.G, on, stream())

    def _stage(self, batches):
        """Copy the active slots' frames into the persistent (G b, ...) batch; the rows of idle slots keep what they held."""
        dev = self.thetas.device
        first = next(b for b in batches if b is not None)
        keys = ('image', 'smpl_j2d') + (GT_KEYS if self.fused_eval != 'none' else ())
        if self._frames is None:
            self._frames = {}
        for k in keys:
            if k not in self._frames:
                self._frames[k] = torch.zeros((self.G * first[k].shape[0],) + tuple(first[k].shape[1:]), dtype=torch.float32, device=dev)
        for g, bt in enumerate(batches):
            if bt is None:
                continue
            for k in keys:
                buf = self._frames[k]
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
        if self.fused_eval not in EVAL_MODES:
            raise ValueError(f'fused_eval must be one of {EVAL_MODES}, got {self.fused_eval!r}')
        if self.fused_eval != 'none':
            for g in self._slots(on):
                missing = [k for k in GT_KEYS if k not in batches[g]]
                if missing:
                    raise ValueError(f'slot {g}: fused_eval={self.fused_eval!r} needs the ground truth {", ".join(missing)} in the batch')
        self._check_runtime()
        self._adapt_staged(on, self._stage(batches))

    def _adapt_staged(self, on, batch):
        """The frame of ``adapt`` on rows already staged in ``batch`` (the persistent staging), for the slots in ``on`` (bit
        mask): a subclass that writes the staged rows itself runs the same step through here."""
        o, G = self.options, self.G
        self._evals, self._gt = [], None
        self._step.eval_mode = self.fused_eval
        self._step.video_options = [self.slot_options(g) if self.hparams[g] else o for g in range(G)]
        f = fused_adapt(self._step, batch, on, self.video_steps)
        self._gt = None
        self.fit_losses, self.kp2dlosses_lower, self.last_upper_loss = slot_records(f, G, self.last_upper_loss)
        self.kp2dlosses_upper = {self.global_step: self.fit_losses['ul/s2dloss']} if 'ul/s2dloss' in self.fit_losses else {}
        if f.picks is not None:
            self.last_retrieval = [p if p is not None else q for p, q in zip(f.picks, self.last_retrieval)]
        if o.dynamic_boa:
            self.optimized_step = [f.steps.get(g) for g in range(G)]
            for g in self._slots(on):
                self.optim_step_record[g].append(f.steps[g])
                self.feat_sims[g][self.video_steps[g] + self.motion_lead] = f.sims[g]
        self._pending.append((on, {g: self.video_steps[g] for g in self._slots(on)}, self.fused_eval == 'all', self._evals,
                              list(self.kp2dlosses_lower), self.kp2dlosses_upper.get(self.global_step)))
        if len(self._pending) >= PENDING_FRAMES:
            self._form_records()
        for g in self._slots(on):
            self.video_steps[g] += 1
        self.global_step += 1

    def _evaluate(self, batch, arena, on, inner):
        """One evaluation of ``arena`` (theta, or the fast weights of inner step ``inner``) for the slots in ``on``: a grouped
        forward, SMPL decode and ``dboa_eval_metrics_active`` (ground truth from the frame's first), kept on the device."""
        with torch.no_grad():
            rot, shape, _, _, _ = hmr_mod.raw_forward(arena, self.buffers, batch['image'], groups=self.G, active=on)
            pred = self.base.decode_smpl_params(rot, shape)['vts']
            if self._gt is None:                             # as Adaptor.inference, for every staged row
                self._gt = self.base._gt_meshes(batch)
            out = self.base.eval_metrics(pred, *self._gt, groups=self.G, active=on)
        self._evals.append((out, on, inner))

    def _form_records(self):
        """File the device records of every frame adapted since the last call into the slots' host records: one copy to the
        host (and so one synchronisation) for all of them."""
        if not self._pending:
            return
        G, b = self.G, self._frames['image'].shape[0] // self.G
        flat = [t.reshape(-1) for _, _, _, evals, low, up in self._pending for t in [e[0] for e in evals] + low + ([up] if up is not None else [])]
        host = torch.cat(flat).cpu().numpy() if flat else None
        off = 0

        def take(n):
            nonlocal off
            off += n
            return host[off - n:off]
        for on, frames, steps, evals, low, up in self._pending:
            evals = [(take(out.numel()).reshape(-1, 3), mask, step) for out, mask, step in evals]
            low = [take(G) for _ in low]
            up = take(G) if up is not None else None
            for g, t in frames.items():
                # Adaptor.inference's values: metrics[:, 0] * 1000, metrics[:, 1] * 1000, float(metrics[:, 2].mean()) * 1000
                mine = [(np.ascontiguousarray(m[g * b:(g + 1) * b]), step) for m, mask, step in evals if (mask >> g) & 1]
                thetas = [(m[:, 0] * 1000, m[:, 1] * 1000, float(m[:, 2].mean()) * 1000) for m, step in mine if step is None]
                for m, step in mine:
                    if step is not None:
                        self.mpjpe_all_lower[g][step].append(m[:, 0] * 1000)
                        self.pampjpe_all_lower[g][step].append(m[:, 1] * 1000)
                if thetas:
                    self.mpjpe_all[g].append(thetas[-1][0])
                    self.pampjpe_all[g].append(thetas[-1][1])
                    self.pve_all[g].append(thetas[-1][2])
                if steps:                                    # 'all': every theta evaluation of the frame
                    self.mpjpe_statistics[g][t] = [x[0] for x in thetas]
                    self.pampjpe_statistics[g][t] = [x[1] for x in thetas]
                self.kp2dloss_lower_all[g] += [float(v[g]) for v in low]
                if up is not None:
                    self.kp2dloss_upper_all[g][t + self.motion_lead] = float(up[g])
        self._pending = []

    def records(self, g):
        """Slot g's records since its ``start`` as host values, under the names ``adaptor.write_records`` takes (the values of
        ``Adaptor.excute``'s records for that video), and ``frames``."""
        self._form_records()
        n = self.video_steps[g]
        return dict(frames=n, mpjpe=list(self.mpjpe_all[g]), pampjpe=list(self.pampjpe_all[g]), pve=list(self.pve_all[g]),
                    mpjpe_all_lower=[list(x) for x in self.mpjpe_all_lower[g]], pampjpe_all_lower=[list(x) for x in self.pampjpe_all_lower[g]],
                    mpjpe_statistics=[self.mpjpe_statistics[g].get(t, []) for t in range(n)],
                    pampjpe_statistics=[self.pampjpe_statistics[g].get(t, []) for t in range(n)],
                    feat_sims=dict(self.feat_sims[g]), optim_step_record=list(self.optim_step_record[g]),
                    kp2dlosses_lower=list(self.kp2dloss_lower_all[g]), kp2dlosses_upper=dict(self.kp2dloss_upper_all[g]))

    def run(self, videos, exppath=None, names=None, checkpoint=None, every=0, hparams=None, models=None):
        """Adapt every video of ``videos`` (a list of iterables of batch dicts with batch size 1: a ``DataLoader`` over a
        sequence, a ``SyntheticStream``) through the G slots.  Slots are filled in order and refilled from the queue as soon as
        their video ends; video i starts with ``start(g, seed=options.seed * 1000 + i)``, so its seed follows the video, and
        ``slot_video[g]`` is the index of the video slot g holds (for a ``mask_provider``).  Returns one summary per video, in
        order: name, frames, and the mean MPJPE, PA-MPJPE and PVE of its frames (``res.txt``'s; NaN without evaluation).  With
        ``exppath``, each video's eight result files go to ``exppath/<name>/`` when it finishes (``names``: default the
        video's index).

        ``checkpoint``: a directory of pool checkpoints (``save``), written every ``every`` ticks and once more at the end.  When it
        holds a complete checkpoint the run resumes from it: the finished videos' summaries are returned as recorded (their
        result files are left alone), every video in flight continues in its slot from its own frame, and the queue goes on
        from there.  The summaries and result files are those of a run that was never interrupted.

        ``hparams``: one dict of ``start``'s hparams, or None, per video; the dict follows the video into its slot, as its seed
        does.  A resumed run must be given the hparams of the run it continues.

        ``models``: one checkpoint path, or None for ``options.model_file``, per video; the model follows the video into its slot
        (``start(g, model=...)``) and each summary names it (``model``).  Every distinct path is read and checked once before the
        first tick; a resumed run must be given checkpoints with the weights of the run it continues."""
        from .adaptor import write_records
        videos = list(videos)
        hparams = check_hparams(self.options, hparams, len(videos))
        models = None if models is None else check_models(models, len(videos))
        names = video_names(videos, names, default=[str(i) for i in range(len(videos))])
        mean = lambda v: float(np.mean(v)) if len(v) else float('nan')

        def finish(i, g):
            if g is None:                                    # an empty video
                out = dict(name=names[i], frames=0, mpjpe=float('nan'), pampjpe=float('nan'), pve=float('nan'))
            else:
                rec = self.records(g)
                if exppath is not None:
                    d = os.path.join(exppath, names[i])
                    os.makedirs(d, exist_ok=True)
                    write_records(d, rec['frames'] - 1, rec)
                out = dict(name=names[i], frames=rec['frames'], mpjpe=mean(rec['mpjpe']), pampjpe=mean(rec['pampjpe']), pve=mean(rec['pve']))
            if models is not None:
                out['model'] = models[i]
            return out
        return self._queue(videos, self.adapt, finish, checkpoint=checkpoint, every=every, hparams=hparams, models=models)

    def _queue(self, videos, tick, finish, checkpoint=None, every=0, items_from=None, barrier=None, hparams=None, models=None):
        """``run``'s queue: the slots are filled in order and refilled as soon as their video ends; video i starts with
        ``start(g, seed=options.seed * 1000 + i)`` and ``slot_video[g] = i``.  ``tick(items)`` advances the pool by one frame,
        ``items[g]`` being slot g's next item of its video (None: an idle slot); ``finish(i, g)`` returns video i's summary once
        it ended in slot g (g None: video i was empty), before the slot is refilled.  Returns the summaries in order.

        ``checkpoint`` / ``every``: ``run``'s.  ``items_from(i, k)``: an iterator over video i's items from item k on (default
        ``items_from``); ``barrier()``: futures of files a checkpoint taken now covers (``save``); ``hparams``: video i's
        ``start`` hparams (checked; None: none); ``models``: video i's checkpoint path (None: the pool's), each distinct one read and
        checked here, before the first tick, with only its digest kept."""
        n = len(videos)
        hparams = check_hparams(self.options, hparams, n)
        own = [own_values(self.options, h) for h in hparams]
        paths = check_models(models, n)
        digests = {p: self._read_model(p)[1] for p in dict.fromkeys(p for p in paths if p is not None)}
        # per video: (path, digest) of its own checkpoint, None on the pool's (a checkpoint with the pool's weights is the pool's)
        own_models = [None if p is None or digests[p] == self._pool_model_digest() else (p, digests[p]) for p in paths]
        queue, its, nxt, out = list(range(n)), [None] * self.G, [None] * self.G, [None] * n
        items_from = items_from or (lambda i, k: _items_from(videos[i], k))

        def check_run(run):                                  # before the checkpoint's slots are restored
            if run is None:
                return
            if run['videos'] != n:
                raise ValueError(f'{checkpoint}: the checkpoint is of a queue of {run["videos"]} videos, not {n}')
            if run.get('hparams', [{}] * n) != own:
                raise ValueError(f'{checkpoint}: the checkpoint is of a run with hparams {run.get("hparams")!r}, not {own!r}')
            saved = [None if m is None else m[1] for m in run.get('models', [None] * n)]
            if saved != [None if m is None else m[1] for m in own_models]:
                raise ValueError(f'{checkpoint}: the checkpoint is of a run with models {run.get("models")!r}, whose weights differ from '
                                 f'{[None if m is None else m[0] for m in own_models]!r}')
        run = self.load(checkpoint, check_run, models=paths) if checkpoint is not None else None
        if run is not None:
            queue, out = list(run['queue']), list(run['out'])
            for g in range(self.G):
                if self.slot_video[g] is not None:
                    its[g] = items_from(self.slot_video[g], self.video_steps[g])
                    nxt[g] = next(its[g], None)

        def save():
            rec = dict(videos=n, queue=queue, out=out, hparams=own)
            if any(m is not None for m in own_models):
                rec['models'] = own_models
            self.save(checkpoint, run=rec, barrier=barrier, wait=False)

        def fill(g):
            self.slot_video[g] = None
            while queue:
                i = queue.pop(0)
                its[g] = items_from(i, 0)
                nxt[g] = next(its[g], None)
                if nxt[g] is None:
                    out[i] = finish(i, None)
                    continue
                self._start(g, seed=self.options.seed * 1000 + i, hparams=hparams[i], model=paths[i], expect=digests.get(paths[i]))
                self.slot_video[g] = i
                return

        try:
            if run is None:
                for g in range(self.G):
                    fill(g)
            while any(i is not None for i in self.slot_video):
                tick([nxt[g] if self.slot_video[g] is not None else None for g in range(self.G)])
                for g in range(self.G):
                    if self.slot_video[g] is None:
                        continue
                    nxt[g] = next(its[g], None)
                    if nxt[g] is None:
                        out[self.slot_video[g]] = finish(self.slot_video[g], g)
                        fill(g)
                if checkpoint is not None and every and self.global_step % every == 0:
                    save()
            if checkpoint is not None:
                save()
        finally:
            self._writer.wait()                              # no checkpoint is still being written when run returns or raises
        return out

    # ------------------------------------------------------------------ saved state (state.py, DESIGN.md section 11)
    def _slot_state(self, g, copy):
        """Slot g's video state, its arenas brought to the host by ``copy(key, device tensor)`` and its history frames by
        ``state.host_copy``, both on the current stream (the records must have been formed)."""
        G, small = self.G, state_mod.host_copy
        hist = []
        for k, (image, kp) in sorted(self.histories[g].items()):
            b = image.shape[0] // G
            hist.append((k, small(image[g * b:(g + 1) * b]), small(kp[g * b:(g + 1) * b])))
        records = {name: getattr(self, name)[g] for name in SLOT_RECORDS}
        records['last_upper_loss'] = small(self.last_upper_loss[g:g + 1])
        return state_mod.video_state(self.slot_options(g), 'slot', G, copy(('theta', g), self.thetas[g]),
                                     None if self.teachers is None else copy(('teacher', g), self.teachers[g]),
                                     copy(('m', g), self.m[g]), copy(('v', g), self.v[g]), self.step_counts[g], self.video_steps[g], hist,
                                     dict(random=self.rngs[g].getstate()), records, model=self.slot_models[g])

    def _restore_slot(self, g, st):
        G, dev = self.G, self.thetas.device
        self.thetas[g].copy_(st['theta'])
        if self.teachers is not None:
            self.teachers[g].copy_(st['teacher'])
        self.m[g].copy_(st['m'])
        self.v[g].copy_(st['v'])
        self.step_counts[g], self.video_steps[g] = st['step_count'], st['frames']
        h = self.histories[g]
        for k, rows in st['history'].items():                 # the pool's history frames hold every slot's rows: slot g's filled
            full = []
            for t in rows:
                b = t.shape[0]
                f = torch.zeros((G * b,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
                f[g * b:(g + 1) * b].copy_(t)
                full.append(f)
            h[k] = tuple(full)
        self.rngs[g].setstate(st['rng']['random'])
        rec = st['records']
        for name in SLOT_RECORDS:
            getattr(self, name)[g] = rec[name]
        self.last_upper_loss[g] = rec['last_upper_loss'].to(dev)[0]

    def save_slot(self, g, path):
        """Write slot g's video as a video state to ``path`` (durably and atomically): what ``start(g', state=path)`` continues
        from in any slot of a pool with the same G.  Between frames: the copies wait for the slot's last write."""
        self._check_slot(g)
        self._check_runtime()
        self._form_records()
        st = self._slot_state(g, lambda key, t: state_mod.host_copy(t))
        torch.cuda.current_stream().synchronize()
        state_mod.write(path, st)

    def save(self, root, slots=None, run=None, barrier=None, wait=True):
        """Write a pool checkpoint under the directory ``root``: one video state per slot of ``slots`` (default: every slot that
        holds a video of ``run``, or all G slots of a pool driven by ``adapt``), a pool file (``global_step``, torch's CUDA
        generator state -- the teacher masks of every slot are drawn from it in slot order --, ``slot_video`` and ``run``) and
        the manifest, written last.  The arenas come to the host through pinned buffers on the current stream and the files are
        written on a background thread, after the futures of ``barrier()`` (files the checkpoint covers) are done; a new save
        waits for the previous one.  ``wait``: return once the checkpoint is durable."""
        self._check_runtime()
        self._writer.wait()                                  # the pinned buffers are free again
        if slots is None:
            slots = [g for g in range(self.G) if self.slot_video[g] is not None] if run is not None else list(range(self.G))
        self._form_records()
        states = {g: self._slot_state(g, self._pinned.copy) for g in slots}
        pool = state_mod.header(state_mod.POOL, self.options)
        pool.update(G=self.G, global_step=self.global_step, cuda_rng=torch.cuda.get_rng_state(self.thetas.device),
                    slot_video=list(self.slot_video), run=state_mod.plain(run))
        done = torch.cuda.Event()
        done.record()
        waits = list(barrier()) if barrier is not None else []

        def job():
            for f in waits:
                f.result()
            path = state_mod.new_checkpoint(root)
            for g, st in states.items():
                state_mod.write(os.path.join(path, f'slot{g}.pt'), st)
            state_mod.write(os.path.join(path, 'pool.pt'), pool)
            state_mod.commit(root, path, {g: f'slot{g}.pt' for g in states})
        self._writer.submit(job, done)
        if wait:
            self._writer.wait()

    def load(self, root, check_run=None, models=None):
        """Continue from the newest complete checkpoint ``save`` wrote under ``root``: every file is checked first (ValueError),
        then the saved slots are restored with ``start(g, state=...)``, the others marked empty in ``slot_video``, and
        ``global_step`` and torch's CUDA generator set.  Returns the checkpoint's ``run`` (None without a checkpoint).
        ``check_run(run)``: raises for a ``run`` the caller cannot continue, after the files are checked and before anything is
        restored.  ``models``: per video of the run, the checkpoint path its slot is restored with (None: the path its state
        records, if any)."""
        found = state_mod.latest(root)
        if found is None:
            return None
        path, man = found
        self._check_runtime()
        pool = state_mod.read(os.path.join(path, man['pool']), state_mod.POOL, self.options)
        if pool.get('G') != self.G:
            raise ValueError(f'{path}: a checkpoint of a {pool.get("G")}-slot pool cannot be loaded into {self.G} slots')
        states = {g: state_mod.read_video(os.path.join(path, f), self.options, 'slot', self.G, own=PER_VIDEO) for g, f in man['slots'].items()}
        run = state_mod.unplain(pool['run'])
        if check_run is not None:
            check_run(run)
        for g in range(self.G):
            self.slot_video[g] = pool['slot_video'][g] if g in states else None
            if g in states:
                self.start(g, state=states[g], model=None if models is None else models[self.slot_video[g]])
        self.global_step = pool['global_step']
        torch.cuda.set_rng_state(pool['cuda_rng'], self.thetas.device)
        torch.cuda.synchronize(self.thetas.device)
        return run

    def export_model(self, g, path):
        """Write video g's adapted weights as a checkpoint in the reference's format (``Adaptor.export_model``)."""
        self._check_slot(g)
        state_mod.write(path, {'model': layout.state_dict(self.thetas[g], self.buffers, prefix='module.')})

    def predict(self, images, active=None):
        """Every video's prediction for its rows of ``images`` with its current weights: a list of G dicts with rotmat, betas,
        cam, joints (49) and vertices.  ``active`` (bit mask; None: every slot): one grouped forward of only those slots
        (``dboa_hmr_forward_active``), then the SMPL decode; the entries of the other slots are None."""
        rot, shape, cam, out = self._outputs(images, active)
        b = rot.shape[0] // self.G
        s = [slice(g * b, (g + 1) * b) for g in range(self.G)]
        return [dict(rotmat=rot[q], betas=shape[q], cam=cam[q], joints=out['s3d'][q], vertices=out['vts'][q])
                if active is None or (active >> g) & 1 else None for g, q in enumerate(s)]

    def _outputs(self, images, active=None):
        """``predict``'s grouped forward and SMPL decode as whole (G b, ...) tensors: rotmat, betas, cam and the decode's dict
        (rows of slots outside ``active`` hold no prediction)."""
        with torch.no_grad():
            image = images.to(self.thetas.device).contiguous().float()
            rot, shape, cam, _, _ = hmr_mod.raw_forward(self.thetas, self.buffers, image, groups=self.G, active=active)
            return rot, shape, cam, self.base.decode_smpl_params(rot, shape)
