"""Saved adaptation state: the one module that knows the file layout (DESIGN.md section 11).

A *video state* is one ``torch.save`` file holding everything one video's adaptation continues from: its theta, teacher, Adam
moments and step count, its frame count, its history ring, its retrieval generator and its records, and, for a pool slot
started from a checkpoint of its own, that checkpoint's path and digest (``model``).  ``Adaptor.save_state`` /
``load_state`` and the pools' ``save_slot`` / ``start(g, state=...)`` write and read them through ``video_state`` /
``read_video``.  A *pool checkpoint* is a directory of numbered checkpoints, each one video state per occupied slot, one pool
file and a manifest written last: ``latest`` returns the newest checkpoint whose manifest is complete.

Files hold tensors and plain containers only and are read with ``torch.load(weights_only=True)``: a state file is input from
outside the program.  Every check -- format, version, arena size, parameter table, options -- runs on the host before any
device work and raises ``ValueError``.  Writes go to a temporary file in the same directory, are fsynced and renamed over the
target, so a crash mid-write leaves the previous file as it was.
"""
import os
import re
import shutil
import sys
import tempfile
import threading

import numpy as np
import torch

from . import layout

VIDEO, POOL, MANIFEST = 'dynaboa_b200.video_state', 'dynaboa_b200.pool_state', 'dynaboa_b200.pool_manifest'
VERSION = 1
MANIFEST_FILE = 'MANIFEST.pt'
# Options that may differ between the run that saved a state and the run that loads it: where results and logs go, the
# checkpoint a fresh slot starts from and the length of the synthetic stand-in stream.  None of them enters the arithmetic of
# a frame; every other option does, and a difference in it is refused.
MAY_DIFFER = frozenset({'expdir', 'expname', 'tensorboard', 'save_res', 'cache_results', 'model_file', 'synthetic_frames'})
VIDEO_FIELDS = ('kind', 'G', 'theta', 'teacher', 'm', 'v', 'step_count', 'frames', 'history', 'rng', 'records')


# ------------------------------------------------------------------ plain containers
def plain(x):
    """``x`` as tensors and plain containers: host copies of tensors, numpy arrays and scalars tagged so that ``unplain`` gives
    them back with their dtype and shape (a record file written from them is byte-identical).  A host tensor that is the whole
    of its own storage (a ``Pinned`` buffer still being filled) is kept as it is, not copied."""
    if isinstance(x, torch.Tensor):
        t = x.detach()
        if t.is_cuda:
            return t.cpu()
        whole = t.is_contiguous() and t.storage_offset() == 0 and t.untyped_storage().nbytes() == t.numel() * t.element_size()
        return t if whole else t.clone()
    if isinstance(x, np.ndarray):
        return {'__ndarray__': torch.from_numpy(np.ascontiguousarray(x).copy())}
    if isinstance(x, np.generic):
        return {'__npscalar__': torch.from_numpy(np.asarray(x).reshape(1).copy())}
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, list):
        return [plain(v) for v in x]
    if isinstance(x, tuple):
        return tuple(plain(v) for v in x)
    if x is None or isinstance(x, (bool, int, float, str)):
        return x
    raise TypeError(f'a state holds tensors and plain containers, not {type(x).__name__}')


def unplain(x):
    if isinstance(x, dict):
        if set(x) == {'__ndarray__'}:
            return x['__ndarray__'].numpy()
        if set(x) == {'__npscalar__'}:
            return x['__npscalar__'].numpy()[0]
        return {unplain(k): unplain(v) for k, v in x.items()}
    if isinstance(x, list):
        return [unplain(v) for v in x]
    if isinstance(x, tuple):
        return tuple(unplain(v) for v in x)
    if isinstance(x, str):
        return sys.intern(x)        # as the literals of the records ('cos', the summaries' keys): pickles of them stay byte-identical
    return x


def options_dict(options):
    """The options namespace as a plain dict (a value that is no plain container is kept as its repr)."""
    out = {}
    for k, v in sorted(vars(options).items()):
        try:
            out[k] = plain(v)
        except TypeError:
            out[k] = repr(v)
    return out


def check_options(saved, options, own=frozenset()):
    """Raise ValueError naming every option that differs between ``saved`` (a state's options) and ``options`` outside
    ``MAY_DIFFER`` and ``own``."""
    now, missing = options_dict(options), object()
    bad = sorted(k for k in set(saved) | set(now) if k not in MAY_DIFFER and k not in own and not _same(saved.get(k, missing), now.get(k, missing)))
    if bad:
        detail = ', '.join(f'{k} (saved {saved.get(k, "unset")!r}, now {now.get(k, "unset")!r})' for k in bad)
        raise ValueError(f'the state was saved with different options: {detail}')


def _same(a, b):
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        return isinstance(a, torch.Tensor) and isinstance(b, torch.Tensor) and torch.equal(a, b)
    return type(a) is type(b) and a == b


# ------------------------------------------------------------------ files
def header(fmt, options):
    """The fields every file starts with: format, version, arena size P, parameter-table digest and the options."""
    return {'format': fmt, 'version': VERSION, 'P': int(layout.arena_layout().floats), 'layout': layout.digest(),
            'options': options_dict(options)}


def write(path, obj):
    """``torch.save(obj)`` to ``path`` durably and atomically: a temporary file in the same directory, fsync, ``os.replace``,
    fsync of the directory."""
    d = os.path.dirname(os.path.abspath(path))
    os.makedirs(d, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix='.' + os.path.basename(path) + '.', suffix='.tmp', dir=d)
    try:
        with os.fdopen(fd, 'wb') as f:
            torch.save(obj, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    _fsync_dir(d)


def _fsync_dir(d):
    fd = os.open(d, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def read(path, fmt, options=None, own=frozenset()):
    """Load ``path`` with ``weights_only=True`` and check it: format ``fmt``, this version, this library's arena size and
    parameter table and, given ``options``, options that differ only in ``MAY_DIFFER`` and ``own``.  ValueError otherwise."""
    try:
        obj = torch.load(path, map_location='cpu', weights_only=True)
    except FileNotFoundError:
        raise
    except Exception as e:                                     # truncated, not a torch file, or a pickled object
        raise ValueError(f'{path}: not a readable state file (truncated or malformed): {type(e).__name__}: {e}') from None
    if not isinstance(obj, dict) or obj.get('format') != fmt:
        got = obj.get('format') if isinstance(obj, dict) else type(obj).__name__
        raise ValueError(f'{path}: unknown format {got!r}, expected {fmt!r}')
    if obj.get('version') != VERSION:
        raise ValueError(f'{path}: format version {obj.get("version")!r}, this library reads version {VERSION}')
    P = int(layout.arena_layout().floats)
    if obj.get('P') != P:
        raise ValueError(f'{path}: saved for an arena of {obj.get("P")!r} floats, this library has {P}')
    if obj.get('layout') != layout.digest():
        raise ValueError(f'{path}: saved with a different parameter table (layout digest {str(obj.get("layout"))[:12]}...)')
    if not isinstance(obj.get('options'), dict):
        raise ValueError(f'{path}: malformed state: no options')
    if options is not None:
        check_options(obj['options'], options, own)
    return obj


# ------------------------------------------------------------------ video states
def video_state(options, kind, G, theta, teacher, m, v, step_count, frames, history, rng, records, model=None):
    """A video state as a dict of host tensors and plain containers.  ``kind``: 'adaptor' (``Adaptor``) or 'slot' (a pool slot
    of a G-slot pool); ``theta``, ``teacher`` (None without one), ``m``, ``v``: (P,) arenas; ``frames``: the video's frame count;
    ``history``: {frame: (image, keypoints)}; ``rng``: generator states; ``records``: the adaptor's records of the video.
    ``model``: (path, digest) of the slot's own checkpoint, kept as the ``model`` entry; None (no entry): the pool's."""
    out = header(VIDEO, options)
    out.update(kind=kind, G=int(G), theta=plain(theta), teacher=None if teacher is None else plain(teacher), m=plain(m), v=plain(v),
               step_count=int(step_count), frames=int(frames), history={int(k): (plain(a), plain(b)) for k, a, b in history},
               rng=plain(rng), records=plain(records))
    if model is not None:
        out['model'] = {'path': str(model[0]), 'digest': str(model[1])}
    return out


def read_video(path, options, kind, G=1, own=frozenset()):
    """A video state checked against ``options``, its ``kind`` and pool width ``G``, with its records unpacked.  ``own``: options
    the video may carry values of its own in (a pool slot's per-video hyperparameters; its state holds the slot's effective
    options), which ``saved_options`` returns."""
    st = read(path, VIDEO, options, own)
    missing = [k for k in VIDEO_FIELDS if k not in st]
    if missing:
        raise ValueError(f'{path}: malformed video state: no {", ".join(missing)}')
    if st['kind'] != kind:
        raise ValueError(f'{path}: a state of kind {st["kind"]!r} cannot be loaded as {kind!r}')
    if st['G'] != G:
        raise ValueError(f'{path}: saved from a pool of {st["G"]} slots, this pool has {G}')
    P = st['P']
    for k in ('theta', 'teacher', 'm', 'v'):
        t = st[k]
        if t is None and k == 'teacher':
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.shape != (P,):
            raise ValueError(f'{path}: malformed video state: {k} is not a ({P},) float32 tensor')
    if (st['teacher'] is None) != (not getattr(options, 'use_meanteacher', 0)):
        raise ValueError(f'{path}: malformed video state: teacher does not match use_meanteacher')
    saved_model(st, path)
    st['records'] = unplain(st['records'])
    st['rng'] = unplain(st['rng'])
    return st


def saved_model(st, where='state'):
    """(path, digest) of the slot's own checkpoint a video state ``st`` records, or None for the pool's (no ``model`` entry, or
    None).  ValueError for a malformed entry (``where`` names the file)."""
    m = st.get('model')
    if m is None:
        return None
    if (not isinstance(m, dict) or set(m) != {'path', 'digest'} or not isinstance(m['path'], str) or not isinstance(m['digest'], str)
            or not re.fullmatch(r'[0-9a-f]{64}', m['digest'])):
        raise ValueError(f'{where}: malformed video state: the model entry must be None or {{path, digest}} with a sha256 digest, '
                         f'got {m!r}')
    return m['path'], m['digest']


def saved_options(st, keys):
    """The values of the options ``keys`` a video state ``st`` was saved with (those it holds)."""
    return {k: unplain(st['options'][k]) for k in keys if k in st['options']}


# ------------------------------------------------------------------ background writes
class Writer:
    """Writes files on a background thread, one job at a time: ``submit`` waits for the previous job (and raises its error)
    before it starts the next; ``wait`` waits for the last one.  A job waits for ``event`` (the device-to-host copies of its
    tensors) first, so the caller's stream is never blocked by the file write."""

    def __init__(self):
        self._thread, self._error = None, None

    def submit(self, job, event=None):
        self.wait()

        def run():
            try:
                if event is not None:
                    event.synchronize()
                job()
            except BaseException as e:                         # raised by the next wait()
                self._error = e
        self._thread = threading.Thread(target=run, name='dboa-state-writer', daemon=True)
        self._thread.start()

    def wait(self):
        if self._thread is not None:
            self._thread.join()
            self._thread = None
        if self._error is not None:
            e, self._error = self._error, None
            raise e


class Pinned:
    """Reusable page-locked host buffers by key, for device-to-host copies that do not block the caller's stream."""

    def __init__(self):
        self._bufs = {}

    def copy(self, key, t):
        """A pinned host copy of the device tensor ``t`` enqueued on the current stream (valid once the stream reaches it)."""
        buf = self._bufs.get(key)
        if buf is None or buf.shape != t.shape or buf.dtype != t.dtype:
            buf = self._bufs[key] = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        buf.copy_(t, non_blocking=True)
        return buf


def host_copy(t):
    """A fresh pinned host copy of a small device tensor, enqueued on the current stream."""
    out = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    out.copy_(t, non_blocking=True)
    return out


# ------------------------------------------------------------------ pool checkpoints
def _numbered(root):
    if not os.path.isdir(root):
        return []
    return sorted((int(n), os.path.join(root, n)) for n in os.listdir(root) if re.fullmatch(r'\d{8}', n))


def new_checkpoint(root):
    """A new, empty checkpoint directory under ``root``, numbered after the last one."""
    n = _numbered(root)
    path = os.path.join(root, f'{(n[-1][0] + 1) if n else 0:08d}')
    if os.path.exists(path):
        shutil.rmtree(path)
    os.makedirs(path)
    return path


def commit(root, path, slots):
    """Complete the checkpoint ``path``: its manifest (``slots``: {slot: file name}) written last, atomically; then every
    older checkpoint under ``root`` is removed."""
    write(os.path.join(path, MANIFEST_FILE), {'format': MANIFEST, 'version': VERSION, 'pool': 'pool.pt',
                                              'slots': {int(g): str(f) for g, f in slots.items()}})
    for _, old in _numbered(root):
        if old != path and int(os.path.basename(old)) < int(os.path.basename(path)):
            shutil.rmtree(old, ignore_errors=True)


def latest(root):
    """(path, manifest) of the newest checkpoint under ``root`` with a readable manifest, or None.  A checkpoint without one
    (a write cut short) is ignored in favour of the one before it."""
    for _, path in reversed(_numbered(root)):
        try:
            man = torch.load(os.path.join(path, MANIFEST_FILE), map_location='cpu', weights_only=True)
        except Exception:
            continue
        if isinstance(man, dict) and man.get('format') == MANIFEST and man.get('version') == VERSION:
            return path, man
    return None
