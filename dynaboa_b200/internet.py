"""Several Internet videos adapted side by side on one GPU: ``MultiInternetAdaptor``, a ``multivideo.MultiVideoAdaptor`` pool
with the Internet client's semantics per video (``adaptor.InternetAdaptor``, reference dynaboa_internet.py), fed from the
folder layout of ``run_on_internet.sh`` (``datasets.internet_videos``) and writing each video's ``Pred_<t>.pt`` files and, with
``save_res=1``, its rendered frames.

Per tick the active slots' frames are uploaded once, cropped in one grouped call and their keypoints transformed in another
(``dataprocess.crop_groups`` / ``j2d_processing_groups``); the bilevel step (and the dynamic loop) runs over the pool; one
masked output forward gives every mesh; each output tensor comes to the host in one copy; with ``save_res`` every mesh is drawn
over its device frame in one grouped overlay call.  Decoding the frames and writing the files run on a small thread pool, so
the host I/O of one tick overlaps the device work of the next.  DESIGN.md section 10, "Internet videos".
"""
import os
from concurrent.futures import Future, ThreadPoolExecutor

import numpy as np
import torch

from . import constants, dataprocess, render as render_mod
from .adaptor import InternetAdaptor
from .multivideo import MultiVideoAdaptor, check_hparams, check_models, check_options as pool_check_options, video_names

COLOR = (205, 129, 98)       # the mesh colour of BaseAdaptor.save_results, in the order it is given there
PRED_KEYS = ('verts', 'cam', 'rotmat', 'beta')


def check_options(options, n_videos, dynamic_loop=False):
    """Raise ValueError for what the Internet pool does not support (no device needed): every ``multivideo.check_options``
    rejection, and a ``batch_size`` other than 1 (a slot adapts one frame of its video per tick)."""
    if int(getattr(options, 'batch_size', 1)) != 1:
        raise ValueError(f'batch_size={options.batch_size}: the Internet pool adapts one frame per video and tick (batch_size=1)')
    pool_check_options(options, n_videos, dynamic_loop)


def output_paths(exppath, name, t):
    """Where frame t of video ``name`` goes: (``exppath/name/result/Pred_t.pt``, ``exppath/name/image/Pred_t.png``)."""
    d = os.path.join(exppath, name)
    return os.path.join(d, 'result', f'Pred_{t}.pt'), os.path.join(d, 'image', f'Pred_{t}.png')


def decode(path):
    """The frame at ``path`` as ``Internet_dataset`` reads it: cv2's BGR decode, reversed to a contiguous RGB uint8 array."""
    import cv2
    bgr = cv2.imread(path)
    if bgr is None:
        raise FileNotFoundError(path)
    return np.ascontiguousarray(bgr[:, :, ::-1])


class FileWriter:
    """The files of the pool: ``pred`` dumps the reference's joblib dict, ``image`` writes a BGR uint8 array with cv2."""

    def pred(self, path, arrays):
        import joblib
        joblib.dump(arrays, path)

    def image(self, path, bgr):
        import cv2
        if not cv2.imwrite(path, bgr):
            raise OSError(f'cv2.imwrite could not write {path}')


class _PoolBase(InternetAdaptor):
    """The pool's ``InternetAdaptor``: checkpoint, SMPL models, prior and exemplar bank; no data loader of its own."""

    def set_dataloader(self):
        self.dataloader, self.imgdir = [], None


class MultiInternetAdaptor(MultiVideoAdaptor):
    """``MultiInternetAdaptor(options, n_videos, dynamic_loop=False)``: G slots, each adapting one Internet video as its own
    ``InternetAdaptor.excute(fused=True)`` does: the 24 ground-truth-layout joints in the 2D and motion terms, the teacher's
    dropout live (the reference never puts the teacher in eval mode), retrieval and mix-training as the options say, no
    evaluation (there is no ground truth).  ``options`` is the Internet driver's namespace; ``dynamic_loop=True`` accepts
    ``dynamic_boa=1`` (``run_on_internet.sh``'s flags) and runs the re-adaptation loop per video.

    ``run(videos, exppath, names=None)`` adapts ``datasets.internet_videos(root)`` through the slots and writes each video's
    files under ``exppath/<name>/``: ``result/Pred_<t>.pt`` (unless ``cache_results=0``) and, with ``save_res=1``,
    ``image/Pred_<t>.png``, the mesh drawn over the frame bit for bit as ``BaseAdaptor.save_results`` draws it.  The pool
    writes no ``demo.obj``: G videos would overwrite one file in the working directory.

    ``input_side(frames)`` is a tick's input side alone and ``tick(frames)`` a whole tick without the thread pool.  ``writer``
    (a ``FileWriter``) writes the files; ``workers`` threads decode and write during ``run``."""
    kp_range = (25, 24)
    motion_lead = 0
    workers = 4

    def __init__(self, options, n_videos, dynamic_loop=False):
        check_options(options, n_videos, dynamic_loop)
        super().__init__(options, n_videos, dynamic_loop)
        self.fused_eval = 'none'
        self.writer = FileWriter()

    def _make_base(self, options):
        return _PoolBase(options)

    def _rows(self):
        """The pool's persistent staging rows, (G, 3, 224, 224) images and the (G, 49, 3) keypoint block."""
        if self._frames is None:
            dev = self.thetas.device
            self._frames = {'image': torch.zeros(self.G, 3, 224, 224, device=dev), 'smpl_j2d': torch.zeros(self.G, 49, 3, device=dev)}
        return self._frames

    # ------------------------------------------------------------------ one tick
    def input_side(self, frames):
        """Stage one frame per active slot.  ``frames[g]``: None (slot g sits the tick out), or ``(video, t)`` / ``(video, t,
        image)`` with ``video`` an ``InternetVideo`` and ``image`` frame t as ``decode`` returns it (or a Future of it; None:
        decoded here).  Each frame is uploaded once; one grouped crop and one grouped keypoint call (49 rows) write the active
        slots' staging rows, each bit-identical to ``Internet_dataset``'s item of that frame.  Returns (the active bit mask,
        per slot the device RGB frame and the (1, 3) bbox, None for idle slots)."""
        G = self.G
        if len(frames) != G:
            raise ValueError(f'expected {G} frames, one per slot, got {len(frames)}')
        on, recs = 0, [None] * G
        for g, f in enumerate(frames):
            if f is None:
                continue
            if not isinstance(f, (tuple, list)) or len(f) not in (2, 3):
                raise ValueError(f'slot {g}: expected (video, t) or (video, t, image), got {type(f).__name__}')
            video, t = f[0], f[1]
            recs[g] = video.frame(t) + (f[2] if len(f) == 3 else None,)
            on |= 1 << g
        if on == 0:
            return 0, [None] * G, [None] * G
        self._check_runtime()
        dev, rows = self.thetas.device, self._rows()
        imgs, centers, scales, bboxes, kps = [None] * G, [None] * G, [None] * G, [None] * G, np.zeros((G, 49, 3), np.float32)
        for g, r in enumerate(recs):
            if r is None:
                continue
            path, centers[g], scales[g], kps[g], bboxes[g], image = r
            if image is None:
                image = decode(path)
            elif isinstance(image, Future):
                image = image.result()
            imgs[g] = self._upload(image)
        dataprocess.crop_groups(imgs, centers, scales, rows['image'], on)
        dataprocess.j2d_processing_groups(torch.from_numpy(kps).to(dev), centers, scales, rows['smpl_j2d'], on)
        return on, imgs, bboxes

    def _upload(self, image):
        """A decoded frame on the device (kept there for the tick's drawing)."""
        return torch.from_numpy(image).to(self.thetas.device)

    def tick(self, frames, exppath=None, names=None):
        """One tick of the active slots (``input_side``'s ``frames``): the input side, the bilevel step, one masked output
        forward and, with ``save_res``, one grouped overlay.  Returns the tick's files as (slot, path of Pred_<t>.pt, its dict of
        host arrays, path of the PNG or None, the BGR image or None) without writing them; paths are None without ``exppath``
        (``names[g]``: slot g's directory, default its video's name)."""
        on, imgs, bboxes = self.input_side(frames)
        if on == 0:
            return []
        return self._output_side(on, frames, imgs, bboxes, exppath, names)

    def _output_side(self, on, frames, imgs, bboxes, exppath, names):
        G = self.G
        self._adapt_staged(on, self._frames)
        rot, shape, cam, out = self._outputs(self._frames['image'], on)
        verts = out['vts']
        cam_t = torch.stack([cam[:, 1], cam[:, 2], 2 * 5000. / (constants.IMG_RES * cam[:, 0] + 1e-9)], dim=-1)   # InternetAdaptor.inference
        slots = self._slots(on)
        drawn = {}
        if getattr(self.options, 'save_res', 0):
            # save_results draws the RGB-ordered colour into cv2's BGR frame; the shading is per channel, so drawing the RGB
            # device frame in the reversed colour and returning BGR (render_groups) gives the same bytes
            res = render_mod.render_groups([verts[g:g + 1] for g in slots], [cam[g:g + 1] for g in slots], [imgs[g] for g in slots],
                                           [bboxes[g] for g in slots], [COLOR[::-1]] * len(slots))
            flat = torch.cat([r.reshape(-1) for r in res]).cpu().numpy()                     # one copy for every frame
            off = 0
            for g, r in zip(slots, res):
                drawn[g] = flat[off:off + r.numel()].reshape(tuple(r.shape))
                off += r.numel()
        host = [t.cpu().numpy() for t in (verts, cam_t, rot, shape)]                          # one copy per output tensor
        files = []
        for g in slots:
            video, t = frames[g][0], frames[g][1]
            name = video.name if names is None else names[g]
            pred_path, png_path = output_paths(exppath, name, t) if exppath is not None else (None, None)
            files.append((g, pred_path, {k: np.array(h[g:g + 1]) for k, h in zip(PRED_KEYS, host)}, png_path if g in drawn else None,
                          drawn.get(g)))
        return files

    def write(self, files):
        """Write a tick's ``files`` (``tick``'s list) with ``writer``: each Pred dict unless ``cache_results=0``, each PNG."""
        cache = getattr(self.options, 'cache_results', 1)
        for _, pred_path, pred, png_path, image in files:
            if cache:
                self.writer.pred(pred_path, pred)
            if png_path is not None:
                self.writer.image(png_path, image)

    # ------------------------------------------------------------------ videos
    def run(self, videos, exppath, names=None, checkpoint=None, every=0, hparams=None, models=None):
        """Adapt every video of ``videos`` (``datasets.InternetVideo``s) through the G slots with ``MultiVideoAdaptor.run``'s
        queue (slots filled in order and refilled as soon as their video ends; video i starts with seed ``options.seed * 1000 +
        i``) and write each video's files under ``exppath/<name>/`` (``names``: default the videos' names).  The frames of
        the next tick are decoded, and the files written, on ``workers`` threads; a tick enqueues its device work before it
        waits for the previous tick's files, and the files of one video are written in frame order.  Returns once every file
        is on disk (an exception of a writer is raised here) with one summary per video: name, frames and, with the dynamic
        loop, ``optim_step_record`` (the trip count of each frame).

        ``checkpoint`` / ``every``: ``MultiVideoAdaptor.run``'s pool checkpoints.  A checkpoint is complete only once every
        ``Pred_<t>`` file of the frames it covers is written; a resumed video is advanced to its frame by index, without
        decoding the frames before it.  ``hparams``: ``MultiVideoAdaptor.run``'s, one dict (or None) per video.  ``models``:
        ``MultiVideoAdaptor.run``'s, one checkpoint path (or None) per video, read and checked before the first tick; each summary
        then names its video's (``model``)."""
        videos = list(videos)
        for i, v in enumerate(videos):
            if not callable(getattr(v, 'frame', None)) or not hasattr(v, '__len__') or not hasattr(v, 'name'):
                raise ValueError(f'video {i} is a {type(v).__name__}, expected an InternetVideo (datasets.internet_videos)')
        names = video_names(videos, names, default=[v.name for v in videos])
        hparams = check_hparams(self.options, hparams, len(videos))
        models = None if models is None else check_models(models, len(videos))
        if len(set(names)) != len(names):
            raise ValueError(f'two videos would write to one directory: names {names}')
        dirs = ('result',) if getattr(self.options, 'cache_results', 1) else ()
        dirs += ('image',) if getattr(self.options, 'save_res', 0) else ()
        for name in names:
            for sub in dirs:
                os.makedirs(os.path.join(exppath, name, sub), exist_ok=True)
        with ThreadPoolExecutor(max_workers=self.workers, thread_name_prefix='dboa-io') as io:
            pending = []                                     # the previous tick's writes

            def frames_of(i, k=0):
                """Video i's frames from frame k on as (video, t, Future of the decoded frame), frame t + 1 submitted when frame t
                is taken."""
                v = videos[i]
                if len(v) <= k:
                    return
                nxt = io.submit(decode, v.frame(k)[0])
                for t in range(k, len(v)):
                    cur, nxt = nxt, (io.submit(decode, v.frame(t + 1)[0]) if t + 1 < len(v) else None)
                    yield (v, t, cur)

            def tick(items):
                on, imgs, bboxes = self.input_side(items)
                files = self._output_side(on, items, imgs, bboxes, exppath, [None if x is None else names[self.slot_video[g]]
                                                                            for g, x in enumerate(items)])
                for f in pending:
                    f.result()
                pending[:] = [io.submit(self.write, [f]) for f in files]          # one job per video: its frames stay in order

            def finish(i, g):
                out = dict(name=names[i], frames=0 if g is None else self.video_steps[g])
                if getattr(self.options, 'dynamic_boa', 0):
                    out['optim_step_record'] = [] if g is None else list(self.optim_step_record[g])
                if models is not None:
                    out['model'] = models[i]
                return out

            out = self._queue([_Frames(frames_of, i) for i in range(len(videos))], tick, finish, checkpoint=checkpoint, every=every,
                              items_from=frames_of, barrier=lambda: pending, hparams=hparams, models=models)
            for f in pending:
                f.result()
        return out


class _Frames:
    """Iterable over video i's frames (``make(i)``), started anew by every ``iter``."""

    def __init__(self, make, i):
        self.make, self.i = make, i

    def __iter__(self):
        return self.make(self.i)
