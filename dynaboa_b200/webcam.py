"""Third client of the adaptation path: frames + OpenPose detections instead of a dataset (the role of reference
dynaboa_webcam.py ``Adaptor`` :36-337; the capture / OpenPose / viewer loop :373-447 stays with the caller).

What differs from the benchmark client, and where it lands here:

* the 2D re-projection and motion terms compare the 25 OpenPose joints ``pred_s2d[:, :25]`` with the detections
  (reference :236,246,262 and :161-181) instead of the 24 ground-truth joints 25..48: ``kp_range = (0, 25)`` selects the
  joints inside the loss kernels (``dboa_loss_args.kp_first / kp_count``, ``dboa_loss_motion_joints``); the detections
  travel in rows 0..24 of the usual (B, 49, 3) keypoint block;
* the lower level has the frame losses only, the upper level adds motion and mean-teacher terms (:228-271);
* the teacher runs in eval mode (:69) -- no dropout masks; no exemplar retrieval;
* ``save_hist`` advances ``global_step`` itself (:105-108), so the motion term looks ``interval - 1`` frames back and
  starts one frame earlier than in the benchmark driver;
* the input side (``dataprocess`` :185-206: bounding box from the detections, confidence threshold 0.3, crop / resize /
  normalise) runs on the GPU through dynaboa_b200.dataprocess.

``online_adaptation(frame, detections)`` returns the reference's result dictionary (``vts``, ``cam``, ``bbox`` and, with
``test_basemodel``, ``vts_base`` / ``cam_base``).

``MultiWebcamAdaptor`` serves several live streams from one GPU: a ``multivideo.MultiVideoAdaptor`` pool with the webcam
client's semantics per stream, whose input side crops every stream's frame in one grouped call (DESIGN.md section 10,
"Webcam streams").
"""
from types import SimpleNamespace

import numpy as np
import torch

from . import config, dataprocess, hmr as hmr_mod, render as render_mod
from .adaptor import Adaptor
from .hmr import hmr
from .multivideo import MultiVideoAdaptor


def webcam_options(o):
    """The webcam script's flag namespace (reference dynaboa_webcam.py:339-371) completed with the fields ``BaseAdaptor``
    reads, set to what the webcam ``Adaptor`` hard-codes."""
    d = dict(vars(o))
    d.update(use_frame_losses_lower=1, use_frame_losses_upper=1, use_temporal_losses_lower=0, use_temporal_losses_upper=1,
             retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0, sample_num=1, inner_step=1, batch_size=1,
             teacher_dropout=0, dataset='webcam')
    for k, v in dict(labelloss_weight=0.0, tensorboard=0, expdir='exps', expname='webcam', use_meanteacher=0, use_motion=0,
                     dynamic_boa=0, cos_sim_threshold=3.1e-4, optim_steps=7, interval=5, alpha=0.1, test_basemodel=0,
                     motionloss_weight=0.8, teacherloss_weight=0.1, seed=22).items():
        d.setdefault(k, v)
    return SimpleNamespace(**d)


class WebcamAdaptor(Adaptor):
    kp_range = (0, 25)
    motion_lead = 1                                         # save_hist advances global_step before the levels
    step_graph = False                                      # a replayed frame could not advance it

    def __init__(self, options):
        super().__init__(webcam_options(options))
        self.fused_eval = 'none'
        self.basemodel = None
        if self.options.test_basemodel:                     # frozen copy of the base model, shown side by side (:71-74)
            ck = torch.load(self.options.model_file, map_location='cpu', weights_only=False)
            self.basemodel = hmr(config.SMPL_MEAN_PARAMS).to(self.device)
            self.basemodel.load_state_dict({k.replace('module.', ''): v for k, v in ck['model'].items()}, strict=True)
            self.basemodel.eval()

    def set_dataloader(self):
        self.dataloader, self.imgdir = [], None

    def save_hist(self, image, s2d):
        super().save_hist(image, s2d)
        self.global_step += 1                               # reference :105-108

    def reload(self):
        """Key ``r`` of the demo (:184-195): back to the base checkpoint, fresh Adam state."""
        self.set_model_optim()
        self.model.eval()
        if self.options.use_meanteacher:
            self.set_teacher()
        self.history = {}

    def dataprocess(self, image, gtkp2d, scaleFactor=1.0):
        """reference :197-218.  ``image``: (H, W, 3) RGB uint8 / float32 frame (numpy or CUDA tensor); ``gtkp2d``: (25, 3) OpenPose
        detections (x, y, confidence) in frame pixels.  Returns the (1, 3, 224, 224) network input, the (1, 49, 3) keypoint
        block (rows 0..24 filled) and the (1, 3) bounding box."""
        center, scale, bbox, kp = _box(gtkp2d, scaleFactor)
        img = image if torch.is_tensor(image) else torch.from_numpy(np.ascontiguousarray(image))
        img = img.to(self.device, non_blocking=True)
        net_in = dataprocess.crop(img, center, scale)
        kp25 = dataprocess.j2d_processing(torch.from_numpy(kp).float().to(self.device), center, scale)
        kp49 = torch.zeros(1, 49, 3, dtype=torch.float32, device=self.device)
        kp49[0, :25] = kp25
        return net_in.unsqueeze(0), kp49, bbox

    def online_adaptation(self, ori_image, gtkp2d):
        """reference :221-337: one adaptation step on the frame, then the adapted model's mesh."""
        image, kp, bbox = self.dataprocess(ori_image, np.asarray(gtkp2d)[0], scaleFactor=1.2)
        return self.adapt_processed(image, kp, bbox)

    def adapt_processed(self, image, kp, bbox=None):
        """The same on an already cropped frame and a (B, 49, 3) keypoint block (rows 0..24 = OpenPose joints in [-1, 1])."""
        self.fit_losses = {}
        self.model.eval()
        self.adapt({'image': image, 'smpl_j2d': kp})        # fused path: bilevel step (+ dynamic loop), no evaluation
        with torch.no_grad():
            rot, shape, cam = self.model(image)
            res = {'vts': self.decode_smpl_params(rot, shape)['vts'], 'cam': cam, 'bbox': bbox}
            if self.basemodel is not None:
                rot_b, shape_b, cam_b = self.basemodel(image)
                res.update(vts_base=self.decode_smpl_params(rot_b, shape_b)['vts'], cam_base=cam_b)
        return res


def _box(det, scaleFactor=1.2):
    """``WebcamAdaptor.dataprocess``'s host side for one stream: (center, scale, bbox (1, 3), keypoints with the 0.3 confidence
    threshold applied in double)."""
    kp = np.array(det, dtype=np.float64, copy=True)
    x0, y0, x1, y1 = kp[:, 0].min(), kp[:, 1].min(), kp[:, 0].max(), kp[:, 1].max()
    center = [(x1 + x0) / 2, (y1 + y0) / 2]
    scale = scaleFactor * max(x1 - x0, y1 - y0) / 200
    kp[:, 2] = kp[:, 2] > 0.3
    return center, scale, np.stack([center[0], center[1], scale * 200])[None, :], kp


def _frame_ok(f):
    dt = f.dtype if torch.is_tensor(f) else np.dtype(f.dtype)
    ok = (torch.uint8, torch.float32) if torch.is_tensor(f) else (np.dtype(np.uint8), np.dtype(np.float32))
    return f.ndim == 3 and f.shape[2] == 3 and dt in ok


class MultiWebcamAdaptor(MultiVideoAdaptor):
    """``MultiWebcamAdaptor(options, n_streams, dynamic_loop=False)``: G live streams (cameras, or people's recorded clips)
    adapted in lockstep, each with the semantics of its own ``WebcamAdaptor``: the 25 OpenPose joints in the 2D and motion
    terms (``kp_range``), the teacher in eval mode, no retrieval, and the motion term ``interval - 1`` frames back, live one
    frame earlier (``motion_lead = 1``).  ``options`` is the webcam script's namespace (completed by ``webcam_options``);
    ``dynamic_loop=True`` accepts ``dynamic_boa=1`` and runs the re-adaptation loop per stream.

    ``online_adaptation(frames, detections)`` advances every stream that has a frame and detections by one tick: the boxes on
    the host, one grouped crop and one grouped keypoint call into the pool's staging rows, the bilevel step, one masked output
    forward.  ``adapt_processed`` does the same on already cropped rows.  ``render(frames, results)`` draws the tick's meshes
    in one grouped overlay call.  ``reload(g)`` is the demo's key ``r`` for stream g; ``start(g)`` puts a new camera into slot
    g (``start(g, model=path)``: from a checkpoint of its own, which ``reload`` and the base outputs then use).  Per slot, ``video_steps[g]`` counts the stream's frames."""
    colors = ((205, 129, 98), (100, 100, 200))             # adapted and base mesh (reference dynaboa_webcam.py:410,416)
    kp_range = (0, 25)
    motion_lead = 1

    def __init__(self, options, n_streams, dynamic_loop=False):
        self._base_stack = None              # (G, P) base arenas of the streams, while one holds a model of its own (test_basemodel)
        super().__init__(webcam_options(options), n_streams, dynamic_loop)
        self.fused_eval = 'none'

    def _make_base(self, options):
        return WebcamAdaptor(SimpleNamespace(**dict(vars(options), test_basemodel=0)))     # base outputs: its own checkpoint arena

    def _rows(self):
        """The pool's persistent staging rows, (G, 3, 224, 224) images and the (G, 49, 3) keypoint block."""
        if self._frames is None:
            dev = self.thetas.device
            self._frames = {'image': torch.zeros(self.G, 3, 224, 224, device=dev), 'smpl_j2d': torch.zeros(self.G, 49, 3, device=dev)}
        return self._frames

    def _slot_model_set(self, g):
        """With ``test_basemodel``: the (G, P) stack of base arenas the tick's base outputs read while any stream holds a model
        of its own, allocated when the first one does (every row filled) and freed when none does; otherwise row g is filled."""
        if not self.options.test_basemodel:
            return
        if all(m is None for m in self.slot_models):
            self._base_stack = None
        elif self._base_stack is None:
            self._base_stack = torch.stack([self._model_arena(h) for h in range(self.G)])
        else:
            self._base_stack[g].copy_(self._model_arena(g))

    def reload(self, g):
        """Key ``r`` of the demo for stream g (reference dynaboa_webcam.py:184-194): theta and teacher back to the stream's
        checkpoint (``slot_model(g)``, else the pool's) and a fresh Adam (zero moments, step count 0).  The stream's history, frame count and hparams (``start(g, hparams=...)``) are
        kept, so its motion term stays as it was; the other streams are left alone."""
        self._reset_weights(g)

    def online_adaptation(self, frames, detections):
        """One tick of every stream (reference :221-337 per stream).  ``frames[g]``: an (H, W, 3) RGB uint8 / float32 frame (numpy
        or CUDA tensor), ``detections[g]``: its (1, 25, 3) or (25, 3) OpenPose detections in frame pixels; a None frame or None
        detections (no person found) leaves stream g as it was.  Returns per stream the reference's result dictionary, or None
        for a stream that sat the tick out (all None when no stream has a frame)."""
        on, bboxes = self.input_side(frames, detections)
        return self._tick(on, bboxes) if on else [None] * self.G

    def input_side(self, frames, detections):
        """The input side of ``online_adaptation`` alone: the boxes on the host (``WebcamAdaptor.dataprocess``'s arithmetic),
        then one grouped crop and one grouped keypoint call into the staging rows of the streams that have a frame and
        detections.  Returns (their bit mask, per stream the (1, 3) bbox or None)."""
        G = self.G
        if len(frames) != G or len(detections) != G:
            raise ValueError(f'expected {G} frames and {G} detections, one per stream, got {len(frames)} and {len(detections)}')
        on, centers, scales, bboxes, kps = 0, [None] * G, [None] * G, [None] * G, np.zeros((G, 25, 3))
        for g, (f, d) in enumerate(zip(frames, detections)):
            if f is None or d is None:
                continue
            det = np.asarray(d.cpu() if torch.is_tensor(d) else d)
            if det.shape == (1, 25, 3):
                det = det[0]
            if det.shape != (25, 3):
                raise ValueError(f'stream {g}: detections of shape {det.shape}, expected (1, 25, 3) or (25, 3)')
            if not _frame_ok(f):
                raise ValueError(f'stream {g}: expected an (H, W, 3) uint8 / float32 frame, got {tuple(f.shape)} {f.dtype}')
            centers[g], scales[g], bboxes[g], kps[g] = _box(det)
            on |= 1 << g
        if on == 0:
            return 0, bboxes
        self._check_runtime()
        dev, rows = self.thetas.device, self._rows()
        imgs = [None if not (on >> g) & 1 else (f if torch.is_tensor(f) else torch.from_numpy(np.ascontiguousarray(f))).to(dev, non_blocking=True)
                for g, f in enumerate(frames)]
        dataprocess.crop_groups(imgs, centers, scales, rows['image'], on)
        dataprocess.j2d_processing_groups(torch.from_numpy(kps).float().to(dev), centers, scales, rows['smpl_j2d'], on)
        return on, bboxes

    def adapt_processed(self, images, kps, bboxes=None, active=None):
        """The same on already cropped frames: ``images`` (G, 3, 224, 224) and ``kps`` (G, 49, 3) (rows 0..24 = OpenPose joints in
        [-1, 1]) with ``active`` (bit mask; None: every stream), or lists of G (1, 3, 224, 224) / (1, 49, 3) entries with None
        for a stream that sits the tick out.  ``bboxes[g]`` goes to stream g's result."""
        G = self.G
        if isinstance(images, (list, tuple)) != isinstance(kps, (list, tuple)):
            raise ValueError('images and kps must both be lists or both be tensors')
        if isinstance(images, (list, tuple)):
            if len(images) != G or len(kps) != G:
                raise ValueError(f'expected {G} images and {G} keypoint blocks, one per stream, got {len(images)} and {len(kps)}')
            pairs = [None if i is None or k is None else (i, k) for i, k in zip(images, kps)]
        else:
            if tuple(images.shape) != (G, 3, 224, 224) or tuple(kps.shape) != (G, 49, 3):
                raise ValueError(f'expected ({G}, 3, 224, 224) images and a ({G}, 49, 3) keypoint block, got {tuple(images.shape)} '
                                 f'and {tuple(kps.shape)}')
            active = (1 << G) - 1 if active is None else int(active)
            pairs = [(images[g:g + 1], kps[g:g + 1]) if (active >> g) & 1 else None for g in range(G)]
        for g, p in enumerate(pairs):
            if p is not None and (tuple(p[0].shape) != (1, 3, 224, 224) or tuple(p[1].shape) != (1, 49, 3)):
                raise ValueError(f'stream {g}: image {tuple(p[0].shape)} and keypoints {tuple(p[1].shape)}, expected (1, 3, 224, 224) '
                                 'and (1, 49, 3)')
        on = sum(1 << g for g, p in enumerate(pairs) if p is not None)
        if on == 0:
            return [None] * G
        self._check_runtime()
        self._rows()
        self._stage([None if p is None else {'image': p[0], 'smpl_j2d': p[1]} for p in pairs])
        return self._tick(on, [None] * G if bboxes is None else bboxes)

    def _tick(self, on, bboxes):
        """The pool step on the staged rows, then one masked forward of the adapted weights and the result dictionaries.  With
        ``test_basemodel``, the base outputs: one forward of the checkpoint arena the base adaptor holds while no active stream
        holds a model of its own, else one grouped forward of the active streams over the stack of base arenas."""
        rows = self._frames
        self._adapt_staged(on, rows)
        preds = self.predict(rows['image'], on)
        base = None
        if self.options.test_basemodel:
            with torch.no_grad():
                if any(self.slot_models[g] is not None for g in self._slots(on)):
                    rot, shape, cam, _, _ = hmr_mod.raw_forward(self._base_stack, self.buffers, rows['image'], groups=self.G, active=on)
                else:
                    rot, shape, cam, _, _ = hmr_mod.raw_forward(self.base.model.module.arena, self.buffers, rows['image'])
                base = (self.base.decode_smpl_params(rot, shape)['vts'], cam)
        out = []
        for g, p in enumerate(preds):
            if p is None:
                out.append(None)
                continue
            res = {'vts': p['vertices'], 'cam': p['cam'], 'bbox': bboxes[g]}
            if base is not None:
                res.update(vts_base=base[0][g:g + 1], cam_base=base[1][g:g + 1])
            out.append(res)
        return out

    def render(self, frames, results):
        """The viewer's drawing for one tick (reference dynaboa_webcam.py:409-418 per stream): ``frames`` as passed to
        ``online_adaptation`` (the (H, W, 3) RGB uint8 frames, numpy or CUDA), ``results`` the list it returned.  Returns per
        stream ``(rendered, rendered_base)``, BGR like ``render.render`` and on the frame's side (numpy or CUDA);
        ``rendered_base`` is None without ``test_basemodel``, and a stream without a result gives None.  Every mesh of the tick
        is drawn in one ``dboa_render_overlay_groups`` call (one per 64 meshes), with all cameras brought to the host in one
        copy; each image is bit-identical to ``render.render`` on that stream's result alone."""
        G = self.G
        if len(frames) != G or len(results) != G:
            raise ValueError(f'expected {G} frames and {G} results, one per stream, got {len(frames)} and {len(results)}')
        base = bool(self.options.test_basemodel)
        vts, cams, images, bboxes, colors, owner = [], [], [], [], [], []
        for g, (f, res) in enumerate(zip(frames, results)):
            if res is None:
                continue
            if f is None or not _frame_ok(f) or (f.dtype != torch.uint8 if torch.is_tensor(f) else np.dtype(f.dtype) != np.uint8):
                raise ValueError(f'stream {g}: expected the (H, W, 3) uint8 frame of its result, got '
                                 f'{None if f is None else (tuple(f.shape), f.dtype)}')
            for key, col in (('', self.colors[0]), ('_base', self.colors[1])) if base else (('', self.colors[0]),):
                vts.append(res['vts' + key])
                cams.append(res['cam' + key])
                images.append(f)
                bboxes.append(res['bbox'])
                colors.append(col)
                owner.append(g)
        drawn = render_mod.render_groups(vts, cams, images, bboxes, colors)
        out = [None] * G
        for i, g in enumerate(owner):
            if out[g] is None:
                out[g] = (drawn[i], None)
            else:
                out[g] = (out[g][0], drawn[i])
        return out
