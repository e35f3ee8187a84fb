"""Mesh overlay on the GPU (drop-in for reference render_demo.py:33-153 and utils/webcam_utils.py:71-79).

``Renderer(resolution, orig_img, wireframe).render(img, verts, cam, angle, axis, mesh_filename, color)`` keeps the reference's
signature and defaults; the drawing is one ``dboa_render_overlay`` call (csrc/render.cu) instead of trimesh + pyrender + EGL.
``img`` is an (H, W, 3) uint8 frame: a numpy array gives a numpy result (the reference's contract), a CUDA tensor gives a
CUDA tensor, so a frame that is already on the device is drawn on and stays there.  The reference builds a new ``Renderer``
for every frame (base_adaptor.py:441, webcam_utils.py:77), so construction does no work: the device copy of the faces and
their vertex->face adjacency are cached per faces array, the scratch buffer per (W, H, samples, mesh size).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr, stream

_faces_cache = {}        # (id(faces), NV, device) -> (faces array kept alive, faces, vf_offsets, vf_faces)
_scratch_cache = {}      # (W, H, samples, NV, NF, device) -> uint8 tensor
_smpl_faces = {}         # SMPL model directory -> faces


def convert_crop_cam_to_orig_img(cam, bbox, img_width, img_height):
    """reference render_demo.py:136-153: weak-perspective camera of the crop (s, tx, ty) -> (sx, sy, tx, ty) in the frame.
    ``cam`` (B, 3), ``bbox`` (B, 3) = (cx, cy, h); every row uses the frame size passed in."""
    cam, bbox = np.asarray(cam), np.asarray(bbox)
    cx, cy, h = bbox[:, 0], bbox[:, 1], bbox[:, 2]
    hw, hh = img_width / 2., img_height / 2.
    sx = cam[:, 0] * (1. / (img_width / h))
    sy = cam[:, 0] * (1. / (img_height / h))
    tx = ((cx - hw) / hw / sx) + cam[:, 1]
    ty = ((cy - hh) / hh / sy) + cam[:, 2]
    return np.stack([sx, sy, tx, ty]).T


def rotation_matrix(angle_deg, axis):
    """trimesh.transformations.rotation_matrix(math.radians(angle), axis) as a 3 x 3 float64 array."""
    a = math.radians(angle_deg)
    d = np.asarray(axis, dtype=np.float64)[:3]
    d = d / np.sqrt(np.dot(d, d))
    R = np.diag([math.cos(a)] * 3) + np.outer(d, d) * (1.0 - math.cos(a))
    d = d * math.sin(a)
    return R + np.array([[0.0, -d[2], d[1]], [d[2], 0.0, -d[0]], [-d[1], d[0], 0.0]])


def _device_faces(faces, nv, device):
    key = (id(faces), nv, device)
    hit = _faces_cache.get(key)
    if hit is not None and hit[0] is faces:
        return hit[1:]
    f = np.asarray(faces)
    if f.ndim != 2 or f.shape[1] != 3:
        raise ValueError(f'faces must be (NF, 3), got {f.shape}')
    f = f.astype(np.int64)
    if f.size and (f.min() < 0 or f.max() >= nv):
        raise ValueError(f'face indices must lie in [0, {nv})')
    if f.size >= 2 ** 31:
        raise ValueError('at most 2^31 - 1 face corners (the vertex->face adjacency is indexed with int32)')
    flat = f.reshape(-1)
    vf_faces = (np.argsort(flat, kind='stable') // 3).astype(np.int32)       # faces of each vertex in ascending order
    vf_off = np.concatenate([[0], np.cumsum(np.bincount(flat, minlength=nv))]).astype(np.int32)
    dev = tuple(torch.from_numpy(np.ascontiguousarray(a)).to(device) for a in (f.astype(np.int32), vf_off, vf_faces))
    if len(_faces_cache) >= 8:
        _faces_cache.clear()
    _faces_cache[key] = (faces,) + dev
    return dev


def _scratch(W, H, samples, nv, nf, device):
    key = (W, H, samples, nv, nf, device)
    buf = _scratch_cache.get(key)
    if buf is None:
        need = _lib.load().dboa_render_scratch_bytes(W, H, nv, nf, samples)
        _lib.check(int(need) if need < 0 else 0, 'dboa_render_scratch_bytes')
        if len(_scratch_cache) >= 4:
            _scratch_cache.clear()
        buf = _scratch_cache[key] = torch.empty(int(need), dtype=torch.uint8, device=device)
    return buf


def draw(img, verts, faces, cam4, rot=None, color=(1.0, 1.0, 0.9), samples=4, face_ids=False):
    """One ``dboa_render_overlay`` call.  img: (H, W, 3) uint8 CUDA tensor; verts: (NV, 3) CUDA tensor; faces: (NF, 3) integer
    numpy array (cached on the device by identity); cam4 = (sx, sy, tx, ty); rot: optional 3 x 3 rotation applied after
    Rx(180).  Returns the (H, W, 3) uint8 result, and with ``face_ids`` also the (H, W, samples) int32 winning faces."""
    _lib.require_cuda(img, verts)
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError(f'img must be an (H, W, 3) uint8 frame, got {tuple(img.shape)} {img.dtype}')
    if samples not in (1, 4):
        raise ValueError('samples must be 1 or 4')
    H, W = int(img.shape[0]), int(img.shape[1])
    img = img.contiguous()
    v = verts.detach().reshape(-1, 3).to(device=img.device, dtype=torch.float32).contiguous()
    nv = v.shape[0]
    f_dev, vf_off, vf_faces = _device_faces(faces, nv, img.device)
    nf = f_dev.shape[0]
    scratch = _scratch(W, H, samples, nv, nf, img.device)
    out = torch.empty_like(img)
    ids = torch.empty(H, W, samples, dtype=torch.int32, device=img.device) if face_ids else None
    cam = (C.c_float * 4)(*[float(c) for c in np.asarray(cam4, dtype=np.float64).reshape(4)])
    R = None if rot is None else (C.c_float * 9)(*[float(x) for x in np.asarray(rot, dtype=np.float64).reshape(9)])
    col = (C.c_float * 3)(*[float(c) for c in np.asarray(color, dtype=np.float64).reshape(3)])
    _lib.call('dboa_render_overlay', ptr(v), ptr(f_dev), ptr(vf_off), ptr(vf_faces), nv, nf, cam, R, col, ptr(img), W, H, samples,
              ptr(scratch), scratch.numel(), ptr(out), ptr(ids), stream())
    return (out, ids) if face_ids else out


def get_smpl_faces():
    """model.smpl.get_smpl_faces(), read once per SMPL model directory (the reference reloads the model per frame)."""
    from . import config, smpl
    key = config.SMPL_MODEL_DIR
    if key not in _smpl_faces:
        _smpl_faces[key] = smpl.get_smpl_faces()
    return _smpl_faces[key]


def write_obj(path, verts, faces):
    """Wavefront OBJ: ``v`` lines, then 1-based ``f`` lines (the side effect of the reference's ``mesh.export``)."""
    with open(path, 'w') as fh:
        fh.write(''.join(f'v {x:.8f} {y:.8f} {z:.8f}\n' for x, y, z in np.asarray(verts, dtype=np.float64)))
        fh.write(''.join(f'f {a + 1} {b + 1} {c + 1}\n' for a, b, c in np.asarray(faces, dtype=np.int64)))


class Renderer:
    """reference render_demo.py:58-134 on the device; 4x multisampled like pyrender's off-screen framebuffer."""

    samples = 4

    def __init__(self, resolution=(224, 224), orig_img=False, wireframe=False):
        if wireframe:
            raise NotImplementedError('wireframe rendering (RenderFlags.ALL_WIREFRAME) is not supported')
        self.resolution = resolution
        self.faces = get_smpl_faces()
        self.orig_img = orig_img
        self.wireframe = wireframe

    def render(self, img, verts, cam, angle=None, axis=None, mesh_filename=None, color=[1.0, 1.0, 0.9]):
        on_host = not torch.is_tensor(img)
        W, H = self.resolution
        frame = torch.from_numpy(np.ascontiguousarray(img)).cuda() if on_host else img
        if tuple(frame.shape[:2]) != (H, W):
            raise ValueError(f'frame is {tuple(frame.shape[:2])}, the renderer was built for (H, W) = {(H, W)}')
        v = verts if torch.is_tensor(verts) else torch.from_numpy(np.asarray(verts, dtype=np.float32))
        v = v.to(frame.device)
        if mesh_filename is not None:                             # :93-94: the mesh after Rx(180), before the angle/axis rotation
            vh = v.detach().double().cpu().numpy() * np.array([1.0, -1.0, -1.0])
            write_obj(mesh_filename, vh, self.faces)
        rot = rotation_matrix(angle, axis) if angle and axis is not None and len(axis) else None
        cam4 = cam.detach().double().cpu().numpy() if torch.is_tensor(cam) else np.asarray(cam, dtype=np.float64)
        out = draw(frame, v, self.faces, cam4, rot=rot, color=color, samples=self.samples)
        return out.cpu().numpy() if on_host else out


def render(vts, cam, image, bbox, color=[205, 129, 98]):
    """reference utils/webcam_utils.py:71-79: draws the first mesh of the batch over an RGB frame (numpy or CUDA) and returns
    it in BGR order, as the webcam viewer shows it."""
    cam = cam.detach().cpu().numpy() if torch.is_tensor(cam) else np.asarray(cam)
    ori_h, ori_w = image.shape[:2]
    ori_pred_cams = convert_crop_cam_to_orig_img(cam, bbox, ori_w, ori_h)
    renderer = Renderer(resolution=(ori_w, ori_h), orig_img=True, wireframe=False)
    rendered = renderer.render(image, vts[0], ori_pred_cams[0], color=np.array(color) / 255)
    return rendered.flip(-1) if torch.is_tensor(rendered) else rendered[:, :, ::-1]
