"""Mesh overlay on the GPU (drop-in for reference render_demo.py:33-153 and utils/webcam_utils.py:71-79).

``Renderer(resolution, orig_img, wireframe).render(img, verts, cam, angle, axis, mesh_filename, color)`` keeps the reference's
signature and defaults; the drawing is one ``dboa_render_overlay`` call (csrc/render.cu) instead of trimesh + pyrender + EGL.
``img`` is an (H, W, 3) uint8 frame: a numpy array gives a numpy result (the reference's contract), a CUDA tensor gives a
CUDA tensor, so a frame that is already on the device is drawn on and stays there.  The reference builds a new ``Renderer``
for every frame (base_adaptor.py:441, webcam_utils.py:77), so construction does no work: the device copy of the faces and
their vertex->face adjacency are cached per faces array, the scratch buffer per (frame sizes, samples, mesh size).

``draw_groups`` / ``render_groups`` draw many meshes of one topology, each over its own frame, in one
``dboa_render_overlay_groups`` call (the adapted and base meshes of every stream of a webcam pool); ``draw`` is its
one-mesh case.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from ._lib import ptr, stream

_faces_cache = {}        # (id(faces), NV, device) -> (faces array kept alive, faces, vf_offsets, vf_faces)
_scratch_cache = {}      # (((W, H), ...), samples, NV, NF, device) -> uint8 tensor
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


def _scratch(sizes, samples, nv, nf, device):
    """Scratch of one grouped call over frames of the (W, H) ``sizes``, cached per (sizes, samples, mesh size, device)."""
    key = (tuple(sizes), samples, nv, nf, device)
    buf = _scratch_cache.get(key)
    if buf is None:
        M = len(sizes)
        W, H = (C.c_int * M)(*[w for w, _ in sizes]), (C.c_int * M)(*[h for _, h in sizes])
        need = _lib.load().dboa_render_scratch_bytes_groups(W, H, M, nv, nf, samples)
        _lib.check(int(need) if need < 0 else 0, 'dboa_render_scratch_bytes_groups')
        if len(_scratch_cache) >= 4:
            _scratch_cache.clear()
        buf = _scratch_cache[key] = torch.empty(int(need), dtype=torch.uint8, device=device)
    return buf


MAX_MESHES = 64


def draw_groups(imgs, verts, faces, cam4s, colors, rots=None, samples=4, face_ids=False):
    """One ``dboa_render_overlay_groups`` call: M <= 64 meshes of one topology, mesh k drawn over ``imgs[k]``.  imgs: M (H_k,
    W_k, 3) uint8 CUDA tensors (one tensor may appear several times: entries that share a frame each get their own output);
    verts: M (NV, 3) CUDA tensors, or one (M, NV, 3) tensor; faces: (NF, 3) integer numpy array; cam4s: host (M, 4) array of
    (sx, sy, tx, ty); colors: host (M, 3) base colours in 0..1; rots: None or M optional 3 x 3 rotations.  Returns the M (H_k,
    W_k, 3) results, and with ``face_ids`` also the M (H_k, W_k, samples) int32 winning faces.  Each entry is bit-identical to
    ``draw`` on that entry alone."""
    M = len(imgs)
    if not 1 <= M <= MAX_MESHES:
        raise ValueError(f'draw_groups draws 1 to {MAX_MESHES} meshes per call, got {M}')
    cam4s = np.asarray(cam4s, dtype=np.float64).reshape(-1, 4) if len(cam4s) else np.zeros((0, 4))
    colors = np.asarray(colors, dtype=np.float64).reshape(-1, 3) if len(colors) else np.zeros((0, 3))
    rots = [None] * M if rots is None else list(rots)
    if len(verts) != M or len(cam4s) != M or len(colors) != M or len(rots) != M:
        raise ValueError(f'expected {M} vertex sets, cameras, colours and rotations, one per frame, got {len(verts)}, '
                         f'{len(cam4s)}, {len(colors)} and {len(rots)}')
    if samples not in (1, 4):
        raise ValueError('samples must be 1 or 4')
    for k, img in enumerate(imgs):
        if not torch.is_tensor(img) or img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
            raise ValueError(f'entry {k}: img must be an (H, W, 3) uint8 frame, got {tuple(img.shape)} {img.dtype}')
    _lib.require_cuda(*imgs, *verts)
    dev = imgs[0].device
    imgs = [i.contiguous() for i in imgs]
    vs = [v.detach().reshape(-1, 3).to(device=dev, dtype=torch.float32).contiguous() for v in verts]
    nv = vs[0].shape[0]
    if any(v.shape[0] != nv for v in vs):
        raise ValueError('every mesh of a grouped call has the same number of vertices')
    f_dev, vf_off, vf_faces = _device_faces(faces, nv, dev)
    nf = f_dev.shape[0]
    sizes = [(int(i.shape[1]), int(i.shape[0])) for i in imgs]
    scratch = _scratch(sizes, samples, nv, nf, dev)
    outs = [torch.empty_like(i) for i in imgs]
    ids = [torch.empty(i.shape[0], i.shape[1], samples, dtype=torch.int32, device=dev) for i in imgs] if face_ids else [None] * M
    desc = (_lib.RenderDescStruct * M)()
    for k in range(M):
        d = desc[k]
        d.verts, d.img, d.out, d.face_ids = ptr(vs[k]), ptr(imgs[k]), ptr(outs[k]), ptr(ids[k])
        d.cam4[:] = [float(c) for c in cam4s[k]]
        d.has_rot = int(rots[k] is not None)
        if rots[k] is not None:
            d.rot3x3[:] = [float(x) for x in np.asarray(rots[k], dtype=np.float64).reshape(9)]
        d.color3[:] = [float(c) for c in colors[k]]
        d.W, d.H = sizes[k]
    _lib.call('dboa_render_overlay_groups', desc, M, ptr(f_dev), ptr(vf_off), ptr(vf_faces), nv, nf, samples, ptr(scratch),
              scratch.numel(), stream())
    return (outs, ids) if face_ids else outs


def draw(img, verts, faces, cam4, rot=None, color=(1.0, 1.0, 0.9), samples=4, face_ids=False):
    """The one-mesh case of ``draw_groups``.  img: (H, W, 3) uint8 CUDA tensor; verts: (NV, 3) CUDA tensor; faces: (NF, 3)
    integer numpy array (cached on the device by identity); cam4 = (sx, sy, tx, ty); rot: optional 3 x 3 rotation applied after
    Rx(180).  Returns the (H, W, 3) uint8 result, and with ``face_ids`` also the (H, W, samples) int32 winning faces."""
    _lib.require_cuda(img, verts)
    r = draw_groups([img], [verts], faces, [np.asarray(cam4, dtype=np.float64).reshape(4)],
                    [np.asarray(color, dtype=np.float64).reshape(3)], rots=[rot], samples=samples, face_ids=face_ids)
    return (r[0][0], r[1][0]) if face_ids else r[0]


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


def render_groups(vts, cams, images, bboxes, colors):
    """``render`` for many meshes at once: entry k draws the first mesh of ``vts[k]`` with the crop camera ``cams[k]`` and box
    ``bboxes[k]`` over ``images[k]`` (RGB, numpy or CUDA; entries may share a frame) in ``colors[k]`` (0..255), and returns it
    in BGR order, numpy in -> numpy out, CUDA in -> CUDA out.  Each result is bit-identical to ``render`` on that entry.  The
    device cameras come to the host in one copy; the meshes are drawn in one ``dboa_render_overlay_groups`` call per 64."""
    n = len(images)
    if len(vts) != n or len(cams) != n or len(bboxes) != n or len(colors) != n:
        raise ValueError(f'expected {n} meshes, cameras, boxes and colours, one per image, got {len(vts)}, {len(cams)}, '
                         f'{len(bboxes)} and {len(colors)}')
    if n == 0:
        return []
    dev_cams = [k for k, c in enumerate(cams) if torch.is_tensor(c)]
    host_cams = list(cams)
    if dev_cams:
        dts = {cams[k].dtype for k in dev_cams}
        rows = [cams[k].detach()[:1] for k in dev_cams]
        flat = torch.cat(rows).cpu().numpy() if len(dts) == 1 else [r.cpu().numpy() for r in rows]
        for i, k in enumerate(dev_cams):
            host_cams[k] = flat[i:i + 1]
    uploads, frames, on_host = {}, [], []
    for img in images:
        on_host.append(not torch.is_tensor(img))
        if on_host[-1]:
            key = id(img)
            if key not in uploads:
                uploads[key] = (img, torch.from_numpy(np.ascontiguousarray(img)).cuda())
            frames.append(uploads[key][1])
        else:
            frames.append(img)
    cam4s, verts = [], []
    for k in range(n):
        ori_h, ori_w = images[k].shape[:2]
        cam4s.append(convert_crop_cam_to_orig_img(np.asarray(host_cams[k])[:1], bboxes[k], ori_w, ori_h)[0])
        v = vts[k][0]
        verts.append((v if torch.is_tensor(v) else torch.from_numpy(np.asarray(v, dtype=np.float32))).to(frames[k].device))
    cols = [np.array(c) / 255 for c in colors]
    faces, outs = get_smpl_faces(), []
    for a in range(0, n, MAX_MESHES):
        b = min(n, a + MAX_MESHES)
        outs += draw_groups(frames[a:b], verts[a:b], faces, cam4s[a:b], cols[a:b], samples=Renderer.samples)
    return [o.cpu().numpy()[:, :, ::-1] if h else o.flip(-1) for o, h in zip(outs, on_host)]
