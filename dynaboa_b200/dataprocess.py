"""Input side of the hot path on the GPU (drop-in for the pieces of reference utils/dataprocess.py and boa_dataset/pw3d.py the
benchmark path uses: ``get_transform`` :13-37, ``transform`` :39-46, ``crop`` :48-96 at rot = 0, ``rgb_processing`` /
``j2d_processing`` / ``process_sample`` pw3d.py:127-163).

``skimage.transform.resize`` is linear and separable: a Gaussian pre-filter (sigma = (in / out - 1) / 2 per axis when
down-scaling, mirror boundary) followed by an order-1 zoom with pixel-centre alignment.  Per crop size the HOST composes the
banded matrix of one axis once (cached): row o holds the weights with which crop pixels contribute to output pixel o.  The GPU
applies the two matrices (``dboa_crop_resize_normalize``) fused with the crop itself (zero fill outside the frame), /255, the
channel normalisation and the HWC -> CHW transpose; the image never leaves the device.  The keypoint transform keeps the
reference's double-precision truncation (``dboa_keypoint_transform``).  ``crop_groups`` / ``j2d_processing_groups`` do the same
for the frames of several streams at once, one launch per pass for all of them (the webcam pool, webcam.MultiWebcamAdaptor).
"""
import ctypes as C
import functools

import numpy as np
import torch

from . import _lib, constants
from ._lib import ptr, stream

IMG_NORM_MEAN = (0.485, 0.456, 0.406)        # reference constants.py:6-7
IMG_NORM_STD = (0.229, 0.224, 0.225)


def get_transform(center, scale, res):
    """reference utils/dataprocess.py:13-37 at rot = 0."""
    h = 200 * scale
    t = np.zeros((3, 3))
    t[0, 0] = float(res[1]) / h
    t[1, 1] = float(res[0]) / h
    t[0, 2] = res[1] * (-float(center[0]) / h + .5)
    t[1, 2] = res[0] * (-float(center[1]) / h + .5)
    t[2, 2] = 1
    return t


def transform(pt, center, scale, res, invert=0):
    """reference utils/dataprocess.py:39-46 (host scalar version, used for the crop corners)."""
    t = get_transform(center, scale, res)
    if invert:
        t = np.linalg.inv(t)
    new_pt = np.dot(t, np.array([pt[0] - 1, pt[1] - 1, 1.]).T)
    return new_pt[:2].astype(int) + 1


@functools.lru_cache(maxsize=256)
def _axis_matrix(n_in, n_out):
    """Banded matrix (start[n_out] int32, weights[n_out][T] float32) of skimage's resize along one axis of length ``n_in``:
    Gaussian pre-filter (mirror) then order-1 zoom with grid_mode (mirror), composed by pushing the identity through the same
    two scipy.ndimage calls skimage makes (skimage/transform/_warps.py::resize)."""
    import scipy.ndimage as ndi
    factor = n_in / n_out
    sigma = max(0.0, (factor - 1) / 2)
    eye = np.eye(n_in)
    if sigma > 0:
        eye = ndi.gaussian_filter1d(eye, sigma, axis=0, mode='mirror')
    M = ndi.zoom(eye, (n_out / n_in, 1.0), order=1, mode='mirror', cval=0, grid_mode=True)       # (n_out, n_in)
    nz = M != 0
    lo = nz.argmax(1)
    hi = n_in - 1 - nz[:, ::-1].argmax(1)
    T = int((hi - lo).max()) + 1
    w = np.zeros((n_out, T), np.float32)
    for o in range(n_out):
        w[o, :hi[o] - lo[o] + 1] = M[o, lo[o]:hi[o] + 1]
    return lo.astype(np.int32), w


_TABLES = {}


def _tables(n_in, n_out, device):
    key = (n_in, n_out, device.index)
    if key not in _TABLES:
        lo, w = _axis_matrix(n_in, n_out)
        _TABLES[key] = (torch.from_numpy(lo).to(device), torch.from_numpy(w).to(device).contiguous())
    return _TABLES[key]


def _box(center, scale, res):
    """Integer upper-left corner and size (ul_x, ul_y, Wc, Hc) of the reference ``crop``'s box (host arithmetic)."""
    ul = np.array(transform([1, 1], center, scale, res, invert=1)) - 1
    br = np.array(transform([res[0] + 1, res[1] + 1], center, scale, res, invert=1)) - 1
    Wc, Hc = int(br[0] - ul[0]), int(br[1] - ul[1])
    if Wc < 2 or Hc < 2:
        raise ValueError('degenerate bounding box')
    return int(ul[0]), int(ul[1]), Wc, Hc


def _check_frame(img):
    _lib.require_cuda(img)
    if img.dim() != 3 or img.shape[2] != 3 or img.dtype not in (torch.float32, torch.uint8):
        raise ValueError('crop expects an (H, W, 3) float32 / uint8 image and a square output')


def crop(img, center, scale, res=(constants.IMG_RES, constants.IMG_RES)):
    """GPU version of reference ``crop`` + ``rgb_processing`` + ``Normalize``: ``img`` is a CUDA tensor (H, W, 3) RGB, float32
    0..255 or uint8; returns the normalised (3, res, res) float32 network input."""
    _check_frame(img)
    if res[0] != res[1]:
        raise ValueError('crop expects an (H, W, 3) float32 / uint8 image and a square output')
    img = img.contiguous()
    H, W = int(img.shape[0]), int(img.shape[1])
    ul_x, ul_y, Wc, Hc = _box(center, scale, res)
    dev = img.device
    sx, wx = _tables(Wc, res[1], dev)
    sy, wy = _tables(Hc, res[0], dev)
    tmp = torch.empty(Hc * res[1] * 3, dtype=torch.float32, device=dev)
    out = torch.empty(3, res[0], res[1], dtype=torch.float32, device=dev)
    mean, std = (C.c_float * 3)(*IMG_NORM_MEAN), (C.c_float * 3)(*IMG_NORM_STD)
    _lib.call('dboa_crop_resize_normalize', ptr(img), int(img.dtype == torch.uint8), H, W, ul_x, ul_y, Hc, ptr(wx), ptr(sx),
              int(wx.shape[1]), ptr(wy), ptr(sy), int(wy.shape[1]), int(res[0]), mean, std, ptr(tmp), ptr(out), stream())
    return out


def _mask(active, n, present=None):
    """``active`` as an int bit mask over n entries (None: the entries of ``present`` that are not None, else all)."""
    if active is None:
        return sum(1 << g for g in range(n) if present is None or present[g] is not None)
    return int(active)


def crop_groups(frames, centers, scales, out, active=None, res=constants.IMG_RES):
    """``crop`` of the frames of G streams in two launches (``dboa_crop_resize_normalize_groups``): ``frames[g]`` is a CUDA
    (H_g, W_g, 3) float32 / uint8 frame (sizes and dtypes may differ), cropped at ``centers[g]`` / ``scales[g]`` into row g of
    ``out``, a (G, 3, res, res) float32 CUDA tensor.  ``active``: bit mask of the streams to crop (None: every frame that is
    not None); the other frames are not read and their rows of ``out`` keep what they held.  Row g is bit-identical to
    ``crop(frames[g], centers[g], scales[g])``.  Returns ``out``."""
    G = len(frames)
    active = _mask(active, G, frames)
    _lib.require_cuda(out)
    if tuple(out.shape) != (G, 3, res, res) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError(f'out must be a contiguous ({G}, 3, {res}, {res}) float32 tensor')
    descs, keep, total = (_lib.CropDescStruct * max(G, 1))(), [], 0
    for g in range(G):
        if not (active >> g) & 1:
            continue
        if frames[g] is None:
            raise ValueError(f'stream {g} is active but has no frame')
        _check_frame(frames[g])
        img = frames[g].contiguous()
        ul_x, ul_y, Wc, Hc = _box(centers[g], scales[g], (res, res))
        sx, wx = _tables(Wc, res, out.device)
        sy, wy = _tables(Hc, res, out.device)
        keep.append(img)
        d = descs[g]
        d.img, d.wx, d.sx, d.wy, d.sy = img.data_ptr(), wx.data_ptr(), sx.data_ptr(), wy.data_ptr(), sy.data_ptr()
        d.is_u8, d.H, d.W, d.ul_x, d.ul_y = int(img.dtype == torch.uint8), int(img.shape[0]), int(img.shape[1]), ul_x, ul_y
        d.Hc, d.Tx, d.Ty = Hc, int(wx.shape[1]), int(wy.shape[1])
        total += Hc * res * 3
    tmp = torch.empty(max(total, 1), dtype=torch.float32, device=out.device)
    mean, std = (C.c_float * 3)(*IMG_NORM_MEAN), (C.c_float * 3)(*IMG_NORM_STD)
    _lib.call('dboa_crop_resize_normalize_groups', descs, G, active, int(res), mean, std, ptr(tmp), tmp.numel(), ptr(out), stream())
    return out


def j2d_processing(kp, center, scale, res=constants.IMG_RES):
    """GPU version of reference ``j2d_processing`` (pw3d.py:151-163, no flip): (N, 3) pixel keypoints + confidence on the device
    -> integer crop pixels mapped to [-1, 1]."""
    _lib.require_cuda(kp)
    kp = kp.contiguous().float()
    t = get_transform(center, scale, [res, res])
    out = torch.empty_like(kp)
    _lib.call('dboa_keypoint_transform', ptr(kp), int(kp.shape[0]), float(t[0, 0]), float(t[0, 2]), float(t[1, 1]), float(t[1, 2]), int(res),
              ptr(out), stream())
    return out


def j2d_processing_groups(kps, centers, scales, out, active=None, res=constants.IMG_RES):
    """``j2d_processing`` of G streams in one launch (``dboa_keypoint_transform_groups``): ``kps`` (G, n, 3) CUDA keypoints
    (n <= 49) of stream g mapped through its box into rows [0, n) of ``out[g]``, a (G, 49, 3) float32 CUDA block whose rows
    [n, 49) are zeroed.  ``active``: bit mask (None: all); idle streams' keypoints are not read and their rows keep what they
    held.  Row g is bit-identical to ``j2d_processing(kps[g], centers[g], scales[g])``.  Returns ``out``."""
    _lib.require_cuda(kps, out)
    G = int(kps.shape[0])
    if kps.dim() != 3 or kps.shape[2] != 3 or tuple(out.shape) != (G, 49, 3) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError('j2d_processing_groups expects (G, n, 3) keypoints and a contiguous (G, 49, 3) float32 block')
    active = _mask(active, G)
    kps = kps.contiguous().float()
    t4 = (C.c_double * (4 * max(G, 1)))()
    for g in range(G):
        if (active >> g) & 1:
            t = get_transform(centers[g], scales[g], [res, res])
            t4[4 * g:4 * g + 4] = [float(t[0, 0]), float(t[0, 2]), float(t[1, 1]), float(t[1, 2])]
    _lib.call('dboa_keypoint_transform_groups', ptr(kps), int(kps.shape[1]), t4, int(res), ptr(out), G, active, stream())
    return out


def process_sample(image, keypoints, smpl_j2ds, center, scale):
    """reference pw3d.py:127-136 for the benchmark path (no augmentation): (op_j2d, image, smpl_j2d) on the device."""
    return j2d_processing(keypoints, center, scale), crop(image, center, scale), j2d_processing(smpl_j2ds, center, scale)
