"""Scaffolding shared by the test modules and the timing scripts.  A plain module, not a test module: pytest does not collect it,
and no test module imports another.

- Helpers: ``bits``, ``same_bits``, ``fetch``, ``stream``, ``golden_options`` and its presets, ``state``.
- Guard-banded device buffers: ``Buf`` (an output starts as NaN, its tail of ``GUARD`` ``SENTINEL`` elements must survive).
- The device-free ABI tests: ``built_lib``, the stand-in pointer ``FAKE``, the ``ERR_*`` codes, ``cpu_options`` and ``idle_pool``.
- The per-video pool runs: ``video_masks`` / ``video_seed`` and the golden-aware ``masks_for`` / ``seed_for``, ``PoolRun`` (a
  MultiVideoAdaptor whose slots carry videos) and ``SingleRun`` (the same video through the single-video ``Adaptor.adapt``).
- The grouped HMR plan tests: the ``model`` fixture body, ``stacked``, ``inputs``, the fp64 bounds of the layer tests, the
  fp64 GroupNorm ``gn_stats`` / ``gn_apply`` and ``tape_pattern``, the kink pattern of a GPU forward for oracle/hmr_frozen.py.
- The grouped input side: the mixed frames and boxes of ``scene``, their ``crop_kind`` and the fp64 ``crop_oracle``.
- The exact references of the step's sweeps (``f32``, ``sgd_ref``, ``ema_ref``, ``adam_ref``), the fp64 bounds of the cosine
  feature test and the pose prior's near-tie rule ``selected``.
- Rendering: the analytic scene helpers, ``sphere``, ``posed_smpl_mesh``, ``check_against_oracle``, and the synthetic Internet
  video of the unchanged-driver tests."""
import ast
import ctypes
import math
import os
import random
from types import SimpleNamespace

import numpy as np
import torch

from dynaboa_b200 import _lib
from oracle import ref_harness


def bits(t):
    """The bits of `t`, for bit-for-bit comparison: float64 viewed as int64, float32 as int32, other dtypes as they are."""
    t = t.contiguous()
    if t.dtype == torch.float64:
        return t.view(torch.int64)
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same_bits(a, b):
    """a and b have the same dtype, shape and bits (NaN payloads included); b may live on another device."""
    a, b = a.contiguous(), b.to(a.device).contiguous()
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    return torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------ guard-banded device buffers
GUARD = 64
SENTINEL = {torch.float32: -1.2345678e33, torch.float64: -1.25e300, torch.int32: 0x5A5A5A5A, torch.uint8: 0xA5}
UNSET = {torch.int32: -7, torch.uint8: 0xEE}            # the fill of an output buffer of an integer type (floats: NaN)


class Buf:
    """A device buffer of n elements (``x``'s values, else NaN / UNSET) followed by GUARD sentinel elements."""

    def __init__(self, x=None, n=None, dtype=torch.float32):
        if x is not None:
            dtype, n = x.dtype, x.numel()
        self.n, self.dtype = n, dtype
        self.whole = torch.empty(n + GUARD, dtype=dtype, device='cuda')
        self.whole[n:] = SENTINEL[dtype]
        self.t = self.whole[:n]
        if x is not None:
            self.t.copy_(x.reshape(-1))
        else:
            self.t.fill_(UNSET.get(dtype, float('nan')))

    @property
    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def cpu(self):
        return self.t.cpu()

    def intact(self):
        tail = self.whole[self.n:].cpu()
        return same_bits(tail, torch.full_like(tail, SENTINEL[self.dtype]))


def fetch(batch):
    """A batch dict with its tensors on the device."""
    return {k: v.cuda() if torch.is_tensor(v) else v for k, v in batch.items()}


def stream(vid, n):
    from dynaboa_b200 import synthetic
    return synthetic.SyntheticStream(length=n, batch_size=1, rank=vid)


# ------------------------------------------------------------------ options
def golden_options(tmp, gd, **overrides):
    """The options a golden was recorded with (``gd``: the loaded golden, or the repr of its options), with ``expdir=tmp`` and
    ``overrides``."""
    o = dict(ast.literal_eval(gd if isinstance(gd, str) else str(gd['options'])))
    o.update(expdir=str(tmp), **overrides)
    return SimpleNamespace(**o)


def adapt_options(tmp, gd, **overrides):
    """An adapt_*.npz golden's options for an adaptation run of the synthetic checkpoint under ``tmp``."""
    from dynaboa_b200 import config
    return golden_options(tmp, gd, expname='run', tensorboard=0, synthetic_frames=8, cache_results=0, model_file=config.BASE_MODEL,
                          **overrides)


def pool_options(tmp, golden, tag, name, **overrides):
    """``adapt_options`` of adapt_{tag}.npz under tmp / name: C2 and C3 without the dynamic loop, C5 with it."""
    o = adapt_options(tmp / name, golden(f'adapt_{tag}'), **overrides)
    if tag == 'c5':
        assert o.dynamic_boa
    else:
        assert not o.dynamic_boa
    return o


def cam_options(tmp, gd, **overrides):
    """adapt_webcam.npz's options for a webcam run of the synthetic checkpoint under ``tmp``."""
    from dynaboa_b200 import config
    return golden_options(tmp, gd, expname='cam', tensorboard=0, model_file=config.BASE_MODEL, **overrides)


def webcam_pool(tmp, gd, G, name, **overrides):
    from dynaboa_b200.webcam import MultiWebcamAdaptor
    return MultiWebcamAdaptor(cam_options(tmp / name, gd, **overrides), G, dynamic_loop=True)


# ------------------------------------------------------------------ device-free ABI tests
# stand-in device pointer: every call it is passed to rejects its arguments before a pointer is dereferenced or a device touched
FAKE = ctypes.c_void_p(0x1000)
# the codes of _lib._ERRORS, which test_cabi.py holds to the header's DBOA_ERR_* (None for a name the binding lacks: no status is None)
_CODE = {name: code for code, name in _lib._ERRORS.items()}
ERR_ARG, ERR_SHAPE, ERR_CUDA, ERR_UNSUPPORTED = (_CODE.get('DBOA_ERR_' + n) for n in ('ARG', 'SHAPE', 'CUDA', 'UNSUPPORTED'))


def built_lib():
    """The library, built for sm_90a and loaded with its ctypes signatures: the body of the device-free modules' ``lib`` fixtures."""
    from dynaboa_b200 import build
    build.build()
    return _lib.load()


def cpu_options(workload, **extra):
    """bench.py's options of `workload` with ``extra`` on top, for checks that run before any device or file is touched."""
    from bench import WORKLOADS, default_options
    return default_options(expdir='/nonexistent', expname='x', model_file='unused', synthetic_frames=2,
                           **{**WORKLOADS[workload], **extra})


def idle_pool(cls, G, **attrs):
    """A ``cls`` pool (MultiVideoAdaptor, MultiWebcamAdaptor) of G slots with ``attrs`` set and no device: only its checks that
    run before any device work can be called."""
    pool = cls.__new__(cls)
    vars(pool).update(G=G, **attrs)
    return pool


# ------------------------------------------------------------------ per-video pool runs
def video_masks(vid, t, call):
    """Teacher keep-masks of video `vid`, its own frame t, teacher forward `call`."""
    gen = torch.Generator().manual_seed(1000003 * vid + 1009 * t + call)
    return (torch.rand(3, 2, 1, 1024, generator=gen) >= 0.5).float() * 2.0


def video_seed(vid, t):
    """Retrieval seed of video `vid`, its own frame t."""
    return 7919 * vid + t


def masks_for(g, t, call, gd):
    """Teacher keep-masks of video g, frame t, teacher forward `call`: the golden's for video 0, seeded for the others."""
    if g == 0:
        m = torch.from_numpy(gd['teacher_masks']).float()
        return m[t, min(call, m.shape[1] - 1)]
    gen = torch.Generator().manual_seed(100000 * g + 100 * t + call)
    return (torch.rand(3, 2, 1, 1024, generator=gen) >= 0.5).float() * 2.0


def seed_for(g, t):
    return 1000 + t if g == 0 else 1000 * (g + 1) + t


# cos_sim_threshold for videos 0..3 (SyntheticStream(rank=g), video_masks, seeds 7919 g + t) at adapt_c5.npz's options over 8
# frames, calibrated once on an H100 80GB HBM3: the single-video loops run different numbers of iterations in frames 1 and 2
# (trip counts [1, 1, 2, 1] and [0, 0, 0, 3]), and the closest of all 1 - cos12 decisions lies 2.1 % from it.
# test_gpu_multivideo_dynamic.py::test_mixed_trip_counts_follow_the_single_video_runs checks both.
MIXED_THRESHOLD = 7e-5
N_FRAMES = 8


def state(mv, g):
    """Slot g's theta, teacher and Adam moments."""
    return [mv.thetas[g].clone(), mv.teachers[g].clone(), mv.m[g].clone(), mv.v[g].clone()]


class PoolRun:
    """A MultiVideoAdaptor whose slots carry (video id, stream, own frame); teacher masks ``masks(vid, t, call)`` and retrieval
    seeds ``seed(vid, t)`` follow the video."""

    def __init__(self, opts, G, dynamic_loop=False, masks=video_masks, seed=video_seed):
        from dynaboa_b200.multivideo import MultiVideoAdaptor
        self.mv = MultiVideoAdaptor(opts, G, dynamic_loop=dynamic_loop)
        self.masks, self.seed = masks, seed
        self.slot, self.calls = [None] * G, [0] * G
        self.mv.mask_provider = self.provider

    def provider(self, g, B, dev):
        vid, _, t = self.slot[g]
        m = self.masks(vid, t, self.calls[g])
        self.calls[g] += 1
        return m.to(dev)

    def start(self, g, vid, stream):
        self.mv.start(g)
        self.slot[g] = [vid, stream, 0]

    def step(self, run):
        """One pool frame: the slots in `run` advance by one frame of their video.  Returns {slot: (vid, own frame, batch)}."""
        batches, done = [None] * self.mv.G, {}
        for g in run:
            vid, s, t = self.slot[g]
            batches[g] = fetch(s[t])
            self.calls[g] = 0
            self.mv.rngs[g].seed(self.seed(vid, t))
            done[g] = (vid, t, batches[g])
        self.mv.adapt(batches)
        for g in run:
            self.slot[g][2] += 1
        return done

    def state(self, g):
        return state(self.mv, g)


class SingleRun:
    """``Adaptor.adapt`` of video `vid` alone, with the teacher masks and retrieval seeds a PoolRun gives it."""

    def __init__(self, opts, vid, masks=video_masks, seed=video_seed):
        from dynaboa_b200.adaptor import Adaptor
        self.ad = Adaptor(opts)
        self.ad.fused_eval = 'none'
        self.vid, self.masks, self.seed = vid, masks, seed

    def step(self, t, batch):
        calls, ad = {'i': 0}, self.ad

        def provider(B, dev):
            m = self.masks(self.vid, t, calls['i'])
            calls['i'] += 1
            return m.to(dev)
        ad.teacher.mask_provider = provider
        random.seed(self.seed(self.vid, t))
        ad.global_step, ad.fit_losses = t, {}
        ad.model.eval()
        ad.adapt(batch)


# ------------------------------------------------------------------ grouped HMR plan
def hmr_model():
    """Body of the grouped-plan tests' module fixture: the synthetic checkpoint's HMR with the fused plans off, the library's modes
    restored afterwards."""
    from dynaboa_b200 import _lib, synthetic
    from dynaboa_b200.hmr import hmr
    from oracle import hmr_ref
    lib = _lib.load()
    m = hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    prev = lib.dboa_get_fused_forward(), lib.dboa_get_fused_backward()
    lib.dboa_set_fused_forward(0)
    lib.dboa_set_fused_backward(0)
    yield m
    lib.dboa_set_tensor_core_conv(3)          # library default: later test modules must not inherit this module's mode
    lib.dboa_set_fused_forward(prev[0])
    lib.dboa_set_fused_backward(prev[1])


def stacked(m, G, seed):
    """(G, P) arena stack: video g's weights are the checkpoint's scaled element-wise by 1 + 0.05 N(0, 1) (seeded per video;
    the zero padding of the arena stays zero)."""
    P = m.arena.numel()
    out = torch.empty(G, P, device='cuda')
    for g in range(G):
        gen = torch.Generator(device='cuda').manual_seed(seed + g)
        out[g] = m.arena * (1 + 0.05 * torch.randn(P, generator=gen, device='cuda'))
    return out


def inputs(B, seed, masked):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, 224, 224, generator=g).cuda()
    masks = (torch.rand(3, 2, B, 1024, generator=g) >= 0.5).float().cuda() * 2 if masked else None
    d = [torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda(), torch.randn(B, 3, generator=g).cuda()]
    return x, masks, d


# Forward bounds of the HMR plan against fp64, each relative to the largest value of the layer's fp64 result ('stats': mean error
# in units of the group's standard deviation, and relative rstd error).  Worst measured over test_gpu_hmr_layers' configurations
# on an H100 80GB HBM3 (400 W): y 2.8e-6 (CUDA-core convs, B = 64), stats 1.9e-7, a 2.4e-7, head 3.4e-7, rotmat 6.1e-7.
FWD_TOL = {'y': 6e-6, 'stats': 5e-7, 'a': 6e-7, 'head': 1e-6, 'out': 2e-6}
# Backward: max |g - ref| <= GRAD_TOL * max |ref| for every one of the 169 tensors, and whole-arena relative L2 below
# GRAD_L2.  Worst measured: 1.6e-5 per tensor (tensor-core mode 1, B = 64) and 2.0e-6 relative L2 (dropout, B = 9).
GRAD_TOL = 5e-5
GRAD_L2 = 1e-5


def structure():
    """Convolution geometry plus the bottleneck blocks as (c1, c2, c3, downsample or None) conv indices."""
    from dynaboa_b200.hmr import conv_geometry
    geo = conv_geometry()
    blocks = []
    for i, g in enumerate(geo):
        if g[0].endswith('.conv1'):
            blocks.append([i, i + 1, i + 2, i + 3 if i + 3 < len(geo) and 'downsample' in geo[i + 3][0] else None])
    return geo, blocks


def nchw(t):
    return t.permute(0, 3, 1, 2).double()


def rel(a, ref, scale=None):
    s = ref.abs().max() if scale is None else scale
    return float((a.double() - ref).abs().max() / s.clamp_min(1e-30))


def gn_stats(y):
    """fp64 GroupNorm (4 groups) statistics (mean, rstd) of an NCHW tensor, per sample and group."""
    v = y.reshape(y.shape[0], 4, -1)
    return v.mean(-1), (v.var(-1, unbiased=False) + 1e-5).rsqrt()


def gn_apply(y, mean, rstd, gamma, beta):
    B, C = y.shape[:2]
    v = ((y.reshape(B, 4, -1) - mean[..., None]) * rstd[..., None]).reshape(y.shape)
    return v * gamma.double().view(1, C, 1, 1) + beta.double().view(1, C, 1, 1)


def tape_pattern(tape, B, rows=slice(None), masks=None):
    """The kink pattern (oracle/hmr_frozen.py) of the samples ``rows`` of the GPU forward whose tape is ``tape`` (batch B):
    each ReLU's ``a > 0``, the max-pool's window positions and the dropout keep-masks ``masks`` (None: no dropout)."""
    from dynaboa_b200.hmr import tape_views
    v = tape_views(tape, B)
    geo, _ = structure()
    return {'relu': {g[0]: nchw(v['a'][i][rows]) > 0 for i, g in enumerate(geo) if v['a'][i] is not None},
            'pool': v['p0_idx'][rows].permute(0, 3, 1, 2).long(),
            'drop': None if masks is None else masks[:, :, rows].double()}


# ------------------------------------------------------------------ the step's sweeps and the pose prior's choice
def f32(x):
    """A Python double rounded once to fp32: the scalar torch hands its fp32 kernels."""
    return float(np.float32(x))


def sgd_ref(p, g, lr):
    return torch.add(p, torch.mul(g, f32(-lr)))


def ema_ref(t, p, alpha):
    return torch.add(torch.mul(t, f32(alpha)), torch.mul(p, f32(1.0 - alpha)))


def adam_ref(p, g, m, v, t, lr, betas, eps, step, alpha=0.1, gscale=1.0):
    """torch's single-tensor Adam (lerp_, mul_ + addcmul_, sqrt / bias_correction2_sqrt + eps, addcdiv_) op by op in fp32,
    then the EMA teacher on the new weights (t None: no teacher).  Returns (p, m, v, t)."""
    beta1, beta2 = betas
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    w1 = f32(1.0 - beta1)
    g = torch.mul(g, f32(gscale))
    diff = torch.sub(g, m)
    # ATen's lerp: w < 0.5 ? a + w (b - a) : b - (b - a)(1 - w), with 1 - w formed in fp32
    m = torch.add(m, torch.mul(diff, w1)) if w1 < 0.5 else torch.sub(g, torch.mul(diff, f32(1.0 - w1)))
    v = torch.add(torch.mul(v, f32(beta2)), torch.mul(torch.mul(g, f32(1.0 - beta2)), g))
    # ATen's vectorised CPU sqrt is not correctly rounded (a few elements in 10^3 are 1 ulp off); the fp64 square root of an
    # fp32 value, rounded to fp32, is
    denom = torch.add(torch.div(torch.sqrt(v.double()).float(), f32(math.sqrt(bc2))), f32(eps))
    p = torch.add(p, torch.mul(torch.div(m, denom), f32(-(lr / bc1))))
    return p, m, v, (None if t is None else ema_ref(t, p, alpha))


# The cosine feature test's sums against fp64 sums of the same fp32 inputs: |terms - fp64| <= TERMS_TOL * scale (sum |a_k b_k|,
# |a|^2, |b|^2).  Worst measured on an H100 80GB HBM3 (700 W) over test_gpu_step_kernels.py: 1.3e-7 (G = 8, b = 2).
# |delta(1 - cos)| from the device sums: worst measured 1.4e-7 (G = 8, b = 1); the fp32 cosine the loop tests adds up to 3e-8.
TERMS_TOL = 1e-6
COS_TOL = 1e-6


def selected(ll, prior_b):
    """The component each body's GPU prior value belongs to: the fp64 component value closest to it."""
    return (ll.detach() - prior_b.double().cpu()[:, None]).abs().argmin(1)


# ------------------------------------------------------------------ rendering
COLOR = (205 / 255, 129 / 255, 98 / 255)
CAM = np.array([1.0, 1.0, 0.0, 0.0])
# frame sizes (H, W) the grouped input side and the grouped overlay cycle through
SIZES = [(240, 320), (1080, 1920), (720, 1280), (480, 640), (300, 400), (1080, 1920), (256, 256), (600, 800)]


def scene(G, seed):
    """G frames (sizes of SIZES, uint8 and float32 mixed) with boxes inside, partly outside and wholly outside the frame, and
    scales that up-scale (box smaller than 224) and down-scale."""
    rng = np.random.default_rng(seed)
    frames, centers, scales = [], [], []
    for g in range(G):
        H, W = SIZES[(g + seed) % len(SIZES)]
        img = rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8)
        t = torch.from_numpy(img).cuda()
        frames.append(t if g % 2 == 0 else t.float())
        kind = (g + seed) % 4
        if kind == 0:
            c, s = [W / 2 + rng.uniform(-20, 20), H / 2 + rng.uniform(-20, 20)], min(H, W) / 200 * rng.uniform(0.3, 0.9)
        elif kind == 1:
            c, s = [rng.uniform(0, 0.1) * W, rng.uniform(0.9, 1.0) * H], min(H, W) / 200 * 0.8
        elif kind == 2:
            c, s = [W + 300.0, -250.0], 1.2                                  # wholly outside: zeros
        else:
            c, s = [rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H], 0.5  # 100-pixel box: up-scales
        centers.append(c)
        scales.append(s)
    return frames, centers, scales


# |GPU crop - oracle| of a 1080p uint8 frame (test_dataprocess.py), the bound of every scene() frame
CROP_TOL = 3e-5


def crop_kind(frame, center, scale):
    """How the box of ``center`` / ``scale`` meets the (H, W, 3) frame: 'outside' (no pixel of the frame), 'partial' or
    'inside', and whether the crop is resized 'up' (smaller than 224 pixels) or 'down'."""
    from dynaboa_b200 import dataprocess as D
    H, W = frame.shape[:2]
    ul_x, ul_y, Wc, Hc = D._box(center, scale, (224, 224))
    if ul_x >= W or ul_y >= H or ul_x + Wc <= 0 or ul_y + Hc <= 0:
        where = 'outside'
    else:
        where = 'inside' if ul_x >= 0 and ul_y >= 0 and ul_x + Wc <= W and ul_y + Hc <= H else 'partial'
    return where, 'up' if Hc < 224 else ('down' if Hc > 224 else 'same')


def crop_oracle(frame, center, scale):
    """oracle/dataprocess_ref.py's normalised (3, 224, 224) crop of a device frame, in fp64 from its float32 values.  A box
    that misses the frame crops zeros; the reference's slicing cannot express an empty overlap, so that crop is the oracle's
    crop of a zero frame of the same size through a box inside it."""
    from oracle import dataprocess_ref as R
    img = frame.float().cpu().numpy()
    if crop_kind(frame, center, scale)[0] == 'outside':
        H, W = img.shape[:2]
        return R.rgb_processing(np.zeros_like(img), [W / 2, H / 2], scale)
    return R.rgb_processing(img, center, scale)


def px_verts(pts, W, H):
    """Vertices whose window position is (u, r) pixels and whose ndc_z is d, under cam4 = (1, 1, 0, 0) and no rotation."""
    pts = np.asarray(pts, dtype=np.float64)
    return np.stack([2 * pts[:, 0] / W - 1, 2 * pts[:, 1] / H - 1, pts[:, 2]], 1).astype(np.float32)


def quad(x0, y0, x1, y1, d, first=0, flip=False):
    """Two front-facing triangles (image-space signed area < 0) sharing the diagonal (x0, y0)-(x1, y1)."""
    pts = [(x0, y0, d), (x1, y0, d), (x1, y1, d), (x0, y1, d)]
    f = [[0, 3, 2], [0, 2, 1]]
    if flip:
        f = [[a, c, b] for a, b, c in f]
    return pts, (np.array(f) + first).tolist()


def frame(H, W, seed=0):
    return np.random.default_rng(seed).integers(0, 256, size=(H, W, 3), dtype=np.uint8)


def gpu_draw(img, verts, faces, cam4, rot=None, color=COLOR, samples=4):
    from dynaboa_b200 import render
    out, ids = render.draw(torch.from_numpy(img).cuda(), torch.as_tensor(verts).cuda(), faces, cam4, rot=rot, color=color,
                           samples=samples, face_ids=True)
    return out.cpu().numpy(), ids.cpu().numpy()


def check_against_oracle(img, verts, faces, cam4, rot=None, color=COLOR, samples=4, min_covered=1):
    from oracle import render_ref
    out, ids = gpu_draw(img, verts, faces, cam4, rot, color, samples)
    ref_out, ref_ids = render_ref.render(img, np.asarray(verts), faces, cam4, rot=rot, color=color, samples=samples)
    mism = ids != ref_ids
    assert not mism.any(), f'{mism.sum()} samples pick a different face than the oracle, first at {np.argwhere(mism)[0]}'
    covered = (ids >= 0).any(2)
    assert covered.sum() >= min_covered
    assert np.array_equal(out[~covered], img[~covered])
    diff = np.abs(out.astype(int) - ref_out.astype(int))[covered]
    assert diff.max() <= 1, f'byte differs by {diff.max()}'
    return out, ids


def sphere(n_lat=24, n_lon=48, radius=0.6):
    """Closed UV sphere, faces wound counter-clockwise seen from outside."""
    v = [(0.0, 0.0, radius)]
    for i in range(1, n_lat):
        th = np.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * np.pi * j / n_lon
            v.append((radius * np.sin(th) * np.cos(ph), radius * np.sin(th) * np.sin(ph), radius * np.cos(th)))
    v.append((0.0, 0.0, -radius))
    f, last = [], len(v) - 1
    ring = lambda i, j: 1 + (i - 1) * n_lon + (j % n_lon)
    for j in range(n_lon):
        f.append((0, ring(1, j), ring(1, j + 1)))
        f.append((last, ring(n_lat - 1, j + 1), ring(n_lat - 1, j)))
    for i in range(1, n_lat - 1):
        for j in range(n_lon):
            f.append((ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)))
            f.append((ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)))
    return np.array(v, dtype=np.float32), np.array(f, dtype=np.int64)


def posed_smpl_mesh():
    """The synthetic SMPL mesh posed by an HMR forward of the synthetic base model on a seeded image, as (device vertices, faces,
    cam4), cam4 the camera of a 400-pixel crop of a 1920 x 1080 frame (a fixed crop camera: the random-weight regressor's own
    camera is arbitrary).  Reads the synthetic asset directory ``config.set_data_root`` points at."""
    from dynaboa_b200 import config, render, synthetic
    from dynaboa_b200.hmr import hmr
    from dynaboa_b200.smpl import SMPL
    from oracle import hmr_ref
    m = hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    x = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    with torch.no_grad():
        rot, shape, _ = m(x)
        smpl = SMPL(config.SMPL_MODEL_DIR, create_transl=False).cuda()
        verts = smpl(betas=shape, body_pose=rot[:, 1:], global_orient=rot[:, 0].unsqueeze(1), pose2rot=False).vertices[0].contiguous()
    cam4 = render.convert_crop_cam_to_orig_img(np.array([[0.9, 0.05, 0.1]]), np.array([[900.0, 560.0, 400.0]]), 1920, 1080)[0]
    return verts, render.get_smpl_faces(), cam4


# ------------------------------------------------------------------ the unchanged Internet driver
DRIVER = os.path.join(ref_harness.REF or '', 'dynaboa_internet.py')
SHADOWED = ('constants', 'config', 'model', 'utils', 'base_adaptor', 'boa_dataset', 'learn2learn')
FLAGS = dict(inner_step=1, retrieval=0, lower_level_mixtrain=0, upper_level_mixtrain=0, dynamic_boa=0)
N = 3


def make_video(root):
    """N frames 240 x 320 (smooth content, moving box), 49 keypoints projected inside the box, reference npz layout."""
    import cv2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    rng = np.random.default_rng(11)
    base = cv2.GaussianBlur(rng.uniform(0, 255, size=(240, 320, 3)).astype(np.float32), (0, 0), 3)
    names, centers, scales, parts, frames = [], [], [], [], []
    for t in range(N):
        frame = np.clip(np.roll(base, 3 * t, axis=1) + rng.normal(0, 2, base.shape), 0, 255).astype(np.uint8)
        name = f'f{t:03d}.png'
        cv2.imwrite(os.path.join(root, 'images', name), frame[:, :, ::-1])
        center, scale = np.array([150.0 + 4 * t, 118.0 + t]), 0.9 + 0.01 * t
        kp = np.concatenate([center + rng.uniform(-70, 70, size=(49, 2)), np.ones((49, 1))], 1)
        names.append(name); centers.append(center); scales.append(scale); parts.append(kp); frames.append(frame)
    np.savez(os.path.join(root, 'video.npz'), imgname=np.array(names), center=np.stack(centers), scale=np.array(scales), part=np.stack(parts))
    return frames, centers, scales, parts
