"""HMR regressor (GroupNorm ResNet-50 + iterative SMPL-parameter head) on the CUDA library.

Drop-in for reference model/hmr.py: ``hmr(smpl_mean_params)`` (:314-323) returns an ``nn.Module`` whose
``state_dict`` names/shapes, ``parameters()`` order and ``forward`` signature/returns (:127-181) match the
reference, so ``load_state_dict(ckpt['model'], strict=True)`` and the unchanged driver work.

GPU-first design: all 169 parameters are strided views of ONE flat fp32 arena (conv weights stored
[Cout][kh][kw][Cin] for K-major GEMM tiles, fc1 rows padded to 2208 for 16-byte row pitch), so the
inner SGD step, Adam, the EMA teacher and the gradient all-reduce are single sweeps.  The forward and the
hand-written backward are single C-ABI calls (``dboa_hmr_forward`` / ``dboa_hmr_backward``); torch autograd
only sees one ``Function`` node per forward.
"""
import ctypes as C
import math
import weakref

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import ptr, stream
from .layout import ArenaLayout, arena_layout as layout  # noqa: F401  (the arena's parameter table)

# callable(B, device) -> (3,2,B,1024) scaled keep-masks used by every HMR in train mode that has no mask_provider of its own
# (parity tests replay the reference's recorded teacher dropout masks through the UNCHANGED driver this way)
DEFAULT_MASK_PROVIDER = None


_FEATURE_INFO = {}
_TAPE_FLOATS = {}
_SCRATCH = {}


def _feature_views(tape, B):
    if B not in _FEATURE_INFO:
        lib = _lib.load()
        off, nd = C.c_longlong(), C.c_int()
        shp, strd = (C.c_longlong * 4)(), (C.c_longlong * 4)()
        info = []
        for i in range(15):
            _lib.check(lib.dboa_hmr_feature_info(B, i, C.byref(off), C.byref(nd), shp, strd), 'dboa_hmr_feature_info')
            info.append((off.value, tuple(shp[k] for k in range(nd.value)), tuple(strd[k] for k in range(nd.value))))
        _FEATURE_INFO[B] = info
    return [tape.as_strided(s, st, o) for o, s, st in _FEATURE_INFO[B]]


def tape_floats(B):
    if B not in _TAPE_FLOATS:
        _TAPE_FLOATS[B] = _lib.load().dboa_hmr_tape_floats(B)
        if _TAPE_FLOATS[B] < 0:
            raise RuntimeError(f'unsupported batch size {B} (1..64)')
    return _TAPE_FLOATS[B]


# region kinds of dboa_hmr_tape_offset (include/dynaboa_b200.h, DBOA_TAPE_*)
TAPE_Y, TAPE_STATS, TAPE_A = 0, 1, 2
TAPE_WHOLE = {'x0': 3, 'p0': 4, 'p0_idx': 5, 'xc': 6, 'h1pre': 7, 'h1post': 8, 'h2pre': 9, 'h2post': 10, 'params': 11, 'masks': 12}


def conv_geometry():
    """Per convolution i (weight = parameter 3*i): (name, Cin, Cout, k, stride, Hout), from the parameter table and the
    ResNet-50 rule that the first block of layers 2..4 downsamples in its conv2 and its shortcut."""
    lay = layout()
    out = []
    for i in range(0, lay.n - 10, 3):
        name = lay.names[i][:-len('.weight')]
        cout, cin, k, _ = lay.shapes[i]
        if name == 'conv1':
            out.append((name, cin, cout, k, 2, 112))
            continue
        li, bi, part = int(name[5]), int(name.split('.')[1]), name.split('.')[2]
        down = li > 1 and bi == 0
        stride = 2 if down and part in ('conv2', 'downsample') else 1
        out.append((name, cin, cout, k, stride, 56 >> (li - 2 if down and part == 'conv1' else li - 1)))
    return out


def tape_views(tape, B):
    """Named NHWC views of a forward's tape (dboa_hmr_tape_offset): 'y', 'stats', 'a' are lists over the 53 convolutions
    ('a' is None for the downsample convs), plus the whole-tape regions.  'p0_idx' is a uint8 view."""
    lib = _lib.load()

    def off(kind, conv=0):
        o = lib.dboa_hmr_tape_offset(B, kind, conv)
        if o < 0:
            raise RuntimeError(f'dboa_hmr_tape_offset({B}, {kind}, {conv}) failed: {o}')
        return o

    def view(o, shape):
        return tape.as_strided(shape, [math.prod(shape[d + 1:]) for d in range(len(shape))], o)
    v = {'y': [], 'stats': [], 'a': []}
    for i, (name, _, cout, _, _, h) in enumerate(conv_geometry()):
        v['y'].append(view(off(TAPE_Y, i), (B, h, h, cout)))
        v['stats'].append(view(off(TAPE_STATS, i), (B, 4, 2)))
        v['a'].append(None if 'downsample' in name else view(off(TAPE_A, i), (B, h, h, cout)))
    v['x0'] = view(off(TAPE_WHOLE['x0']), (B, 224, 224, 3))
    v['p0'] = view(off(TAPE_WHOLE['p0']), (B, 56, 56, 64))
    n = B * 56 * 56 * 64
    v['p0_idx'] = tape.view(torch.uint8)[4 * off(TAPE_WHOLE['p0_idx']):][:n].view(B, 56, 56, 64)
    v['xc'] = view(off(TAPE_WHOLE['xc']), (3, B, 2208))
    for k in ('h1pre', 'h1post', 'h2pre', 'h2post'):
        v[k] = view(off(TAPE_WHOLE[k]), (3, B, 1024))
    v['params'] = view(off(TAPE_WHOLE['params']), (4, B, 160))
    v['masks'] = view(off(TAPE_WHOLE['masks']), (3, 2, B, 1024))
    return v


def scratch_for(B, device):
    """Per-(device, B, stream) scratch shared by forward and backward; stream-ordered reuse is safe, and forwards
    issued concurrently on different streams (teacher next to the fast-weight forward) get separate buffers."""
    key = (device.index, B, torch.cuda.current_stream(device).cuda_stream)
    if key not in _SCRATCH:
        _SCRATCH[key] = torch.empty(_lib.load().dboa_hmr_scratch_floats(B), dtype=torch.float32, device=device)
    return _SCRATCH[key]


def _check_groups(arena, B, groups):
    if groups < 1 or B % groups:
        raise ValueError(f'{B} samples do not split into {groups} videos')
    if groups > 1 and (not arena.is_contiguous() or arena.numel() != groups * layout().floats):
        raise ValueError(f'a grouped call needs one contiguous ({groups}, {layout().floats}) arena stack')


def raw_forward(arena, buffers, image, masks=None, tape=None, groups=1, active=None):
    """One ``dboa_hmr_forward_active`` call.  Returns (rotmat, shape, cam, pose6d, tape).  No autograd.

    ``groups`` > 1: ``arena`` is a (groups, P) stack, and video g's weights ``arena[g]`` see the samples
    [g * B / groups, (g + 1) * B / groups) of ``image`` (and of ``masks`` and the outputs).  ``active``: an int whose bit g
    means video g takes part; the rows of the other videos are left unspecified.  None: all."""
    _lib.require_cuda(arena, image)
    B = image.shape[0]
    if tuple(image.shape[1:]) != (3, 224, 224):
        raise ValueError(f'HMR expects (B,3,224,224) images, got {tuple(image.shape)}')
    _check_groups(arena, B, groups)
    image = image.contiguous().float()
    dev = image.device
    if tape is None:
        tape = torch.empty(tape_floats(B), dtype=torch.float32, device=dev)
    rot = torch.empty(B, 24, 3, 3, dtype=torch.float32, device=dev)
    shape = torch.empty(B, 10, dtype=torch.float32, device=dev)
    cam = torch.empty(B, 3, dtype=torch.float32, device=dev)
    pose6d = torch.empty(B, 144, dtype=torch.float32, device=dev)
    if masks is not None:
        masks = masks.contiguous().float()
        if tuple(masks.shape) != (3, 2, B, 1024):
            raise ValueError('dropout masks must be (3,2,B,1024)')
    args = (ptr(arena), ptr(buffers['init_pose']), ptr(buffers['init_shape']), ptr(buffers['init_cam']), ptr(image), B, ptr(masks),
            ptr(tape), ptr(scratch_for(B, dev)), ptr(rot), ptr(shape), ptr(cam), ptr(pose6d), stream(), groups)
    _lib.call('dboa_hmr_forward_active', *args, (1 << groups) - 1 if active is None else int(active))
    return rot, shape, cam, pose6d, tape


def raw_backward(arena, tape, B, masked, d_rot, d_shape, d_cam, grad_arena, groups=1, active=None):
    """One ``dboa_hmr_backward_active`` call: accumulates into ``grad_arena`` (flat, arena layout).  ``groups`` > 1: ``arena``
    and ``grad_arena`` are both (groups, P) stacks (see ``raw_forward``).  ``active``: as in ``raw_forward``; the gradient
    arenas of the other videos are not written."""
    _check_groups(arena, B, groups)
    _check_groups(grad_arena, B, groups)
    c = lambda t: None if t is None else t.contiguous().float()
    d_rot, d_shape, d_cam = c(d_rot), c(d_shape), c(d_cam)
    args = (ptr(arena), ptr(tape), B, int(masked), ptr(d_rot), ptr(d_shape), ptr(d_cam), ptr(grad_arena), ptr(scratch_for(B, tape.device)),
            stream(), groups)
    _lib.call('dboa_hmr_backward_active', *args, (1 << groups) - 1 if active is None else int(active))


class _HMRFunction(torch.autograd.Function):
    """Autograd node of one forward.  ``weights`` is either the single flat fast-weight tensor of a MAML
    learner or the 169 leaf parameters (views of ``owner._arena``)."""

    @staticmethod
    def forward(ctx, image, masks, owner, flat_mode, *weights):
        arena = weights[0] if flat_mode else owner._arena
        if flat_mode and not arena.is_contiguous():
            raise RuntimeError('fast weights must be a contiguous flat arena')
        rot, shape, cam, _, tape = raw_forward(arena, owner._buffers, image, masks)
        ctx.arena, ctx.tape, ctx.B, ctx.masked, ctx.flat_mode = arena, tape, image.shape[0], masks is not None, flat_mode
        feats = _feature_views(tape, image.shape[0])
        ctx.mark_non_differentiable(*feats)
        return (rot, shape, cam) + tuple(feats)

    @staticmethod
    def backward(ctx, d_rot, d_shape, d_cam, *_):
        lay = layout()
        g = torch.zeros(lay.floats, dtype=torch.float32, device=ctx.tape.device)
        raw_backward(ctx.arena, ctx.tape, ctx.B, ctx.masked, d_rot, d_shape, d_cam, g)
        if ctx.flat_mode:
            return (None, None, None, None, g)
        return (None, None, None, None) + tuple(lay.views(g))


class _CloneArena(torch.autograd.Function):
    """learn2learn ``clone_module``: fast = clone(theta), with d fast / d theta = I routed to the 169 leaves."""

    @staticmethod
    def forward(ctx, owner, *params):
        return owner._arena.clone()

    @staticmethod
    def backward(ctx, g):
        return (None,) + tuple(layout().views(g.contiguous()))


class _SgdStep(torch.autograd.Function):
    """learn2learn ``maml_update`` with first-order gradients: out = fast + (-lr * g); d out / d fast = I."""

    @staticmethod
    def forward(ctx, fast, g, lr):
        out = torch.empty_like(fast)
        _lib.call('dboa_sgd_update', ptr(fast), ptr(g.contiguous()), ptr(out), float(lr), fast.numel(), stream())
        return out

    @staticmethod
    def backward(ctx, go):
        return go, None, None


class _Holder(nn.Module):
    """Name-space node so that state_dict keys follow the reference (conv1.weight, layer1.0.bn1.bias, ...)."""


class HMR(nn.Module):
    """SMPL iterative regressor with a GroupNorm(4) ResNet-50 backbone (reference model/hmr.py:63-181)."""

    def __init__(self, smpl_mean_params):
        super().__init__()
        lay = layout()
        self._lay = lay
        object.__setattr__(self, '_arena', torch.zeros(lay.floats, dtype=torch.float32))
        object.__setattr__(self, '_fast', None)          # flat fast weights when this instance is a MAML learner
        object.__setattr__(self, '_grad_arena', None)
        self.mask_provider = None                          # callable(B, device) -> (3,2,B,1024) scaled keep-masks
        self._param_list = []
        for name, view in zip(lay.names, lay.views(self._arena)):
            node, parts = self, name.split('.')
            for part in parts[:-1]:
                if part not in node._modules:
                    node.add_module(part, _Holder())
                node = node._modules[part]
            p = nn.Parameter(view)
            p._dboa_owner = weakref.ref(self)
            node.register_parameter(parts[-1], p)
            self._param_list.append(p)
        self._init_parameters()
        mean = np.load(smpl_mean_params) if isinstance(smpl_mean_params, str) else smpl_mean_params
        self.register_buffer('init_pose', torch.as_tensor(np.asarray(mean['pose'][:]), dtype=torch.float32).unsqueeze(0))
        self.register_buffer('init_shape', torch.as_tensor(np.asarray(mean['shape'][:]).astype('float32')).unsqueeze(0))
        self.register_buffer('init_cam', torch.as_tensor(np.asarray(mean['cam']), dtype=torch.float32).unsqueeze(0))

    # ------------------------------------------------------------------ construction helpers
    def _init_parameters(self):
        """Same distributions as the reference constructor (model/hmr.py:85-96 and nn defaults)."""
        with torch.no_grad():
            for name, p in zip(self._lay.names, self._param_list):
                head = name.split('.')[0]
                if p.dim() == 4:
                    cout, _, k, _ = p.shape
                    p.copy_(torch.randn(tuple(p.shape)) * math.sqrt(2.0 / (k * k * cout)))
                elif head in ('fc1', 'fc2'):
                    fan_in = 2205 if head == 'fc1' else 1024
                    p.copy_((torch.rand(tuple(p.shape)) * 2 - 1) / math.sqrt(fan_in))
                elif head in ('decpose', 'decshape', 'deccam'):
                    if p.dim() == 2:
                        bound = 0.01 * math.sqrt(6.0 / (p.shape[0] + p.shape[1]))
                    else:
                        bound = 1.0 / math.sqrt(1024)
                    p.copy_((torch.rand(tuple(p.shape)) * 2 - 1) * bound)
                elif name.endswith('weight'):
                    p.fill_(1.0)      # GroupNorm affine
                else:
                    p.zero_()

    def _rebind(self):
        for p, view in zip(self._param_list, self._lay.views(self._arena)):
            p.data = view
            p.grad = None
        object.__setattr__(self, '_grad_arena', None)

    def _apply(self, fn, recurse=True):
        new = fn(self._arena)
        if new.dtype != torch.float32:
            raise RuntimeError('HMR parameters are fp32 master weights; other dtypes are not supported')
        object.__setattr__(self, '_arena', new.contiguous())
        self._rebind()
        for k, b in self._buffers.items():
            if b is not None:
                self._buffers[k] = fn(b)
        return self

    # ------------------------------------------------------------------ flat access (optimiser / DP all-reduce)
    @property
    def arena(self):
        return self._arena

    def grad_arena(self):
        """Flat gradient arena; the ``.grad`` of every parameter is a view of it."""
        if self._grad_arena is None:
            g = torch.zeros_like(self._arena)
            object.__setattr__(self, '_grad_arena', g)
            for p, view in zip(self._param_list, self._lay.views(g)):
                p.grad = view
        return self._grad_arena

    # ------------------------------------------------------------------ forward
    def _masks(self, B, device):
        if not self.training:
            return None
        if self.mask_provider is not None:
            return self.mask_provider(B, device)
        if DEFAULT_MASK_PROVIDER is not None:
            return DEFAULT_MASK_PROVIDER(B, device)
        return (torch.rand(3, 2, B, 1024, device=device) >= 0.5).float() * 2.0      # nn.Dropout(p=0.5)

    def forward(self, x, need_feature=False, init_pose=None, init_shape=None, init_cam=None, n_iter=3):
        if init_pose is not None or init_shape is not None or init_cam is not None or n_iter != 3:
            raise NotImplementedError('the CUDA plan implements the reference call pattern: default init_*, n_iter=3')
        _lib.require_cuda(x, self._arena)
        masks = self._masks(x.shape[0], x.device)
        if self._fast is not None:
            out = _HMRFunction.apply(x, masks, self, True, self._fast)
        elif torch.is_grad_enabled() and any(p.requires_grad for p in self._param_list):
            out = _HMRFunction.apply(x, masks, self, False, *self._param_list)
        else:
            rot, shape, cam, _, tape = raw_forward(self._arena, self._buffers, x, masks)
            out = (rot, shape, cam) + tuple(_feature_views(tape, x.shape[0]))
        if need_feature:
            return out[0], out[1], out[2], list(out[3:])
        return out[0], out[1], out[2]

    # ------------------------------------------------------------------ MAML support (see maml.py)
    def clone_as_learner(self):
        """Structural copy sharing buffers whose weights are a differentiable clone of this model's arena."""
        new = HMR.__new__(HMR)
        new.__dict__ = self.__dict__.copy()
        new._parameters = dict(self._parameters)
        new._buffers = self._buffers           # shared, read-only
        base = self._fast if self._fast is not None else _CloneArena.apply(self, *self._param_list)
        if self._fast is not None:
            base = self._fast.clone()
        object.__setattr__(new, '_fast', base)
        return new

    def fast_parameters(self):
        return self._lay.views(self._fast)

    def parameters(self, recurse=True):
        if self._fast is not None:
            return iter(self.fast_parameters())
        return super().parameters(recurse)

    def named_parameters(self, prefix='', recurse=True, remove_duplicate=True):
        if self._fast is not None:
            return iter([(prefix + ('.' if prefix else '') + n, v) for n, v in zip(self._lay.names, self.fast_parameters())])
        return super().named_parameters(prefix, recurse, remove_duplicate)

    def sgd_step(self, grad_flat, lr):
        object.__setattr__(self, '_fast', _SgdStep.apply(self._fast, grad_flat, lr))


def hmr(smpl_mean_params, pretrained=False, **kwargs):
    """Constructs the HMR model (reference model/hmr.py:314-323; ``pretrained`` is accepted and ignored --
    ImageNet weights are never used by the reference drivers, which load data/basemodel.pt)."""
    return HMR(smpl_mean_params, **kwargs)
