"""Parameter table of the HMR regressor (names, shapes, order).

Single Python-side statement of the state_dict contract of reference
model/hmr.py:67-124 (``HMR.__init__`` / ``_make_layer``) and SURVEY.md §8(a1):
169 parameter tensors, 26 977 501 scalars, in module-registration order, plus
the three ``init_*`` buffers.  The CUDA library holds the same table
(csrc/hmr_plan.cu) and ``tests/test_layout.py`` checks they agree.

``ArenaLayout`` is that table as the library stores it (offset, logical shape and strides of every
parameter inside the one flat fp32 arena); ``state_dict`` maps an arena to named tensors with it, the
mapping ``HMR``'s parameters use, ``arena_from_state_dict`` maps them back, ``read_checkpoint`` reads and checks a
checkpoint file into an arena for a pool slot, and ``digest`` fingerprints the table for saved states (state.py).
"""
import ctypes as C
import hashlib
from collections import OrderedDict

import torch

BLOCKS = (3, 4, 6, 3)            # reference model/hmr.py:322  hmr() -> HMR(Bottleneck, [3, 4, 6, 3])
PLANES = (64, 128, 256, 512)
EXPANSION = 4
GN_GROUPS = 4                    # reference model/hmr.py:18  nn.GroupNorm(32 // 8, planes)
GN_EPS = 1e-5
NPOSE = 24 * 6
FEAT_DIM = 2048
HEAD_IN = FEAT_DIM + NPOSE + 10 + 3   # 2205
HEAD_HID = 1024
N_ITER = 3


def conv_specs():
    """Yield (name_prefix, norm_prefix, cin, cout, k, stride, pad, hin) for all 53 convs
    in forward order (stem; per block conv1, conv2, conv3, [downsample])."""
    specs = [('conv1', 'bn1', 3, 64, 7, 2, 3, 224)]
    inplanes, h = 64, 56
    for li, (nblk, planes) in enumerate(zip(BLOCKS, PLANES)):
        lstride = 1 if li == 0 else 2
        for bi in range(nblk):
            s = lstride if bi == 0 else 1
            pre = f'layer{li + 1}.{bi}'
            specs.append((f'{pre}.conv1', f'{pre}.bn1', inplanes, planes, 1, 1, 0, h))
            specs.append((f'{pre}.conv2', f'{pre}.bn2', planes, planes, 3, s, 1, h))
            hout = h // s
            specs.append((f'{pre}.conv3', f'{pre}.bn3', planes, planes * EXPANSION, 1, 1, 0, hout))
            if bi == 0:
                specs.append((f'{pre}.downsample.0', f'{pre}.downsample.1', inplanes,
                              planes * EXPANSION, 1, s, 0, h))
            inplanes, h = planes * EXPANSION, hout
    return specs


def param_shapes():
    """OrderedDict name -> shape, in ``nn.Module.parameters()`` order of the reference."""
    out = OrderedDict()
    specs = conv_specs()
    i = 0
    # stem
    name, norm, cin, cout, k, *_ = specs[i]
    out[f'{name}.weight'] = (cout, cin, k, k)
    out[f'{norm}.weight'] = (cout,)
    out[f'{norm}.bias'] = (cout,)
    i += 1
    while i < len(specs):
        name, norm, cin, cout, k, *_ = specs[i]
        out[f'{name}.weight'] = (cout, cin, k, k)
        out[f'{norm}.weight'] = (cout,)
        out[f'{norm}.bias'] = (cout,)
        i += 1
    for lin, (n, kdim) in (('fc1', (HEAD_HID, HEAD_IN)), ('fc2', (HEAD_HID, HEAD_HID)),
                           ('decpose', (NPOSE, HEAD_HID)), ('decshape', (10, HEAD_HID)),
                           ('deccam', (3, HEAD_HID))):
        out[f'{lin}.weight'] = (n, kdim)
        out[f'{lin}.bias'] = (n,)
    return out


def buffer_shapes():
    return OrderedDict(init_pose=(1, NPOSE), init_shape=(1, 10), init_cam=(1, 3))


def num_params():
    n = 0
    for shp in param_shapes().values():
        c = 1
        for d in shp:
            c *= d
        n += c
    return n


# feature list layout of HMR.forward(need_feature=True): reference model/hmr.py:138-168
FEATURE_NAMES = ['stem_conv', 'layer1', 'layer2', 'layer3', 'layer4', 'pooled',
                 'fc1_it0', 'drop1_it0', 'fc2_it0', 'fc1_it1', 'drop1_it1', 'fc2_it1',
                 'fc1_it2', 'drop1_it2', 'fc2_it2']


class ArenaLayout:
    """Parameter table queried from the library (names, offsets, logical shapes, strides)."""

    def __init__(self):
        from . import _lib
        lib = _lib.load()
        self.n = lib.dboa_hmr_num_params()
        self.floats = lib.dboa_hmr_arena_floats()
        self.names, self.offsets, self.shapes, self.strides = [], [], [], []
        name = C.create_string_buffer(128)
        off, nd = C.c_longlong(), C.c_int()
        shp, strd = (C.c_longlong * 4)(), (C.c_longlong * 4)()
        for i in range(self.n):
            _lib.check(lib.dboa_hmr_param_info(i, name, 128, C.byref(off), C.byref(nd), shp, strd), 'dboa_hmr_param_info')
            self.names.append(name.value.decode())
            self.offsets.append(off.value)
            self.shapes.append(tuple(shp[k] for k in range(nd.value)))
            self.strides.append(tuple(strd[k] for k in range(nd.value)))

    def views(self, flat):
        return [flat.as_strided(s, st, o) for s, st, o in zip(self.shapes, self.strides, self.offsets)]


_LAYOUT = None


def arena_layout():
    """The library's ``ArenaLayout``, queried once."""
    global _LAYOUT
    if _LAYOUT is None:
        _LAYOUT = ArenaLayout()
    return _LAYOUT


def digest():
    """sha256 of the arena's parameter table (name, shape, offset and strides of every parameter, the arena size) and of the
    buffer shapes: two arenas with the same digest hold the same parameter at the same place."""
    lay = arena_layout()
    rows = [lay.floats] + list(zip(lay.names, lay.shapes, lay.offsets, lay.strides)) + list(buffer_shapes().items())
    return hashlib.sha256(repr(rows).encode()).hexdigest()


def state_dict(arena, buffers, prefix=''):
    """The reference's state_dict of the weights in the flat ``arena``: ``prefix + name`` -> a contiguous copy of each of the
    169 parameters (the ``HMR`` parameter views of the arena), then the ``init_*`` buffers of ``buffers``, on the host."""
    lay = arena_layout()
    if arena.dim() != 1 or arena.numel() != lay.floats:
        raise ValueError(f'expected a flat arena of {lay.floats} floats, got shape {tuple(arena.shape)}')
    def own(t):                       # a host tensor with a storage of its own (a saved view would carry the whole arena)
        t = t.detach().contiguous()
        return t.cpu() if t.is_cuda else t.clone()
    out = OrderedDict((prefix + n, own(v)) for n, v in zip(lay.names, lay.views(arena)))
    for k in buffer_shapes():
        out[prefix + k] = own(buffers[k])
    return out


def arena_from_state_dict(sd, out, prefix=''):
    """The inverse of ``state_dict``: each of the 169 parameters ``sd[prefix + name]`` copied into its view of the flat arena
    ``out`` (cast to fp32 as ``load_state_dict`` does; the arena's padding is not written).  Returns ``out``."""
    lay = arena_layout()
    if out.dim() != 1 or out.numel() != lay.floats or out.dtype != torch.float32:
        raise ValueError(f'expected a flat fp32 arena of {lay.floats} floats, got {out.dtype} of shape {tuple(out.shape)}')
    for n, v in zip(lay.names, lay.views(out)):
        v.copy_(sd[prefix + n])
    return out


def read_checkpoint(path, buffers):
    """A checkpoint in the reference's format (``{'model': {'module.<name>': tensor}}``: what ``export_model`` writes and
    ``model_file`` names) read into a host arena and checked against the pool whose ``init_*`` buffers are ``buffers``.
    Returns (the (P,) fp32 host arena, its digest).  The arena is zero outside the parameters, as the arena of a model loaded
    with ``load_state_dict``.

    Every check runs on the host and raises ValueError naming the file and the key: a file that is no readable checkpoint, a
    missing or extra key (strict, as ``load_state_dict(strict=True)``), a shape other than ``param_shapes()`` /
    ``buffer_shapes()``, a value that is not finite float data, ``init_*`` buffers that differ in any bit from ``buffers`` (the
    grouped forward reads one buffer set for every video).  The digest is the sha256 of the arena's and the buffers' bytes:
    two files with the same weights are one model, whatever their path, pickling or key order."""
    try:
        obj = torch.load(path, map_location='cpu', weights_only=True)
    except Exception as e:                                     # missing, truncated, not a torch file, or a pickled object
        raise ValueError(f'{path}: not a readable checkpoint: {type(e).__name__}: {e}') from None
    sd = obj.get('model') if isinstance(obj, dict) else None
    if not isinstance(sd, dict):
        raise ValueError(f'{path}: not a checkpoint: expected a dict with a \'model\' state dict, got {type(obj).__name__}'
                         + (f' with keys {sorted(map(str, obj))[:8]}' if isinstance(obj, dict) else ''))
    want = OrderedDict(('module.' + k, s) for k, s in list(param_shapes().items()) + list(buffer_shapes().items()))
    missing, extra = [k for k in want if k not in sd], sorted(str(k) for k in sd if k not in want)
    if missing:
        raise ValueError(f'{path}: missing key {missing[0]!r}' + (f' and {len(missing) - 1} more' if len(missing) > 1 else ''))
    if extra:
        raise ValueError(f'{path}: unexpected key {extra[0]!r}' + (f' and {len(extra) - 1} more' if len(extra) > 1 else ''))
    for k, shp in want.items():
        t = sd[k]
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise ValueError(f'{path}: {k} is not float data ({type(t).__name__}{"" if not isinstance(t, torch.Tensor) else " " + str(t.dtype)})')
        if tuple(t.shape) != tuple(shp):
            raise ValueError(f'{path}: {k} has shape {tuple(t.shape)}, expected {tuple(shp)}')
        if not bool(torch.isfinite(t).all()):
            raise ValueError(f'{path}: {k} holds values that are not finite')
    for k in buffer_shapes():
        mine, pool = sd['module.' + k].float().contiguous(), buffers[k].detach().float().cpu().contiguous()
        if not torch.equal(mine.view(torch.int32), pool.view(torch.int32)):
            raise ValueError(f'{path}: module.{k} differs from the pool\'s {k}: every slot reads the pool\'s init_* buffers')
    arena = arena_from_state_dict(sd, torch.zeros(arena_layout().floats, dtype=torch.float32), prefix='module.')
    return arena, arena_digest(arena, buffers)


def arena_digest(arena, buffers):
    """sha256 of a flat arena's bytes and of the ``init_*`` buffers': the identity of a model (``read_checkpoint``)."""
    h = hashlib.sha256(arena.detach().float().cpu().contiguous().numpy().tobytes())
    for k in buffer_shapes():
        h.update(buffers[k].detach().float().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()
