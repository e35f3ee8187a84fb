"""Parameter table of the HMR regressor (names, shapes, order).

Single Python-side statement of the state_dict contract of reference
model/hmr.py:67-124 (``HMR.__init__`` / ``_make_layer``) and SURVEY.md §8(a1):
169 parameter tensors, 26 977 501 scalars, in module-registration order, plus
the three ``init_*`` buffers.  The CUDA library holds the same table
(csrc/hmr_plan.cu) and ``tests/test_layout.py`` checks they agree.

``ArenaLayout`` is that table as the library stores it (offset, logical shape and strides of every
parameter inside the one flat fp32 arena); ``state_dict`` maps an arena to named tensors with it, the
mapping ``HMR``'s parameters use, and ``digest`` fingerprints it for saved states (state.py).
"""
import ctypes as C
import hashlib
from collections import OrderedDict

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
