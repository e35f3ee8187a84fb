"""The C-ABI library loads on a CPU-only machine and exports every symbol the public header declares; the ctypes binding
(signatures, struct mirrors, error codes, tape kinds) follows the header; the layout table the library reports matches the
Python-side statement of the reference's state_dict contract."""
import ctypes
import os
import re
import subprocess
from types import SimpleNamespace

import pytest

from dynaboa_b200 import _lib, hmr, layout
from harness import built_lib

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, 'include', 'dynaboa_b200.h')


@pytest.fixture(scope='module')
def lib():
    return built_lib()


# ------------------------------------------------------------------ the header, parsed
# ctypes does not notice a binding that disagrees with the header (a truncated long long, a double read as a float, a misplaced
# field), so the binding is checked against the header text.  The parser knows every C type the header uses and fails on any other,
# naming its entry, rather than skip it.  A C type is (base, pointer depth), const dropped.
SCALARS = {'int': ctypes.c_int, 'long long': ctypes.c_longlong, 'unsigned long long': ctypes.c_ulonglong, 'float': ctypes.c_float,
           'double': ctypes.c_double}
OPAQUE = {('dboa_stream_t', 0): ctypes.c_void_p, ('void', 1): ctypes.c_void_p, ('unsigned char', 1): ctypes.c_void_p,
          ('char', 1): ctypes.c_char_p}
MIRRORS = {'dboa_smpl_model': _lib.SmplModelStruct, 'dboa_loss_args': _lib.LossArgsStruct, 'dboa_fused_conv': _lib.FusedConvStruct,
           'dboa_dgrad_args': _lib.DgradFusedStruct, 'dboa_crop_desc': _lib.CropDescStruct, 'dboa_render_desc': _lib.RenderDescStruct}


def declaration(decl, entry, structs):
    """[(name, type, array length or None)] of one C declaration.  Declarators after a comma share the first one's base type, as
    in 'const float *x, *res, *w' or 'const float *prep_y[2], *prep_stats[2]'."""
    out, base = [], None
    for part in decl.split(','):
        toks = re.findall(r'\[\s*\d+\s*\]|\w+|\S', part)
        words = [t for t in toks if re.fullmatch(r'\w+', t)]
        arrays = [int(t[1:-1]) for t in toks if t[0] == '[']
        stars = toks.count('*')
        own = ' '.join(w for w in words[:-1] if w != 'const')
        base = own if base is None else base
        known = base in SCALARS and stars <= 2 or base in structs and stars == 1 or (base, stars) in OPAQUE
        if not known or (own and own != base) or len(words) + stars + len(arrays) != len(toks) or len(arrays) > 1:
            raise ValueError(f'{entry}: unknown C type or declarator {part.strip()!r}')
        out.append((words[-1], (base, stars), arrays[0] if arrays else None))
    return out


def parse_header(text):
    """The header text's prototypes (name -> (return type, [(parameter, type)]), an array parameter being a pointer), structs
    (name -> [(field, type, array length or None)]) and DBOA_OK / DBOA_ERR_* / DBOA_TAPE_* macros (name -> value)."""
    src = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    macros = {k: int(v) for k, v in re.findall(r'^\s*#\s*define\s+(DBOA_OK|DBOA_ERR_\w+|DBOA_TAPE_\w+)\s+\(?(-?\d+)\)?\s*$', src, re.M)}
    src = re.sub(r'^\s*#.*$', '', src, flags=re.M)
    structs = {}
    for body, name in re.findall(r'typedef\s+struct\s+\w*\s*\{([^{}]*)\}\s*(\w+)\s*;', src):
        structs[name] = [f for decl in body.split(';') if decl.strip() for f in declaration(decl, name, structs)]
    src = re.sub(r'typedef\s+struct\s+\w*\s*\{[^{}]*\}\s*\w+\s*;', ';', src)
    protos = {}
    for head, params in re.findall(r'([^;{}()]*\bdboa_\w+)\s*\(([^()]*)\)\s*;', src):
        (name, ret, _), = declaration(head, re.search(r'dboa_\w+$', head).group(), structs)
        decls = [] if params.strip() == 'void' else [declaration(p, name, structs)[0] for p in params.split(',')]
        protos[name] = (ret, [(arg, (base, stars + (n is not None))) for arg, (base, stars), n in decls])
    missed = set(re.findall(r'\b(dboa_\w+)\s*\(', src)) - set(protos)
    if missed:
        raise ValueError(f'not read as prototypes: {sorted(missed)}')
    return SimpleNamespace(protos=protos, structs=structs, macros=macros)


def binding_ctypes(t):
    """The ctypes a parameter or return value of C type t may be bound as.  The header does not say which pointers are host and
    which device pointers, so a pointer to a scalar may be c_void_p or a typed POINTER; a struct pointer must be its mirror's."""
    base, stars = t
    if t in OPAQUE:
        return [OPAQUE[t]]
    if base in MIRRORS:
        return [ctypes.POINTER(MIRRORS[base])]
    if stars == 0:
        return [SCALARS[base]]
    return [ctypes.c_void_p, ctypes.POINTER(SCALARS[base] if stars == 1 else ctypes.c_void_p)]


def field_ctype(t, n):
    ct = SCALARS[t[0]] if t[1] == 0 else ctypes.c_void_p
    return ct if n is None else ct * n


@pytest.fixture(scope='module')
def header():
    return parse_header(open(HEADER).read())


@pytest.fixture(scope='module')
def c_layout(header, tmp_path_factory):
    """{struct: {field: (offsetof, sizeof), 'struct': (sizeof, _Alignof)}} of every header struct, printed by one C program
    compiled against the header (no CUDA needed)."""
    rows = [f'"{s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s} *)0)->{f})' for s in header.structs for f, _, _ in header.structs[s]]
    rows += [f'"{s} struct %zu %zu\\n", sizeof({s}), _Alignof({s})' for s in header.structs]
    d = tmp_path_factory.mktemp('layout')
    (d / 'layout.c').write_text('#include <stddef.h>\n#include <stdio.h>\n#include "dynaboa_b200.h"\nint main(void) {\n'
                                + ''.join(f'    printf({r});\n' for r in rows) + '    return 0;\n}\n')
    subprocess.check_call(['gcc', '-I', os.path.dirname(HEADER), str(d / 'layout.c'), '-o', str(d / 'layout')])
    out = {}
    for row in subprocess.check_output([str(d / 'layout')], text=True).splitlines():
        s, f, a, b = row.split()
        out.setdefault(s, {})[f] = (int(a), int(b))
    return out


def test_header_symbols_exported(lib, header):
    syms = sorted(header.protos)
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/dynaboa_b200.h but not exported'
    assert set(syms) == set(_lib.SIGNATURES), 'ctypes signature table out of sync with the header'


def test_signatures_follow_the_header(header):
    for name, (ret, params) in header.protos.items():
        res, args = _lib.SIGNATURES[name]
        assert res in binding_ctypes(ret), (name, 'returns', ret, res)
        assert len(args) == len(params), (name, f'{len(args)} argtypes for {len(params)} parameters')
        for (arg, t), a in zip(params, args):
            assert a in binding_ctypes(t), (name, arg, t, a)


def test_structs_follow_the_header(header, c_layout):
    """Every struct's mirror has the header's fields in order, each of the header's type (scalars exactly, pointers as c_void_p,
    T x[N] as ctype(T) * N) and at the compiled offset and size; the struct's size and alignment are the compiled ones."""
    assert set(header.structs) == set(MIRRORS)
    for name, fields in header.structs.items():
        m, c = MIRRORS[name], c_layout[name]
        want = [(f, field_ctype(t, n), c[f]) for f, t, n in fields]
        got = [(f, ct, (getattr(m, f).offset, getattr(m, f).size)) for f, ct in m._fields_]
        assert got + [(ctypes.sizeof(m), ctypes.alignment(m))] == want + [c['struct']], name
    for name in ('dboa_crop_desc', 'dboa_render_desc'):       # 64 of them go by value in the 32 KB kernel parameter space
        assert 64 * c_layout[name]['struct'][0] < 32 * 1024, name


def test_constants_follow_the_header(header):
    m = header.macros
    assert m['DBOA_OK'] == 0
    assert _lib._ERRORS == {v: k for k, v in m.items() if k.startswith('DBOA_ERR_')}
    tape = {k[len('DBOA_TAPE_'):].lower(): v for k, v in m.items() if k.startswith('DBOA_TAPE_')}
    assert dict(y=hmr.TAPE_Y, stats=hmr.TAPE_STATS, a=hmr.TAPE_A, **hmr.TAPE_WHOLE) == tape


def test_grouped_entries_extend_the_one_video_entries(header):
    """Every grouped or masked entry point is its one-video or grouped entry with the grouping arguments added (types only),
    and returns a status; the per-frame parameters of the one-frame crop lead its parameter list in the descriptor's order."""
    sig = {name: [t for _, t in params] for name, (_, params) in header.protos.items()}
    INT, ULL, STREAM = ('int', 0), ('unsigned long long', 0), ('dboa_stream_t', 0)
    extends = {'dboa_hmr_forward_groups': sig['dboa_hmr_forward'] + [INT],
               'dboa_hmr_backward_groups': sig['dboa_hmr_backward'] + [INT],
               'dboa_hmr_forward_active': sig['dboa_hmr_forward_groups'] + [ULL],
               'dboa_hmr_backward_active': sig['dboa_hmr_backward_groups'] + [ULL],
               'dboa_loss_motion_active': sig['dboa_loss_motion_groups'][:-1] + [ULL] + sig['dboa_loss_motion_groups'][-1:],
               'dboa_eval_metrics_active': sig['dboa_eval_metrics'][:-1] + [INT, ULL, STREAM],
               'dboa_cosine_terms_active': sig['dboa_cosine_terms'] + [INT, ULL]}
    for name, want in extends.items():
        assert sig[name] == want, name
        assert header.protos[name][0] == INT, name
    assert sig['dboa_cosine_partial_floats_groups'][:2] == sig['dboa_cosine_partial_floats']
    assert sig['dboa_loss_motion_groups'][:12] == sig['dboa_loss_motion_joints'][:12]
    desc = [(f, t) for f, t, _ in header.structs['dboa_crop_desc']]
    one = header.protos['dboa_crop_resize_normalize'][1]
    assert [d for d in desc if d in one[:7]] == one[:7]
    assert set(desc) <= set(one)


@pytest.mark.parametrize('decl', ['int dboa_new(size_t n, dboa_stream_t stream);', 'typedef struct dboa_new { short n; } dboa_new;',
                                  'int dboa_new(void (*callback)(int));'], ids=['parameter', 'field', 'function-pointer'])
def test_an_unknown_declaration_fails_the_parse(decl):
    with pytest.raises(ValueError, match='dboa_new'):
        parse_header(open(HEADER).read() + decl)


def test_version_and_counters(lib):
    assert b'sm_90a' in lib.dboa_version()
    assert lib.dboa_launch_count() >= 0


def test_layout_matches_reference_contract(lib):
    from dynaboa_b200.hmr import ArenaLayout
    lay = ArenaLayout()
    ref = layout.param_shapes()
    assert lay.n == 169 and lay.names == list(ref.keys())
    assert [tuple(s) for s in lay.shapes] == [tuple(v) for v in ref.values()]
    assert sum(int(__import__('numpy').prod(s)) for s in lay.shapes) == layout.num_params() == 26977501
    # views must not overlap and must stay inside the arena
    spans = sorted((o, o + 1 + sum((s - 1) * st for s, st in zip(sh, stv))) for o, sh, stv in zip(lay.offsets, lay.shapes, lay.strides))
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 <= b0
    assert spans[-1][1] <= lay.floats


def test_size_queries(lib):
    assert lib.dboa_hmr_tape_floats(1) > 20_000_000 and lib.dboa_hmr_tape_floats(0) < 0
    assert lib.dboa_hmr_scratch_floats(2) > 0
    assert lib.dboa_smpl_tape_floats(2) == 2 * (8 * 20670 + 648)      # 7 blend-shape row splits + posed vertices, chain state


@pytest.mark.parametrize('B', [1, 2, 9, 22, 64])
def test_tape_offsets_cover_disjoint_regions_of_the_layer_shapes(lib, B):
    """dboa_hmr_tape_offset: every region lies inside dboa_hmr_tape_floats(B), no two overlap, and each is as large as
    the layer it holds (shapes from the parameter table); the convolution output sizes agree with dboa_hmr_feature_info."""
    geo = hmr.conv_geometry()
    assert len(geo) == 53 and sum('downsample' in g[0] for g in geo) == 4
    regions = []
    for i, (name, cin, cout, k, stride, h) in enumerate(geo):
        n = B * h * h * cout
        regions += [(lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y, i), n, ('y', name)),
                    (lib.dboa_hmr_tape_offset(B, hmr.TAPE_STATS, i), B * 8, ('stats', name))]
        if 'downsample' in name:
            assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_A, i) == -1, name
        else:
            regions.append((lib.dboa_hmr_tape_offset(B, hmr.TAPE_A, i), n, ('a', name)))
    # consecutive convolutions chain: Cin of each conv is the channel count of its input, Hin = Hout * stride
    for (n0, _, c0, _, _, h0), (n1, cin1, _, _, s1, h1) in zip(geo, geo[1:]):
        if n1.endswith('conv2') or n1.endswith('conv3'):
            assert cin1 == c0 and h0 == h1 * s1, (n0, n1)
    sizes = {'x0': B * 224 * 224 * 3, 'p0': B * 56 * 56 * 64, 'p0_idx': (B * 56 * 56 * 64 + 3) // 4, 'xc': 3 * B * 2208,
             'h1pre': 3 * B * 1024, 'h1post': 3 * B * 1024, 'h2pre': 3 * B * 1024, 'h2post': 3 * B * 1024, 'params': 4 * B * 160,
             'masks': 6 * B * 1024}
    for kind, n in sizes.items():
        regions.append((lib.dboa_hmr_tape_offset(B, hmr.TAPE_WHOLE[kind], 0), n, (kind,)))
    assert all(o >= 0 for o, _, _ in regions), [r for r in regions if r[0] < 0]
    regions.sort()
    for (o0, n0, w0), (o1, _, w1) in zip(regions, regions[1:]):
        assert o0 + n0 <= o1, (w0, w1)
    assert regions[-1][0] + regions[-1][1] <= lib.dboa_hmr_tape_floats(B)
    off, nd = ctypes.c_longlong(), ctypes.c_int()
    shp, st = (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
    firsts = [0] + [i for i, g in enumerate(geo) if g[0].endswith('.conv3') and g[0].split('.')[1] == {1: '2', 2: '3', 3: '5', 4: '2'}[int(g[0][5])]]
    for feat, ci in enumerate(firsts):
        assert lib.dboa_hmr_feature_info(B, feat, ctypes.byref(off), ctypes.byref(nd), shp, st) == 0
        assert (shp[1], shp[2]) == (geo[ci][2], geo[ci][5]), feat
        assert off.value == lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y if feat == 0 else hmr.TAPE_A, ci), feat


def test_tape_offset_errors(lib):
    for B in (0, -1, 65):
        assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_Y, 0) == -2
        assert lib.dboa_hmr_tape_offset(B, hmr.TAPE_WHOLE['x0'], 0) == -2
    for kind in (-1, 13, 99):
        assert lib.dboa_hmr_tape_offset(1, kind, 0) == -1
    for conv in (-1, 53, 1000):
        for kind in (hmr.TAPE_Y, hmr.TAPE_STATS, hmr.TAPE_A):
            assert lib.dboa_hmr_tape_offset(1, kind, conv) == -1
    assert lib.dboa_hmr_tape_offset(1, hmr.TAPE_A, 4) == -1            # layer1.0.downsample.0
    assert lib.dboa_hmr_tape_offset(1, hmr.TAPE_Y, 4) >= 0


def test_argument_errors_do_not_need_a_gpu(lib):
    assert lib.dboa_rot6d_fwd(None, None, 4, None) == -1
    assert lib.dboa_sgd_update(None, None, None, 0.1, 8, None) == -1
    off, nd = ctypes.c_longlong(), ctypes.c_int()
    shp, st = (ctypes.c_longlong * 4)(), (ctypes.c_longlong * 4)()
    assert lib.dboa_hmr_param_info(999, None, 0, ctypes.byref(off), ctypes.byref(nd), shp, st) == -1

