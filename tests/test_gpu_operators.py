"""The single-operator entry points (include/dynaboa_b200.h "single operators") against fp64 on the CPU, computed from the
GPU's own fp32 inputs, over the shapes their launchers accept rather than ResNet-50's 53 layers at 224 x 224:

- the fp32 CUDA-core convolution (csrc/conv.cu) and the wgmma TF32x3 convolution (csrc/conv_tc.cu), forward, data gradient
  and weight gradient: non-square frames, odd extents, k 1 / 3 / 5 / 7, stride 1 / 2 / 3, pad 0 or k / 2, row tails against
  both tile heights, K tails, accumulation, and every split-K cluster size the launchers pick;
- GroupNorm forward and backward (csrc/groupnorm.cu): 1 to 16 CTAs per cluster, B up to 64, means far from zero, a constant
  group, and the per-sample ticket path of the B > 1 backward called twice in a row;
- the 3 x 3 / stride 2 max-pool (csrc/norm_pool.cu): non-square extents, negative inputs, ties, NaN and the overlapping
  windows of the backward.

Every output lives in a guard-banded buffer that starts as NaN (harness.Buf): the guard must be bit-intact and no NaN may
be left in the output.  The convolutions are held per element to the fp64 result in units of the fp64 sum of the absolute
products (conv of |x| and |w|): a wrong tap, a swapped extent or a lost tail moves an element by a whole product, not by a
rounding error.  Each bound is about 3x the worst error measured on an H100 80GB HBM3, which is written beside it; every
test prints its worst errors."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from harness import Buf, same_bits

pytestmark = pytest.mark.gpu

OK = 0


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    lib = _lib.load()
    yield _lib
    lib.dboa_set_tensor_core_conv(3)          # the library default: later test modules must not inherit this module's mode


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# =====================================================================================================================
# convolutions
# =====================================================================================================================
# B, Hi, Wi, Cin, Cout, k, stride, pad
CASES = [
    # non-square frames, every product
    (1, 14, 22, 64, 64, 3, 1, 1),
    (2, 9, 7, 64, 192, 3, 2, 1),         # odd extents at stride 2 (the wgmma data gradient refuses them)
    (1, 28, 12, 128, 64, 5, 2, 2),       # k = 5 at stride 2: parity classes of 3 x 3, 3 x 2, 2 x 3 and 2 x 2 taps
    (1, 13, 11, 64, 64, 7, 3, 3),        # k = 7 at stride 3
    (1, 10, 14, 64, 128, 5, 1, 0),       # pad 0 != k / 2
    (1, 16, 10, 64, 64, 1, 2, 0),        # 1 x 1 at stride 2: three of the four parity classes receive nothing
    (1, 15, 9, 64, 64, 3, 3, 0),
    (2, 12, 6, 64, 192, 3, 2, 0),        # even extents at stride 2 with pad 0
    (1, 11, 16, 64, 64, 5, 2, 2),        # odd H, even W at stride 2
    # row tails against the 64-row fp32 tile and the 128-row wgmma tile (M = B * Ho * Wo for the forward)
    (1, 1, 1, 64, 64, 3, 1, 1),          # M = 1: only the centre tap is inside the frame
    (1, 7, 9, 64, 64, 3, 1, 1),          # 63
    (1, 4, 16, 64, 64, 1, 1, 0),         # 64
    (1, 5, 13, 64, 64, 3, 1, 1),         # 65
    (1, 127, 1, 64, 64, 3, 1, 1),        # 127, a one-pixel-wide frame
    (1, 16, 8, 64, 192, 1, 1, 0),        # 128
    (1, 3, 43, 64, 64, 3, 1, 1),         # 129
    (3, 8, 8, 64, 64, 3, 1, 1),          # 192 over three samples
    # long K, few tiles: the split-K clusters of 8
    (1, 7, 5, 256, 64, 3, 1, 1),
    (1, 8, 6, 64, 128, 3, 2, 1),
    (1, 24, 22, 64, 64, 1, 1, 0),
    (2, 14, 10, 128, 128, 3, 1, 1),
    (1, 18, 14, 64, 64, 3, 2, 1),
    (1, 30, 34, 64, 64, 3, 1, 1),
    (4, 28, 20, 64, 128, 3, 1, 1),
    (2, 30, 26, 128, 64, 3, 2, 1),
    (1, 10, 12, 128, 256, 1, 1, 0),
    (1, 12, 10, 64, 192, 1, 2, 0),
    # K tails of the fp32 forward and weight gradient: Cin % 4 != 0 (scalar gather) and Cin % 16 != 0, padded pitch
    (1, 11, 17, 3, 64, 7, 2, 3),
    (2, 9, 14, 12, 64, 3, 1, 1),
    (1, 13, 10, 20, 128, 5, 2, 2),
    (1, 6, 9, 20, 192, 1, 3, 0),
]


def out_hw(c):
    B, Hi, Wi, Cin, Cout, k, s, p = c
    return (Hi + 2 * p - k) // s + 1, (Wi + 2 * p - k) // s + 1


def pitch_of(c):
    """The weight row pitch a case runs with: k * k * Cin when the wgmma kernels take the case (they need exactly that, and
    it is a multiple of 16 then), else roundup16 + 4, so the fp32 weight gradient has padding columns to leave alone."""
    B, Hi, Wi, Cin, Cout, k, s, p = c
    K = k * k * Cin
    return K if Cin % 64 == 0 else (K + 15) // 16 * 16 + 4


def products(c):
    """The products the launchers take for case c."""
    B, Hi, Wi, Cin, Cout, k, s, p = c
    out = []
    if Cout % 64 == 0:
        out += ['fwd32', 'wgrad32']
    if Cin % 64 == 0 and Cout % 16 == 0:
        out.append('dgrad32')
    if Cin % 64 == 0 and Cout % 64 == 0:
        out += ['fwd_tc', 'wgrad_tc']
        if s != 2:
            out.append('dgrad_tc_s1')
        elif Hi % 2 == 0 and Wi % 2 == 0:
            out.append('dgrad_tc_s2')
    return out


# ---- split-K: the launchers' rules, restated.  A change to pick_split / conv_fwd / conv_dgrad / conv_wgrad (csrc/conv.cu) or
# ---- to tc::launch (csrc/conv_tc.cu) has to be made here too, or the coverage test below stops meaning what it says.
def split32(tiles, kiters, sms):
    """pick_split: a power of two <= 8 that fills ~2 waves and leaves >= 4 k-slabs per slice."""
    ns = 1
    while ns < 8 and tiles * ns * 2 <= 2 * sms + tiles and kiters // (ns * 2) >= 4:
        ns *= 2
    return ns


def split_tc(tiles, nkb, sms):
    """tc::launch: a power of two <= 8 that keeps the grid within about one wave and leaves >= 2 k-blocks per CTA."""
    ns = 1
    while ns < 8 and tiles * ns * 2 <= sms + tiles and nkb // (ns * 2) >= 2:
        ns *= 2
    return ns


def cdiv(a, b):
    return -(-a // b)


def split_of(product, c, sms):
    B, Hi, Wi, Cin, Cout, k, s, p = c
    Ho, Wo = out_hw(c)
    K = k * k * Cin
    if product == 'fwd32':
        return split32(cdiv(B * Ho * Wo, 64) * (Cout // 64), cdiv(K, 16), sms)
    if product == 'dgrad32':
        return split32(cdiv(B * Hi * Wi, 64) * (Cin // 64), k * k * Cout // 16, sms)
    if product == 'wgrad32':
        return split32((Cout // 64) * cdiv(K, 64), cdiv(B * Ho * Wo, 16), sms)
    if product == 'fwd_tc':
        return split_tc(cdiv(B * Ho * Wo, 128) * (Cout // 64), cdiv(K, 32), sms)
    if product == 'dgrad_tc_s1':
        return split_tc(cdiv(B * Hi * Wi, 128) * (Cin // 64), cdiv(k * k * Cout, 32), sms)
    if product == 'dgrad_tc_s2':          # parity classes of B * Hi/2 * Wi/2 rows; the longest tap set sizes the split
        ncls = 4 if k >= 2 else 1
        return split_tc(ncls * cdiv(B * (Hi // 2) * (Wi // 2), 128) * (Cin // 64), cdiv(((k + 1) // 2) ** 2 * Cout, 32), sms)
    if product == 'wgrad_tc':
        return split_tc(cdiv(Cout, 128) * (K // 64), cdiv(B * Ho * Wo, 32), sms)
    raise ValueError(product)


PRODUCTS = ('fwd32', 'dgrad32', 'wgrad32', 'fwd_tc', 'dgrad_tc_s1', 'dgrad_tc_s2', 'wgrad_tc')


def test_split_k_coverage():
    """Every product meets cluster sizes 1, 2, 4 and 8 over CASES on this device."""
    sms = num_sms()
    reached = {pr: {} for pr in PRODUCTS}
    for c in CASES:
        for pr in products(c):
            reached[pr].setdefault(split_of(pr, c, sms), c)
    for pr in PRODUCTS:
        print(f'split-K {pr:12s} ({sms} SMs): ' + ', '.join(f'{ns}: {c}' for ns, c in sorted(reached[pr].items())))
    for pr in PRODUCTS:
        assert set(reached[pr]) == {1, 2, 4, 8}, (pr, sorted(reached[pr]))


# ---- the data of a case and its fp64 references
class Conv:
    def __init__(self, c, seed):
        B, Hi, Wi, Cin, Cout, k, s, p = c
        self.c, (self.Ho, self.Wo) = c, out_hw(c)
        self.K, self.pitch = k * k * Cin, pitch_of(c)
        g = torch.Generator().manual_seed(seed)
        self.x = torch.randn(B, Cin, Hi, Wi, generator=g)
        self.w = torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(k * k * Cin)
        self.dy = torch.randn(B, Cout, self.Ho, self.Wo, generator=g)
        self.base_x = torch.randn(B, Hi, Wi, Cin, generator=g)               # accumulation bases
        self.base_w = torch.randn(Cout, self.K, generator=g) * 0.1
        rows = self.w.permute(0, 2, 3, 1).reshape(Cout, self.K)
        self.wrows = torch.zeros(Cout, self.pitch)
        self.wrows[:, :self.K] = rows
        self.xd = Buf(self.x.permute(0, 2, 3, 1).contiguous())
        self.wd = Buf(self.wrows)
        self.dyd = Buf(self.dy.permute(0, 2, 3, 1).contiguous())
        self._ref = {}

    def args(self):
        B, Hi, Wi, Cin, Cout, k, s, p = self.c
        return B, Hi, Wi, Cin, Cout, k, s, p, self.pitch

    def ref(self, what, x=None):
        """fp64 result and the fp64 sum of absolute products, in the kernels' layouts: y (B, Ho, Wo, Cout), dx (B, Hi, Wi,
        Cin), dw (Cout, K).  ``x``: a stand-in input of the same numel read with other extents (negative controls)."""
        key = what if x is None else None
        if key in self._ref:
            return self._ref[key]
        B, Hi, Wi, Cin, Cout, k, s, p = self.c
        xs = (self.x if x is None else x).double()
        w, dy = self.w.double(), self.dy.double()
        out = []
        for a, b, d in ((xs, w, dy), (xs.abs(), w.abs(), dy.abs())):
            if what == 'y':
                r = F.conv2d(a, b, stride=s, padding=p).permute(0, 2, 3, 1)
            elif what == 'dx':
                r = conv2d_input(a.shape, b, d, stride=s, padding=p).permute(0, 2, 3, 1)
            else:
                r = conv2d_weight(a, b.shape, d, stride=s, padding=p).permute(0, 2, 3, 1).reshape(Cout, self.K)
            out.append(r.contiguous())
        if key is not None:
            self._ref[key] = tuple(out)
        return tuple(out)


def elem_err(got, ref, absref, base=None):
    """max over elements of |got (- base) - ref| / (sum of |products| (+ |base|)).  An element no product reaches must be
    exactly zero."""
    got = got.double().reshape(ref.shape)
    scale = absref
    if base is not None:
        got = got - base.double().reshape(ref.shape)
        scale = absref + base.double().abs().reshape(ref.shape)
    d = (got - ref).abs()
    return float(torch.where(scale > 0, d / scale.clamp_min(1e-300), d * 1e300).max())


# Bounds on the per-element error in units of the sum of |products|.  Worst measured over CASES on an H100 80GB HBM3 (700 W):
#   fp32 CUDA cores:  forward 2.7e-7, data gradient 2.6e-7, weight gradient 3.3e-7
#   wgmma TF32x3:     forward 6.2e-7, data gradient 6.7e-7, weight gradient 1.4e-6 (accumulating splits: out - base)
# A product lost or taken twice moves an element by about 1 / (k * k * Cin) of that unit or more.
TOL = {'fwd32': 8e-7, 'dgrad32': 8e-7, 'wgrad32': 1e-6, 'fwd_tc': 2e-6, 'dgrad_tc': 2e-6, 'wgrad_tc': 4e-6}
WORST = {}


def note(name, err, tol, c):
    WORST[name] = max(WORST.get(name, 0.0), err)
    assert err <= tol, (name, c, err, tol)


def no_nan(buf):
    return not bool(torch.isnan(buf.t).any())


def lib_call(L, name, *args):
    st = getattr(L.load(), name)(*args, L.stream())
    assert st == OK, (name, st)


def run_fwd(L, cv, tc):
    B, Hi, Wi, Cin, Cout, k, s, p, pitch = cv.args()
    y = Buf(n=B * cv.Ho * cv.Wo * Cout)
    if tc:
        lib_call(L, 'dboa_conv2d_tc_fwd', cv.xd.ptr, cv.wd.ptr, y.ptr, *cv.args())
    else:
        lib_call(L, 'dboa_conv2d_fwd', cv.xd.ptr, cv.wd.ptr, y.ptr, *cv.args(), None, 0)
    return y


def run_dgrad(L, cv, tc, acc):
    B, Hi, Wi, Cin = cv.c[:4]
    dx = Buf(cv.base_x) if acc else Buf(n=B * Hi * Wi * Cin)
    if tc:
        lib_call(L, 'dboa_conv2d_tc_dgrad', cv.dyd.ptr, cv.wd.ptr, dx.ptr, *cv.args(), acc)
    else:
        lib_call(L, 'dboa_conv2d_dgrad', cv.dyd.ptr, cv.wd.ptr, dx.ptr, *cv.args(), acc, None, 0)
    return dx


PAD_FILL = -3.75                 # the weight-gradient padding columns: never written


def run_wgrad(L, cv, tc, base):
    """dw += dy^T im2col(x) on `base` (Cout, K); padding columns hold PAD_FILL."""
    Cout = cv.c[4]
    init = torch.full((Cout, cv.pitch), PAD_FILL)
    init[:, :cv.K] = base
    dw = Buf(init)
    if tc:
        lib_call(L, 'dboa_conv2d_tc_wgrad', cv.dyd.ptr, cv.xd.ptr, dw.ptr, *cv.args())
    else:
        lib_call(L, 'dboa_conv2d_wgrad', cv.dyd.ptr, cv.xd.ptr, dw.ptr, *cv.args(), None, 0)
    return dw


def check_out(buf, what):
    assert buf.intact(), f'{what}: guard written'
    assert no_nan(buf), f'{what}: NaN left in the output'


@pytest.mark.parametrize('c', CASES, ids=[f'{c[0]}x{c[1]}x{c[2]}x{c[3]}-{c[4]}-k{c[5]}s{c[6]}p{c[7]}' for c in CASES])
def test_conv(L, c):
    prods = products(c)
    cv = Conv(c, seed=hash(c) % 100003)
    Cout = c[4]
    L.load().dboa_set_tensor_core_conv(2)                    # forward, data and weight gradient on the tensor cores
    errs = {}
    for tc in (False, True):
        sfx = '_tc' if tc else '32'
        if 'fwd' + sfx in prods:
            y = run_fwd(L, cv, tc)
            check_out(y, 'fwd' + sfx)
            errs['fwd' + sfx] = elem_err(y.cpu(), *cv.ref('y'))
            note('fwd' + sfx, errs['fwd' + sfx], TOL['fwd' + sfx], c)
        dname = 'dgrad32' if not tc else ('dgrad_tc_s2' if c[6] == 2 else 'dgrad_tc_s1')
        if dname in prods:
            tol = TOL['dgrad32' if not tc else 'dgrad_tc']
            over = run_dgrad(L, cv, tc, 0)
            check_out(over, dname)
            ref, absref = cv.ref('dx')
            e0 = elem_err(over.cpu(), ref, absref)
            accd = run_dgrad(L, cv, tc, 1)
            check_out(accd, dname + ' acc')
            if tc:                     # the split-K reduction starts from the base: out - base against fp64
                e1 = elem_err(accd.cpu(), ref, absref, base=cv.base_x)
            else:                      # base + the overwriting call's result, rounded once: bit for bit
                assert same_bits(accd.cpu(), cv.base_x.reshape(-1) + over.cpu()), (c, 'dgrad32 accumulate')
                e1 = 0.0
            errs[dname] = max(e0, e1)
            note('dgrad32' if not tc else 'dgrad_tc', errs[dname], tol, c)
        if 'wgrad' + sfx in prods:
            ref, absref = cv.ref('dw')
            zero = run_wgrad(L, cv, tc, torch.zeros(Cout, cv.K))
            based = run_wgrad(L, cv, tc, cv.base_w)
            for b, what in ((zero, 'zero base'), (based, 'base')):
                check_out(b, f'wgrad{sfx} {what}')
                whole = b.cpu().reshape(Cout, cv.pitch)
                assert bool((whole[:, cv.K:] == PAD_FILL).all()), (c, 'padding columns written')
            e0 = elem_err(zero.cpu().reshape(Cout, cv.pitch)[:, :cv.K], ref, absref)
            got = based.cpu().reshape(Cout, cv.pitch)[:, :cv.K]
            if tc and split_of('wgrad_tc', c, num_sms()) > 1:
                e1 = elem_err(got, ref, absref, base=cv.base_w)
            else:                      # one slice (wgmma) or any split (fp32): base + the zero-base result, rounded once
                assert same_bits(got.contiguous(), cv.base_w + zero.cpu().reshape(Cout, cv.pitch)[:, :cv.K]), (c, 'wgrad' + sfx)
                e1 = 0.0
            errs['wgrad' + sfx] = max(e0, e1)
            note('wgrad' + sfx, errs['wgrad' + sfx], TOL['wgrad' + sfx], c)
        for b in (cv.xd, cv.wd, cv.dyd):
            assert b.intact()
    print(c, ' '.join(f'{k} {v:.2e}' for k, v in errs.items()))


# ---- negative controls: the comparisons above can fail
def test_conv_negative_controls(L):
    c = (1, 14, 22, 64, 64, 3, 1, 1)
    cv = Conv(c, seed=5)
    L.load().dboa_set_tensor_core_conv(2)
    for tc in (False, True):
        tol = TOL['fwd_tc' if tc else 'fwd32']
        y = run_fwd(L, cv, tc)
        ref, absref = cv.ref('y')
        got = y.cpu()
        assert elem_err(got, ref, absref) <= tol
        # a reference that reads the NHWC input with H and W swapped (an index computation of the kernel that swaps them)
        B, Hi, Wi, Cin = c[:4]
        swapped = cv.x.permute(0, 2, 3, 1).reshape(B, Wi, Hi, Cin).permute(0, 3, 1, 2)
        sref, sabs = cv.ref('y', x=swapped)
        assert elem_err(got, sref.reshape(ref.shape), sabs.reshape(ref.shape)) > 100 * tol
        # one output element moved by a thousandth of its scale
        bad = got.clone().reshape(ref.shape)
        i = (0, 7, 13, 40)
        bad[i] += 1e-3 * float(absref[i])
        assert elem_err(bad, ref, absref) > tol
        # an element past the output written
        assert y.intact()
        y.whole[y.n + 17] = 0.0
        assert not y.intact()
        # an element left unwritten
        y.t[123] = float('nan')
        assert not no_nan(y)


# =====================================================================================================================
# GroupNorm
# =====================================================================================================================
GN_NT, GN_V, GN_MAXCL = 1024, 4, 16


def gn_chunks(HW, C):
    """gn_plan (csrc/groupnorm.cu): CTAs per (sample, group), or None for a shape the launchers refuse."""
    cg4 = C // 16
    if C % 16 or cg4 < 1 or cg4 > GN_NT or cg4 & (cg4 - 1):
        return None
    chunks = min(max(cdiv(HW * cg4, GN_NT * 2), 1), GN_MAXCL)
    rows = cdiv(HW, chunks)
    if rows * cg4 > GN_NT * GN_V:
        return None
    return cdiv(HW, rows)


# B, C, HW
GN_CASES = [
    (1, 16, 1), (2, 32, 3), (5, 64, 49), (17, 128, 50), (64, 256, 1), (64, 64, 49), (1, 2048, 49), (2, 1024, 196),
    (1, 16, 12544), (1, 64, 12544), (3, 32, 3136), (1, 256, 3136), (2, 512, 196), (5, 2048, 50), (17, 16, 196), (2, 64, 3136),
    (2, 1024, 50), (1, 128, 3136),
]

# Bounds relative to the largest fp64 value of each output (mean: in units of the group's standard deviation; rstd relative).
# Worst measured on an H100 80GB HBM3 (700 W) over GN_CASES, the constant group and the ticket test:
#   out 1.9e-7, dy 6.4e-7, dgamma / dbeta 4.1e-7, mean 2.0e-7, rstd 1.5e-7.
GN_TOL = {'out': 6e-7, 'dy': 2e-6, 'dgb': 1.2e-6, 'mean': 6e-7, 'rstd': 5e-7}
# Means 1e3 and 1e4 times the spread: the output, gradient and mean errors follow the spacing of the fp32 inputs, which grows
# with |mean| / std; these bounds are per unit of 1 + |mean| / std.  Worst measured: out 3.6e-8, dy 2.9e-9, dgamma / dbeta
# 6.4e-8, mean 1.1e-7 (all at 1e3).  rstd is held to its own bound, not scaled: worst 9.2e-7 (at 1e4).  A variance formed as
# E[y^2] - E[y]^2 in fp32 would lose every digit of rstd at these means.
GN_BIG_TOL = {'out': 1e-7, 'dy': 1e-8, 'dgb': 2e-7, 'mean': 3e-7}
GN_BIG_RSTD = 3e-6


def gn_ref(y, gamma, beta, dz):
    """fp64 GroupNorm(4) of NHWC fp32 `y`: normalised output, (mean, rstd) per (sample, group) and the backward of sum(z * dz)."""
    B, HW, C = y.shape
    yd = y.double().requires_grad_(True)
    v = yd.reshape(B, HW, 4, C // 4)
    mean = v.mean(dim=(1, 3), keepdim=True)
    var = ((v - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    g, b = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = ((v - mean) * rstd).reshape(B, HW, C) * g + b
    (z * dz.double()).sum().backward()
    return z.detach(), mean.detach().reshape(B, 4), rstd.detach().reshape(B, 4), yd.grad, g.grad, b.grad


def gn_run(L, y, gamma, beta, res, relu, dout, mask, dg0, db0):
    """One forward and one backward call; mask: use the forward's output as mask_src.  dg0 / db0: dgamma / dbeta bases."""
    B, HW, C = y.shape
    yd, gd, bd = Buf(y), Buf(gamma), Buf(beta)
    rd = Buf(res) if res is not None else None
    out, stats = Buf(n=y.numel()), Buf(n=B * 8)
    part = L.load().dboa_gn_partial_floats(B, HW, C)
    lib_call(L, 'dboa_groupnorm_fwd', yd.ptr, gd.ptr, bd.ptr, rd.ptr if rd else None, out.ptr, stats.ptr, None, B, HW, C, relu)
    dod = Buf(dout)
    dy, dg, db = Buf(n=y.numel()), Buf(dg0), Buf(db0)
    bpart = Buf(n=max(1, L.load().dboa_gn_bwd_partial_floats(B, HW, C)))
    lib_call(L, 'dboa_groupnorm_bwd', dod.ptr, out.ptr if mask else None, yd.ptr, stats.ptr, gd.ptr, dy.ptr, dg.ptr, db.ptr, bpart.ptr,
             B, HW, C)
    for b in (out, stats, dy, dg, db):
        check_out(b, 'groupnorm')
    for b in (yd, gd, bd, dod, bpart) + ((rd,) if rd else ()):
        assert b.intact()
    assert part == 0
    return out.cpu().reshape(B, HW, C), stats.cpu().reshape(B, 4, 2), dy.cpu().reshape(B, HW, C), dg.cpu(), db.cpu()


def rel(got, ref):
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


def gn_check(L, B, C, HW, seed, relu, with_res, mask, mean=0.0, std=1.0, const_group=False):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B, HW, C, generator=g) * std + mean
    if const_group:
        y[:, :, :C // 4] = 3.25
    gamma, beta = torch.randn(C, generator=g) * 0.3 + 1, torch.randn(C, generator=g) * 0.2
    res = torch.randn(B, HW, C, generator=g) if with_res else None
    dout = torch.randn(B, HW, C, generator=g)
    dg0, db0 = torch.randn(C, generator=g), torch.randn(C, generator=g)
    out, stats, dy, dg, db = gn_run(L, y, gamma, beta, res, relu, dout, mask, dg0, db0)
    z, rmean, rrstd, rdy, rdg, rdb = gn_ref(y, gamma, beta, dout * (out > 0) if mask else dout)
    rout = z + (res.double() if with_res else 0)
    if relu:
        rout = rout.clamp_min(0)
    sd = y.double().reshape(B, HW, 4, C // 4).std(dim=(1, 3), unbiased=False).clamp_min(1e-30)
    e = {'out': rel(out, rout), 'dy': rel(dy, rdy),
         'dgb': max(rel(dg - dg0, rdg), rel(db - db0, rdb)),
         'mean': float(((stats[..., 0].double() - rmean).abs() / sd).max()) if not const_group else float((stats[..., 0].double() - rmean).abs().max()),
         'rstd': rel(stats[..., 1], rrstd)}
    return e, out, rout


GN_WORST = {}


def gn_note(e, tol, scale, what):
    for k, v in e.items():
        GN_WORST[k] = max(GN_WORST.get(k, 0.0), v / scale)
        assert v <= tol[k] * scale, (what, k, v, tol[k] * scale)


@pytest.fixture(scope='module', autouse=True)
def worst_report():
    """After the module: the worst errors the convolution and GroupNorm sweeps met, the numbers the bounds above quote."""
    yield
    if WORST:
        print('\nconv worst per-element errors:', ' '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))
    if GN_WORST:
        print('GroupNorm worst errors:', ' '.join(f'{k} {v:.2e}' for k, v in sorted(GN_WORST.items())))


@pytest.mark.parametrize('case', GN_CASES, ids=[f'B{b}-C{c}-HW{h}' for b, c, h in GN_CASES])
def test_groupnorm(L, case):
    B, C, HW = case
    assert gn_chunks(HW, C) is not None
    worst = {}
    for relu in (0, 1):
        for with_res in (False, True):
            for mask in (False, True):
                e, _, _ = gn_check(L, B, C, HW, seed=B * 7919 + C * 31 + HW + relu * 3 + with_res * 5 + mask * 11, relu=relu, with_res=with_res,
                                   mask=mask)
                gn_note(e, GN_TOL, 1.0, (case, relu, with_res, mask))
                worst = {k: max(worst.get(k, 0.0), v) for k, v in e.items()}
    print(case, f'chunks {gn_chunks(HW, C)}', ' '.join(f'{k} {v:.2e}' for k, v in worst.items()))


def test_groupnorm_cluster_sizes():
    """GN_CASES cover one CTA per cluster, the 16-CTA limit and sizes in between."""
    sizes = {gn_chunks(HW, C) for _, C, HW in GN_CASES}
    print('GroupNorm CTAs per cluster:', sorted(sizes))
    assert {1, 2, 16} <= sizes and len(sizes) >= 6


@pytest.mark.parametrize('ratio', [1e3, 1e4])
@pytest.mark.parametrize('case', [(1, 64, 3136), (5, 256, 49), (17, 2048, 3)], ids=['B1-C64-HW3136', 'B5-C256-HW49', 'B17-C2048-HW3'])
def test_groupnorm_large_mean(L, case, ratio):
    """Means of 1e3 and 1e4 times the spread: the statistics are (count, mean, M2) merged pairwise, so the error stays at the
    spacing of the fp32 inputs instead of growing with mean^2 / var as a sum of squares would."""
    B, C, HW = case
    e, _, _ = gn_check(L, B, C, HW, seed=int(ratio) + B, relu=0, with_res=False, mask=False, mean=0.37 * ratio, std=0.37)
    print(case, ratio, ' '.join(f'{k} {v:.2e}' for k, v in e.items()))
    for k, v in e.items():
        assert v <= (GN_BIG_RSTD if k == 'rstd' else GN_BIG_TOL[k] * (1 + ratio)), (k, v)


@pytest.mark.parametrize('case', [(1, 64, 49), (3, 256, 196)], ids=['B1', 'B3'])
def test_groupnorm_constant_group(L, case):
    """Group 0 of every sample is one value: its variance is 0, rstd = 1 / sqrt(eps) and its output is beta."""
    B, C, HW = case
    e, out, rout = gn_check(L, B, C, HW, seed=3, relu=0, with_res=False, mask=False, const_group=True)
    print(case, ' '.join(f'{k} {v:.2e}' for k, v in e.items()))
    gn_note(e, GN_TOL, 1.0, ('constant', case))


@pytest.mark.parametrize('case', [(2, 64, 49), (17, 256, 196), (64, 16, 3), (5, 2048, 50)], ids=['B2', 'B17', 'B64', 'B5-C2048'])
def test_groupnorm_bwd_tickets_reset(L, case):
    """Two B > 1 backward calls in a row, on one stream, into dgamma / dbeta that start at zero: the first leaves the
    increment a, the second 2a exactly.  A ticket counter left behind would make the second call's last-CTA pass fire early
    (a partial sum) or never (a again)."""
    B, C, HW = case
    g = torch.Generator().manual_seed(B + C)
    y, dout = torch.randn(B, HW, C, generator=g), torch.randn(B, HW, C, generator=g)
    gamma, beta = torch.randn(C, generator=g) * 0.3 + 1, torch.randn(C, generator=g) * 0.2
    yd, gd, bd, dod = Buf(y), Buf(gamma), Buf(beta), Buf(dout)
    out, stats = Buf(n=y.numel()), Buf(n=B * 8)
    lib_call(L, 'dboa_groupnorm_fwd', yd.ptr, gd.ptr, bd.ptr, None, out.ptr, stats.ptr, None, B, HW, C, 1)
    dg, db = Buf(torch.zeros(C)), Buf(torch.zeros(C))
    bpart = Buf(n=L.load().dboa_gn_bwd_partial_floats(B, HW, C))
    got = []
    for _ in range(2):
        dy = Buf(n=y.numel())
        lib_call(L, 'dboa_groupnorm_bwd', dod.ptr, out.ptr, yd.ptr, stats.ptr, gd.ptr, dy.ptr, dg.ptr, db.ptr, bpart.ptr, B, HW, C)
        got.append((dy.cpu(), dg.cpu(), db.cpu()))
        check_out(dy, 'dy')
    for b in (dg, db, bpart, out, stats):
        assert b.intact()
    (dy1, g1, b1), (dy2, g2, b2) = got
    assert same_bits(dy1, dy2)
    assert same_bits(g2, g1 * 2) and same_bits(b2, b1 * 2)
    _, _, _, _, rdg, rdb = gn_ref(y, gamma, beta, dout * (out.cpu().reshape(B, HW, C) > 0))
    e = max(rel(g1, rdg), rel(b1, rdb))
    print(case, f'dgamma/dbeta {e:.2e}')
    assert e <= GN_TOL['dgb']


def test_groupnorm_negative_controls(L):
    B, C, HW = 2, 64, 49
    g = torch.Generator().manual_seed(1)
    y, dout = torch.randn(B, HW, C, generator=g), torch.randn(B, HW, C, generator=g)
    gamma, beta = torch.randn(C, generator=g) * 0.3 + 1, torch.randn(C, generator=g) * 0.2
    out, stats, dy, _, _ = gn_run(L, y, gamma, beta, None, 0, dout, False, torch.zeros(C), torch.zeros(C))
    z, _, _, rdy, _, _ = gn_ref(y, gamma, beta, dout)
    assert rel(out, z) <= GN_TOL['out'] and rel(dy, rdy) <= GN_TOL['dy']
    # one output element moved by a thousandth of the output's scale
    bad = out.clone()
    bad[1, 10, 5] += 1e-3 * float(z.abs().max())
    assert rel(bad, z) > GN_TOL['out']
    # a reference that groups the channels the other way (channel c in group c % 4, not c // (C / 4)): the kernel's channel
    # indexing, the one spatial-free index GroupNorm has, gone wrong
    perm = torch.arange(C).reshape(C // 4, 4).t().reshape(-1)
    inv = torch.argsort(perm)
    zi, _, _, dyi, _, _ = gn_ref(y[..., perm], gamma[perm], beta[perm], dout[..., perm])
    assert rel(out, zi[..., inv]) > 100 * GN_TOL['out'] and rel(dy, dyi[..., inv]) > 100 * GN_TOL['dy']


# =====================================================================================================================
# max-pool 3 x 3, stride 2, pad 1
# =====================================================================================================================
POOL_CASES = [(2, 112, 112, 64), (1, 14, 22, 8), (3, 6, 10, 4), (1, 2, 2, 4), (2, 8, 30, 12), (1, 28, 12, 16)]


def pool_input(kind, shape, g):
    B, H, W, C = shape
    x = torch.randn(B, C, H, W, generator=g)
    if kind == 'negative':
        x = -(x.abs() + 0.1)
    elif kind == 'ties':                       # few distinct values: most windows hold several copies of their maximum
        x = torch.round(x * 1.5) / 2
    elif kind == 'nan':
        x = torch.round(x * 1.5) / 2
        x[torch.rand(x.shape, generator=g) < 0.04] = float('nan')
        x[:, 0, 0, 0] = float('nan')           # at least one, in the corner window
    return x


def pool_ref(x):
    """fp64 MaxPool2d(3, 2, 1) with ATen's flat indices turned into the window position r * 3 + s, NHWC."""
    B, C, H, W = x.shape
    y, flat = F.max_pool2d(x.double(), 3, 2, 1, return_indices=True)
    Ho, Wo = y.shape[2:]
    hi, wi = flat // W, flat % W
    r = hi - (2 * torch.arange(Ho).view(1, 1, Ho, 1) - 1)
    s = wi - (2 * torch.arange(Wo).view(1, 1, 1, Wo) - 1)
    assert bool(((r >= 0) & (r < 3) & (s >= 0) & (s < 3)).all())
    return y.permute(0, 2, 3, 1), (r * 3 + s).permute(0, 2, 3, 1).to(torch.uint8), flat


def same_values(a, b):
    """Equal as numbers, NaN where the other is NaN."""
    a, b = a.double(), b.double()
    na, nb = torch.isnan(a), torch.isnan(b)
    return bool(torch.equal(na, nb)) and bool(torch.equal(a[~na], b[~nb]))


# backward: |dx - fp64 scatter| <= POOL_TOL * (sum of |dy| over the windows that picked the element), a sum of at most 4 fp32
# terms.  Worst measured on an H100 80GB HBM3 (700 W): 1.4e-7.
POOL_TOL = 4e-7


@pytest.mark.parametrize('kind', ['randn', 'negative', 'ties', 'nan'])
@pytest.mark.parametrize('shape', POOL_CASES, ids=[f'{b}x{h}x{w}x{c}' for b, h, w, c in POOL_CASES])
def test_maxpool(L, shape, kind):
    B, H, W, C = shape
    g = torch.Generator().manual_seed(B * 100 + H + W + C)
    x = pool_input(kind, shape, g)
    Ho, Wo = H // 2, W // 2
    xd = Buf(x.permute(0, 2, 3, 1).contiguous())
    y, idx = Buf(n=B * Ho * Wo * C), Buf(n=B * Ho * Wo * C, dtype=torch.uint8)
    lib_call(L, 'dboa_maxpool_fwd', xd.ptr, y.ptr, idx.ptr, B, H, W, C)
    ry, ridx, flat = pool_ref(x)
    assert y.intact() and idx.intact() and xd.intact()
    assert kind == 'nan' or no_nan(y)
    assert same_values(y.cpu(), ry.reshape(-1)), 'max'
    assert torch.equal(idx.cpu(), ridx.reshape(-1)), 'window index (first maximum in scan order; the last NaN)'
    if kind == 'nan':
        assert bool(torch.isnan(ry).any())
    dy = torch.randn(B, C, Ho, Wo, generator=g)
    dyd = Buf(dy.permute(0, 2, 3, 1).contiguous())
    dx = Buf(n=x.numel())
    lib_call(L, 'dboa_maxpool_bwd', dyd.ptr, idx.ptr, dx.ptr, B, H, W, C)
    check_out(dx, 'maxpool bwd')
    assert dyd.intact() and idx.intact()
    ref = torch.zeros(B, C, H * W, dtype=torch.float64)
    scale = torch.zeros(B, C, H * W, dtype=torch.float64)
    ref.scatter_add_(2, flat.reshape(B, C, -1), dy.double().reshape(B, C, -1))
    scale.scatter_add_(2, flat.reshape(B, C, -1), dy.double().abs().reshape(B, C, -1))
    ref, scale = ref.reshape(B, C, H, W).permute(0, 2, 3, 1).reshape(-1), scale.reshape(B, C, H, W).permute(0, 2, 3, 1).reshape(-1)
    got = dx.cpu().double()
    assert bool((got[scale == 0] == 0).all()), 'gradient where no window picked the element'
    err = float(((got - ref).abs() / scale.clamp_min(1e-300))[scale > 0].max())
    print(shape, kind, f'bwd {err:.2e}')
    assert err <= POOL_TOL


def test_maxpool_negative_controls(L):
    B, H, W, C = 1, 14, 22, 8
    g = torch.Generator().manual_seed(3)
    x = pool_input('ties', (B, H, W, C), g)
    xd = Buf(x.permute(0, 2, 3, 1).contiguous())
    y, idx = Buf(n=B * 7 * 11 * C), Buf(n=B * 7 * 11 * C, dtype=torch.uint8)
    lib_call(L, 'dboa_maxpool_fwd', xd.ptr, y.ptr, idx.ptr, B, H, W, C)
    ry, ridx, _ = pool_ref(x)
    assert same_values(y.cpu(), ry.reshape(-1)) and torch.equal(idx.cpu(), ridx.reshape(-1))
    # H and W swapped: the NHWC input read as (W, H)
    sw = x.permute(0, 2, 3, 1).reshape(B, W, H, C).permute(0, 3, 1, 2)
    sy, sidx, _ = pool_ref(sw)
    assert not torch.equal(idx.cpu(), sidx.reshape(-1))
    # the input has windows whose maximum occurs more than once, so the first-in-scan-order rule is exercised
    pad = F.pad(x, (1, 1, 1, 1), value=float('-inf'))
    win = pad.unfold(2, 3, 2).unfold(3, 3, 2).reshape(B, C, 7, 11, 9)
    ties = (win == win.max(-1, keepdim=True).values).sum(-1) > 1
    assert int(ties.sum()) > 50
    bad_idx = idx.cpu().clone()
    bad_idx[ties.permute(0, 2, 3, 1).reshape(-1).nonzero()[0]] += 1
    assert not torch.equal(bad_idx, ridx.reshape(-1))
    bad = y.cpu().clone()
    bad[5] += 0.5
    assert not same_values(bad, ry.reshape(-1))
    y.whole[y.n] = 0.0
    assert not y.intact()
