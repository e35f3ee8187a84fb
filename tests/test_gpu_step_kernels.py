"""The kernels of an adapted frame outside the HMR plan and the loss head, through the C ABI, against exact references at
the sizes the step runs: the whole-arena sweeps (inner SGD, Adam + EMA teacher, EMA; csrc/optim.cu), the 15-pair cosine
feature test of the dynamic loop, retrieval's nearest centre, and the evaluation metrics (MPJPE, PA-MPJPE, PVE;
csrc/eval.cu).

The sweeps round every operation on its own (__fmul_rn, __fadd_rn, __fsub_rn, __fdiv_rn, __fsqrt_rn), so their results are
fully determined: they must equal, bit for bit, an op-by-op fp32 restatement on the CPU that uses only single-rounding
torch ops (no lerp / addcmul / addcdiv and no alpha=, which ATen's vectorised CPU kernels may evaluate with an FMA; the
square root is taken in fp64 and rounded once, since ATen's vectorised fp32 sqrt is not correctly rounded) and
derives Adam's scalars the way torch's single-tensor Adam does, in Python doubles cast once to fp32.  CPU tests pin the
restatement itself against fp64 Adam and against torch.optim.Adam.  The reductions (cosines, retrieval, evaluation) are
compared with fp64 sums of the same fp32 inputs, and their discrete decisions (the dynamic loop's threshold test, the
cluster pick) with the fp64 decision wherever the fp64 margin exceeds the measured error.

Every output buffer starts as NaN and is followed by a guard of sentinel values that must survive the call."""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from harness import COS_TOL, TERMS_TOL, Buf, adam_ref, ema_ref, f32, same_bits, sgd_ref

U32 = 2.0 ** -24                                   # unit roundoff of fp32
OK, ERR_ARG, ERR_SHAPE = 0, -1, -2
THRESHOLD = 3.1e-4                                 # bench.py's cos_sim_threshold


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    _lib.load()
    return _lib


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def sweep_sizes(L):
    """4, 1020, the grid cap of the sweeps (num_sms * 16 blocks of 256 float4) and its neighbours, the HMR arena."""
    cap = 4 * 256 * 16 * num_sms()
    return [4, 1020, cap - 4, cap, cap + 4, L.load().dboa_hmr_arena_floats()]


# ---------------------------------------------------------------------------------------------------------------------
# fp32 restatements of the sweeps (CPU), the fp64 Adam they must mean
# ---------------------------------------------------------------------------------------------------------------------
def adam_fp64(p, g, m, v, lr, betas, eps, step, gscale=1.0):
    """Adam in fp64 on the same fp32 inputs: (p, m, v, denom)."""
    beta1, beta2 = betas
    p, g, m, v = p.double(), g.double() * gscale, m.double(), v.double()
    m = m + (1.0 - beta1) * (g - m)
    v = beta2 * v + (1.0 - beta2) * g * g
    denom = v.sqrt() / math.sqrt(1.0 - beta2 ** step) + eps
    return p - lr / (1.0 - beta1 ** step) * m / denom, m, v, denom


def adam_state(n, step, seed, zero_block=0):
    """Seeded (p, g, m, v) of n floats.  Gradients span exact zeros, subnormals (g*g underflows), ~eps, ~1e3 and mixed
    signs; m and v are a plausible moment state after step - 1 steps (zero before the first).  The first ``zero_block``
    entries have g = m = v = 0."""
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen)
    mag = 10.0 ** (torch.rand(n, generator=gen) * 12 - 9)           # 1e-9 .. 1e3
    g = torch.randn(n, generator=gen) * mag
    kind = torch.randint(0, 8, (n,), generator=gen)
    g = torch.where(kind == 0, torch.zeros(()), g)
    g = torch.where(kind == 1, torch.randn(n, generator=gen) * 1e-40, g)  # subnormal
    g = torch.where(kind == 2, torch.randn(n, generator=gen) * 1e-8, g)   # about eps
    if step == 1:
        m, v = torch.zeros(n), torch.zeros(n)
    else:
        m = g * torch.rand(n, generator=gen) + torch.randn(n, generator=gen) * mag * 0.1
        v = m * m * (1 + 3 * torch.rand(n, generator=gen))
    if zero_block:
        g[:zero_block] = 0
        m[:zero_block] = 0
        v[:zero_block] = 0
    return p, g, m, v


def adam_units(p_in, g, m_in, ref, got, lr, betas, step, gscale=1.0):
    """Errors of (p, m, v) against the fp64 ``ref`` (p, m, v, denom) in units of the fp32 roundoff of their natural scales:
    for p its magnitude, its step and the step the roundoff of m can make (m's scale over denom), for m |m_in| + |g| (the
    lerp cancels), for v its magnitude (every term of v is non-negative)."""
    p, m, v = got
    rp, rm, rv, denom = ref
    g = g.double() * gscale
    m_scale = m_in.double().abs() + g.abs()
    p_scale = rp.abs() + 8 * (rp - p_in.double()).abs() + 4 * lr / (1.0 - betas[0] ** step) * m_scale / denom
    up = ((p.double() - rp).abs() / (U32 * p_scale).clamp_min(1e-45)).max().item()
    um = ((m.double() - rm).abs() / (U32 * m_scale).clamp_min(1e-45)).max().item()
    uv = ((v.double() - rv).abs() / (U32 * rv.abs()).clamp_min(1e-45)).max().item()
    return up, um, uv


# The fp32 restatement against fp64 Adam on the same fp32 inputs, in the units of adam_units.  Worst measured over the
# cases below: p 1.0, m 1.3, v 6.1 (at gscale 1/3, whose fp32 rounding v squares).
ADAM_FP64_UNITS = {'p': 2.0, 'm': 3.0, 'v': 10.0}
# The fp32 restatement against torch.optim.Adam(foreach=False) on the CPU, whose vectorised lerp_ / addcmul_ / addcdiv_
# may fuse: worst measured p 2.0, m 1.8, v 2.0 units.
ADAM_TORCH_UNITS = 4.0
BETAS = [(0.5, 0.9), (0.9, 0.999)]                 # bench.py's (lerp weight exactly 0.5: ATen's second branch); torch's default
STEPS = [1, 2, 3, 100, 10000]


@pytest.mark.parametrize('betas', BETAS)
@pytest.mark.parametrize('step', STEPS)
@pytest.mark.parametrize('gscale', [1.0, 0.5, 1.0 / 3.0])
def test_adam_restatement_means_adam(betas, step, gscale):
    """CPU: the restatement the GPU sweep is held to is Adam -- against fp64, and against torch.optim.Adam(foreach=False)."""
    n, lr, eps = 1 << 18, 3e-6, 1e-8
    p, g, m, v = adam_state(n, step, seed=step * 7 + int(betas[1] * 1000), zero_block=64 if step == 1 else 0)
    rp, rm, rv, _ = adam_ref(p, g, m, v, None, lr, betas, eps, step, gscale=gscale)
    ref64 = adam_fp64(p, g, m, v, lr, betas, eps, step, gscale=gscale)
    up, um, uv = adam_units(p, g, m, ref64, (rp, rm, rv), lr, betas, step, gscale)
    assert up <= ADAM_FP64_UNITS['p'] and um <= ADAM_FP64_UNITS['m'] and uv <= ADAM_FP64_UNITS['v'], (up, um, uv)
    pc = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([pc], lr=lr, betas=betas, eps=eps, foreach=False)
    opt.state[pc] = {'step': torch.tensor(float(step - 1)), 'exp_avg': m.clone(), 'exp_avg_sq': v.clone()}
    pc.grad = torch.mul(g, f32(gscale))
    opt.step()
    st = opt.state[pc]
    tp, tm, tv = adam_units(p, g, m, (rp.double(), rm.double(), rv.double(), ref64[3]), (pc.detach(), st['exp_avg'], st['exp_avg_sq']),
                            lr, betas, step, gscale)
    assert max(tp, tm, tv) <= ADAM_TORCH_UNITS, (tp, tm, tv)
    if step == 1:                                  # zero gradient on zero moments: nothing moves
        assert same_bits(rp[:64], p[:64]) and same_bits(rm[:64], m[:64]) and same_bits(rv[:64], v[:64])


def test_ema_restatement_means_ema():
    gen = torch.Generator().manual_seed(3)
    t, p = torch.randn(1 << 16, generator=gen), torch.randn(1 << 16, generator=gen)
    for alpha in (0.1, 0.99):
        got = ema_ref(t, p, alpha).double()
        ref = alpha * t.double() + (1 - alpha) * p.double()
        # three roundings of terms of the scale |t| + |p|: worst measured 2.0 units
        assert ((got - ref).abs() / (U32 * (t.double().abs() + p.double().abs()))).max().item() <= 4.0


# ---------------------------------------------------------------------------------------------------------------------
# sweeps on the GPU: bit equality
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sgd_sweep_bits(L):
    lr = 8e-6
    sizes = sweep_sizes(L)
    P = sizes[-1]
    for n in sizes + [8 * P]:                      # the last: an (8, P) stack of fast weights
        gen = torch.Generator().manual_seed(n % 9973)
        p, g = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-3
        g[: min(n, 16)] = 0
        pd, gd, out = Buf(p), Buf(g), Buf(n=n)
        L.call('dboa_sgd_update', pd.ptr, gd.ptr, out.ptr, lr, n, L.stream())
        assert same_bits(out.cpu(), sgd_ref(p, g, lr)), n
        assert out.intact() and pd.intact() and gd.intact() and same_bits(pd.cpu(), p)
    for n in (1, 2, 3, 5, 1022):
        out = Buf(n=n)
        assert L.load().dboa_sgd_update(Buf(n=n).ptr, Buf(n=n).ptr, out.ptr, lr, n, L.stream()) == ERR_SHAPE
        assert torch.isnan(out.cpu()).all() and out.intact()


def run_adam(L, bufs, n, lr, betas, eps, step, alpha, gscale, teacher=True):
    """dboa_adam_ema_scaled, or dboa_adam_ema for gscale None."""
    p, g, m, v, t = bufs
    args = [p.ptr, g.ptr, m.ptr, v.ptr, t.ptr if teacher else None, n, lr, betas[0], betas[1], eps, step, alpha]
    if gscale is None:
        L.call('dboa_adam_ema', *args, L.stream())
    else:
        L.call('dboa_adam_ema_scaled', *args, gscale, L.stream())


def check_adam_step(L, state, n, betas, step, gscale, teacher, alpha=0.1, lr=3e-6, eps=1e-8):
    """One Adam + EMA sweep from the device state ``state`` (p, g, m, v, t on the CPU) against adam_ref, bit for bit;
    returns the new state, read back from the device.  gscale None: the unscaled entry point."""
    p, g, m, v, t = state
    bufs = [Buf(x) for x in (p, g, m, v, t)]
    run_adam(L, bufs, n, lr, betas, eps, step, alpha, gscale, teacher)
    rp, rm, rv, rt = adam_ref(p, g, m, v, t if teacher else None, lr, betas, eps, step, alpha, 1.0 if gscale is None else gscale)
    got = [b.cpu() for b in bufs]
    tag = (n, betas, step, gscale, teacher)
    assert same_bits(got[0], rp) and same_bits(got[2], rm) and same_bits(got[3], rv), tag
    assert same_bits(got[4], rt if teacher else t), tag
    assert same_bits(got[1], g) and all(b.intact() for b in bufs), tag
    return got


@pytest.mark.gpu
@pytest.mark.parametrize('betas', BETAS)
def test_adam_ema_sweep_bits(L, betas):
    """Every (step, gscale, teacher) at a size past the grid cap; steps 1..3 at every sweep size, each step from the
    device's own state; the first entries have zero gradients and moments and must not move."""
    sizes = sweep_sizes(L)
    cap4 = sizes[4]
    for step in STEPS:
        for gscale in (1.0, 0.5, 1.0 / 3.0):
            p, g, m, v = adam_state(cap4, step, seed=step + 11, zero_block=64 if step == 1 else 0)
            t = p + 0.01 * torch.randn(cap4, generator=torch.Generator().manual_seed(5))
            with_t = check_adam_step(L, (p, g, m, v, t), cap4, betas, step, gscale, True)
            without = check_adam_step(L, (p, g, m, v, t), cap4, betas, step, gscale, False)
            for a, b in zip(with_t[:4], without[:4]):               # the teacher never changes p, m, v
                assert same_bits(a, b)
            if step == 1:
                assert same_bits(with_t[0][:64], p[:64]) and same_bits(with_t[2][:64], m[:64]) and same_bits(with_t[3][:64], v[:64])
        check_adam_step(L, (p, g, m, v, t), cap4, betas, step, None, True)         # dboa_adam_ema: gscale 1 implied
    for n in sizes:
        p, g, m, v = adam_state(n, 1, seed=n % 7919)
        state = (p, g, m, v, p.clone())
        for step in (1, 2, 3):
            got = check_adam_step(L, state, n, betas, step, 1.0, True)
            g = torch.randn(n, generator=torch.Generator().manual_seed(step)) * 1e-3
            state = (got[0], g, got[2], got[3], got[4])


@pytest.mark.gpu
def test_adam_ema_argument_checks(L):
    lib, bufs = L.load(), [Buf(n=8) for _ in range(5)]
    p, g, m, v, t = (b.ptr for b in bufs)
    assert lib.dboa_adam_ema(p, g, m, v, t, 6, 3e-6, 0.5, 0.9, 1e-8, 1, 0.1, L.stream()) == ERR_ARG      # n % 4
    assert lib.dboa_adam_ema(p, g, m, v, t, 8, 3e-6, 0.5, 0.9, 1e-8, 0, 0.1, L.stream()) == ERR_ARG      # step < 1
    assert lib.dboa_adam_ema(p, None, m, v, t, 8, 3e-6, 0.5, 0.9, 1e-8, 1, 0.1, L.stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert all(torch.isnan(b.cpu()).all() and b.intact() for b in bufs)


@pytest.mark.gpu
def test_ema_sweep_bits(L):
    for n in sweep_sizes(L):
        gen = torch.Generator().manual_seed(n % 6007)
        t, p = torch.randn(n, generator=gen), torch.randn(n, generator=gen)
        for alpha in (0.1, 0.99):
            td, pd = Buf(t), Buf(p)
            L.call('dboa_ema_update', td.ptr, pd.ptr, n, alpha, L.stream())
            assert same_bits(td.cpu(), ema_ref(t, p, alpha)), (n, alpha)
            assert td.intact() and pd.intact() and same_bits(pd.cpu(), p)
    out = Buf(n=6)
    assert L.load().dboa_ema_update(out.ptr, Buf(n=6).ptr, 6, 0.1, L.stream()) == ERR_SHAPE


@pytest.mark.gpu
def test_pool_adam_runs(L):
    """A (G, P) pool stack swept as MultiVideoAdaptor._adam_ema does it: one dboa_adam_ema_groups call, every active video at
    its own step count.  Each video's rows equal a one-video call at its own step; idle videos keep every bit."""
    G, P = 6, L.load().dboa_hmr_arena_floats()
    steps = [3, 1, 1, 5, 2, 2]
    on = 0b110111                                     # video 3 idle
    lr, betas, alpha = 3e-6, (0.5, 0.9), 0.1
    stack = [torch.empty(G, P, device='cuda') for _ in range(5)]     # theta, grad, m, v, teacher
    for k in range(G):
        for x, y in zip(stack, adam_state(P, steps[k], seed=100 + k)):
            x[k] = y.cuda()
    stack[4].copy_(stack[0] * 0.999)
    bufs = [Buf(x) for x in stack]
    rows, row = (C.c_float * (G * L.ADAM_SCALARS))(), (C.c_float * L.ADAM_SCALARS)()
    for k in range(G):
        if (on >> k) & 1:
            L.call('dboa_adam_scalars', row, lr, betas[0], betas[1], 1e-8, steps[k], alpha, 1.0)
            rows[k * L.ADAM_SCALARS:(k + 1) * L.ADAM_SCALARS] = row[:]
    L.call('dboa_adam_ema_groups', *(b.ptr for b in bufs), P, rows, G, on, L.stream())
    got = [b.t.view(G, P) for b in bufs]
    assert all(b.intact() for b in bufs)
    for k in range(G):
        if (on >> k) & 1:
            one = [Buf(x[k]) for x in stack]
            run_adam(L, one, P, lr, betas, 1e-8, steps[k], alpha, 1.0)
            for x, y in zip(got, one):
                assert same_bits(x[k], y.t), k
        else:
            for x, y in zip(got, stack):
                assert same_bits(x[k], y[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# the feature test
# ---------------------------------------------------------------------------------------------------------------------
def feature_lengths(L, b):
    lib = L.load()
    off, nd = C.c_longlong(), C.c_int()
    shp, strd = (C.c_longlong * 4)(), (C.c_longlong * 4)()
    out = []
    for i in range(15):
        L.check(lib.dboa_hmr_feature_info(b, i, C.byref(off), C.byref(nd), shp, strd), 'dboa_hmr_feature_info')
        out.append(math.prod(shp[k] for k in range(nd.value)))
    return out


def cosine_terms(L, A, B, G, active, partial_floats=None):
    """dboa_cosine_terms_active on lists of dense device tensors: (status, terms Buf (G, n, 3), partial Buf)."""
    lib, n = L.load(), len(A)
    pa = (C.c_void_p * n)(*[t.data_ptr() for t in A])
    pb = (C.c_void_p * n)(*[t.data_ptr() for t in B])
    ln = (C.c_longlong * n)(*[t.numel() for t in A])
    need = lib.dboa_cosine_partial_floats_groups(ln, n, G) if n <= 16 else 3 * 4096
    part = Buf(n=need if partial_floats is None else partial_floats)
    terms = Buf(n=G * n * 3, dtype=torch.float64)
    st = lib.dboa_cosine_terms_active(pa, pb, ln, n, part.ptr, part.n, terms.ptr, L.stream(), G, active)
    torch.cuda.synchronize()
    return st, terms, part


def fp64_terms(A, B, G):
    """(G, n, 3) fp64 sums (a.b, |a|^2, |b|^2) of each video's part, and the (G, n) scales sum |a_k b_k|, |a|^2, |b|^2."""
    rows = []
    for a, b in zip(A, B):
        a, b = a.double().view(G, -1), b.double().view(G, -1)
        rows.append(torch.stack([(a * b).sum(1), (a * a).sum(1), (b * b).sum(1), (a * b).abs().sum(1)], 1).cpu())
    t = torch.stack(rows, 1)
    return t[..., :3], torch.stack([t[..., 3], t[..., 1], t[..., 2]], -1)


def one_minus_cos(t):
    return 1.0 - t[..., 0] / (t[..., 1].sqrt().clamp_min(1e-12) * t[..., 2].sqrt().clamp_min(1e-12))


def feature_pairs(lengths, G, seed):
    """Pairs b = a + delta * noise per video, with delta set so that fp64 1 - cos spans 1e-6 .. 1e-2, half of the pairs
    within 3% of the benchmark threshold."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    cpu = torch.Generator().manual_seed(seed)
    A, B = [], []
    for n in lengths:
        k = n // G
        target = torch.where(torch.rand(G, 1, generator=cpu) < 0.5, 10.0 ** (torch.rand(G, 1, generator=cpu) * 4 - 6),
                             THRESHOLD * (1 + 0.06 * (torch.rand(G, 1, generator=cpu) - 0.5)))
        a = torch.randn(G, k, device='cuda', generator=gen)
        b = a + (2 * target).sqrt().cuda() * torch.randn(G, k, device='cuda', generator=gen)
        A.append(a.reshape(-1))
        B.append(b.reshape(-1))
    return A, B


# TERMS_TOL, COS_TOL (harness.py): the bounds against fp64 sums of the same fp32 inputs.  dboa_cosine_terms equals the grouped
# call at G = 1 bit for bit.
def check_cosine_case(L, A, B, G, active, record):
    st, terms, part = cosine_terms(L, A, B, G, active)
    assert st == OK and terms.intact() and part.intact()
    ref, scale = fp64_terms(A, B, G)
    got = terms.cpu().view(G, len(A), 3)
    on = [g for g in range(G) if (active >> g) & 1]
    off = [g for g in range(G) if not (active >> g) & 1]
    assert torch.isnan(got[off]).all()                              # idle videos' rows are not written
    err = ((got[on] - ref[on]).abs() / scale[on]).max().item()
    dcos = (one_minus_cos(got[on]) - one_minus_cos(ref[on])).abs().max().item()
    record['terms'] = max(record.get('terms', 0.0), err)
    record['cos'] = max(record.get('cos', 0.0), dcos)
    assert err <= TERMS_TOL and dcos <= COS_TOL, (err, dcos)
    return ref, on


def check_decisions(A, B, G, active, ref, on):
    """fused.cosines + fused._continuing on the device sums take the fp64 branch for every pair clear of the bound."""
    from dynaboa_b200 import fused
    cos, _ = fused.cosines(A, B, G, active, None)
    d64 = one_minus_cos(ref)
    o = SimpleNamespace(cos_sim_threshold=THRESHOLD, optim_steps=1 << 30)
    checked = 0
    for i in range(len(A)):
        # the loop tests one feature's cosine (pair 12): put pair i in its place
        mask = fused._continuing(o, {g: {12: {'cos': float(cos[g, i])}} for g in on}, [0] * G)
        for g in on:
            if abs(d64[g, i].item() - THRESHOLD) > COS_TOL + 3e-8:
                assert ((mask >> g) & 1) == (d64[g, i].item() > THRESHOLD), (g, i, d64[g, i].item(), float(cos[g, i]))
                checked += 1
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize('G,b,active', [(1, 1, 1), (1, 2, 1), (1, 9, 1), (1, 64, 1), (2, 1, 0b10), (2, 2, 0b01), (2, 8, 0b11),
                                        (4, 1, 0b1101), (4, 2, 0b1011), (4, 8, 0b0110), (8, 1, 0b10110101), (8, 2, 0xFF),
                                        (8, 8, 0b01011100)])
def test_cosine_terms_at_feature_lengths(L, G, b, active):
    lengths = [n * G for n in feature_lengths(L, b)]
    A, B = feature_pairs(lengths, G, seed=G * 100 + b)
    record = {}
    ref, on = check_cosine_case(L, A, B, G, active, record)
    assert check_decisions(A, B, G, active, ref, on) >= len(on) * len(A) // 2
    if G == 1:                                  # dboa_cosine_terms is the grouped call at G = 1; and the float cosines of dboa_cosine_pairs
        n = len(A)
        st, terms, _ = cosine_terms(L, A, B, 1, 1)
        one = Buf(n=n * 3, dtype=torch.float64)
        part = Buf(n=L.load().dboa_cosine_partial_floats((C.c_longlong * n)(*[t.numel() for t in A]), n))
        L.call('dboa_cosine_terms', (C.c_void_p * n)(*[t.data_ptr() for t in A]), (C.c_void_p * n)(*[t.data_ptr() for t in B]),
               (C.c_longlong * n)(*[t.numel() for t in A]), n, part.ptr, part.n, one.ptr, L.stream())
        assert st == OK and same_bits(one.cpu(), terms.cpu()) and one.intact() and part.intact()
        out = Buf(n=n)
        pa = (C.c_void_p * n)(*[t.data_ptr() for t in A])
        pb = (C.c_void_p * n)(*[t.data_ptr() for t in B])
        ln = (C.c_longlong * n)(*[t.numel() for t in A])
        part = Buf(n=L.load().dboa_cosine_partial_floats(ln, n))
        L.call('dboa_cosine_pairs', pa, pb, ln, n, part.ptr, part.n, out.ptr, 1e-12, L.stream())
        assert out.intact() and part.intact()
        assert ((1.0 - out.cpu().double()) - one_minus_cos(ref[0])).abs().max().item() <= COS_TOL + 6e-8
    print(f'cosines G={G} b={b}: terms {record["terms"]:.2e}, 1 - cos {record["cos"]:.2e}')


@pytest.mark.gpu
def test_cosine_edges(L):
    lib = L.load()
    record = {}
    for G in (1, 2):
        lengths = [G * n for n in (1, 7, 4095, 4096, 4097, 8191, 8192, 12289)]
        A, B = feature_pairs(lengths, G, seed=7 + G)
        check_cosine_case(L, A, B, G, (1 << G) - 1, record)
    gen = torch.Generator(device='cuda').manual_seed(1)
    A16 = [torch.randn(4096 + 4 * i, device='cuda', generator=gen) for i in range(17)]
    B16 = [a + 0.01 * torch.randn(a.shape, device='cuda', generator=gen) for a in A16]
    check_cosine_case(L, A16[:16], B16[:16], 1, 1, record)          # 16 pairs: accepted
    st, terms, part = cosine_terms(L, A16, B16, 1, 1)               # 17: rejected before any launch
    assert st == ERR_ARG and torch.isnan(terms.cpu()).all() and torch.isnan(part.cpu()).all()
    ln = (C.c_longlong * 17)(*[t.numel() for t in A16])
    assert lib.dboa_cosine_partial_floats_groups(ln, 17, 1) == ERR_ARG
    need = lib.dboa_cosine_partial_floats_groups(ln, 16, 1)
    st, terms, part = cosine_terms(L, A16[:16], B16[:16], 1, 1, partial_floats=need - 1)
    assert st == ERR_ARG and torch.isnan(terms.cpu()).all() and torch.isnan(part.cpu()).all() and terms.intact()
    # an all-zero pair: cos = 0, as F.cosine_similarity(eps=1e-12)
    z = [torch.zeros(4096, device='cuda')]
    st, terms, _ = cosine_terms(L, z, z, 1, 1)
    assert st == OK and torch.equal(terms.cpu(), torch.zeros(3, dtype=torch.float64))
    from dynaboa_b200 import fused
    assert float(fused.cosines(z, z, 1, 1, None)[0][0, 0]) == 0.0
    assert float(torch.nn.functional.cosine_similarity(z[0], z[0], dim=0, eps=1e-12)) == 0.0
    out, part = Buf(n=1), Buf(n=lib.dboa_cosine_partial_floats((C.c_longlong * 1)(4096), 1))
    L.call('dboa_cosine_pairs', (C.c_void_p * 1)(z[0].data_ptr()), (C.c_void_p * 1)(z[0].data_ptr()), (C.c_longlong * 1)(4096), 1,
           part.ptr, part.n, out.ptr, 1e-12, L.stream())
    assert float(out.cpu()[0]) == 0.0 and out.intact()
    print(f'cosine edges: terms {record["terms"]:.2e}, 1 - cos {record["cos"]:.2e}')


# ---------------------------------------------------------------------------------------------------------------------
# retrieval
# ---------------------------------------------------------------------------------------------------------------------
# |dists - fp64 (1 - cos)| (norms clamped at 1e-8 each): worst measured 1.9e-7 (K = 64, D = 2047; exact at D = 1).
RETRIEVAL_TOL = 1e-6


def retrieval(L, feat, centers):
    K, D = centers.shape
    best, dists = Buf(n=1, dtype=torch.int32), Buf(n=K)
    fd, cd = Buf(feat), Buf(centers)
    st = L.load().dboa_retrieval_nearest(fd.ptr, cd.ptr, K, D, best.ptr, dists.ptr, L.stream())
    torch.cuda.synchronize()
    assert best.intact() and dists.intact()
    return st, int(best.cpu()[0]), dists.cpu()


def retrieval_fp64(feat, centers):
    f, c = feat.double(), centers.double()
    return 1.0 - (c @ f) / (f.norm().clamp_min(1e-8) * c.norm(dim=1).clamp_min(1e-8))


@pytest.mark.gpu
@pytest.mark.parametrize('D', [2048, 2047, 1])
@pytest.mark.parametrize('K', [1, 7, 8, 9, 33, 64])
def test_retrieval_nearest(L, K, D):
    gen = torch.Generator().manual_seed(K * 4099 + D)
    feat = torch.rand(D, generator=gen)
    # centres at graded distances from the feature (relative noise 10^-3 .. 10^0), shuffled
    noise = 10.0 ** (-3 + 3 * torch.rand(K, 1, generator=gen))
    centers = (feat * (0.5 + torch.rand(K, 1, generator=gen)) + noise * torch.rand(K, D, generator=gen))[torch.randperm(K, generator=gen)]
    st, best, d = retrieval(L, feat, centers.contiguous())
    assert st == OK
    ref = retrieval_fp64(feat, centers)
    err = (d.double() - ref).abs().max().item()
    assert err <= RETRIEVAL_TOL, err
    assert best == int(torch.nonzero(d == d.min())[0])              # the first minimum of what it returns
    srt = ref.sort().values
    if K == 1 or (srt[1] - srt[0]).item() > 2 * RETRIEVAL_TOL:
        assert best == int(ref.argmin())
    print(f'retrieval K={K} D={D}: {err:.2e}')


@pytest.mark.gpu
def test_retrieval_edges(L):
    gen = torch.Generator().manual_seed(17)
    feat = torch.rand(2048, generator=gen)
    centers = torch.rand(40, 2048, generator=gen)
    centers[13] = feat * 2 + 1e-3 * torch.rand(2048, generator=gen)
    centers[29] = centers[13]                                       # a duplicate of the nearest: the lower index wins
    centers[21] = centers[13]
    centers[5] = 0                                                  # a zero centre: distance exactly 1
    st, best, d = retrieval(L, feat, centers)
    assert st == OK and best == 13 and d[13] == d[21] == d[29] and float(d[5]) == 1.0
    centers[3] = centers[13]                                        # ... also when the duplicate comes first
    st, best, d = retrieval(L, feat, centers)
    assert best == 3
    for K in (0, 65):
        c = torch.rand(max(K, 1), 64, generator=gen)
        best, dists = Buf(n=1, dtype=torch.int32), Buf(n=max(K, 1))
        assert L.load().dboa_retrieval_nearest(Buf(feat[:64].clone()).ptr, Buf(c).ptr, K, 64, best.ptr, dists.ptr, L.stream()) == ERR_SHAPE
        torch.cuda.synchronize()
        assert int(best.cpu()[0]) == -7 and torch.isnan(dists.cpu()).all() and best.intact() and dists.intact()


# ---------------------------------------------------------------------------------------------------------------------
# evaluation: MPJPE, PA-MPJPE, PVE
# ---------------------------------------------------------------------------------------------------------------------
# Against oracle/eval_ref.py in fp64, relative to the largest ground-truth joint distance from the pelvis.  The joints are
# exact here (one-hot regressor rows), so what remains is the fp64 Procrustes and the final cast to fp32: worst measured
# 6.0e-8 over MPJPE and PA-MPJPE (64 axis-aligned collinear predictions; 64 planar ones 4.9e-8, the edge cases 3.1e-8,
# idle-video rows 1.2e-8); PVE 2.6e-8 relative to itself.
EVAL_TOL = 5e-7
# With a dense regressor the fp32 joint sums round too: |out - fp64| <= EVAL_DENSE_TOL * max |fp64| over MPJPE, PA-MPJPE
# and PVE.  Worst measured: 1.5e-7 (NJ = 32), 1.0e-7 (NV = 5 < NJ).
EVAL_DENSE_TOL = 1e-5


def eval_call(L, pred, gt, gtn, J, jmap, groups=1, active=None):
    """dboa_eval_metrics(_active) on fp32 numpy inputs: (status, (B,3) output with NaN where unwritten)."""
    B, NV, NJ = pred.shape[0], pred.shape[1], J.shape[0]
    args = [Buf(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))) for x in (pred, gt, gtn, J)]
    jm = Buf(torch.from_numpy(np.asarray(jmap, dtype=np.int32)))
    scratch = Buf(n=max(1, L.load().dboa_eval_scratch_floats(B, min(NJ, 32))))
    out = Buf(n=B * 3)
    lib = L.load()
    common = [a.ptr for a in args] + [NJ, NV, jm.ptr, jm.n, scratch.ptr, out.ptr, B]
    if active is None:
        st = lib.dboa_eval_metrics(*common, L.stream())
    else:
        st = lib.dboa_eval_metrics_active(*common, groups, active, L.stream())
    torch.cuda.synchronize()
    assert out.intact() and scratch.intact() and all(a.intact() for a in args) and jm.intact()
    return st, out.cpu().view(B, 3).double().numpy()


def eval_ref64(pred, gt, gtn, J, jmap):
    from oracle import eval_ref
    p, g, n, Jd = (x.astype(np.float64) for x in (pred, gt, gtn, J))
    m, pa, _ = eval_ref.eval_metrics(p, g, n, Jd, np.asarray(jmap))
    pve = np.sqrt(((n - p) ** 2).sum(2)).mean(1)
    return np.stack([m, pa, pve], 1)


def eval_scale(joints, jmap):
    """The largest distance of an evaluation joint from the pelvis (regressor joint 0)."""
    j = np.asarray(joints, dtype=np.float64)
    return np.linalg.norm(j[jmap] - j[0], axis=1).max()


def one_hot_regressor(NJ, NV, rng):
    """Joint j is vertex idx[j] exactly (weight 1, all others 0): the regressed joints equal the chosen vertices bit for bit."""
    idx = rng.choice(NV, NJ, replace=False)
    J = np.zeros((NJ, NV), np.float32)
    J[np.arange(NJ), idx] = 1
    return J, idx


def rotation(rng):
    q, r = np.linalg.qr(rng.randn(3, 3))
    q = q * np.sign(np.diag(r))
    return q * np.sign(np.linalg.det(q))


def edge_predictions(gt_joints, rng):
    """Eval-joint sets of the predictions, from (NJ, 3) ground-truth joints: identical, an exact similarity transform, a
    mirror image, planar (axis-aligned: exactly rank 2 after centring, and tilted), collinear (along an axis: exactly rank
    1, and oblique), generic."""
    NJ = gt_joints.shape[0]
    R, s, t = rotation(rng), 1.3, np.array([0.2, -0.1, 0.4])
    plane = gt_joints.copy()
    plane[:, 2] = 0.37
    axis_line = np.zeros_like(gt_joints)
    axis_line[:, 0] = rng.randn(NJ) * 0.4
    axis_line[:, 1:] = (0.11, -0.23)
    d = rng.randn(3)
    return {
        'identical': gt_joints,
        'similarity': (s * gt_joints @ R.T + t),
        'mirror': gt_joints * np.array([-1.0, 1.0, 1.0]),
        'planar': plane,
        'planar_tilted': (gt_joints * np.array([1.0, 1.0, 0.0])) @ rotation(rng).T,
        'collinear': axis_line,
        'collinear_oblique': rng.randn(NJ, 1) * 0.4 * d / np.linalg.norm(d) + rng.randn(3) * 0.1,
        'generic': gt_joints * 1.1 + rng.randn(NJ, 3) * 0.05,
    }


@pytest.mark.gpu
def test_eval_procrustes_edges(L):
    from dynaboa_b200 import constants as K
    rng = np.random.RandomState(5)
    NV, NJ = 6890, 17
    jmap = np.asarray(K.H36M_TO_J14)
    J, idx = one_hot_regressor(NJ, NV, rng)
    gt = (rng.randn(NV, 3) * 0.5).astype(np.float32)
    preds = edge_predictions(gt[idx].astype(np.float64), rng)
    names = list(preds)
    P = np.repeat(gt[None], len(names), 0) + (rng.randn(len(names), NV, 3) * 0.03).astype(np.float32)
    for k, name in enumerate(names):
        P[k, idx] = preds[name]
    GT = np.repeat(gt[None], len(names), 0)
    GTN = (GT + 0.01).astype(np.float32)
    st, out = eval_call(L, P, GT, GTN, J, jmap)
    assert st == OK and np.isfinite(out).all(), dict(zip(names, out.tolist()))
    ref = eval_ref64(P, GT, GTN, J, jmap)
    scale = eval_scale(gt[idx], jmap)
    err = np.abs(out[:, :2] - ref[:, :2]).max(1) / scale
    worst = {n: float(e) for n, e in zip(names, err)}
    assert (err <= EVAL_TOL).all(), worst
    assert (np.abs(out[:, 2] - ref[:, 2]) <= EVAL_TOL * ref[:, 2]).all()
    i = names.index('identical')
    assert out[i, 0] == 0.0 and out[i, 1] <= EVAL_TOL * scale
    assert out[names.index('similarity'), 1] <= EVAL_TOL * scale
    print('eval edges:', {n: f'{e:.1e}' for n, e in worst.items()}, f'pve {(np.abs(out[:, 2] - ref[:, 2]) / ref[:, 2]).max():.1e}')


@pytest.mark.gpu
def test_eval_degenerate_ground_truth_is_finite(L):
    """With planar, collinear or coincident ground-truth joints the optimal rotation is not unique: no reference value,
    but the metrics must be finite."""
    from dynaboa_b200 import constants as K
    rng = np.random.RandomState(6)
    NV, NJ = 500, 17
    J, idx = one_hot_regressor(NJ, NV, rng)
    base = rng.randn(NV, 3).astype(np.float32) * 0.5
    GT = np.repeat(base[None], 3, 0)
    GT[0, idx, 2] = 0.5                                               # planar
    GT[1, idx, 1:] = (0.1, 0.2)                                       # collinear
    GT[2, idx] = (0.3, 0.1, -0.2)                                     # coincident: zero covariance
    P = np.repeat(base[None], 3, 0) + (rng.randn(3, NV, 3) * 0.05).astype(np.float32)
    jmap = np.asarray(K.H36M_TO_J14)
    st, out = eval_call(L, P, GT, GT, J, jmap)                        # generic predictions
    assert st == OK and np.isfinite(out).all(), out
    st, out = eval_call(L, GT[:2].copy(), GT[:2], GT[:2], J, jmap)    # predictions as degenerate as the ground truth
    assert st == OK and np.isfinite(out).all(), out


@pytest.mark.gpu
def test_eval_shapes_and_active(L):
    from dynaboa_b200 import constants as K
    rng = np.random.RandomState(7)
    # NJ = n_map = 32 is accepted, 33 is not
    for NJ, want in ((32, OK), (33, ERR_SHAPE)):
        NV = 300
        J = rng.rand(NJ, NV).astype(np.float32) ** 8
        J /= J.sum(1, keepdims=True)
        gt = (rng.randn(2, NV, 3) * 0.5).astype(np.float32)
        pred = (gt * 1.05 + rng.randn(2, NV, 3) * 0.05).astype(np.float32)
        jmap = np.arange(NJ)
        st, out = eval_call(L, pred, gt, gt, J, jmap)
        assert st == want, NJ
        if want == OK:
            ref = eval_ref64(pred, gt, gt, J, jmap)
            e32 = np.abs(out - ref).max() / np.abs(ref).max()
            assert e32 <= EVAL_DENSE_TOL, (out, ref)
        else:
            assert np.isnan(out).all()
    # fewer vertices than joints: the PVE slices of joints >= NV are empty
    NV, NJ = 5, 17
    J = rng.rand(NJ, NV).astype(np.float32)
    J /= J.sum(1, keepdims=True)
    gt = (rng.randn(3, NV, 3) * 0.5).astype(np.float32)
    pred = (gt + rng.randn(3, NV, 3) * 0.1).astype(np.float32)
    gtn = (gt + 0.02).astype(np.float32)
    jmap = np.asarray(K.H36M_TO_J14)
    st, out = eval_call(L, pred, gt, gtn, J, jmap)
    ref = eval_ref64(pred, gt, gtn, J, jmap)
    e5 = np.abs(out - ref).max() / np.abs(ref).max()
    assert st == OK and e5 <= EVAL_DENSE_TOL, (out, ref)
    # three videos of two rows, the middle one idle: its rows are not written
    NV, NJ = 2000, 17
    J, idx = one_hot_regressor(NJ, NV, rng)
    gt = (rng.randn(6, NV, 3) * 0.5).astype(np.float32)
    pred = (gt * 0.9 + rng.randn(6, NV, 3) * 0.05).astype(np.float32)
    pred[4, idx, 1:] = (0.2, 0.3)                                     # a collinear prediction in an active video
    st, out = eval_call(L, pred, gt, gt, J, jmap, groups=3, active=0b101)
    assert st == OK and np.isnan(out[2:4]).all() and np.isfinite(out[[0, 1, 4, 5]]).all()
    ref = eval_ref64(pred, gt, gt, J, jmap)
    rows = [0, 1, 4, 5]
    scale = np.array([eval_scale(gt[r, idx], jmap) for r in rows])   # one-hot regressor: the bound of the edge test
    e_act = (np.abs(out[rows, :2] - ref[rows, :2]).max(1) / scale).max()
    assert e_act <= EVAL_TOL and (np.abs(out[rows, 2] - ref[rows, 2]) <= EVAL_TOL * ref[rows, 2]).all()
    print(f'eval shapes: NJ = 32 {e32:.1e}, NV = 5 {e5:.1e}, active rows {e_act:.1e}')


@pytest.mark.gpu
def test_eval_rank_deficient_batches(L):
    """64 seeded predictions whose evaluation joints lie on a coordinate axis line (covariance of rank 1) and 64 on a
    coordinate plane (rank 2), each against its own full-rank ground truth and oracle/eval_ref.  The Jacobi sweeps leave
    spare columns anywhere from exactly zero down to underflow; every one must be completed to an orthonormal U."""
    from dynaboa_b200 import constants as K
    rng = np.random.RandomState(8)
    NV, NJ, n = 200, 17, 64
    jmap = np.asarray(K.H36M_TO_J14)
    J, idx = one_hot_regressor(NJ, NV, rng)
    GT = (rng.randn(2 * n, NV, 3) * 0.5).astype(np.float32)
    P = (rng.randn(2 * n, NV, 3) * 0.5).astype(np.float32)
    for k in range(2 * n):
        axis = rng.randint(3)
        fixed = [c for c in range(3) if c != axis] if k < n else [axis]
        P[k][np.ix_(idx, fixed)] = rng.randn(len(fixed)).astype(np.float32)    # constant coordinates across the joints
    st, out = eval_call(L, P, GT, GT, J, jmap)
    assert st == OK and np.isfinite(out).all()
    ref = eval_ref64(P, GT, GT, J, jmap)
    scale = np.array([eval_scale(GT[k, idx], jmap) for k in range(2 * n)])
    err = np.abs(out[:, :2] - ref[:, :2]).max(1) / scale
    print(f'rank-deficient predictions: collinear {err[:n].max():.1e}, planar {err[n:].max():.1e}')
    assert (err <= EVAL_TOL).all(), {k: float(err[k]) for k in np.nonzero(err > EVAL_TOL)[0]}
