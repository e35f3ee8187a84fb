"""Fused convolution (csrc/conv_tc.cu with an operand transform): GroupNorm of the operand applied on load,
GroupNorm statistics of the output as fixed-point sums from the epilogue.  Checked against torch (fp64 convolution,
F.group_norm) on the device, one problem and two problems per launch, every transform mode, and end to end against the
unfused plan."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    _lib.load()
    return _lib


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def wmat(w):
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


def merged_stats(part, B, n_per_group):
    """fixed-point (sum, sum of squares) accumulators, long long [B][4][2], scale 2^24 -> mean, biased variance (fp64)."""
    acc = part.view(torch.int64)[:B * 8].view(B, 4, 2).double().cpu() / 2.0 ** 24
    mean = acc[..., 0] / n_per_group
    var = acc[..., 1] / n_per_group - mean ** 2
    return mean, var


def group_stats(y_nchw):
    B, Cc = y_nchw.shape[:2]
    g = y_nchw.double().reshape(B, 4, -1)
    return g.mean(-1).cpu(), g.var(-1, unbiased=False).cpu()


class Prob:
    """One problem of a fused launch: keeps every tensor alive and builds the C struct."""

    def __init__(self, L, B, Hi, Cin, Cout, k, stride, pad, mode, x, w, res=None, part_in=None, gamma=None, beta=None,
                 part2_in=None, gamma2=None, beta2=None, want_a=True):
        self.L, self.B, self.mode = L, B, mode
        self.Ho = (Hi + 2 * pad - k) // stride + 1
        dev = 'cuda'
        self.x, self.w, self.res = x, w, res
        self.y = torch.full((B, self.Ho, self.Ho, Cout), float('nan'), device=dev)
        self.part_out = torch.zeros(L.load().dboa_conv_fused_part_floats(B, self.Ho, Cout), device=dev)
        self.a_out = torch.full_like(x, float('nan')) if (mode >= 1 and want_a) else None
        self.stats_out = torch.full((B, 4, 2), float('nan'), device=dev) if mode >= 1 and want_a else None
        self.stats2_out = torch.full((B, 4, 2), float('nan'), device=dev) if mode == 3 and want_a else None
        self.keep = (part_in, gamma, beta, part2_in, gamma2, beta2)
        s = L.FusedConvStruct()
        for name, t in (('x', x), ('res', res), ('w', w), ('a_out', self.a_out), ('stats_out', self.stats_out), ('stats2_out', self.stats2_out),
                        ('part_in', part_in), ('part2_in', part2_in), ('gamma', gamma), ('beta', beta), ('gamma2', gamma2), ('beta2', beta2),
                        ('y', self.y), ('part_out', self.part_out)):
            setattr(s, name, None if t is None else t.data_ptr())
        s.mode = mode
        s.Hi, s.Cin, s.Cout, s.k, s.stride, s.pad = Hi, Cin, Cout, k, stride, pad
        self.struct = s


def launch(L, probs):
    B = probs[0].B
    arr = (L.FusedConvStruct * len(probs))(*[p.struct for p in probs])
    L.call('dboa_conv_fused_fwd', arr, len(probs), B, L.stream())
    torch.cuda.synchronize()


def check_output(p, a_nchw, w_nchw, stride, pad, tag):
    ref = F.conv2d(a_nchw.double(), w_nchw.double(), stride=stride, padding=pad)
    assert torch.isfinite(p.y).all(), tag
    # TF32x3 with fp32 accumulation in the tensor core: ~1e-6 for short reductions, up to ~2e-5 for K = 4608 in one chain
    assert rel_err(p.y.permute(0, 3, 1, 2), ref) < 3e-5, tag
    mean, var = merged_stats(p.part_out, p.B, ref[0].numel() / 4)
    rm, rv = group_stats(ref)
    assert (mean - rm).abs().max() <= 1e-5 * rv.sqrt().max() + 1e-6, tag
    assert ((var - rv).abs() / rv).max() < 3e-5, tag


CASES = [  # B, H, Cin, Cout, k, stride, pad
    (1, 56, 64, 64, 1, 1, 0), (1, 56, 64, 256, 1, 1, 0), (1, 56, 64, 64, 3, 1, 1), (2, 28, 128, 128, 3, 1, 1), (1, 28, 512, 128, 1, 1, 0),
    (1, 14, 256, 256, 3, 1, 1), (3, 14, 1024, 256, 1, 1, 0), (1, 7, 512, 2048, 1, 1, 0), (2, 7, 2048, 512, 1, 1, 0),
    (1, 7, 512, 512, 3, 1, 1), (9, 7, 512, 512, 3, 1, 1), (2, 28, 128, 512, 1, 1, 0),
    (1, 56, 128, 128, 3, 2, 1), (2, 28, 256, 256, 3, 2, 1), (1, 14, 512, 512, 3, 2, 1), (1, 56, 256, 512, 1, 2, 0), (3, 14, 1024, 2048, 1, 2, 0)]


@pytest.mark.parametrize('case', CASES)
def test_plain_operand_and_statistics(L, case):
    """mode 0: convolution of an existing activation; output and the per-group statistics its epilogue leaves."""
    B, H, Cin, Cout, k, s, pd = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, Cin, H, H, generator=g).cuda() + 0.3
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (k * k * Cin) ** 0.5).cuda()
    p = Prob(L, B, H, Cin, Cout, k, s, pd, 0, nhwc(x), wmat(w))
    launch(L, [p])
    check_output(p, x, w, s, pd, case)


CHAINS = [  # B, H, C0 (input of the producer), C1 (its output = operand channels), C2, k, stride of the consumer
    (1, 56, 64, 64, 64, 3, 1), (2, 56, 64, 128, 128, 1, 1), (1, 28, 128, 128, 512, 1, 1), (2, 14, 256, 256, 256, 3, 1), (1, 14, 256, 1024, 256, 1, 1),
    (1, 28, 128, 128, 128, 3, 1), (3, 7, 512, 512, 2048, 1, 1), (1, 7, 512, 2048, 512, 1, 1), (2, 7, 256, 512, 512, 3, 1),
    (1, 56, 64, 128, 128, 3, 2), (2, 28, 128, 256, 256, 3, 2), (1, 14, 256, 512, 512, 3, 2)]


@pytest.mark.parametrize('case', CHAINS)
def test_groupnorm_on_load(L, case):
    """producer (mode 0) -> consumer (mode 1): the consumer normalises with the producer's partial statistics, writes the
    activation and (mean, rstd) to the tape, and convolves the normalised operand."""
    B, H, C0, C1, C2, k, s = case
    g = torch.Generator().manual_seed(sum(case) + 1)
    x = torch.randn(B, C0, H, H, generator=g).cuda()
    w0 = (torch.randn(C1, C0, 1, 1, generator=g) / C0 ** 0.5).cuda()
    gamma = (1 + 0.3 * torch.randn(C1, generator=g)).cuda()
    beta = (0.2 * torch.randn(C1, generator=g)).cuda()
    w1 = (torch.randn(C2, C1, k, k, generator=g) / (k * k * C1) ** 0.5).cuda()
    p0 = Prob(L, B, H, C0, C1, 1, 1, 0, 0, nhwc(x), wmat(w0))
    launch(L, [p0])
    p1 = Prob(L, B, H, C1, C2, k, s, k // 2, 1, p0.y, wmat(w1), part_in=p0.part_out, gamma=gamma, beta=beta)
    launch(L, [p1])
    y0 = p0.y.permute(0, 3, 1, 2)
    a_ref = F.relu(F.group_norm(y0.double(), 4, gamma.double(), beta.double(), eps=1e-5))
    assert torch.isfinite(p1.a_out).all(), case
    assert rel_err(p1.a_out.permute(0, 3, 1, 2), a_ref) < 1e-5, case
    rm, rv = group_stats(y0)
    assert (p1.stats_out[..., 0].double().cpu() - rm).abs().max() < 1e-5 * rv.sqrt().max() + 1e-6
    assert rel_err(p1.stats_out[..., 1], 1.0 / (rv + 1e-5).sqrt()) < 2e-5
    check_output(p1, p1.a_out.permute(0, 3, 1, 2), w1, s, k // 2, case)


@pytest.mark.parametrize('B,H,C,planes,stride', [(1, 56, 256, 128, 2), (2, 14, 1024, 512, 2), (1, 28, 512, 128, 1), (1, 7, 2048, 512, 1), (1, 28, 512, 256, 2)])
@pytest.mark.parametrize('mode', [2, 3])
def test_block_output_on_load_two_problems(L, B, H, C, planes, stride, mode):
    """conv1 (+ the down-sampling 1x1 conv, second problem of the launch) of a bottleneck: the operand is the previous block's
    output relu(gn(y3) + shortcut), formed on load from y3 and either the materialised shortcut (mode 2) or the raw output
    of the previous block's down-sampling convolution and ITS GroupNorm (mode 3)."""
    g = torch.Generator().manual_seed(B + H + C + mode)
    Cq = C // 4
    xin = torch.randn(B, Cq, H, H, generator=g).cuda()
    w3 = (torch.randn(C, Cq, 1, 1, generator=g) / Cq ** 0.5).cuda()
    wd = (torch.randn(C, Cq, 1, 1, generator=g) / Cq ** 0.5).cuda()
    ga3, be3 = (1 + 0.3 * torch.randn(C, generator=g)).cuda(), (0.2 * torch.randn(C, generator=g)).cuda()
    gad, bed = (1 + 0.3 * torch.randn(C, generator=g)).cuda(), (0.2 * torch.randn(C, generator=g)).cuda()
    xin_d = nhwc(xin)                                               # both problems of a launch read the SAME operand tensor
    p3 = Prob(L, B, H, Cq, C, 1, 1, 0, 0, xin_d, wmat(w3))
    pdn = Prob(L, B, H, Cq, C, 1, 1, 0, 0, xin_d, wmat(wd))
    launch(L, [p3, pdn])                                            # two problems, mode 0
    y3, yd = p3.y.permute(0, 3, 1, 2).double(), pdn.y.permute(0, 3, 1, 2).double()
    if mode == 2:
        res = torch.randn(B, H, H, C, generator=g).cuda().abs()
        block_out = F.relu(F.group_norm(y3, 4, ga3.double(), be3.double(), eps=1e-5) + res.permute(0, 3, 1, 2).double())
        extra = dict(res=res)
    else:
        block_out = F.relu(F.group_norm(y3, 4, ga3.double(), be3.double(), eps=1e-5) + F.group_norm(yd, 4, gad.double(), bed.double(), eps=1e-5))
        extra = dict(res=pdn.y, part2_in=pdn.part_out, gamma2=gad, beta2=bed)
    w1 = (torch.randn(planes, C, 1, 1, generator=g) / C ** 0.5).cuda()
    wds = (torch.randn(planes * 4, C, 1, 1, generator=g) / C ** 0.5).cuda()
    common = dict(part_in=p3.part_out, gamma=ga3, beta=be3, **extra)
    c1 = Prob(L, B, H, C, planes, 1, 1, 0, mode, p3.y, wmat(w1), **common)
    ds = Prob(L, B, H, C, planes * 4, 1, stride, 0, mode, p3.y, wmat(wds), want_a=False, **common)
    launch(L, [c1, ds])
    assert rel_err(c1.a_out.permute(0, 3, 1, 2), block_out) < 1e-5
    check_output(c1, block_out, w1, 1, 0, 'conv1')
    check_output(ds, block_out, wds, stride, 0, 'downsample')
    if mode == 3:
        rm, rv = group_stats(yd)
        assert rel_err(c1.stats2_out[..., 1], 1.0 / (rv + 1e-5).sqrt()) < 2e-5


def test_fused_forward_fills_the_same_tape_as_the_unfused_plan(L):
    """Whole HMR forward: fused plan (one launch per convolution) against the unfused plan (conv + GroupNorm launches);
    outputs, all 15 features and the complete tape (y, statistics, activations: what the backward reads)."""
    from dynaboa_b200 import hmr as hmr_mod, synthetic
    from oracle import hmr_ref
    m = hmr_mod.hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    lib = L.load()
    for B in (1, 2, 9):
        x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(B)).cuda()
        outs = {}
        prev = lib.dboa_get_fused_forward()
        for fused in (0, 1):
            lib.dboa_set_fused_forward(fused)
            try:
                n0 = lib.dboa_launch_count()
                outs[fused] = hmr_mod.raw_forward(m.arena, m._buffers, x)
                torch.cuda.synchronize()
                outs[fused] += (lib.dboa_launch_count() - n0,)
            finally:
                lib.dboa_set_fused_forward(prev)
        (r0, s0, c0, p0, t0, n_un), (r1, s1, c1, p1, t1, n_fu) = outs[0], outs[1]
        print(f'B={B}: launches unfused {n_un} fused {n_fu}')
        assert n_fu <= n_un - 40
        assert rel_err(r1, r0) < 1e-4 and rel_err(s1, s0) < 1e-4 and rel_err(c1, c0) < 1e-4
        f0, f1 = hmr_mod._feature_views(t0, B), hmr_mod._feature_views(t1, B)
        for i in range(15):
            assert rel_err(f1[i], f0[i]) < 2e-4, (B, i)
        # the tape holds per-layer partial-statistics slots the unfused plan never writes: compare everything else through the
        # backward, which reads y, (mean, rstd) and the activations of every layer
        G0, G1 = torch.zeros_like(m.arena), torch.zeros_like(m.arena)
        dr, dsh, dc = torch.randn_like(r0), torch.randn_like(s0), torch.randn_like(c0)
        hmr_mod.raw_backward(m.arena, t0, B, False, dr, dsh, dc, G0)
        hmr_mod.raw_backward(m.arena, t1, B, False, dr, dsh, dc, G1)
        torch.cuda.synchronize()
        assert ((G1 - G0).norm() / G0.norm()).item() < 2e-3, B


WGRAD = [  # B, H (input), Cin, Cout, k, stride
    (1, 56, 64, 256, 1, 1), (1, 28, 128, 128, 3, 1), (2, 28, 512, 128, 1, 1), (1, 14, 256, 256, 3, 1), (3, 14, 1024, 256, 1, 1), (1, 7, 512, 512, 3, 1),
    (2, 7, 512, 2048, 1, 1), (9, 7, 2048, 512, 1, 1), (1, 14, 256, 1024, 1, 1), (1, 56, 128, 128, 3, 2), (2, 28, 256, 256, 3, 2), (1, 14, 512, 512, 3, 2),
    (1, 56, 256, 512, 1, 2), (2, 14, 1024, 2048, 1, 2)]


@pytest.mark.parametrize('case', WGRAD)
def test_weight_gradient_on_tensor_cores_mn_major(L, case):
    """Tensor-core weight gradient (dboa_conv2d_wgrad_tma: the wgmma kernel of csrc/conv_tc.cu) against the fp32 CUDA-core kernel and an fp64
    reference; dw is accumulated."""
    B, H, Cin, Cout, k, st = case
    g = torch.Generator().manual_seed(sum(case) + 3)
    Ho = H // st
    x = torch.randn(B, H, H, Cin, generator=g).cuda()
    dy = torch.randn(B, Ho, Ho, Cout, generator=g).cuda()
    K = k * k * Cin
    base = (torch.randn(Cout, K, generator=g) * 0.1).cuda()
    dw_tma, dw32 = base.clone(), base.clone()
    L.call('dboa_conv2d_wgrad_tma', L.ptr(dy), L.ptr(x), L.ptr(dw_tma), B, H, H, Cin, Cout, k, st, k // 2, K, L.stream())
    ws = torch.empty(8 << 20, device='cuda')
    L.call('dboa_conv2d_wgrad', L.ptr(dy), L.ptr(x), L.ptr(dw32), B, H, H, Cin, Cout, k, st, k // 2, K, L.ptr(ws), ws.numel(), L.stream())
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2).double(), (Cout, Cin, k, k), dy.permute(0, 3, 1, 2).double(), stride=st, padding=k // 2)
    ref = ref.permute(0, 2, 3, 1).reshape(Cout, K)
    assert rel_err(dw_tma - base, ref) < 2e-5, case
    assert rel_err(dw_tma - base, dw32 - base) < 2e-5, case


DGRAD = [  # B, H, Cin, Cout, k, nprep, addend
    (1, 56, 64, 64, 3, 1, False), (1, 56, 256, 64, 1, 1, True), (2, 28, 128, 128, 3, 1, False), (1, 28, 128, 512, 1, 0, False),
    (1, 14, 256, 256, 3, 1, False), (3, 14, 1024, 256, 1, 2, True), (1, 7, 512, 512, 3, 1, False), (2, 7, 2048, 512, 1, 1, True),
    (1, 7, 512, 2048, 1, 1, False), (9, 7, 512, 512, 3, 1, False)]
FIX = 2.0 ** 28


def _group_sums(q, xh, B):
    """(sum q, sum q x^) per (sample, group) of an NHWC tensor pair, fp64."""
    Cc = q.shape[-1]
    qg = q.double().reshape(B, -1, 4, Cc // 4).permute(0, 2, 1, 3).reshape(B, 4, -1)
    xg = xh.double().reshape(B, -1, 4, Cc // 4).permute(0, 2, 1, 3).reshape(B, 4, -1)
    return torch.stack([qg.sum(-1), (qg * xg).sum(-1)], -1)


def _stats(y, B):
    Cc = y.shape[-1]
    g = y.double().reshape(B, -1, 4, Cc // 4).permute(0, 2, 1, 3).reshape(B, 4, -1)
    mean, var = g.mean(-1), g.var(-1, unbiased=False)
    return torch.stack([mean, 1.0 / (var + 1e-5).sqrt()], -1)              # (B, 4, 2)


def _expand(st, Cc):                                                         # (B,4) -> (B,1,1,C)
    return st.repeat_interleave(Cc // 4, dim=1)[:, None, None, :]


@pytest.mark.parametrize('case', DGRAD)
def test_fused_data_gradient(L, case):
    """Fused data gradient (csrc/conv_tc.cu) against an fp64 torch restatement: GroupNorm_c backward on load, transposed convolution,
    shortcut addend, ReLU mask, and the fixed-point sums of the producing layer's GroupNorm backward(s)."""
    B, H, Cin, Cout, k, nprep, with_add = case
    g = torch.Generator().manual_seed(sum(case[:5]) + 17)
    rn = lambda *s: torch.randn(*s, generator=g).cuda()
    dz, y_c = rn(B, H, H, Cout) * 0.1, rn(B, H, H, Cout) + 0.2
    gamma_c = 1 + 0.3 * rn(Cout)
    w = rn(Cout, Cin, k, k) / (k * k * Cin) ** 0.5
    st_c = _stats(y_c, B)
    xh_c = (y_c.double() - _expand(st_c[..., 0], Cout)) * _expand(st_c[..., 1], Cout)
    q_c = dz.double() * gamma_c.double()
    sums_c = _group_sums(q_c, xh_c, B)
    N = H * H * Cout // 4
    dy = _expand(st_c[..., 1], Cout) * (q_c - _expand(sums_c[..., 0] / N, Cout) - xh_c * _expand(sums_c[..., 1] / N, Cout))
    dX = torch.nn.grad.conv2d_input((B, Cin, H, H), w.double(), dy.permute(0, 3, 1, 2), padding=k // 2).permute(0, 2, 3, 1)
    addend = rn(B, H, H, Cin) * 0.05 if with_add else None
    if addend is not None:
        dX = dX + addend.double()
    f = L.DgradFusedStruct()
    sums_c_fix = (sums_c * FIX).round().long().cuda().contiguous()
    st_c32 = st_c.float().cuda().contiguous()
    dy_out = torch.full((B, H, H, Cout), float('nan'), device='cuda')
    out = torch.full((B, H, H, Cin), float('nan'), device='cuda')
    keep = [dz, y_c, gamma_c, sums_c_fix, st_c32, dy_out, out, addend]
    wm = wmat(w)
    for name, t in (('dz', dz), ('y_c', y_c), ('w', wm), ('stats_c', st_c32), ('sums_c', sums_c_fix), ('gamma_c', gamma_c), ('dy_out', dy_out),
                    ('addend', addend), ('out', out)):
        setattr(f, name, None if t is None else t.data_ptr())
    preps = []
    if nprep > 0:
        a_p = rn(B, H, H, Cin)
        f.mask = a_p.data_ptr()
        for j in range(nprep):
            y_p, gamma_p = rn(B, H, H, Cin) - 0.1, 1 + 0.3 * rn(Cin)
            st_p = _stats(y_p, B).float().cuda().contiguous()
            sums_p = torch.zeros(B, 4, 2, dtype=torch.int64, device='cuda')
            dgb_p = torch.zeros(Cin, 2, dtype=torch.int64, device='cuda')
            f.prep_y[j], f.prep_stats[j], f.prep_gamma[j] = y_p.data_ptr(), st_p.data_ptr(), gamma_p.data_ptr()
            f.prep_sums[j], f.prep_dgb[j] = sums_p.data_ptr(), dgb_p.data_ptr()
            preps.append((y_p, gamma_p, st_p, sums_p, dgb_p))
        keep.append(a_p)
    f.nprep, f.accumulate = nprep, 0
    L.call('dboa_dgrad_fused', C.byref(f), B, H, Cin, Cout, k, L.stream())
    torch.cuda.synchronize()
    assert rel_err(dy_out, dy) < 2e-5, case
    if nprep == 0:
        assert rel_err(out, dX) < 3e-5, case
        return
    dz_p = dX * (a_p > 0)
    assert rel_err(out, dz_p) < 3e-5, case
    for y_p, gamma_p, st_p, sums_p, dgb_p in preps:
        xh = (y_p.double() - _expand(st_p[..., 0].double(), Cin)) * _expand(st_p[..., 1].double(), Cin)
        ref_sums = _group_sums(dz_p * gamma_p.double(), xh, B)
        got = sums_p.double() / FIX
        assert (got - ref_sums).abs().max() <= 3e-5 * ref_sums.abs().max() + 1e-6, case
        ref_dg, ref_db = (dz_p * xh).sum((0, 1, 2)), dz_p.sum((0, 1, 2))
        got_g = dgb_p.double() / FIX
        assert (got_g[:, 0] - ref_dg).abs().max() <= 3e-5 * ref_dg.abs().max() + 1e-6, case
        assert (got_g[:, 1] - ref_db).abs().max() <= 3e-5 * ref_db.abs().max() + 1e-6, case


def test_fused_backward_chain_matches_the_unfused_chain(L):
    """dboa_hmr_backward through the fused data-gradient chain (conv_tc.cu + gn_bwd_prep seams) against the default chain, same
    tape, B = 1, 2 and 9: the complete gradient arena."""
    from dynaboa_b200 import hmr as hmr_mod, synthetic
    from oracle import hmr_ref
    m = hmr_mod.hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    lib = L.load()
    for B in (1, 2, 9):
        x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(40 + B)).cuda()
        rot, shp, cam, _, tape = hmr_mod.raw_forward(m.arena, m._buffers, x)
        dr, dsh, dc = torch.randn_like(rot), torch.randn_like(shp), torch.randn_like(cam)
        G = []
        for fused in (0, 1):
            lib.dboa_set_fused_backward(fused)
            try:
                g = torch.zeros_like(m.arena)
                hmr_mod.raw_backward(m.arena, tape, B, False, dr, dsh, dc, g)
                torch.cuda.synchronize()
                G.append(g)
            finally:
                lib.dboa_set_fused_backward(0)          # the library default
        assert ((G[1] - G[0]).norm() / G[0].norm()).item() < 1e-4, B
        lay = hmr_mod.layout()
        for name, a, b in zip(lay.names, lay.views(G[0]), lay.views(G[1])):
            assert ((a - b).norm() <= 2e-3 * a.norm() + 1e-12), (B, name)
