"""wgmma TF32x3 GEMM path (csrc/conv_tc.cu) validated on the device against the exact-fp32 CUDA-core conv
(csrc/conv.cu) and against the CPU oracle, then end to end through the HMR forward."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

SHAPES = [  # M, Cin, Cout
    (3136, 64, 256), (3136, 256, 64), (784, 512, 128), (196, 1024, 256), (49, 2048, 512), (49, 512, 2048), (2 * 196, 256, 1024), (130, 64, 64)]


@pytest.fixture(scope='module')
def L():
    from dynaboa_b200 import _lib
    lib = _lib.load()
    yield _lib
    lib.dboa_set_tensor_core_conv(3)          # the library default: later test modules must not inherit this module's mode


def run_tc(L, mode, M, Cin, Cout, x, w, ws):
    L.load().dboa_set_tensor_core_conv(mode)
    y = torch.full((M, Cout), float('nan'), device='cuda')
    st = L.load().dboa_conv1x1_tc_fwd(L.ptr(x), L.ptr(w), L.ptr(y), M, Cin, Cout, L.ptr(ws), ws.numel(), L.stream())
    torch.cuda.synchronize()
    return st, y


def test_descriptor_convention_and_accuracy(L):
    """K-major no-swizzle descriptors (LBO = k-chunk step, SBO = 8-row group step, as CUTLASS documents): accuracy of the
    3xTF32 split against an fp64 product."""
    torch.manual_seed(0)
    ws = torch.empty(8 << 20, device='cuda')
    results = {}
    for mode in (1,):
        errs = []
        for M, Cin, Cout in SHAPES:
            x = torch.randn(M, Cin, device='cuda')
            w = torch.randn(Cout, Cin, device='cuda') / Cin ** 0.5
            st, y = run_tc(L, mode, M, Cin, Cout, x, w, ws)
            assert st == 0, (mode, M, Cin, Cout, st)
            ref = (x.double() @ w.double().t())
            errs.append(((y.double() - ref).abs().max() / ref.abs().max()).item())
        results[mode] = max(errs)
        print(f'tensor-core mode {mode}: max rel err over shapes = {results[mode]:.3e}  per-shape {[f"{e:.1e}" for e in errs]}')
    assert results[1] < 5e-6, f'documented descriptor convention failed: {results}'


def test_matches_fp32_cuda_core_path(L):
    torch.manual_seed(1)
    ws = torch.empty(8 << 20, device='cuda')
    for M, Cin, Cout in SHAPES:
        x = torch.randn(M, Cin, device='cuda')
        w = torch.randn(Cout, Cin, device='cuda') / Cin ** 0.5
        st, y = run_tc(L, 1, M, Cin, Cout, x, w, ws)
        assert st == 0
        y32 = torch.empty(M, Cout, device='cuda')
        L.call('dboa_conv2d_fwd', L.ptr(x), L.ptr(w), L.ptr(y32), 1, M, 1, Cin, Cout, 1, 1, 0, Cin, L.ptr(ws), ws.numel(), L.stream())
        assert rel_err(y, y32) < 5e-6, (M, Cin, Cout)


CONV_SHAPES = [  # B, H, Cin, Cout, k, stride, pad
    (1, 56, 64, 64, 3, 1, 1), (2, 28, 128, 128, 3, 2, 1), (1, 56, 256, 512, 1, 2, 0), (1, 7, 512, 512, 3, 1, 1), (3, 14, 256, 256, 3, 1, 1),
    (1, 14, 1024, 256, 1, 1, 0), (2, 7, 2048, 512, 1, 1, 0), (1, 14, 512, 512, 3, 2, 1), (2, 28, 512, 1024, 1, 2, 0)]


@pytest.mark.parametrize('case', CONV_SHAPES)
def test_implicit_gemm_conv_matches_fp32_path_and_oracle(L, case):
    import torch.nn.functional as F
    B, H, Cin, Cout, k, s, p = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, Cin, H, H, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (k * k * Cin) ** 0.5
    ref = F.conv2d(x, w, stride=s, padding=p)
    Ho = ref.shape[2]
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    wd = w.permute(0, 2, 3, 1).reshape(Cout, -1).contiguous().cuda()
    K = wd.shape[1]
    ws = torch.empty(8 << 20, device='cuda')
    y32 = torch.empty(B, Ho, Ho, Cout, device='cuda')
    L.call('dboa_conv2d_fwd', L.ptr(xd), L.ptr(wd), L.ptr(y32), B, H, H, Cin, Cout, k, s, p, K, L.ptr(ws), ws.numel(), L.stream())
    L.load().dboa_set_tensor_core_conv(1)
    ytc = torch.full((B, Ho, Ho, Cout), float('nan'), device='cuda')
    L.call('dboa_conv2d_tc_fwd', L.ptr(xd), L.ptr(wd), L.ptr(ytc), B, H, H, Cin, Cout, k, s, p, K, L.stream())
    torch.cuda.synchronize()
    assert rel_err(ytc, y32) < 5e-6, case
    assert rel_err(ytc.permute(0, 3, 1, 2), ref) < 2e-5, case
    # data and weight gradients on the tensor cores against the fp32 CUDA-core kernels
    L.load().dboa_set_tensor_core_conv(2)
    dy = torch.randn(B, Ho, Ho, Cout, generator=g).cuda()
    for acc in (0, 1):
        base = torch.randn(B, H, H, Cin, generator=g).cuda()
        dx32, dxtc = base.clone(), base.clone()
        L.call('dboa_conv2d_dgrad', L.ptr(dy), L.ptr(wd), L.ptr(dx32), B, H, H, Cin, Cout, k, s, p, K, acc, L.ptr(ws), ws.numel(), L.stream())
        L.call('dboa_conv2d_tc_dgrad', L.ptr(dy), L.ptr(wd), L.ptr(dxtc), B, H, H, Cin, Cout, k, s, p, K, acc, L.stream())
        assert rel_err(dxtc - (base if acc else 0), dx32 - (base if acc else 0)) < 1e-5, (case, 'dgrad', acc)
    basew = torch.randn(Cout, K, generator=g).cuda() * 0.1
    dw32, dwtc = basew.clone(), basew.clone()
    L.call('dboa_conv2d_wgrad', L.ptr(dy), L.ptr(xd), L.ptr(dw32), B, H, H, Cin, Cout, k, s, p, K, L.ptr(ws), ws.numel(), L.stream())
    L.call('dboa_conv2d_tc_wgrad', L.ptr(dy), L.ptr(xd), L.ptr(dwtc), B, H, H, Cin, Cout, k, s, p, K, L.stream())
    torch.cuda.synchronize()
    assert rel_err(dwtc - basew, dw32 - basew) < 1e-5, (case, 'wgrad')


def test_hmr_forward_with_tensor_core_convs(L, golden):
    from dynaboa_b200 import synthetic
    from dynaboa_b200.hmr import hmr
    from oracle import hmr_ref
    gd = golden('hmr_forward')
    m = hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(24)).cuda()
    L.load().dboa_set_tensor_core_conv(2)
    try:
        with torch.no_grad():
            rot, shape, cam, feats = m(x, need_feature=True)
        assert rel_err(rot, gd['rotmat']) < 1e-4 and rel_err(shape, gd['shape']) < 1e-4 and rel_err(cam, gd['cam']) < 1e-4
        for i in range(5, 15):
            assert rel_err(feats[i], gd[f'feat{i}']) < 1e-4, i
        # backward through tensor-core dgrad / wgrad against the reference's golden gradient digest
        for p in m.parameters():
            p.grad = None
        object.__setattr__(m, '_grad_arena', None)
        rot, shape, cam = m(x[:1])
        loss = (rot * torch.from_numpy(gd['w_r']).cuda()).sum() + (shape * torch.from_numpy(gd['w_s']).cuda()).sum() \
            + (cam * torch.from_numpy(gd['w_c']).cuda()).sum()
        loss.backward()
        params = dict(m.named_parameters())
        for key in gd:
            if key.startswith('grad_'):
                gflat = params[key[5:]].grad.contiguous().flatten().double().cpu()
                assert abs(gflat.norm().item() - gd[key][0]) <= 2e-3 * gd[key][0], key
    finally:
        L.load().dboa_set_tensor_core_conv(3)             # the library default
