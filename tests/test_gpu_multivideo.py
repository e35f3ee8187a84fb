"""Grouped HMR plan (dboa_hmr_forward_groups / dboa_hmr_backward_groups): G videos, each with its own weights, in one
launch sequence.

- Layer parity: every video's convolution outputs and regressor rows (from the GPU's own inputs, read from the tape) and
  all 169 gradient tensors (oracle/hmr_frozen.py on the GPU's own ReLU / max-pool / dropout pattern) against fp64 with that
  video's own weights, to the bounds of tests/test_gpu_hmr_layers.py, in every convolution mode, with and without dropout.
- Isolation: identical videos give bit-identical results; changing one video changes no bit of any other.
- groups = 1 is bit-identical to dboa_hmr_forward / dboa_hmr_backward, and grouped calls are bit-reproducible."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_hmr_layers import FWD_TOL, GRAD_TOL, nchw, rel, structure

pytestmark = pytest.mark.gpu

# (videos G, samples per video b, tensor-core mode, dropout masks)
CONFIGS = [(2, 1, 3, False), (4, 2, 3, False), (8, 8, 3, False), (4, 1, 0, False), (2, 8, 0, False), (8, 1, 1, False),
           (2, 2, 1, False), (4, 8, 2, False), (8, 2, 2, False), (2, 1, 3, True), (8, 2, 3, True), (4, 2, 0, True), (2, 8, 1, True)]
IDS = [f'G{g}-b{b}-tc{m}' + ('-masked' if k else '') for g, b, m, k in CONFIGS]


@pytest.fixture(scope='module')
def model():
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


def run(m, arenas, x, masks, d, groups):
    from dynaboa_b200.hmr import raw_backward, raw_forward, tape_floats
    B = x.shape[0]
    tape = torch.full((tape_floats(B),), float('nan'), device='cuda')
    rot, shape, cam, _, _ = raw_forward(arenas, m._buffers, x, masks, tape, groups=groups)
    grad = torch.zeros_like(arenas)
    raw_backward(arenas, tape, B, masks is not None, d[0], d[1], d[2], grad, groups=groups)
    torch.cuda.synchronize()
    return (rot, shape, cam), tape, grad


def inputs(B, seed, masked):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, 224, 224, generator=g).cuda()
    masks = (torch.rand(3, 2, B, 1024, generator=g) >= 0.5).float().cuda() * 2 if masked else None
    d = [torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda(), torch.randn(B, 3, generator=g).cuda()]
    return x, masks, d


@pytest.mark.parametrize('cfg', CONFIGS, ids=IDS)
def test_every_video_against_fp64_with_its_own_weights(model, cfg):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import layout, tape_views
    from oracle import hmr_frozen
    G, b, mode, masked = cfg
    B = G * b
    _lib.load().dboa_set_tensor_core_conv(mode)
    m, lay = model, layout()
    arenas = stacked(m, G, 100 * G + 10 * b + mode)
    x, masks, d = inputs(B, 4000 + B + mode, masked)
    _, tape, grad = run(m, arenas, x, masks, d, G)
    v = tape_views(tape, B)
    geo, blocks = structure()
    block_in = [v['p0']] + [v['a'][bl[2]] for bl in blocks[:-1]]
    conv_in = {0: v['x0']}
    for bi, (c1, c2, c3, cd) in enumerate(blocks):
        conv_in.update({c1: block_in[bi], c2: v['a'][c1], c3: v['a'][c2]})
        if cd is not None:
            conv_in[cd] = block_in[bi]
    names = lay.names
    worst = {'y': 0.0, 'head': 0.0, 'grad': 0.0}
    for g in range(G):
        s = slice(g * b, (g + 1) * b)
        P = lay.views(arenas[g].clone())                 # views() offsets are absolute: give it a tensor of its own
        for i, (name, _, _, k, stride, _) in enumerate(geo):
            ref = F.conv2d(nchw(conv_in[i][s]), P[3 * i].double(), stride=stride, padding=k // 2)
            e = rel(nchw(v['y'][i][s]), ref)
            assert e <= FWD_TOL['y'], (g, name, e)
            worst['y'] = max(worst['y'], e)
        W = {n: P[names.index(n)].double() for n in ('fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias')}
        for it in range(3):
            e = max(rel(v['h1pre'][it][s], v['xc'][it][s, :2205].double() @ W['fc1.weight'].t() + W['fc1.bias']),
                    rel(v['h2pre'][it][s], v['h1post'][it][s].double() @ W['fc2.weight'].t() + W['fc2.bias']))
            assert e <= FWD_TOL['head'], (g, it, e)
            worst['head'] = max(worst['head'], e)
        # gradient of video g: fp64 on the GPU's own pattern of its samples, with its own weights
        p = {n: w.detach().double().requires_grad_(True) for n, w in zip(names, P)}
        bufs = {k: m._buffers[k].double() for k in ('init_pose', 'init_shape', 'init_cam')}
        pattern = {'relu': {gg[0]: nchw(v['a'][i][s]) > 0 for i, gg in enumerate(geo) if v['a'][i] is not None},
                   'pool': v['p0_idx'][s].permute(0, 3, 1, 2).long(),
                   'drop': None if masks is None else masks[:, :, s].double()}
        rot, shape, cam, _ = hmr_frozen.forward(x[s].double(), dict(p, **bufs), pattern)
        ((rot * d[0][s].double()).sum() + (shape * d[1][s].double()).sum() + (cam * d[2][s].double()).sum()).backward()
        for n, gv in zip(names, lay.views(grad[g].clone())):
            e = rel(gv, p[n].grad)
            assert e <= GRAD_TOL, (g, n, e)
            worst['grad'] = max(worst['grad'], e)
    print(f'\nGROUPED {IDS[CONFIGS.index(cfg)]} worst ' + ' '.join(f'{k} {e:.2e}' for k, e in worst.items()))


def test_videos_are_isolated(model):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import tape_views
    _lib.load().dboa_set_tensor_core_conv(3)
    m, G, b = model, 4, 2
    B = G * b
    x1, masks1, d1 = inputs(b, 5000, True)
    rep = lambda t, dim=0: torch.cat([t] * G, dim)
    x, masks, d = rep(x1), rep(masks1, 2), [rep(t) for t in d1]
    arenas = m.arena.repeat(G, 1)
    out, tape, grad = run(m, arenas, x, masks, d, G)
    v = tape_views(tape, B)
    sl = [slice(g * b, (g + 1) * b) for g in range(G)]
    for g in range(1, G):
        for t in out:
            assert torch.equal(t[sl[g]], t[sl[0]]), g
        for i in range(len(v['y'])):
            assert torch.equal(v['y'][i][sl[g]], v['y'][i][sl[0]]), (g, i)
            assert torch.equal(v['stats'][i][sl[g]], v['stats'][i][sl[0]]), (g, i)
        for k, n in (('xc', 2205), ('h1post', 1024), ('h2post', 1024), ('params', 157)):     # without the never-written padding
            assert torch.equal(v[k][:, sl[g], :n], v[k][:, sl[0], :n]), (g, k)
        assert torch.equal(grad[g], grad[0]), g
    # change only video 1: its weights and its upstream gradient
    arenas2 = arenas.clone()
    arenas2[1] = stacked(m, 1, 77)[0]
    d2 = [t.clone() for t in d]
    for t in d2:
        t[sl[1]] *= -1.5
    out2, tape2, grad2 = run(m, arenas2, x, masks, d2, G)
    v2 = tape_views(tape2, B)
    for g in (0, 2, 3):
        for t, t2 in zip(out, out2):
            assert torch.equal(t2[sl[g]], t[sl[g]]), g
        for i in range(len(v['y'])):
            assert torch.equal(v2['y'][i][sl[g]], v['y'][i][sl[g]]), (g, i)
        assert torch.equal(grad2[g], grad[g]), g
    assert not torch.equal(grad2[1], grad[1]) and not torch.equal(out2[0][sl[1]], out[0][sl[1]])


@pytest.mark.parametrize('B', [1, 9])
def test_one_group_is_the_single_video_plan(model, B):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import ptr, scratch_for, stream, tape_floats
    lib = _lib.load()
    lib.dboa_set_tensor_core_conv(3)
    m = model
    x, _, d = inputs(B, 6000 + B, False)
    res = []
    for grouped in (False, True):
        tape = torch.zeros(tape_floats(B), device='cuda')
        o = [torch.empty(B, 24, 3, 3, device='cuda'), torch.empty(B, 10, device='cuda'), torch.empty(B, 3, device='cuda'),
             torch.empty(B, 144, device='cuda')]
        grad = torch.zeros_like(m.arena)
        fa = (ptr(m.arena), ptr(m._buffers['init_pose']), ptr(m._buffers['init_shape']), ptr(m._buffers['init_cam']), ptr(x), B, None,
              ptr(tape), ptr(scratch_for(B, x.device)), *[ptr(t) for t in o], stream())
        ba = (ptr(m.arena), ptr(tape), B, 0, *[ptr(t) for t in d], ptr(grad), ptr(scratch_for(B, x.device)), stream())
        if grouped:
            _lib.call('dboa_hmr_forward_groups', *fa, 1)
            _lib.call('dboa_hmr_backward_groups', *ba, 1)
        else:
            _lib.call('dboa_hmr_forward', *fa)
            _lib.call('dboa_hmr_backward', *ba)
        torch.cuda.synchronize()
        res.append(o + [tape, grad])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_grouped_calls_are_bit_reproducible(model):
    from dynaboa_b200 import _lib
    _lib.load().dboa_set_tensor_core_conv(3)
    G, b = 8, 2
    arenas = stacked(model, G, 900)
    x, masks, d = inputs(G * b, 7000, True)
    r1, r2 = run(model, arenas, x, masks, d, G), run(model, arenas, x, masks, d, G)
    for a, c in zip(r1[0], r2[0]):
        assert torch.equal(a, c)
    assert torch.equal(r1[2], r2[2])
