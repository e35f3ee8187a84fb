"""The HMR plan (csrc/hmr_plan.cu) layer by layer against fp64, at batch 1 to 64, in every convolution mode and plan.

Forward: every tape entry the backward reads is recomputed in fp64 from the GPU's own inputs, read from the tape, so
errors do not compound and each bound is the rounding of one layer: every convolution output `y` (from its input
activation), every GroupNorm `(mean, rstd)` (from the GPU's `y`), every post-activation `a`
(relu(gn(y) [+ identity | + gn(y_downsample)])), the max-pool output and indices, the regressor rows and the outputs.

Backward: oracle/hmr_frozen.py evaluates the network in fp64 on the GPU's own ReLU, max-pool and dropout pattern, so its
autograd gradient is the exact derivative of what the GPU computed, with no kink floor (DESIGN.md section 6), and every
one of the 169 gradient tensors is compared element-wise.

The tape is filled with NaN before each forward, so a region the plan fails to write fails its check."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from harness import FWD_TOL, GRAD_L2, GRAD_TOL, nchw, rel, structure

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, tensor-core mode, fused forward, fused backward, dropout masks)
DEFAULT = ('tc3', 3, 0, 0, False)
CONFIGS = ([DEFAULT + (B,) for B in (1, 2, 3, 8, 9, 17, 22, 64)]
           + [c + (B,) for c in (('tc0', 0, 0, 0, False), ('tc1', 1, 0, 0, False), ('tc2', 2, 0, 0, False),
                                 ('fused_fwd', 3, 1, 0, False), ('fused_bwd', 3, 0, 1, False)) for B in (1, 9, 64)]
           + [('masked', 3, 0, 0, True, B) for B in (1, 9)])
IDS = [f'{c[0]}-B{c[5]}' for c in CONFIGS]

@pytest.fixture(scope='module')
def model():
    from dynaboa_b200 import _lib, synthetic
    from dynaboa_b200.hmr import hmr
    from oracle import hmr_ref
    lib = _lib.load()
    m = hmr(synthetic.make_mean_params()).cuda()
    m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
    m.eval()
    yield m
    lib.dboa_set_tensor_core_conv(3)          # library defaults: later test modules must not inherit this module's modes
    lib.dboa_set_fused_forward(0)
    lib.dboa_set_fused_backward(0)


def run_forward(m, cfg):
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import raw_forward, tape_floats
    _, mode, ffwd, fbwd, masked, B = cfg
    lib = _lib.load()
    lib.dboa_set_tensor_core_conv(mode)
    lib.dboa_set_fused_forward(ffwd)
    lib.dboa_set_fused_backward(fbwd)
    g = torch.Generator().manual_seed(1000 + B + 7 * mode + 3 * ffwd + 5 * fbwd + 11 * masked)
    x = torch.randn(B, 3, 224, 224, generator=g).cuda()
    masks = (torch.rand(3, 2, B, 1024, generator=g) >= 0.5).float().cuda() * 2 if masked else None
    tape = torch.full((tape_floats(B),), float('nan'), device='cuda')
    rot, shape, cam, _, _ = raw_forward(m.arena, m._buffers, x, masks, tape)
    torch.cuda.synchronize()
    return x, masks, tape, (rot, shape, cam)


def gn_stats(y):
    v = y.reshape(y.shape[0], 4, -1)
    return v.mean(-1), (v.var(-1, unbiased=False) + 1e-5).rsqrt()


def gn_apply(y, mean, rstd, gamma, beta):
    B, C = y.shape[:2]
    v = ((y.reshape(B, 4, -1) - mean[..., None]) * rstd[..., None]).reshape(y.shape)
    return v * gamma.double().view(1, C, 1, 1) + beta.double().view(1, C, 1, 1)


@pytest.mark.parametrize('cfg', CONFIGS, ids=IDS)
def test_forward_layer_by_layer(model, cfg):
    from dynaboa_b200.hmr import layout, tape_views
    from oracle import geometry_ref
    m, B = model, cfg[5]
    x, masks, tape, (rot, shape, cam) = run_forward(m, cfg)
    v = tape_views(tape, B)
    P = layout().views(m.arena)
    geo, blocks = structure()
    worst = {k: (0.0, '') for k in FWD_TOL}

    def note(kind, err, where):
        if worst[kind][0] == worst[kind][0] and not err <= worst[kind][0]:       # NaN (an unwritten region) sticks
            worst[kind] = (err, where)

    assert torch.equal(v['x0'], x.permute(0, 2, 3, 1))
    block_in = [v['p0']] + [v['a'][b[2]] for b in blocks[:-1]]
    inputs = {0: v['x0']}
    for bi, (c1, c2, c3, cd) in enumerate(blocks):
        inputs.update({c1: block_in[bi], c2: v['a'][c1], c3: v['a'][c2]})
        if cd is not None:
            inputs[cd] = block_in[bi]
    ref_y, ref_stats = {}, {}
    for i, (name, _, _, k, stride, _) in enumerate(geo):
        y = nchw(v['y'][i])
        ref = F.conv2d(nchw(inputs[i]), P[3 * i].double(), stride=stride, padding=k // 2)
        note('y', rel(y, ref), name)
        mean, rstd = gn_stats(y)
        st = v['stats'][i].double()
        note('stats', float(torch.cat([((st[..., 0] - mean).abs() * rstd).flatten(), (st[..., 1] / rstd - 1).abs().flatten()]).max()), name)
        ref_y[i], ref_stats[i] = y, (mean, rstd)

    def gn(i):
        return gn_apply(ref_y[i], *ref_stats[i], P[3 * i + 1], P[3 * i + 2])
    note('a', rel(nchw(v['a'][0]), torch.relu(gn(0))), 'conv1')
    for bi, (c1, c2, c3, cd) in enumerate(blocks):
        note('a', rel(nchw(v['a'][c1]), torch.relu(gn(c1))), geo[c1][0])
        note('a', rel(nchw(v['a'][c2]), torch.relu(gn(c2))), geo[c2][0])
        res = gn(cd) if cd is not None else nchw(block_in[bi])
        note('a', rel(nchw(v['a'][c3]), torch.relu(gn(c3) + res)), geo[c3][0])

    # max-pool: exact maximum, and the stored index is the first maximum of the window in scan order
    a0 = v['a'][0].permute(0, 3, 1, 2)
    p0 = v['p0'].permute(0, 3, 1, 2)
    assert torch.equal(p0, F.max_pool2d(a0, 3, 2, 1)), 'max-pool output'
    idx = v['p0_idx'].permute(0, 3, 1, 2).long()
    ap = F.pad(a0, (1, 1, 1, 1), value=float('-inf'))
    win = torch.stack([ap[:, :, r:r + 112:2, s:s + 112:2] for r in range(3) for s in range(3)])
    assert int(idx.max()) <= 8
    assert torch.equal(win.gather(0, idx[None]).squeeze(0), p0), 'value at p0_idx'
    earlier = torch.arange(9, device='cuda').view(9, 1, 1, 1, 1) < idx[None]
    assert not bool(((win >= p0[None]) & earlier).any()), 'p0_idx is not the first maximum'

    # regressor: each row from the GPU's previous row, in fp64
    xf = nchw(v['a'][blocks[-1][2]]).mean(dim=(2, 3))
    init = torch.cat([m._buffers['init_pose'], m._buffers['init_shape'], m._buffers['init_cam']], 1).expand(B, -1)
    assert torch.equal(v['params'][0][:, :157], init), 'params[0]'
    names = layout().names
    W = {n: P[names.index(n)].double() for n in ('fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias')}
    Wd = torch.cat([P[names.index(n + '.weight')].double() for n in ('decpose', 'decshape', 'deccam')])
    bd = torch.cat([P[names.index(n + '.bias')].double() for n in ('decpose', 'decshape', 'deccam')])
    for it in range(3):
        xc = v['xc'][it]
        note('head', rel(xc[:, :2048], xf), f'xc[{it}] pooled')
        assert torch.equal(xc[:, 2048:2205], v['params'][it][:, :157]), f'xc[{it}] params'
        h1 = v['h1pre'][it]
        note('head', rel(h1, xc[:, :2205].double() @ W['fc1.weight'].t() + W['fc1.bias']), f'h1pre[{it}]')
        assert torch.equal(v['h1post'][it], h1 * masks[it, 0] if masks is not None else h1), f'h1post[{it}]'
        h2 = v['h2pre'][it]
        note('head', rel(h2, v['h1post'][it].double() @ W['fc2.weight'].t() + W['fc2.bias']), f'h2pre[{it}]')
        assert torch.equal(v['h2post'][it], h2 * masks[it, 1] if masks is not None else h2), f'h2post[{it}]'
        delta = v['h2post'][it].double() @ Wd.t() + bd
        note('head', rel(v['params'][it + 1][:, :157], v['params'][it][:, :157].double() + delta, delta.abs().max()), f'params[{it + 1}]')
    p3 = v['params'][3][:, :157]
    note('out', rel(rot, geometry_ref.rot6d_to_rotmat(p3[:, :144].double()).view(B, 24, 3, 3)), 'rotmat')
    assert torch.equal(shape, p3[:, 144:154]) and torch.equal(cam, p3[:, 154:157]), 'shape / cam'
    print(f'\nFWD {IDS[CONFIGS.index(cfg)]} ' + json.dumps({k: [f'{e:.2e}', w] for k, (e, w) in worst.items()}))
    for k, (e, w) in worst.items():
        assert e <= FWD_TOL[k], (k, e, w)


def frozen_gradient(m, x, masks, tape, B, d):
    """fp64 autograd gradient of hmr_frozen on the GPU's pattern, summed over chunks of samples (the network does not mix
    samples), as {parameter name: gradient}."""
    from dynaboa_b200.hmr import layout, tape_views
    from oracle import hmr_frozen
    lay = layout()
    v = tape_views(tape, B)
    geo, _ = structure()
    p = {n: w.detach().double().requires_grad_(True) for n, w in zip(lay.names, lay.views(m.arena))}
    bufs = {k: m._buffers[k].double() for k in ('init_pose', 'init_shape', 'init_cam')}
    for s0 in range(0, B, 16):
        s = slice(s0, min(B, s0 + 16))
        pattern = {'relu': {g[0]: nchw(v['a'][i][s]) > 0 for i, g in enumerate(geo) if v['a'][i] is not None},
                   'pool': v['p0_idx'][s].permute(0, 3, 1, 2).long(),
                   'drop': None if masks is None else masks[:, :, s].double()}
        rot, shape, cam, _ = hmr_frozen.forward(x[s].double(), dict(p, **bufs), pattern)
        ((rot * d[0][s]).sum() + (shape * d[1][s]).sum() + (cam * d[2][s]).sum()).backward()
    return {n: t.grad for n, t in p.items()}


@pytest.mark.parametrize('cfg', CONFIGS, ids=IDS)
def test_backward_elementwise_on_the_gpu_pattern(model, cfg):
    from dynaboa_b200.hmr import layout, raw_backward
    m, B = model, cfg[5]
    x, masks, tape, _ = run_forward(m, cfg)
    g = torch.Generator().manual_seed(2000 + B)
    d = [torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda(), torch.randn(B, 3, generator=g).cuda()]
    lay = layout()
    grad = torch.zeros(lay.floats, device='cuda')
    raw_backward(m.arena, tape, B, masks is not None, d[0], d[1], d[2], grad)
    ref = frozen_gradient(m, x, masks, tape, B, [t.double() for t in d])
    errs, num, den = [], 0.0, 0.0
    for n, gv in zip(lay.names, lay.views(grad)):
        r = ref[n]
        errs.append((rel(gv, r), n))
        num, den = num + float((gv.double() - r).pow(2).sum()), den + float(r.pow(2).sum())
    errs.sort(key=lambda e: -(e[0] if e[0] == e[0] else float('inf')))
    l2 = (num / den) ** 0.5
    print(f'\nBWD {IDS[CONFIGS.index(cfg)]} rel L2 {l2:.2e} worst ' + json.dumps([(f'{e:.2e}', n) for e, n in errs[:3]]))
    assert l2 <= GRAD_L2, l2
    assert all(e <= GRAD_TOL for e, _ in errs), errs[:6]


@pytest.mark.parametrize('B', [1, 9, 64])
def test_backward_is_bit_reproducible(model, B):
    from dynaboa_b200.hmr import layout, raw_backward
    x, _, tape, _ = run_forward(model, DEFAULT + (B,))
    d = [torch.randn(B, 24, 3, 3, device='cuda'), torch.randn(B, 10, device='cuda'), torch.randn(B, 3, device='cuda')]
    grads = []
    for _ in range(2):
        grads.append(torch.zeros(layout().floats, device='cuda'))
        raw_backward(model.arena, tape, B, False, d[0], d[1], d[2], grads[-1])
    torch.cuda.synchronize()
    assert torch.equal(grads[0], grads[1])


_SYNC_CHILD = r'''
import sys
import torch
from dynaboa_b200 import synthetic
from dynaboa_b200.hmr import hmr, layout, raw_backward, raw_forward
from oracle import hmr_ref
B, out = int(sys.argv[1]), sys.argv[2]
m = hmr(synthetic.make_mean_params()).cuda()
m.load_state_dict(hmr_ref.strip_prefix(synthetic.make_basemodel()['model']), strict=True)
g = torch.Generator().manual_seed(3000 + B)
x = torch.randn(B, 3, 224, 224, generator=g).cuda()
d = [torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda(), torch.randn(B, 3, generator=g).cuda()]
tape = raw_forward(m.arena, m._buffers, x)[4]
grads = []
for _ in range(2):
    grads.append(torch.zeros(layout().floats, device='cuda'))
    raw_backward(m.arena, tape, B, False, d[0], d[1], d[2], grads[-1])
torch.cuda.synchronize()
assert torch.equal(grads[0], grads[1]), 'two backward calls differ'
torch.save(grads[0].cpu(), out)
'''


@pytest.mark.parametrize('B', [1, 9])
def test_backward_without_async_weight_gradients_is_bit_reproducible(model, B, tmp_path):
    """DBOA_ASYNC_WGRAD=0 is read once at library load, so a child process runs the synchronous backward; its arena is
    also compared with the default (side-stream) backward in this process."""
    from dynaboa_b200 import _lib
    from dynaboa_b200.hmr import layout, raw_backward, raw_forward
    env = dict(os.environ, DBOA_ASYNC_WGRAD='0', PYTHONPATH=REPO + os.pathsep + os.environ.get('PYTHONPATH', ''))
    out = str(tmp_path / 'grad_sync.pt')
    r = subprocess.run([sys.executable, '-c', _SYNC_CHILD, str(B), out], env=env, cwd=REPO, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    sync = torch.load(out)
    lib = _lib.load()
    lib.dboa_set_tensor_core_conv(3)
    lib.dboa_set_fused_forward(0)
    lib.dboa_set_fused_backward(0)
    m = model
    g = torch.Generator().manual_seed(3000 + B)
    x = torch.randn(B, 3, 224, 224, generator=g).cuda()
    d = [torch.randn(B, 24, 3, 3, generator=g).cuda(), torch.randn(B, 10, generator=g).cuda(), torch.randn(B, 3, generator=g).cuda()]
    tape = raw_forward(m.arena, m._buffers, x)[4]
    grad = torch.zeros(layout().floats, device='cuda')
    raw_backward(m.arena, tape, B, False, d[0], d[1], d[2], grad)
    torch.cuda.synchronize()
    same = torch.equal(grad.cpu(), sync)
    print(f'\nSYNC B={B} async arena bit-identical to synchronous: {same}')
    assert same
