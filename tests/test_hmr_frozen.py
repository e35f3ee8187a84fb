"""oracle/hmr_frozen.py is the network of oracle/hmr_ref.py: given the pattern of its own fp64 forward, its outputs and its
autograd gradient in all 169 parameters equal hmr_ref's to rounding (CPU, fp64, batch 1)."""
import pytest
import torch


@pytest.mark.parametrize('masked', [False, True])
def test_frozen_pattern_restatement_is_the_reference_network(masked):
    from dynaboa_b200 import synthetic
    from oracle import hmr_frozen, hmr_ref
    sd = hmr_ref.strip_prefix(synthetic.make_basemodel()['model'])
    g = torch.Generator().manual_seed(11 + masked)
    x = torch.randn(1, 3, 224, 224, generator=g, dtype=torch.float64)
    drop = (torch.rand(3, 2, 1, 1024, generator=g) >= 0.5).double() * 2 if masked else None
    w = [torch.randn(1, 24, 3, 3, generator=g, dtype=torch.float64), torch.randn(1, 10, generator=g, dtype=torch.float64),
         torch.randn(1, 3, generator=g, dtype=torch.float64)]

    def run(fn):
        p = {k: v.double().requires_grad_(not k.startswith('init_')) for k, v in sd.items()}
        out = fn(p)
        sum((o * wi).sum() for o, wi in zip(out, w)).backward()
        return [o.detach() for o in out], {k: v.grad for k, v in p.items() if v.grad is not None}

    with torch.no_grad():
        pattern = hmr_frozen.forward(x, {k: v.double() for k, v in sd.items()}, drop=drop)[3]
    assert len(pattern['relu']) == 49 and pattern['pool'].shape == (1, 64, 56, 56)
    assert 0.2 < float(torch.cat([m.flatten() for m in pattern['relu'].values()]).mean()) < 0.8
    out_f, grad_f = run(lambda p: hmr_frozen.forward(x, p, pattern)[:3])
    masks = None if drop is None else [(drop[i, 0], drop[i, 1]) for i in range(3)]
    out_r, grad_r = run(lambda p: hmr_ref.forward(x, p, masks=masks))
    for a, b in zip(out_f, out_r):
        assert (a - b).abs().max() <= 1e-12 * b.abs().max()
    assert len(grad_r) == 169 and set(grad_f) == set(grad_r)
    for k, ref in grad_r.items():
        assert ref.abs().max() > 0, k
        assert (grad_f[k] - ref).abs().max() <= 1e-12 * ref.abs().max(), k
