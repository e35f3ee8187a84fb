"""HMR forward with its piecewise-linear pattern taken as given (test infrastructure only).

The network is piecewise linear in its ReLUs and its max-pool, so its gradient jumps where an activation crosses a kink,
and an fp64 evaluation of ``hmr_ref`` may sit on the other side of a kink than the GPU's fp32 run (DESIGN.md section 6).
This restatement recomputes every convolution, GroupNorm and linear layer in the dtype of its inputs, but takes the
pattern of the kinks from outside:

- each ReLU is a multiplication by a 0/1 mask (on the GPU: ``a > 0`` of that layer's tape entry);
- the max-pool is a gather at the window position ``r*3+s`` the forward chose (the tape's ``p0_idx``);
- dropout multiplies by the given keep-masks.

With the pattern of a GPU forward, its gradient is the exact derivative of the network on the GPU's own activation
pattern, so it and the GPU's hand-written backward differ by rounding only.  With ``pattern=None`` it takes the pattern
from its own values and is the network of ``hmr_ref`` (tests/test_hmr_frozen.py checks both claims).

The pattern is a dict: ``'relu'`` maps the name of each convolution that feeds a ReLU (``conv1``, ``layer1.0.conv1``, ...,
``layerL.B.conv3``; the shortcut joins conv3's ReLU) to an NCHW 0/1 mask, ``'pool'`` is the (B,64,56,56) integer window
position of the max-pool, and ``'drop'`` is None or the (3,2,B,1024) scaled keep-masks.
"""
import torch
import torch.nn.functional as F

from . import geometry_ref, hmr_ref


def _relu(v, name, pattern, own):
    if own:
        pattern['relu'][name] = (v.detach() > 0).to(v.dtype)
    return v * pattern['relu'][name].to(v.dtype)


def _maxpool(a, pattern, own):
    """MaxPool2d(3, 2, 1) as a gather at the given window position (first maximum in scan order when ``own``)."""
    ap = F.pad(a, (1, 1, 1, 1))
    Ho = a.shape[2] // 2
    slices = [ap[:, :, r:r + 2 * Ho:2, s:s + 2 * Ho:2] for r in range(3) for s in range(3)]
    if own:
        neg = F.pad(a.detach(), (1, 1, 1, 1), value=float('-inf'))
        best = torch.full_like(slices[0], float('-inf'))
        idx = torch.zeros(slices[0].shape, dtype=torch.long, device=a.device)
        for k in range(9):
            r, s = divmod(k, 3)
            v = neg[:, :, r:r + 2 * Ho:2, s:s + 2 * Ho:2]
            take = v > best
            best = torch.where(take, v, best)
            idx = torch.where(take, torch.full_like(idx, k), idx)
        pattern['pool'] = idx
    idx = pattern['pool'].to(device=a.device, dtype=torch.long)
    out = torch.zeros_like(slices[0])
    for k, v in enumerate(slices):
        out = torch.where(idx == k, v, out)
    return out


def _bottleneck(x, p, pre, stride, has_ds, pattern, own):
    out = _relu(hmr_ref._gn(F.conv2d(x, p[pre + '.conv1.weight']), p, pre + '.bn1'), pre + '.conv1', pattern, own)
    out = _relu(hmr_ref._gn(F.conv2d(out, p[pre + '.conv2.weight'], stride=stride, padding=1), p, pre + '.bn2'), pre + '.conv2',
                pattern, own)
    out = hmr_ref._gn(F.conv2d(out, p[pre + '.conv3.weight']), p, pre + '.bn3')
    res = x
    if has_ds:
        res = hmr_ref._gn(F.conv2d(x, p[pre + '.downsample.0.weight'], stride=stride), p, pre + '.downsample.1')
    return _relu(out + res, pre + '.conv3', pattern, own)


def forward(x, p, pattern=None, drop=None):
    """(rotmat, shape, cam, pattern) of the HMR forward (hmr_ref.forward with n_iter = 3) on ``pattern``, or on its own
    pattern when None (returned, with ``drop`` as its dropout keep-masks).  ``p`` holds the 169 parameters and the init_*
    buffers by state_dict name."""
    own = pattern is None
    if own:
        pattern = {'relu': {}, 'pool': None, 'drop': drop}
    B = x.shape[0]
    y = _relu(hmr_ref._gn(F.conv2d(x, p['conv1.weight'], stride=2, padding=3), p, 'bn1'), 'conv1', pattern, own)
    y = _maxpool(y, pattern, own)
    for li, nblk in enumerate(hmr_ref.BLOCKS):
        for bi in range(nblk):
            y = _bottleneck(y, p, f'layer{li + 1}.{bi}', 2 if (li > 0 and bi == 0) else 1, bi == 0, pattern, own)
    xf = F.avg_pool2d(y, 7, stride=1).flatten(1)
    drop = pattern['drop']
    masks = None if drop is None else [(drop[i, 0].to(xf), drop[i, 1].to(xf)) for i in range(3)]
    pose, shape, cam, _ = hmr_ref.regressor(xf, p, p['init_pose'].expand(B, -1), p['init_shape'].expand(B, -1),
                                            p['init_cam'].expand(B, -1), 3, masks)
    rotmat = geometry_ref.rot6d_to_rotmat(pose).view(B, 24, 3, 3)
    return rotmat, shape, cam, pattern
