"""PyTorch-op port of the 3D propagation with a K x K x K affinity kernel, K in {3, 5}.  TEST INFRASTRUCTURE ONLY.

The op sequence of oracle/cspn_torch_port.py::cspn3d_torch with K**3-1 taps.  At K = 3 it gives cspn3d_torch's bits; in
fp64 it is the autograd reference for the gradients of the K x K x K path.  Never imported by the product package.
"""
import torch
import torch.nn.functional as F


def offsets_3d(K):
    """(dz, dy, dx) of the K**3-1 taps in raster order over (f, t, l) without the centre (cspn_torch_port.OFFSETS_3D at K = 3)."""
    r = (K - 1) // 2
    return tuple((r - f, r - t, r - l) for f in range(K) for t in range(K) for l in range(K) if (f, t, l) != (r, r, r))


def _shift3d_k(a, dz, dy, dx, r):
    """b[..., z, y, x] = a[..., z+dz, y+dy, x+dx], zero outside (|d| <= r)."""
    D, H, W = a.shape[-3:]
    p = F.pad(a, (r, r, r, r, r, r))
    return p[..., r + dz:r + dz + D, r + dy:r + dy + H, r + dx:r + dx + W]


def cspn3d_torch_k(guidance, feat, prop_time=12, K=5, norm_type=None):
    """cspn3d_torch with a K x K x K kernel (K = 3 gives its bits); in fp64 the autograd reference of the K x K x K path."""
    nt, r = K ** 3 - 1, (K - 1) // 2
    norm_type = norm_type or f'{nt}sum_abs'
    assert K in (3, 5) and norm_type in (f'{nt}sum', f'{nt}sum_abs', 'paddle')
    offs = offsets_3d(K)
    g = guidance[:, :nt]
    if norm_type == 'paddle':
        a = g.abs()
        gate = a / a.sum(1, keepdim=True)
    else:
        if 'abs' in norm_type:
            g = g.abs()
        a = torch.stack([_shift3d_k(g[:, k], *o, r) for k, o in enumerate(offs)], 1)
        gate = a / a.abs().sum(1, keepdim=True)
    gate_sum = gate.sum(1, keepdim=True)
    raw = feat
    result = feat
    for _ in range(prop_time):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + gate[:, k:k + 1] * _shift3d_k(result, *o, r)
        result = acc if norm_type == 'paddle' else (1.0 - gate_sum) * raw + acc
    return result
