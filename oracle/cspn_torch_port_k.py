"""PyTorch-op port of the 2D propagation with a K x K affinity kernel, K in {3, 5, 7}.  TEST INFRASTRUCTURE ONLY.

The op sequence of oracle/cspn_torch_port.py::cspn2d_torch (the reference's cspn.py) with its ZeroPad2d tuples
generalised and a (K*K-1)-way ones conv3d: K*K-1 padded copies per step.  At K = 3 it gives cspn2d_torch's bits; in fp64
it is the autograd reference for the gradients of the K x K path.  Never imported by the product package.
"""
import torch
import torch.nn.functional as F

from .cspn_torch_port import _sum8


def pads_2d(K):
    """ZeroPad2d tuples (left, right, top, bottom) of the K*K-1 taps in raster order without the centre
    (cspn_torch_port.PADS at K = 3)."""
    r = (K - 1) // 2
    return tuple((l, K - 1 - l, t, K - 1 - t) for t in range(K) for l in range(K) if (t, l) != (r, r))


def cspn2d_torch_k(guidance, blur_depth, sparse_depth=None, prop_time=24, K=5, norm_type=None):
    """cspn2d_torch with a K x K kernel: K*K-1 padded copies and a (K*K-1)-way ones conv3d (K = 3 gives its bits)."""
    nt, r = K * K - 1, (K - 1) // 2
    norm_type = norm_type or f'{nt}sum'
    assert K in (3, 5, 7) and norm_type in (f'{nt}sum', f'{nt}sum_abs')
    pads = pads_2d(K)
    ones = torch.ones(1, nt, 1, 1, 1, dtype=blur_depth.dtype, device=blur_depth.device)
    g = guidance.abs() if 'abs' in norm_type else guidance
    gate = torch.cat([F.pad(g.narrow(1, k, 1), pads[k]).unsqueeze(1) for k in range(nt)], 1)
    gate = gate / _sum8(gate.abs(), ones)
    gate_sum = _sum8(gate, ones).squeeze(1)[:, :, r:-r, r:-r]
    raw = blur_depth
    result = blur_depth
    mask = sparse_depth.sign() if sparse_depth is not None else None
    for _ in range(prop_time):
        stacked = torch.cat([F.pad(result, p).unsqueeze(1) for p in pads], 1)
        nb = _sum8(gate * stacked, ones).squeeze(1)[:, :, r:-r, r:-r]
        result = (1.0 - gate_sum) * raw + nb
        if mask is not None:
            result = (1 - mask) * result + mask * raw
    return result
