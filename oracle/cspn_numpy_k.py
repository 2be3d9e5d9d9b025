"""CPU oracle (numpy) of the 2D propagation with a K x K affinity kernel, K in {3, 5, 7}.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and tools/ may import this module; the product path (cspn_b200/) never does.

Parity status: anchored to the pinned 2D arithmetic of oracle/cspn_numpy.py.  cspn2d_k(K=3) gives the bits of
cspn_numpy.cspn2d, which is held to the reference's own outputs; the reference has no K > 3 implementation to pin
against, so K = 5 / 7 are the same op sequence with the ZeroPad2d tuples of cspn.py generalised.
"""
from __future__ import annotations

import numpy as np

from .cspn_numpy import shift2d, sparse_mask


# Tap k enumerates (t, l) over [0, K)^2 in raster order without the centre (r, r), r = (K-1)/2.  Its pad tuple is
# (l, K-1-l, t, K-1-t) followed by the crop [r:-r, r:-r], so it reads the source at (dy, dx) = (r-t, r-l).  At K = 3
# this is cspn_numpy.OFFSETS_2D.
def offsets_2d(K):
    assert K in (3, 5, 7)
    r = (K - 1) // 2
    return tuple((r - t, r - l) for t in range(K) for l in range(K) if (t, l) != (r, r))


def shift2d_k(a, dy, dx):
    """shift2d for offsets that may reach past the image (H or W < K): such a copy is all padding."""
    H, W = a.shape[-2:]
    if abs(dy) >= H or abs(dx) >= W:
        return np.zeros_like(a)
    return shift2d(a, dy, dx)


def norm_names_2d(K):
    """The norm names of a K x K kernel: f'{K*K-1}sum' and f'{K*K-1}sum_abs' ('8sum', '24sum', '48sum', ...)."""
    return (f'{K * K - 1}sum', f'{K * K - 1}sum_abs')


def affinity_normalization_2d_k(guidance, K, norm_type):
    """affinity_normalization_2d with K*K-1 taps: channels 0..K*K-2 of guidance, gathered at offsets_2d(K)."""
    assert norm_type in norm_names_2d(K)
    offs = offsets_2d(K)
    nt = len(offs)
    g = guidance[:, :nt]
    if 'abs' in norm_type:
        g = np.abs(g)
    with np.errstate(divide='ignore', invalid='ignore'):
        a = np.stack([shift2d_k(g[:, k], dy, dx) for k, (dy, dx) in enumerate(offs)], axis=1)
        abs_weight = np.zeros_like(a[:, 0])
        for k in range(nt):
            abs_weight = abs_weight + np.abs(a[:, k])
        gate_wb = a / abs_weight[:, None]
        gate_sum = np.zeros_like(abs_weight)
        for k in range(nt):
            gate_sum = gate_sum + gate_wb[:, k]
    return gate_wb, gate_sum[:, None]


def cspn2d_k(guidance, blur_depth, sparse_depth=None, prop_time=24, K=5, norm_type=None, dtype=np.float32):
    """cspn2d with a K x K kernel, op for op (K = 3 gives cspn2d's bits).  guidance (B, >=K*K-1, H, W); norm_type
    defaults to f'{K*K-1}sum'."""
    norm_type = norm_type or norm_names_2d(K)[0]
    guidance = np.asarray(guidance, dtype=dtype)
    raw = np.asarray(blur_depth, dtype=dtype)
    one = dtype(1.0)
    gate_wb, gate_sum = affinity_normalization_2d_k(guidance, K, norm_type)
    result = raw
    mask = None if sparse_depth is None else sparse_mask(sparse_depth, dtype)
    with np.errstate(invalid='ignore'):
        for _ in range(prop_time):
            acc = np.zeros_like(result)
            for k, (dy, dx) in enumerate(offsets_2d(K)):
                acc = acc + gate_wb[:, k:k + 1] * shift2d_k(result, dy, dx)
            result = (one - gate_sum) * raw + acc
            if mask is not None:
                result = (one - mask) * result + mask * raw
    return result.astype(dtype, copy=False)
