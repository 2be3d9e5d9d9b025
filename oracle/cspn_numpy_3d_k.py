"""CPU oracle (numpy) of the 3D propagation with a K x K x K affinity kernel, K in {3, 5}.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and tools/ may import this module; the product path (cspn_b200/) never does.

Parity status: anchored to the 3D arithmetic of oracle/cspn_numpy.py.  cspn3d_k(K=3) gives the bits of
cspn_numpy.cspn3d; nothing outside this repository pins K = 5, which is the same op sequence over the 5 x 5 x 5 window.
"""
from __future__ import annotations

import numpy as np

from .cspn_numpy import shift3d


# Tap k enumerates (f, t, l) over [0, K)^3 in raster order without the centre (r, r, r) and reads the source at
# (dz, dy, dx) = (r-f, r-t, r-l).  At K = 3 this is cspn_numpy.OFFSETS_3D.
def offsets_3d(K):
    assert K in (3, 5)
    r = (K - 1) // 2
    return tuple((r - f, r - t, r - l) for f in range(K) for t in range(K) for l in range(K) if (f, t, l) != (r, r, r))


def shift3d_k(a, dz, dy, dx):
    """shift3d for offsets that may reach past the volume (D, H or W < K): such a copy is all padding."""
    D, H, W = a.shape[-3:]
    if abs(dz) >= D or abs(dy) >= H or abs(dx) >= W:
        return np.zeros_like(a)
    return shift3d(a, dz, dy, dx)


def norm_names_3d(K):
    """The norm names of a K x K x K kernel: f'{K**3-1}sum', f'{K**3-1}sum_abs' and 'paddle'."""
    return (f'{K ** 3 - 1}sum', f'{K ** 3 - 1}sum_abs', 'paddle')


def affinity_normalization_3d_k(guidance, K, norm_type):
    """cspn_numpy.affinity_normalization_3d with K**3-1 taps.  guidance (B, K**3-1, D, H, W)."""
    assert norm_type in norm_names_3d(K)
    offs = offsets_3d(K)
    nt = len(offs)
    g = guidance[:, :nt]
    with np.errstate(divide='ignore', invalid='ignore'):
        if norm_type == 'paddle':
            g = np.abs(g)
            normalizer = np.zeros_like(g[:, 0])
            for k in range(nt):
                normalizer = normalizer + g[:, k]
            gate = g / normalizer[:, None]
        else:
            if 'abs' in norm_type:
                g = np.abs(g)
            a = np.stack([shift3d_k(g[:, k], *o) for k, o in enumerate(offs)], axis=1)
            abs_weight = np.zeros_like(a[:, 0])
            for k in range(nt):
                abs_weight = abs_weight + np.abs(a[:, k])
            gate = a / abs_weight[:, None]
        gate_sum = np.zeros_like(gate[:, 0])
        for k in range(nt):
            gate_sum = gate_sum + gate[:, k]
    return gate, gate_sum[:, None]


def cspn3d_k(guidance, feat, prop_time=12, K=5, norm_type=None, dtype=np.float32):
    """cspn3d with a K x K x K kernel, op for op (K = 3 gives cspn3d's bits).  guidance (B, K**3-1, D, H, W), one gate
    shared by the channels of feat (B, C, D, H, W); norm_type defaults to f'{K**3-1}sum_abs'."""
    norm_type = norm_type or norm_names_3d(K)[1]
    guidance = np.asarray(guidance, dtype=dtype)
    raw = np.asarray(feat, dtype=dtype)
    one = dtype(1.0)
    gate, gate_sum = affinity_normalization_3d_k(guidance, K, norm_type)
    result = raw
    with np.errstate(invalid='ignore'):
        for _ in range(prop_time):
            acc = np.zeros_like(result)
            for k, o in enumerate(offsets_3d(K)):
                acc = acc + gate[:, k:k + 1] * shift3d_k(result, *o)
            if norm_type == 'paddle':
                result = acc
            else:
                result = (one - gate_sum) * raw + acc
    return result.astype(dtype, copy=False)
