"""CPU oracle (numpy) for the CSPN propagation path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  The product path (cspn_b200/) never does.

Parity status
  2D: PINNED.  Checked against outputs of the reference module itself
      (/root/reference/cspn_pytorch/models/cspn.py executed in the build container,
      fixtures under tests/golden/, generator tests/golden/make_golden.py).
  3D: PARITY UNPINNED.  The reference ships only call sites
      (/root/reference/cspn_paddle/demo.py:41,51) to a Paddle op whose source is not
      in the tree; the arithmetic below is the 26-neighbour generalisation of cspn.py
      (SURVEY.md Appendix A.3) plus the own-location normalisation of demo.py:24,47-49.

Each function cites the reference lines it restates.
"""
from __future__ import annotations

import numpy as np

# (dy, dx) the k-th guidance channel / k-th depth copy is READ FROM, derived from the
# ZeroPad2d tuples (left,right,top,bottom) at cspn.py:105-129 (affinity) and
# cspn.py:149-168 (depth): a pad of (l, r, t, b) followed by the crop [1:-1, 1:-1]
# (cspn.py:72,142) reads the source at (y + 1 - t, x + 1 - l).
OFFSETS_2D = ((1, 1), (1, 0), (1, -1),
              (0, 1),         (0, -1),
              (-1, 1), (-1, 0), (-1, -1))

# 3D: pad triple (f,t,l) in raster order over {0,1,2}^3 without the centre (1,1,1);
# offset (dz,dy,dx) = (1-f, 1-t, 1-l)  (SURVEY.md Appendix A.3).
OFFSETS_3D = tuple((1 - f, 1 - t, 1 - l)
                   for f in range(3) for t in range(3) for l in range(3)
                   if (f, t, l) != (1, 1, 1))


def shift2d(a: np.ndarray, dy: int, dx: int) -> np.ndarray:
    """b[..., y, x] = a[..., y+dy, x+dx], zero outside (ZeroPad2d + crop, cspn.py:105-129,72)."""
    H, W = a.shape[-2:]
    out = np.zeros_like(a)
    ys = slice(max(0, -dy), min(H, H - dy))
    xs = slice(max(0, -dx), min(W, W - dx))
    yd = slice(max(0, -dy) + dy, min(H, H - dy) + dy)
    xd = slice(max(0, -dx) + dx, min(W, W - dx) + dx)
    out[..., ys, xs] = a[..., yd, xd]
    return out


def shift3d(a: np.ndarray, dz: int, dy: int, dx: int) -> np.ndarray:
    D, H, W = a.shape[-3:]
    out = np.zeros_like(a)

    def rng(n, d):
        lo, hi = max(0, -d), min(n, n - d)
        return slice(lo, hi), slice(lo + d, hi + d)
    zs, zd = rng(D, dz)
    ys, yd = rng(H, dy)
    xs, xd = rng(W, dx)
    out[..., zs, ys, xs] = a[..., zd, yd, xd]
    return out


def affinity_normalization_2d(guidance: np.ndarray, norm_type: str):
    """cspn.py:85-144.  guidance (B,>=8,H,W) -> gate_wb (B,8,H,W), gate_sum (B,1,H,W).

    Only channels 0..7 are used (narrow, cspn.py:91-98).  The cropped interior of the
    reference's padded tensors is returned (the padded border never reaches the output,
    cspn.py:72,142)."""
    g = guidance[:, :8]
    if 'abs' in norm_type:                                   # cspn.py:88-89
        g = np.abs(g)
    with np.errstate(divide='ignore', invalid='ignore'):
        a = np.stack([shift2d(g[:, k], dy, dx)               # cspn.py:105-132 (gather)
                      for k, (dy, dx) in enumerate(OFFSETS_2D)], axis=1)
        abs_weight = np.zeros_like(a[:, 0])
        for k in range(8):                                   # cspn.py:135-136 (ones conv = 8-way sum)
            abs_weight = abs_weight + np.abs(a[:, k])
        gate_wb = a / abs_weight[:, None]                    # cspn.py:138 (0/0 -> NaN, kept)
        gate_sum = np.zeros_like(abs_weight)
        for k in range(8):                                   # cspn.py:139
            gate_sum = gate_sum + gate_wb[:, k]
    return gate_wb, gate_sum[:, None]


def sparse_mask(sparse_depth, dtype=np.float32):
    """m = sign(sparse_depth), cspn.py:63-64, as torch.sign computes it on the CPU and on CUDA: 0 for NaN (np.sign gives
    NaN), so a NaN sparse pixel masks nothing."""
    sp = np.asarray(sparse_depth, dtype=dtype)
    return (sp > 0).astype(dtype) - (sp < 0).astype(dtype)


def cspn2d(guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum',
           dtype=np.float32):
    """Affinity_Propagate.forward, cspn.py:42-83, op for op (unfolded mask / centre term).

    guidance (B,>=8,H,W); blur_depth (B,C,H,W); sparse_depth (B,1,H,W) or None.
    dtype=float64 gives the 'exact' spec used to bound fp32 rounding in the tests."""
    assert norm_type in ('8sum', '8sum_abs')                 # cspn.py:36
    guidance = np.asarray(guidance, dtype=dtype)
    raw = np.asarray(blur_depth, dtype=dtype)                # cspn.py:58
    one = dtype(1.0)
    gate_wb, gate_sum = affinity_normalization_2d(guidance, norm_type)   # cspn.py:55
    result = raw                                             # cspn.py:61
    mask = None
    if sparse_depth is not None:
        mask = sparse_mask(sparse_depth, dtype)
    with np.errstate(invalid='ignore'):
        for _ in range(prop_time):                           # cspn.py:66
            acc = np.zeros_like(result)
            for k, (dy, dx) in enumerate(OFFSETS_2D):        # cspn.py:69-72
                acc = acc + gate_wb[:, k:k + 1] * shift2d(result, dy, dx)
            result = (one - gate_sum) * raw + acc            # cspn.py:76
            if mask is not None:                             # cspn.py:80-81
                result = (one - mask) * result + mask * raw
    return result.astype(dtype, copy=False)


def affinity_normalization_3d(guidance, norm_type: str):
    """26-neighbour analogue of cspn.py:85-144 ('26sum', '26sum_abs'), or the Paddle
    demo's own-location normalisation ('paddle', demo.py:24,47-49).
    guidance (B,26,D,H,W) -> gate (B,26,D,H,W), gate_sum (B,1,D,H,W)."""
    g = guidance[:, :26]
    with np.errstate(divide='ignore', invalid='ignore'):
        if norm_type == 'paddle':
            g = np.abs(g)                                    # demo.py:24
            normalizer = np.zeros_like(g[:, 0])
            for k in range(26):                              # demo.py:47 reduce_sum
                normalizer = normalizer + g[:, k]
            gate = g / normalizer[:, None]                   # demo.py:48-49
        else:
            if 'abs' in norm_type:
                g = np.abs(g)
            a = np.stack([shift3d(g[:, k], *o) for k, o in enumerate(OFFSETS_3D)], axis=1)
            abs_weight = np.zeros_like(a[:, 0])
            for k in range(26):
                abs_weight = abs_weight + np.abs(a[:, k])
            gate = a / abs_weight[:, None]
        gate_sum = np.zeros_like(gate[:, 0])
        for k in range(26):
            gate_sum = gate_sum + gate[:, k]
    return gate, gate_sum[:, None]


def cspn3d(guidance, feat, prop_time=12, norm_type='26sum_abs', dtype=np.float32):
    """3D CSPN (SURVEY.md Appendix A.3; call sites demo.py:20-54).

    '26sum' / '26sum_abs': gathered affinities + centre term on the initial volume,
    exactly as cspn.py does in 2D.  'paddle': gate normalised at the voxel's own
    location, out = sum_k gate_k(p) * feat(p+off_k), no centre term (demo.py:50-52:
    the op receives only feat and gate_weight)."""
    assert norm_type in ('26sum', '26sum_abs', 'paddle')
    guidance = np.asarray(guidance, dtype=dtype)
    raw = np.asarray(feat, dtype=dtype)
    one = dtype(1.0)
    gate, gate_sum = affinity_normalization_3d(guidance, norm_type)
    result = raw
    with np.errstate(invalid='ignore'):
        for _ in range(prop_time):
            acc = np.zeros_like(result)
            for k, o in enumerate(OFFSETS_3D):
                acc = acc + gate[:, k:k + 1] * shift3d(result, *o)
            if norm_type == 'paddle':
                result = acc
            else:
                result = (one - gate_sum) * raw + acc
    return result.astype(dtype, copy=False)


def parity_ok(a, b, rtol=1e-4):
    """The parity criterion of BASELINE.md section 4: |a-b| <= rtol*(|b| + mean|b|) elementwise,
    NaNs must coincide.  Returns (ok, max_violation_ratio, normwise_error)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    if not np.array_equal(nan_a, nan_b):
        return False, np.inf, np.inf
    fin = ~nan_b
    if not fin.any():
        return True, 0.0, 0.0
    scale = np.mean(np.abs(b[fin]))
    err = np.abs(a[fin] - b[fin])
    bound = rtol * (np.abs(b[fin]) + scale)
    ratio = float(np.max(err / np.maximum(bound, 1e-300)))
    normwise = float(err.max() / max(np.abs(b[fin]).max(), 1e-300))
    return bool(ratio <= 1.0), ratio, normwise
