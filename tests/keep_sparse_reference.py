"""The keep-sparse mode of the 2D propagation (DESIGN.md section 4.13), restated: the spec's op sequence (autograd-able, any
dtype) and the same forward with its adjoint written out, for step counts where autograd's saved tensors would not fit.
Shared by tests/test_keep_sparse_cpu.py and tests/test_keep_sparse_gpu.py.

    m = 1[sparse > 0];  d_0 = blur;  e_{t+1} = (1 - s) blur + sum_k w_k shift_k(d_t);  d_{t+1} = (1 - m) e_{t+1} + m sparse

with w_k = a_k / sum_j |a_j|, a_k(p) = g'_k(p + off_k) (g' = |g| in the _abs norm, zero outside), s = sum_k w_k, and the
K x K taps of oracle/cspn_numpy_k.py.  The reference module's mode differs only in m = sign(sparse) and "+ m * blur".
"""
import torch

import backward_exact as be
from oracle.cspn_numpy_k import offsets_2d


def _neg(o):
    return tuple(-c for c in o)


def gates(g, K, norm):
    """(a, w, S, s) of the K x K kernel, each (B, taps or 1, H, W)."""
    nt, r = K * K - 1, (K - 1) // 2
    gn = g[:, :nt].abs() if norm.endswith('_abs') else g[:, :nt]
    a = torch.stack([be.shift(gn[:, k], o, r) for k, o in enumerate(offsets_2d(K))], 1)
    S = a.abs().sum(1, keepdim=True)
    w = a / S
    return a, w, S, w.sum(1, keepdim=True)


def mask(sparse, dtype):
    return (sparse > 0).to(dtype)


def op_sequence(g, blur, sparse, N, K=3, norm='8sum'):
    """The spec as written, in the dtype of the inputs: the autograd reference (gradients for g, blur and sparse)."""
    r = (K - 1) // 2
    _, w, _, s = gates(g, K, norm)
    m = mask(sparse, blur.dtype)
    d = blur
    for _ in range(N):
        acc = 0
        for k, o in enumerate(offsets_2d(K)):
            acc = acc + w[:, k:k + 1] * be.shift(d, o, r)
        e = (1 - s) * blur + acc
        d = (1 - m) * e + m * sparse
    return d


def reference(g, blur, sparse, N, K=3, norm='8sum', grad_out=None):
    """op_sequence with its adjoint written out (memory: N + 1 images).  Returns `out`, or with grad_out
    (out, grad_guidance, grad_blur, grad_sparse).  The indicator has zero derivative, so
        dL/dsparse = m sum_t sum_c lambda_{t+1},   dL/dblur = sum_t (1 - m)(1 - s) lambda_{t+1} + lambda_0."""
    r = (K - 1) // 2
    offs = offsets_2d(K)
    nt = len(offs)
    a, w, S, s = gates(g, K, norm)
    m = mask(sparse, blur.dtype)
    ds = [blur]
    for _ in range(N):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + w[:, k:k + 1] * be.shift(ds[-1], o, r)
        ds.append((1 - m) * ((1 - s) * blur + acc) + m * sparse)
    if grad_out is None:
        return ds[-1]
    out = ds[-1]
    lam = grad_out
    gw = torch.zeros_like(w)
    gs = torch.zeros_like(s)
    gblur = torch.zeros_like(blur)
    gsparse = torch.zeros_like(sparse)
    for t in range(N - 1, -1, -1):
        ds.pop()
        mu = (1 - m) * lam                     # dL/de_{t+1}
        gsparse = gsparse + m * lam.sum(1, keepdim=True)
        gblur = gblur + (1 - s) * mu
        gs = gs - (mu * blur).sum(1, keepdim=True)
        for k, o in enumerate(offs):
            gw[:, k] += (mu * be.shift(ds[t], o, r)).sum(1)
        nxt = 0
        for k, o in enumerate(offs):
            nxt = nxt + be.shift(w[:, k:k + 1] * mu, _neg(o), r)
        lam = nxt
    gblur = gblur + lam
    gw = gw + gs
    ga = (gw - a.sign() * (gw * w).sum(1, keepdim=True)) / S
    gn = torch.stack([be.shift(ga[:, k], _neg(o), r) for k, o in enumerate(offs)], 1)
    gg = torch.zeros_like(g)
    gg[:, :nt] = gn * g[:, :nt].sign() if norm.endswith('_abs') else gn
    return out, gg, gblur, gsparse
