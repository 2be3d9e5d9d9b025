"""The aggregation of the 2D propagation's steps (CSPN++'s context-aware CSPN, DESIGN.md section 4.20), restated: the op
sequence (autograd-able, any dtype) and the fp32 sums in the kernels' order.  Shared by tests/test_aggregate_cpu.py and
tests/test_aggregate_gpu.py.

    d_0 = blur;  d_{t+1} = one step of propagate2d_k(..., keep_sparse=keep);  out = sum_j sw[:, j] * d_{s_j}

The step is backward_exact.cspn2d_shift_ref's (the reference module's m = sign(sparse)) or keep_sparse_reference's (the
paper's m = 1[sparse > 0] with the samples kept); a missing sparse in keep mode is the default mode.
"""
import torch

import backward_exact as be
import keep_sparse_reference as ks
from oracle.cspn_numpy_k import offsets_2d


def default_steps(T):
    return tuple(range(1, T + 1))


def step_fn(g, blur, sparse, K, norm, keep):
    """d -> d_{t+1} in the dtype of the inputs."""
    r, offs = (K - 1) // 2, offsets_2d(K)
    _, w, _, s = ks.gates(g, K, norm)
    keep = keep and sparse is not None
    m = None if sparse is None else (ks.mask(sparse, blur.dtype) if keep else sparse.sign())

    def step(d):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + w[:, k:k + 1] * be.shift(d, o, r)
        e = (1 - s) * blur + acc
        if m is None:
            return e
        return (1 - m) * e + m * (sparse if keep else blur)
    return step


def iterates(g, blur, sparse, steps, K=3, norm=None, keep=False):
    """[d_{s_0}, ..., d_{s_{T-1}}] of the op sequence."""
    norm = norm or f'{K * K - 1}sum'
    step = step_fn(g, blur, sparse, K, norm, keep)
    d, out = blur, []
    for t in range(1, steps[-1] + 1):
        d = step(d)
        if t in steps:
            out.append(d)
    return out


def composition(g, blur, sparse, sw, steps=None, K=3, norm=None, keep=False):
    """The op as written: the autograd reference (gradients for g, blur, sw and, in keep mode, sparse)."""
    steps = steps or default_steps(sw.shape[1])
    return aggregate(iterates(g, blur, sparse, steps, K, norm, keep), sw)


def aggregate(ds, sw):
    """out = sw_0 d_{s_0}, then out + sw_j d_{s_j}: the kernels' order, each product and sum rounded on its own in fp32."""
    out = sw[:, 0:1] * ds[0]
    for j in range(1, len(ds)):
        out = out + sw[:, j:j + 1] * ds[j]
    return out


def grad_step_weight(grad_out, ds):
    """grad_sw[:, j] = sum_c grad_out[:, c] d_{s_j}[:, c], c ascending from the first term: the kernels' order."""
    cols = []
    for d in ds:
        a = grad_out[:, 0] * d[:, 0]
        for c in range(1, d.shape[1]):
            a = a + grad_out[:, c] * d[:, c]
        cols.append(a)
    return torch.stack(cols, 1)


def within(ours, ref, rel=2e-3):
    """The K x K backward's tolerance against fp64 autograd: |ours - ref| <= rel (|ref| + mean |ref|)."""
    ours, ref = ours.double().cpu(), ref.double().cpu()
    scale = ref.abs().mean()
    err = (ours - ref).abs()
    return bool((err <= rel * (ref.abs() + scale)).all()), float(err.max()), float(scale)


def dyadic_weights(gen, shape):
    """Step weights in {0, +-1/2, +-1}: products with the dyadic iterates stay on a grid of powers of two."""
    return torch.randint(-2, 3, shape, generator=gen).float() / 2
