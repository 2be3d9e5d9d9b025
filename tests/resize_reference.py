"""Restatements of resize_trilinear (cspn_b200.resize_trilinear, csrc/resize_trilinear.cu; DESIGN.md section 4.14).

- taps(): the per-axis source coordinates, in fp32 with every operation rounded on its own, as the kernels form them.
- forward_fp32 / backward_fp32: numpy fp32 in the kernels' documented operation order; the GPU is held to them bit for bit.
- forward_fp64 / backward_fp64: the same fp32 coordinates and weights, the arithmetic in fp64 (dense per-axis matrices).
- resize_torch: a torch-ops port of forward_fp64 for autograd (any dtype and device).
- bound_fwd / bound_bwd: a-priori bounds of the fp32 evaluation's distance from fp64.
"""
import numpy as np
import torch

F32 = np.float32
U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


def ratio(n_in, n_out, align_corners):
    if n_out == 1:
        return F32(0)
    return F32(n_in - 1) / F32(n_out - 1) if align_corners else F32(n_in) / F32(n_out)


def taps(n_in, n_out, align_corners=True, align_mode=1):
    """(i0, i1, l0, l1) of every output index along one axis: i0 / i1 int64, l0 / l1 float32."""
    r = ratio(n_in, n_out, align_corners)
    o = np.arange(n_out).astype(F32)
    if not align_corners and align_mode == 0:
        s = np.maximum(r * (o + F32(0.5)) - F32(0.5), F32(0))
    else:
        s = r * o
    s = s.astype(F32)
    i0 = np.minimum(s.astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (s - i0.astype(F32)).astype(F32)
    return i0, i1, (F32(1) - l1).astype(F32), l1


def ramp_output(n_in, n_out, align_corners=True, align_mode=1):
    """What a ramp x[i] = i resamples to along one axis, in fp64: the source coordinate s, or n_in-1 where both taps read
    the last index."""
    i0, i1, l0, l1 = taps(n_in, n_out, align_corners, align_mode)
    return i0 * l0.astype(np.float64) + i1 * l1.astype(np.float64)


def _all_taps(in_size, out_size, align_corners, align_mode):
    return [taps(n, m, align_corners, align_mode) for n, m in zip(in_size, out_size)]


def forward_fp32(x, out_size, align_corners=True, align_mode=1):
    """x (B, C, D, H, W) float32 -> (B, C, Do, Ho, Wo), every operation rounded to fp32 in the kernel's order."""
    x = np.asarray(x, dtype=F32)
    (d0, d1, l0d, l1d), (h0, h1, l0h, l1h), (w0, w1, l0w, l1w) = _all_taps(x.shape[2:], out_size, align_corners, align_mode)
    l0d, l1d = l0d[:, None, None], l1d[:, None, None]
    l0h, l1h = l0h[:, None], l1h[:, None]

    def row(di, hi):
        t = x[:, :, di][:, :, :, hi]                                  # (B, C, Do, Ho, W)
        return (l0w * t[..., w0]).astype(F32) + (l1w * t[..., w1]).astype(F32)

    e0 = (l0h * row(d0, h0)).astype(F32) + (l1h * row(d0, h1)).astype(F32)
    e1 = (l0h * row(d1, h0)).astype(F32) + (l1h * row(d1, h1)).astype(F32)
    return ((l0d * e0).astype(F32) + (l1d * e1).astype(F32)).astype(F32)


def _adjoint_axis_fp32(t, axis, n_in, tap):
    """The gather along one axis: out[..., i, ...] = sum over the outputs o that read i, ascending, of t[..., o, ...] * w,
    every operation rounded to fp32; w = l0 if i0(o) == i else l1, and both products (l0 first) where i1 == i0 == i."""
    i0, _, l0, l1 = tap
    t = np.moveaxis(np.asarray(t, dtype=F32), axis, -1)
    i = np.arange(n_in)
    b = np.searchsorted(i0, i - 1, 'left')
    e = np.searchsorted(i0, i + 1, 'left')
    acc = np.zeros(t.shape[:-1] + (n_in,), dtype=F32)
    for k in range(int((e - b).max(initial=0))):
        o = b + k
        valid = o < e
        oc = np.minimum(o, len(i0) - 1)
        v = t[..., oc]
        own = i0[oc] == i
        first = acc + (v * np.where(own, l0[oc], l1[oc])).astype(F32)
        twice = own & (i == n_in - 1)
        second = first + (v * l1[oc]).astype(F32)
        acc = np.where(valid, np.where(twice, second, first), acc).astype(F32)
    return np.moveaxis(acc, -1, axis)


def backward_fp32(g, in_size, align_corners=True, align_mode=1):
    """grad_x (B, C, D, H, W) of grad_out g (B, C, Do, Ho, Wo) in the kernel's order: the W sums of every output row, then
    the H sums of those, then the D sums (each sum from 0, ascending o)."""
    g = np.asarray(g, dtype=F32)
    tap_d, tap_h, tap_w = _all_taps(in_size, g.shape[2:], align_corners, align_mode)
    t = _adjoint_axis_fp32(g, 4, in_size[2], tap_w)
    t = _adjoint_axis_fp32(t, 3, in_size[1], tap_h)
    return _adjoint_axis_fp32(t, 2, in_size[0], tap_d)


def matrices(in_size, out_size, align_corners=True, align_mode=1, abs_=False):
    """Per axis the (n_out, n_in) fp64 matrix M with M[o, i0] += l0, M[o, i1] += l1 (the two taps add at the last index)."""
    ms = []
    for n, m in zip(in_size, out_size):
        i0, i1, l0, l1 = taps(n, m, align_corners, align_mode)
        M = np.zeros((m, n))
        np.add.at(M, (np.arange(m), i0), l0.astype(np.float64))
        np.add.at(M, (np.arange(m), i1), l1.astype(np.float64))
        ms.append(M)
    return ms


def resize_torch(x, out_size, align_corners=True, align_mode=1):
    """forward_fp64 as torch ops (differentiable in x, in x's dtype and on its device)."""
    Md, Mh, Mw = (torch.from_numpy(M).to(x.device, x.dtype) for M in matrices(x.shape[2:], out_size, align_corners, align_mode))
    B, C = x.shape[:2]
    t = x @ Mw.T                                                        # (B, C, D, H, Wo)
    t = Mh @ t                                                          # (B, C, D, Ho, Wo)
    t = Md @ t.reshape(B, C, x.shape[2], -1)                            # (B, C, Do, Ho*Wo)
    return t.reshape(B, C, *out_size)


def adjoint_torch(g, in_size, align_corners=True, align_mode=1):
    """backward_fp64 as torch ops: the transposed matrices applied to g, in g's dtype and on its device."""
    Md, Mh, Mw = (torch.from_numpy(M).to(g.device, g.dtype) for M in matrices(in_size, g.shape[2:], align_corners, align_mode))
    B, C, Do, Ho, Wo = g.shape
    t = g @ Mw                                                          # (B, C, Do, Ho, W)
    t = Mh.T @ t                                                        # (B, C, Do, H, W)
    t = Md.T @ t.reshape(B, C, Do, -1)
    return t.reshape(B, C, *in_size)


def forward_fp64(x, out_size, align_corners=True, align_mode=1):
    return resize_torch(torch.as_tensor(np.asarray(x, dtype=np.float64)), out_size, align_corners, align_mode).numpy()


def backward_fp64(g, in_size, align_corners=True, align_mode=1):
    return adjoint_torch(torch.as_tensor(np.asarray(g, dtype=np.float64)), in_size, align_corners, align_mode).numpy()


def max_range(in_size, out_size, align_corners=True, align_mode=1):
    """The longest run of outputs that read one input index, over the three axes."""
    n = 0
    for (i0, *_), m in zip(_all_taps(in_size, out_size, align_corners, align_mode), in_size):
        i = np.arange(m)
        n = max(n, int((np.searchsorted(i0, i + 1) - np.searchsorted(i0, i - 1)).max()))
    return n


def bound_fwd(x_abs64):
    """|fp32 - fp64| of the forward: 3 products and 3 sums per term, so gamma_6 * forward_fp64(|x|)."""
    return gamma(6) * x_abs64


def bound_bwd(in_size, out_size, align_corners, align_mode):
    """The factor k of |fp32 - fp64| <= gamma_k * adjoint(|g|): 3 products, and per axis at most max_range + 1 additions."""
    return gamma(3 + 3 * (max_range(in_size, out_size, align_corners, align_mode) + 1))
