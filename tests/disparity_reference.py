"""Restatements of disparity_regression (cspn_b200.disparity_regression, csrc/disparity_regression.cu; DESIGN.md section 4.15).

    y[b,c,h,w] = sum_o o * softmax_o(U[b,c,:,h,w]),   U = resize_trilinear(cost, (Do, Ho, Wo), align_corners, align_mode)

- resize_fp32: resize_trilinear in torch fp32, one rounding per operation in the kernels' order: the bits of
  cspn_b200.resize_trilinear (every torch op rounds on its own; nothing is fused in eager mode).
- resize_fp64: the same taps in fp64, as gathers.  It equals resize_reference.resize_torch on finite volumes, and like the
  kernels it reads only the two taps per axis, so a non-finite value reaches only the outputs whose taps read it (the
  dense matrices of resize_torch would multiply it by every zero of its row).
- forward_torch: resize_fp64 -> torch.softmax -> sum o*p, differentiable (any dtype and device).
- softmax_stage_fp32 / softmax_stage_torch: the kernels' softmax stage in fp32 (max, S and N in ascending o, y = N / S),
  in numpy, and in torch on the tensor's device.
- span_in / span_out / fwd_plan / bwd_plan: the kernels' launch plans, and spans(): the spans they bound, from the taps.
- bound_softmax / bound_fwd / bound_bwd: the a-priori bounds of DESIGN.md section 4.15.
"""
import numpy as np
import torch

import resize_reference as rr

U = 2.0 ** -24
TINY = 2.0 ** -148          # twice the smallest subnormal: expf's absolute error where its result is subnormal


def gamma(n):
    return n * U / (1 - n * U)


def _taps(in_size, out_size, align_corners, align_mode, device):
    out = []
    for n, m in zip(in_size, out_size):
        i0, i1, l0, l1 = rr.taps(n, m, align_corners, align_mode)
        out.append((torch.from_numpy(i0).to(device), torch.from_numpy(i1).to(device), torch.from_numpy(l0).to(device),
                    torch.from_numpy(l1).to(device)))
    return out


def _resize(x, out_size, align_corners, align_mode):
    """The nested order of resize_trilinear: the (h, w) blend of every low-resolution plane, then along d."""
    (d0, d1, l0d, l1d), (h0, h1, l0h, l1h), (w0, w1, l0w, l1w) = (
        tuple(t.to(x.dtype) if t.is_floating_point() else t for t in tap)
        for tap in _taps(x.shape[2:], out_size, align_corners, align_mode, x.device))

    def rows(hi):
        t = x[:, :, :, hi]                                            # (B, C, D, Ho, W)
        return l0w * t[..., w0] + l1w * t[..., w1]

    v = l0h[:, None] * rows(h0) + l1h[:, None] * rows(h1)              # (B, C, D, Ho, Wo)
    return l0d[:, None, None] * v[:, :, d0] + l1d[:, None, None] * v[:, :, d1]


def resize_fp32(x, out_size, align_corners=True, align_mode=1):
    return _resize(x.float(), out_size, align_corners, align_mode)


def resize_fp64(x, out_size, align_corners=True, align_mode=1):
    return _resize(x.double() if x.dtype != torch.float64 else x, out_size, align_corners, align_mode)


def regress_torch(u):
    """sum_o o * softmax_o(u) over dim 2 of (B, C, Do, Ho, Wo)."""
    o = torch.arange(u.shape[2], dtype=u.dtype, device=u.device)[:, None, None]
    return (torch.softmax(u, dim=2) * o).sum(2)


def forward_torch(cost, out_size, align_corners=True, align_mode=1):
    return regress_torch(resize_fp64(cost, out_size, align_corners, align_mode))


def softmax_stage_fp32(u):
    """The kernels' softmax stage on fp32 U (B, C, Do, Ho, Wo) in numpy: m = max (NaN if any), S = sum e and N = sum o*e in
    ascending o with e = exp(U - m), y = N / S, every operation rounded to fp32."""
    u = np.asarray(u, dtype=np.float32)
    with np.errstate(invalid='ignore', over='ignore', under='ignore'):
        m = u.max(axis=2)
        S = np.zeros_like(m)
        N = np.zeros_like(m)
        for o in range(u.shape[2]):
            e = np.exp((u[:, :, o] - m).astype(np.float32)).astype(np.float32)
            S = (S + e).astype(np.float32)
            N = (N + (np.float32(o) * e).astype(np.float32)).astype(np.float32)
        return (N / S).astype(np.float32)


def softmax_stage_torch(u):
    """The kernels' softmax stage in torch fp32 on u's device, one rounding per operation in the kernels' order: m = max,
    e = exp(U - m), S = sum e and N = sum o*e in ascending o from 0, y = N / S.  On CUDA, torch.exp of fp32 is the CUDA
    math library's expf, the kernels' own, so with U = cspn_b200.resize_trilinear's output this is the kernels' bits."""
    u = u.float()
    m = u.amax(2)
    S = torch.zeros_like(m)
    N = torch.zeros_like(m)
    for o in range(u.shape[2]):
        e = torch.exp(u[:, :, o] - m)
        S = S + e
        N = N + float(o) * e
    return N / S


def _moments(u):
    """Per column of u (fp64, finite, dim 2): t = u - max, E = exp(t), S, y, p and the disparities o."""
    o = torch.arange(u.shape[2], dtype=torch.float64, device=u.device)[:, None, None]
    t = u - u.amax(2, keepdim=True)
    E = torch.exp(t)
    S = E.sum(2, keepdim=True)
    y = (o * E).sum(2, keepdim=True) / S
    return o, t, E, S, y, E / S


def _stage(u):
    """The softmax stage's bound at fp32 values u: (B_s, and the pieces bound_bwd reuses)."""
    Do = u.shape[2]
    o, t, E, S, y, p = _moments(u)
    a = torch.exp(t * (1 - U)) * (1 + 4 * U) - E + TINY             # |e_hat - exp(t)|: the rounded t, expf's 2 ulp
    A = a.sum(2, keepdim=True)
    num = ((o - y).abs() * a).sum(2, keepdim=True) + gamma(Do) * (y * S + (o * a).sum(2, keepdim=True)) \
        + y * gamma(Do - 1) * (S + A) + Do * 2.0 ** -149
    den = S - A - gamma(Do - 1) * (S + A)
    q = num / den
    return q + U * (y + q), dict(o=o, S=S, y=y, p=p, a=a, theta=(A + gamma(Do - 1) * (S + A)) / S)


def bound_softmax(u32):
    """|y_kernel - y(U)| per pixel (B, C, Ho, Wo) for the fp32 values u32 of U (finite columns), y(U) exact."""
    return _stage(u32.double())[0][:, :, 0]


def _perturbation(cost, out_size, align_corners, align_mode):
    """U* in fp64, and delta, the per-pixel max of resize's bound gamma_6 * resize(|cost|) on |U_fp32 - U*|."""
    ustar = resize_fp64(cost, out_size, align_corners, align_mode)
    delta = (rr.gamma(6) * resize_fp64(cost.double().abs(), out_size, align_corners, align_mode)).amax(2, keepdim=True)
    return ustar, delta


def bound_fwd(cost, out_size, align_corners=True, align_mode=1):
    """|y_kernel - forward_torch(cost)| per pixel: the softmax stage at the fp32 U, plus the move of y from U* to U_fp32,
    at most (e^2delta - e^delta) * sum_o p*_o |o - y*|."""
    ustar, delta = _perturbation(cost, out_size, align_corners, align_mode)
    o, _, _, _, ystar, pstar = _moments(ustar)
    m1 = (pstar * (o - ystar).abs()).sum(2, keepdim=True)
    del ustar, pstar
    stage = _stage(resize_fp32(cost, out_size, align_corners, align_mode).double())[0]
    return (stage + (torch.expm1(2 * delta) - torch.expm1(delta)) * m1)[:, :, 0]


def grad_torch(cost, g, out_size, align_corners=True, align_mode=1):
    """grad_cost of sum(g * y) through forward_torch, in fp64 (autograd)."""
    c = cost.detach().double().requires_grad_(True)
    (forward_torch(c, out_size, align_corners, align_mode) * g.double()).sum().backward()
    return c.grad


def bound_bwd(cost, g, out_size, align_corners=True, align_mode=1):
    """|grad_kernel - grad_torch| per element of cost: a bound e_U on |gU_kernel - gU*| per upsampled element (the softmax
    stage at the fp32 U, then the move from U* to U_fp32), carried through resize's adjoint R^T with its own rounding:
    R^T(e_U) + gamma_k * R^T(|gU*| + e_U), k of resize_reference.bound_bwd."""
    in_size = tuple(cost.shape[2:])
    g = g.double()[:, :, None]
    ustar, delta = _perturbation(cost, out_size, align_corners, align_mode)
    o, _, _, _, ystar, pstar = _moments(ustar)
    del ustar
    m1 = (pstar * (o - ystar).abs()).sum(2, keepdim=True)
    dy = (torch.expm1(2 * delta) - torch.expm1(delta)) * m1
    gstar = g * pstar * (o - ystar)
    e_u = g.abs() * pstar * (torch.expm1(2 * delta) * (o - ystar).abs() + torch.exp(2 * delta) * dy)
    del pstar, ystar
    bs, s = _stage(resize_fp32(cost, out_size, align_corners, align_mode).double())
    p, y, th = s['p'], s['y'], s['theta']
    p_err = s['a'] / (s['S'] * (1 - th)) + p * th / (1 - th)
    dist = (o - y).abs() + bs
    e_u += g.abs() * (p_err * dist + p * bs + (p + p_err) * dist * ((1 + U) ** 3 - 1))
    del p, p_err, dist, s
    k = rr.bound_bwd(in_size, out_size, align_corners, align_mode)
    return rr.adjoint_torch(e_u, in_size, align_corners, align_mode) + k * rr.adjoint_torch(gstar.abs() + e_u, in_size,
                                                                                          align_corners, align_mode)


def sharp_cost(B, C, H, W, seed=0, spike=1000.0):
    """Small integer costs over D = 5 with a spike at one d = k per (b, c) slice, and the k of each slice.  With Do = 17 and
    align_corners (r = 1/4), U at o = 4k is the spike row's blend exactly and every other o is at least 234 below it."""
    gen = torch.Generator().manual_seed(seed)
    cost = torch.randint(-8, 9, (B, C, 5, H, W), generator=gen).float()
    k = torch.randint(0, 5, (B, C), generator=gen)
    for b in range(B):
        for c in range(C):
            cost[b, c, int(k[b, c])] += spike
    return cost, k


def nan_mask_fwd(cost, out_size, align_corners, align_mode):
    """Where the fp64 composition's y is NaN."""
    return torch.isnan(forward_torch(cost, out_size, align_corners, align_mode))


def normwise(got, want):
    return float((got.double() - want).norm() / want.norm())


def max_ratio(got, want, bound):
    """max |got - want| / bound: <= 1 when got is within the bound (an exact 0 where the bound is 0 counts as 0: a cost
    voxel that no output reads has gradient 0 and bound 0)."""
    err = (got.double() - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())



# ---- the launch plans of csrc/disparity_regression.cu, restated: the tile sizes and the spans that size shared memory ----
SMEM_SOFT, SMEM_HARD = 110 * 1024, 227 * 1024
FWD_TILES = [(8, 32), (4, 32), (2, 32), (1, 32), (1, 16), (1, 8), (1, 4), (1, 2), (1, 1)]
BWD_TILES = [(8, 8), (4, 8), (4, 4), (2, 4), (2, 2), (1, 2), (1, 1)]


def span_in(n_in, n_out, align_corners, align_mode, t):
    """The kernels' bound of the low-resolution indices t consecutive outputs read."""
    r = float(rr.ratio(n_in, n_out, align_corners))
    return int(min(n_in, np.floor(r * (t - 1) + (n_in + 2.0) * 2.0 ** -21) + 3))


def span_out(n_in, n_out, align_corners, align_mode, t):
    """The kernels' bound of the outputs that read t consecutive low-resolution indices."""
    r = float(rr.ratio(n_in, n_out, align_corners))
    if r == 0:
        return n_out
    half = not align_corners and align_mode == 0
    return int(min(n_out, np.floor((t + 1.0 + (0.5 if half else 0.0)) / r + (n_out + 2.0) * 2.0 ** -21) + 2))


def spans(n_in, n_out, align_corners, align_mode, t):
    """The largest number of low-resolution indices read by t consecutive outputs, and of outputs that read t consecutive
    low-resolution indices, over every start, from the fp32 taps."""
    i0, i1, _, _ = rr.taps(n_in, n_out, align_corners, align_mode)
    starts = np.arange(0, n_out)
    last = np.minimum(starts + t, n_out) - 1
    read = int((i1[last] - i0[starts] + 1).max())
    cells = np.arange(n_in)
    b = np.searchsorted(i0, cells - 1, 'left')
    e = np.searchsorted(i0, np.minimum(cells + t, n_in) - 1 + 1, 'left')
    return read, int((e - b).max())


def bwd_plan(in_size, out_size, align_corners, align_mode):
    """(tile, (ph, pw), shared bytes) of the backward, or None where no tile fits."""
    (D, H, W), (Do, Ho, Wo) = in_size, out_size
    for th, tw in BWD_TILES:
        ph = span_out(H, Ho, align_corners, align_mode, th)
        pw = span_out(W, Wo, align_corners, align_mode, tw)
        smem = 8 * (Do + ph + pw) + 4 * D * (th + 2) * (tw + 2) + 4 * ph * pw * (D | 1)
        if smem <= SMEM_SOFT or ((th, tw) == (1, 1) and smem <= SMEM_HARD):
            return (th, tw), (ph, pw), smem
    return None


def fwd_plan(in_size, out_size, align_corners, align_mode):
    (D, H, W), (Do, Ho, Wo) = in_size, out_size
    for th, tw in FWD_TILES:
        smem = 8 * Do + 4 * D * span_in(H, Ho, align_corners, align_mode, th) * span_in(W, Wo, align_corners, align_mode, tw)
        if smem <= SMEM_SOFT or ((th, tw) == (1, 1) and smem <= SMEM_HARD):
            return (th, tw), smem
    return None
