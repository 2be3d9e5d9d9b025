"""Restatements of affinity fusion (cspn_b200.affinity_fuse2d, csrc/affinity_fuse.cu; DESIGN.md section 4.18), the CSPN
stereo network's spatial pyramid fusion.  L levels x_l (B, C, h_l, w_l), gate (B, L, H, W):

    a_l = |gate[:, l]|,  S = sum_l a_l,  w_l = a_l / S,  out[:, c] = sum_l w_l * u_l[:, c]

with u_l the level resampled bilinearly to (H, W) by resize_trilinear's per-axis rule (tests/resize_reference.py's taps).

- compose: the torch composition (abs, a sum over the levels, a broadcast divide, L resamplings as dense fp64-exact
  per-axis matrices, L products and a sum), differentiable, in the dtype and on the device of the inputs.  In fp64, with
  its autograd, it is the reference.
- fwd_torch / bwd_torch: the kernels' order in fp32 (eager torch rounds every operation on its own, on the CPU and the GPU
  alike; the level gradients go through resize_reference._adjoint_axis_fp32 in numpy), every sum from its first term:
    S, out      ascending l
    u           l0h*(l0w*x[h0,w0] + l1w*x[h0,w1]) + l1h*(l0w*x[h1,w0] + l1w*x[h1,w1]), left to right
    grad_gate   (t_l / S) * sgn(gate_l),  t_l = sum_c grad_out[c] * (u_l[c] - out[c]) in ascending c
    grad_x_l    sum_oh (sum_ow v * lw) * lh,  v = w_l * grad_out: resize_trilinear's gather over W, then H
- bound_fwd / bound_bwd: the a-priori bounds of the fp32 results against exact arithmetic, u = 2^-24,
  gamma_k = k u / (1 - k u), U_l = upsample(|x_l|), m = sum_l w_l U_l (finite inputs, no underflow):
    out         gamma_{2L+4} m
    grad_gate   |sgn(gate_l)| gamma_{3L+C+5} sum_c |grad_out_c| (U_l,c + m_c) / S
    grad_x_l    gamma_{L+3+2(r+1)} adjoint_l(w_l |grad_out|),  r the longest run of outputs that read one index
"""
import numpy as np
import torch

import resize_reference as rr

U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


def upsample(x, H, W, align_corners=True, align_mode=1):
    """(B, C, h, w) -> (B, C, H, W): the four taps gathered and blended in x's dtype, differentiable.  Its autograd scatters
    into the cells each output reads, as the kernels' gather does, so a NaN gradient reaches those cells only (a dense
    resampling matrix would multiply it into every cell through its zeros)."""
    h0, h1, l0h, l1h = (t.to(x.dtype) if t.is_floating_point() else t for t in _taps(x.shape[2], H, align_corners, align_mode, x.device))
    w0, w1, l0w, l1w = (t.to(x.dtype) if t.is_floating_point() else t for t in _taps(x.shape[3], W, align_corners, align_mode, x.device))
    r0, r1 = x[:, :, h0], x[:, :, h1]
    return l0h[:, None] * (l0w * r0[..., w0] + l1w * r0[..., w1]) + l1h[:, None] * (l0w * r1[..., w0] + l1w * r1[..., w1])


def adjoint(g, hw, align_corners=True, align_mode=1):
    """The transpose of upsample: (B, C, H, W) -> (B, C, h, w), in g's dtype."""
    return rr.adjoint_torch(g[:, :, None], (1, *hw), align_corners, align_mode)[:, :, 0]


def compose(levels, gate, align_corners=True, align_mode=1):
    """The torch composition, differentiable; in fp64 the reference."""
    H, W = gate.shape[2:]
    a = gate.abs()
    w = a / a.sum(dim=1, keepdim=True)
    return sum(w[:, l:l + 1] * upsample(x, H, W, align_corners, align_mode) for l, x in enumerate(levels))


# ---- the kernels' order ---------------------------------------------------------------------------------------------------------
def _taps(n_in, n_out, align_corners, align_mode, device):
    i0, i1, l0, l1 = rr.taps(n_in, n_out, align_corners, align_mode)
    return (torch.from_numpy(i0).to(device), torch.from_numpy(i1).to(device), torch.from_numpy(l0).to(device),
            torch.from_numpy(l1).to(device))


def upsample_fp32(x, H, W, align_corners=True, align_mode=1):
    """u in the kernels' order, every operation rounded to fp32."""
    h0, h1, l0h, l1h = _taps(x.shape[2], H, align_corners, align_mode, x.device)
    w0, w1, l0w, l1w = _taps(x.shape[3], W, align_corners, align_mode, x.device)
    r0, r1 = x[:, :, h0], x[:, :, h1]
    e0 = l0w * r0[..., w0] + l1w * r0[..., w1]
    e1 = l0w * r1[..., w0] + l1w * r1[..., w1]
    return l0h[:, None] * e0 + l1h[:, None] * e1


def weights(gate):
    """(w, S): w (B, L, H, W) = a / S, S (B, H, W) summed in ascending l."""
    a = gate.abs()
    S = a[:, 0]
    for l in range(1, a.shape[1]):
        S = S + a[:, l]
    return a / S[:, None], S


def fwd_torch(levels, gate, align_corners=True, align_mode=1):
    H, W = gate.shape[2:]
    w, _ = weights(gate)
    out = None
    for l, x in enumerate(levels):
        t = w[:, l:l + 1] * upsample_fp32(x, H, W, align_corners, align_mode)
        out = t if out is None else out + t
    return out


def adjoint_fp32(v, hw, align_corners=True, align_mode=1):
    """resize_trilinear's gather restricted to H and W: the W sums of every row, then the H sums of those."""
    H, W = v.shape[2:]
    t = rr._adjoint_axis_fp32(v.detach().cpu().numpy(), 3, hw[1], rr.taps(hw[1], W, align_corners, align_mode))
    t = rr._adjoint_axis_fp32(t, 2, hw[0], rr.taps(hw[0], H, align_corners, align_mode))
    return torch.from_numpy(np.ascontiguousarray(t)).to(v.device)


def bwd_torch(levels, gate, out, grad_out, align_corners=True, align_mode=1):
    """grad_levels (a list), grad_gate in the kernels' order, from the forward's out."""
    H, W = gate.shape[2:]
    w, S = weights(gate)
    gl, gg = [], []
    for l, x in enumerate(levels):
        pr = grad_out * (upsample_fp32(x, H, W, align_corners, align_mode) - out)
        t = pr[:, 0]
        for c in range(1, pr.shape[1]):
            t = t + pr[:, c]
        g = gate[:, l]
        gg.append(t / S * ((g > 0).to(g.dtype) - (g < 0).to(g.dtype)))
        gl.append(adjoint_fp32(w[:, l:l + 1] * grad_out, x.shape[2:], align_corners, align_mode))
    return gl, torch.stack(gg, dim=1)


# ---- a-priori bounds -------------------------------------------------------------------------------------------------------
def bound_fwd(levels, gate, align_corners=True, align_mode=1):
    return gamma(2 * len(levels) + 4) * compose([x.double().abs() for x in levels], gate.double(), align_corners, align_mode)


def bound_bwd(levels, gate, grad_out, align_corners=True, align_mode=1):
    """(bounds of the level gradients, bound of grad_gate)."""
    g, go = gate.double(), grad_out.double().abs()
    L, C = len(levels), grad_out.shape[1]
    H, W = g.shape[2:]
    a = g.abs()
    S = a.sum(dim=1, keepdim=True)
    w = a / S
    ups = [upsample(x.double().abs(), H, W, align_corners, align_mode) for x in levels]
    m = sum(w[:, l:l + 1] * u for l, u in enumerate(ups))
    gb = torch.cat([g[:, l:l + 1].sign().abs() * gamma(3 * L + C + 5) * (go * (u + m)).sum(dim=1, keepdim=True) / S
                    for l, u in enumerate(ups)], dim=1)
    lb = []
    for l, x in enumerate(levels):
        r = rr.max_range((1, *x.shape[2:]), (1, H, W), align_corners, align_mode)
        lb.append(gamma(L + 3 + 2 * (r + 1)) * adjoint(w[:, l:l + 1] * go, x.shape[2:], align_corners, align_mode))
    return lb, gb


def max_ratio(got, want, bound):
    """max |got - want| / bound: <= 1 when got is within the bound (an exact match counts 0)."""
    err = (torch.as_tensor(got).double().cpu() - torch.as_tensor(want).double().cpu()).abs()
    bound = torch.as_tensor(bound).double().cpu()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
