"""Restatements of atrous affinity pooling (cspn_b200.affinity_atrous_pool2d, csrc/affinity_atrous.cu; DESIGN.md section
4.19), the CSPN stereo network's atrous spatial pyramid pooling (ACSPP).  Level l, rate r = rates[l], is one CSPN step over
the 3 x 3 neighbourhood dilated by r, tap t at offset r * (dy_t, dx_t) = r * (t // 3 - 1, t % 3 - 1):

    a_t = |gate[:, 9l + t]|,  S = sum_t a_t,  w_t = a_t / S,  out[:, lC + c] = sum_t w_t * feat[:, c](p + r d_t)

with feat = +0.0 outside the image, that is F.unfold(feat, 3, dilation=r, padding=r).

- compose: the torch composition (F.unfold, abs, a sum, a broadcast divide, a product, a second sum), in the dtype and on
  the device of the inputs, differentiable.  In fp64, with its autograd, it is the reference.
- fwd_torch / bwd_torch: the kernels' order in the dtype and on the device of the inputs (in fp32 the kernels' bits; every
  eager torch op rounds on its own, on the CPU and the GPU alike), every sum started from its first term:
    S, out      taps in ascending t
    grad_gate   ((sum_c grad_out_l[c] * (f_c(p + r d_t) - out_l[c]), ascending c) / S) * sgn(gate), sgn in {-1, 0, 1}
    grad_feat   sum over l ascending, then t ascending, of w_{l,t}(q - r_l d_t) * grad_out_l[c](q - r_l d_t), over the
                terms whose source pixel lies in the image
- bound_fwd / bound_bwd: the a-priori bounds of the fp32 results against exact arithmetic, u = 2^-24,
  gamma_k = k u / (1 - k u), m_c = sum_t w_t |f_c(p + r d_t)| (finite inputs, no underflow):
    out         gamma_18 m_c
    grad_feat   gamma_{9L + 9} sum_{l,t} w_{l,t} |grad_out_l|   (at the source pixels)
    grad_gate   |sgn(gate)| (gamma_k sum_c |g_c| (|f_c(p + r d_t)| + m_c) + (1 + gamma_k) gamma_18 sum_c |g_c| m_c) / S,
                k = C + 10, g = grad_out_l
"""
import torch
import torch.nn.functional as F

U = 2.0 ** -24
OFFSETS = [(t // 3 - 1, t % 3 - 1) for t in range(9)]


def gamma(n):
    return n * U / (1 - n * U)


def compose(feat, gate, rates):
    """The torch composition of every level, (B, L*C, H, W), differentiable; in fp64 the reference."""
    B, C, H, W = feat.shape
    outs = []
    for l, r in enumerate(rates):
        cols = F.unfold(feat, 3, dilation=r, padding=r).view(B, C, 9, H, W)
        a = gate[:, 9 * l:9 * l + 9].abs()
        w = a / a.sum(dim=1, keepdim=True)
        outs.append((w[:, None] * cols).sum(dim=2))
    return torch.cat(outs, dim=1)


# ---- the kernels' order -----------------------------------------------------------------------------------------------------
def shifted(x, oy, ox):
    """y[..., i, j] = x[..., i + oy, j + ox], +0.0 where that lies outside the image."""
    H, W = x.shape[-2:]
    y = torch.zeros_like(x)
    if abs(oy) < H and abs(ox) < W:
        y[..., max(0, -oy):H - max(0, oy), max(0, -ox):W - max(0, ox)] = x[..., max(0, oy):H + min(0, oy), max(0, ox):W + min(0, ox)]
    return y


def inside(H, W, oy, ox, device):
    """The pixels p with p + (oy, ox) in the image."""
    return shifted(torch.ones(H, W, dtype=torch.bool, device=device), oy, ox)


def weights(gate, l):
    """(w, S) of level l: w (B, 9, H, W) = a / S, S (B, H, W), S summed in ascending t."""
    a = gate[:, 9 * l:9 * l + 9].abs()
    S = a[:, 0]
    for t in range(1, 9):
        S = S + a[:, t]
    return a / S[:, None], S


def fwd_torch(feat, gate, rates):
    """(B, L*C, H, W) in the kernels' order."""
    outs = []
    for l, r in enumerate(rates):
        w, _ = weights(gate, l)
        acc = None
        for t, (dy, dx) in enumerate(OFFSETS):
            term = w[:, t:t + 1] * shifted(feat, r * dy, r * dx)
            acc = term if acc is None else acc + term
        outs.append(acc)
    return torch.cat(outs, dim=1)


def bwd_torch(feat, gate, rates, out, grad_out):
    """grad_feat, grad_gate in the kernels' order, from the output and its gradient (B, L*C, H, W)."""
    B, C, H, W = feat.shape
    gf = torch.zeros_like(feat)
    have = torch.zeros(H, W, dtype=torch.bool, device=feat.device)
    gg = torch.empty_like(gate)
    for l, r in enumerate(rates):
        w, S = weights(gate, l)
        o, go = out[:, l * C:(l + 1) * C], grad_out[:, l * C:(l + 1) * C]
        for t, (dy, dx) in enumerate(OFFSETS):
            pr = go * (shifted(feat, r * dy, r * dx) - o)
            T = pr[:, 0]
            for c in range(1, C):
                T = T + pr[:, c]
            g = gate[:, 9 * l + t]
            sgn = (g > 0).to(g.dtype) - (g < 0).to(g.dtype)
            gg[:, 9 * l + t] = T / S * sgn
            # grad_feat at q takes w_t(q - r d_t) * go(q - r d_t) where q - r d_t lies in the image
            term = shifted(w[:, t:t + 1] * go, -r * dy, -r * dx)
            valid = inside(H, W, -r * dy, -r * dx, feat.device)
            gf = torch.where(valid & have, gf + term, torch.where(valid, term, gf))
            have = have | valid
    return gf, gg


# ---- a-priori bounds -------------------------------------------------------------------------------------------------------
def bound_fwd(feat, gate, rates):
    return gamma(18) * compose(feat.double().abs(), gate.double(), rates)


def bound_bwd(feat, gate, rates, grad_out):
    f, g, go = feat.double(), gate.double(), grad_out.double().abs()
    B, C, H, W = f.shape
    m = compose(f.abs(), g, rates)
    wg = torch.zeros_like(f)
    gb = torch.empty_like(g)
    k = C + 10
    for l, r in enumerate(rates):
        a = g[:, 9 * l:9 * l + 9].abs()
        S = a.sum(dim=1)
        ml, gl = m[:, l * C:(l + 1) * C], go[:, l * C:(l + 1) * C]
        for t, (dy, dx) in enumerate(OFFSETS):
            wg = wg + shifted((a[:, t] / S)[:, None] * gl, -r * dy, -r * dx)
            lhs = (gl * (shifted(f, r * dy, r * dx).abs() + ml)).sum(dim=1)
            rhs = (gl * ml).sum(dim=1)
            gb[:, 9 * l + t] = g[:, 9 * l + t].sign().abs() * (gamma(k) * lhs + (1 + gamma(k)) * gamma(18) * rhs) / S
    return gamma(9 * len(rates) + 9) * wg, gb


def max_ratio(got, want, bound):
    """max |got - want| / bound: <= 1 when got is within the bound (an exact match counts 0)."""
    err = (torch.as_tensor(got).double().cpu() - torch.as_tensor(want).double().cpu()).abs()
    bound = torch.as_tensor(bound).double().cpu()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
