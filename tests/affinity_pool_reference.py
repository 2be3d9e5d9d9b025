"""Restatements of affinity pooling (cspn_b200.affinity_pool2d, csrc/affinity_pool.cu; DESIGN.md section 4.17), the CSPN
stereo network's convolutional spatial pyramid pooling.  Level l, window size p = ks[l], pools the windows of
F.avg_pool2d(x, p):

    a = |gate[:, l]|,  S = sum_window a,  w = a / S,  out_l[b, c, i, j] = sum_window w * feat[b, c]

- compose: the torch composition on reshaped windows (abs, a windowed sum, a broadcast divide, a product, a second
  windowed sum), in the dtype and on the device of the inputs, differentiable.  In fp64, with its autograd, it is the
  reference.
- fwd_torch / bwd_torch: the kernels' order in the dtype and on the device of the inputs (in fp32 the kernels' bits; every
  eager torch op rounds on its own, on the CPU and the GPU alike), every sum started from its first term:
    S, out      each window row summed in ascending x, then the row sums in ascending y
    grad_feat   sum over the levels that cover q, ascending l, of w_l(q) * grad_out_l[c, cell]; +0.0 where none covers q
    grad_gate   ((sum_c grad_out_l[c] * (feat[c, q] - out_l[c]), ascending c) / S) * sgn(gate), sgn in {-1, 0, 1};
                +0.0 outside level l's windows
- bound_fwd / bound_bwd: the a-priori bounds of the fp32 results against exact arithmetic, u = 2^-24,
  gamma_k = k u / (1 - k u), m_c = sum_window w |feat_c| (finite inputs, no underflow):
    out_l       gamma_{4p-2} m_c
    grad_feat   gamma_{2 max(p) + L - 1} sum_l w_l |grad_out_l|
    grad_gate   |sgn(gate)| (gamma_k sum_c |g_c| (|feat_c(q)| + m_c) + (1 + gamma_k) gamma_{4p-2} sum_c |g_c| m_c) / S,
                k = C + 2p, g = grad_out_l
- pack / unpack: the C ABI's level-major buffer.
"""
import torch

U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


def windows(t, p):
    """(B, K, H, W) -> (B, K, Hl, p, Wl, p), the floor-mode windows of avg_pool2d(t, p)."""
    B, K, H, W = t.shape
    Hl, Wl = H // p, W // p
    return t[:, :, :Hl * p, :Wl * p].reshape(B, K, Hl, p, Wl, p)


def unwindow(t, H, W):
    """(B, K, Hl, p, Wl, p) -> (B, K, H, W) with +0.0 where no window lies."""
    B, K, Hl, p, Wl, _ = t.shape
    full = t.new_zeros((B, K, H, W))
    full[:, :, :Hl * p, :Wl * p] = t.reshape(B, K, Hl * p, Wl * p)
    return full


def expand(t):
    """(B, K, Hl, Wl) -> (B, K, Hl, 1, Wl, 1), broadcast over the windows."""
    return t[:, :, :, None, :, None]


def compose(feat, gate, ks):
    """The torch composition of every level, differentiable; in fp64 the reference."""
    outs = []
    for l, p in enumerate(ks):
        a = windows(gate[:, l:l + 1], p).abs()
        S = a.sum(dim=(3, 5), keepdim=True)
        outs.append((a / S * windows(feat, p)).sum(dim=(3, 5)))
    return tuple(outs)


# ---- the kernels' order -----------------------------------------------------------------------------------------------------
def ordered_sum(t):
    """(B, K, Hl, p, Wl, p) -> (B, K, Hl, Wl): each window row in ascending x, then the row sums in ascending y."""
    p = t.shape[3]
    r = t[..., 0]
    for x in range(1, p):
        r = r + t[..., x]
    s = r[:, :, :, 0]
    for y in range(1, p):
        s = s + r[:, :, :, y]
    return s


def weights(gate, l, p):
    """(w, S) of level l: w (B, 1, Hl, p, Wl, p) = a / S, S (B, 1, Hl, Wl)."""
    a = windows(gate[:, l:l + 1], p).abs()
    S = ordered_sum(a)
    return a / expand(S), S


def fwd_torch(feat, gate, ks):
    """The L levels in the kernels' order."""
    return tuple(ordered_sum(weights(gate, l, p)[0] * windows(feat, p)) for l, p in enumerate(ks))


def bwd_torch(feat, gate, ks, outs, grads):
    """grad_feat, grad_gate in the kernels' order, from the levels' outputs and gradients."""
    B, C, H, W = feat.shape
    gf = feat.new_zeros(feat.shape)
    have = torch.zeros(H, W, dtype=torch.bool, device=feat.device)
    gg = []
    for l, p in enumerate(ks):
        w, S = weights(gate, l, p)
        go = expand(grads[l])
        term = unwindow(w * go, H, W)
        cov = torch.zeros(H, W, dtype=torch.bool, device=feat.device)
        cov[:(H // p) * p, :(W // p) * p] = True
        gf = torch.where(cov & have, gf + term, torch.where(cov, term, gf))
        have = have | cov
        pr = go * (windows(feat, p) - expand(outs[l]))
        t = pr[:, 0]
        for c in range(1, C):
            t = t + pr[:, c]
        g = windows(gate[:, l:l + 1], p)[:, 0]
        sgn = (g > 0).to(g.dtype) - (g < 0).to(g.dtype)
        gg.append(unwindow((t / S[:, 0, :, None, :, None] * sgn)[:, None], H, W))
    return gf, torch.cat(gg, dim=1)


# ---- a-priori bounds -------------------------------------------------------------------------------------------------------
def bound_fwd(feat, gate, ks):
    m = compose(feat.double().abs(), gate.double(), ks)
    return tuple(gamma(4 * p - 2) * t for t, p in zip(m, ks))


def bound_bwd(feat, gate, ks, grads):
    f, g = feat.double(), gate.double()
    B, C, H, W = f.shape
    wg = f.new_zeros(f.shape)
    gb = []
    m = compose(f.abs(), g, ks)
    for l, p in enumerate(ks):
        a = windows(g[:, l:l + 1], p).abs()
        S = a.sum(dim=(3, 5), keepdim=True)
        ga = expand(grads[l].double().abs())
        wg = wg + unwindow(a / S * ga, H, W)
        k = C + 2 * p
        lhs = (ga * (windows(f, p).abs() + expand(m[l]))).sum(dim=1, keepdim=True)
        rhs = (ga * expand(m[l])).sum(dim=1, keepdim=True)
        gb.append(unwindow(windows(g[:, l:l + 1], p).sign().abs() * (gamma(k) * lhs + (1 + gamma(k)) * gamma(4 * p - 2) * rhs) / S,
                           H, W))
    return gamma(2 * max(ks) + len(ks) - 1) * wg, torch.cat(gb, dim=1)


def max_ratio(got, want, bound):
    """max |got - want| / bound: <= 1 when got is within the bound (an exact match counts 0)."""
    err = (torch.as_tensor(got).double().cpu() - torch.as_tensor(want).double().cpu()).abs()
    bound = torch.as_tensor(bound).double().cpu()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


# ---- the C ABI's packed buffer ------------------------------------------------------------------------------------------------
def pack(levels):
    return torch.cat([t.reshape(-1) for t in levels])


def unpack(flat, B, C, H, W, ks):
    shapes = [(B, C, H // p, W // p) for p in ks]
    sizes = [B * C * (H // p) * (W // p) for p in ks]
    return tuple(v.view(s) for v, s in zip(flat.split(sizes), shapes))
