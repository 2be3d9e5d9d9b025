"""Two restatements of propagate2d_linear (SPN's three-way scans, DESIGN.md section 4.24) in stock torch ops, input makers
and the SPN head of INTEGRATION.md section 2i.

  composition   a port's form in fp64: each direction brought into the l2r frame by flips and transposes, one loop
                iteration per column, h = (1 - g0 - g1 - g2) x + g0 h[i-1] + g1 h[i] + g2 h[i+1], then the node-wise
                merge (first NaN, else first maximum) by an explicit index.  Autograd gives the gradients the op defines.
  kernel_order  the forward and an explicit backward in fp32, every subtraction, product and FMA in the order section
                4.24 and cspn2d_linear.cu state, so on any input it gives the library's bits.  It runs on CUDA tensors.

Every direction is the l2r scan of a flipped and / or transposed plane: r2l = flipW l2r flipW, t2b = T l2r T and
b2t = flipH T l2r T flipH, with tap j at lateral offset j - 1 in every frame."""
import torch
import torch.nn.functional as F

from dynamic_reference import fma

DIRECTIONS = ('l2r', 'r2l', 't2b', 'b2t')


def to_frame(t, d):
    """The (..., H, W) plane as the l2r scan of direction d sees it: rows are lanes, columns are steps in scan order."""
    if d == 'l2r':
        return t
    if d == 'r2l':
        return t.flip(-1)
    if d == 't2b':
        return t.transpose(-1, -2)
    return t.flip(-2).transpose(-1, -2)


def from_frame(t, d):
    if d == 'l2r':
        return t
    if d == 'r2l':
        return t.flip(-1)
    if d == 't2b':
        return t.transpose(-1, -2)
    return t.transpose(-1, -2).flip(-2)


def gate_blocks(gate, C, directions):
    """(B, 3*nd*Cg, H, W) -> per direction a (B, C, 3, H, W) view (a shared gate broadcast over the channels)."""
    B, G, H, W = gate.shape
    nd = len(directions)
    Cg = G // (3 * nd)
    g = gate.reshape(B, nd, Cg, 3, H, W)
    return [g[:, k].expand(B, C, 3, H, W) for k in range(nd)]


def merge_index(hs):
    """d* per node: the first direction that is NaN there, else the first attaining the maximum."""
    best, idx = hs[0], torch.zeros_like(hs[0], dtype=torch.long)
    for k in range(1, len(hs)):
        v = hs[k]
        take = ~torch.isnan(best) & (torch.isnan(v) | (v > best))
        best = torch.where(take, v, best)
        idx = torch.where(take, torch.full_like(idx, k), idx)
    return idx


def _lat(t, j):
    """t (..., L) read at lane i + j - 1, 0 outside."""
    p = F.pad(t, (1, 1))
    return p[..., j:j + t.shape[-1]]


def composition(feat, gate, directions=DIRECTIONS):
    """fp64 (the inputs' dtype) per-column loop under autograd."""
    directions = tuple(directions)
    B, C, H, W = feat.shape
    hs = []
    for d, g in zip(directions, gate_blocks(gate, C, directions)):
        x, gf = to_frame(feat, d), to_frame(g, d)
        h = torch.zeros_like(x[..., 0])
        cols = []
        for t in range(x.shape[-1]):
            g0, g1, g2 = gf[:, :, 0, :, t], gf[:, :, 1, :, t], gf[:, :, 2, :, t]
            h = (1 - g0 - g1 - g2) * x[..., t] + g0 * _lat(h, 0) + g1 * h + g2 * _lat(h, 2)
            cols.append(h)
        hs.append(from_frame(torch.stack(cols, -1), d))
    if len(hs) == 1:
        return hs[0]
    st = torch.stack(hs)
    return st.gather(0, merge_index(hs).unsqueeze(0)).squeeze(0)


def kernel_order(feat, gate, directions=DIRECTIONS, grad_out=None, need_feat=True, need_gate=True):
    """fp32 forward (out, planes) and, given grad_out, the backward (grad_feat, grad_gate) in the library's order."""
    directions = tuple(directions)
    B, C, H, W = feat.shape
    nd = len(directions)
    blocks = gate_blocks(gate, C, directions)
    hs = []
    for d, g in zip(directions, blocks):
        x, gf = to_frame(feat, d), to_frame(g, d)
        h = torch.zeros_like(x[..., 0])
        cols = []
        for t in range(x.shape[-1]):
            g0, g1, g2 = gf[:, :, 0, :, t], gf[:, :, 1, :, t], gf[:, :, 2, :, t]
            c = ((1 - g0) - g1) - g2
            h = fma(g2, _lat(h, 2), fma(g1, h, fma(g0, _lat(h, 0), c * x[..., t])))
            cols.append(h)
        hs.append(from_frame(torch.stack(cols, -1), d))
    idx = merge_index(hs) if nd > 1 else torch.zeros_like(feat, dtype=torch.long)
    out = torch.stack(hs).gather(0, idx.unsqueeze(0)).squeeze(0)
    if grad_out is None:
        return out, torch.stack(hs)
    gxs, ggs = [], []
    for k, (d, g) in enumerate(zip(directions, blocks)):
        x, gf, h = to_frame(feat, d), to_frame(g, d), to_frame(hs[k], d)
        go = to_frame(torch.where(idx == k, grad_out, torch.zeros_like(grad_out)), d)
        S = x.shape[-1]
        zero = torch.zeros_like(x[..., 0])
        dn, g0n, g1n, g2n = zero, zero, zero, zero
        gx = torch.empty_like(x)
        gg = torch.empty_like(gf)
        for t in range(S - 1, -1, -1):
            g0, g1, g2 = gf[:, :, 0, :, t], gf[:, :, 1, :, t], gf[:, :, 2, :, t]
            dl = fma(_lat(g2n, 0), _lat(dn, 0), fma(g1n, dn, fma(_lat(g0n, 2), _lat(dn, 2), go[..., t])))
            gx[..., t] = (((1 - g0) - g1) - g2) * dl
            hp = h[..., t - 1] if t > 0 else zero
            for j in range(3):
                gg[:, :, j, :, t] = dl * (_lat(hp, j) - x[..., t])
            dn, g0n, g1n, g2n = dl, g0, g1, g2
        gxs.append(from_frame(gx, d))
        ggs.append(from_frame(gg, d))
    grad_feat = gxs[0]
    for k in range(1, nd):
        grad_feat = grad_feat + gxs[k]
    Cg = gate.shape[1] // (3 * nd)
    per_block = []
    for k in range(nd):
        gk = ggs[k]                                           # (B, C, 3, H, W)
        if Cg == 1:
            s = gk[:, 0]
            for c in range(1, C):
                s = s + gk[:, c]
            per_block.append(s.unsqueeze(1))
        else:
            per_block.append(gk)
    grad_gate = torch.stack(per_block, 1).reshape(gate.shape)
    return out, torch.stack(hs), (grad_feat if need_feat else None), (grad_gate if need_gate else None)


# ---- inputs -------------------------------------------------------------------------------------------------------------
def random_inputs(B, C, H, W, directions=DIRECTIONS, per_channel=False, seed=0, device='cpu', dtype=torch.float32):
    """feat ~ N(0, 1); gates of random sign with sum_j |g_j| <= 1 at every node (SPN's stability condition)."""
    gen = torch.Generator().manual_seed(seed)
    nd = len(tuple(directions))
    Cg = C if per_channel else 1
    feat = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64)
    g = torch.randn(B, nd * Cg, 3, H, W, generator=gen, dtype=torch.float64)
    scale = torch.rand(B, nd * Cg, 1, H, W, generator=gen, dtype=torch.float64) * 0.8 + 0.2
    g = g / g.abs().sum(2, keepdim=True) * scale
    gate = g.reshape(B, 3 * nd * Cg, H, W)
    return feat.to(device, dtype), gate.to(device, dtype)


def dyadic_inputs(B, C, H, W, directions=DIRECTIONS, per_channel=False, seed=0, device='cpu'):
    """feat in k/4, |k| <= 8, gates in {-1/4, 0, 1/4, 1/2} with sum_j |g_j| <= 1.  A scan of S steps needs about 2S + 6
    significant bits, so for S <= 9 every operation is exact in fp32 and any order gives the fp64 composition's bits."""
    gen = torch.Generator().manual_seed(seed)
    nd = len(tuple(directions))
    Cg = C if per_channel else 1
    feat = torch.randint(-8, 9, (B, C, H, W), generator=gen).double() / 4
    g = torch.randint(-1, 3, (B, nd * Cg, 3, H, W), generator=gen).double() / 4
    over = g.abs().sum(2, keepdim=True) > 1
    g = torch.where(over, g / 2, g)
    gate = g.reshape(B, 3 * nd * Cg, H, W)
    return feat.float().to(device), gate.float().to(device)


def grads(fn, feat, gate, directions, grad_out, dtype=torch.float64):
    """(out, grad_feat, grad_gate) of fn under autograd, computed in dtype."""
    f = feat.detach().to(dtype).requires_grad_(True)
    g = gate.detach().to(dtype).requires_grad_(True)
    out = fn(f, g, directions)
    gf, gg = torch.autograd.grad(out, (f, g), grad_out.to(dtype))
    return out.detach(), gf, gg


def normwise(x, ref):
    """||x - ref|| / ||ref|| in fp64."""
    x, ref = x.detach().double(), ref.detach().double()
    return float((x - ref).norm() / ref.norm().clamp_min(1e-300))


# ---- the SPN head -------------------------------------------------------------------------------------------------------
def normalise_gates(gate, nd):
    """Per direction (and channel) divide the three gates by max(1, sum_j |g_j|): SPN's stability condition."""
    B, G, H, W = gate.shape
    g = gate.reshape(B, G // 3, 3, H, W)
    return (g / g.abs().sum(2, keepdim=True).clamp_min(1)).reshape(B, G, H, W)


def spn_head(guide, feat, weight, bias, directions=DIRECTIONS, use_op=False):
    """A guidance conv emits 3*nd (or 3*nd*C) gate channels, normalised per direction, then four-way propagation."""
    gate = normalise_gates(F.conv2d(guide, weight, bias, padding=1), len(tuple(directions)))
    if use_op:
        import cspn_b200
        return cspn_b200.propagate2d_linear(feat, gate, directions)
    return composition(feat, gate, directions)
