"""Restatements of the stereo cost volumes (cspn_b200.build_concat_volume / build_gwc_volume, csrc/cost_volume.cu; DESIGN.md
section 4.16).

    concat:  out[b, c, d, y, x] = left[b, c, y, x],  out[b, F + c, d, y, x] = right[b, c, y, x - d]      (x >= d, else +0.0)
    gwc:     out[b, g, d, y, x] = (sum_{c in group g} left[b, c, y, x] * right[b, c, y, x - d]) / n      (x >= d, else +0.0)

- concat_loop / gwc_loop: the PSMNet and GwcNet loops over the disparities (new_zeros, then slice writes), in the dtype
  and on the device of the inputs, differentiable.  In fp64 they are the reference.
- gwc_fwd_torch, concat_bwd_torch, gwc_bwd_torch: the kernels' order in the dtype and on the device of the inputs (in fp32
  the kernels' bits), and gwc_fwd_fp32, concat_bwd_fp32, gwc_bwd_fp32 the same on numpy fp32 arrays, every operation rounded on its own and
  every sum started from its first term:
    gwc forward      p_c = L_c * R_c summed in ascending c within the group, then / n
    concat backward  grad_left[c,y,x] = sum_{d=0}^{min(x,D-1)} g[c,d,y,x];  grad_right[c,y,x] = sum_{d=0}^{min(W-1-x,D-1)} g[F+c,d,y,x+d]
    gwc backward     t = g / n;  grad_left[c,y,x] = sum_d t[grp,d,y,x] * R[c,y,x-d];  grad_right[c,y,x] = sum_d t[grp,d,y,x+d] * L[c,y,x+d]
  (ascending d, the ranges of the concat backward).
- bound_gwc_fwd / bound_concat_bwd / bound_gwc_bwd: the a-priori bounds of the fp32 results against exact arithmetic,
  gamma_{n+1} sum|L R| / n, gamma_{D-1} sum|g| and gamma_{D+1} sum|g R| / n (and with L).
- plan / read_span: the kernels' tile plans and the columns a tile reads.
"""
import numpy as np
import torch

U = 2.0 ** -24
SMEM_SOFT = 110 * 1024
SMEM_HARD = 227 * 1024
CONCAT_CHUNK = 4
GWC_BWD_CHUNK = 8


def gamma(n):
    return n * U / (1 - n * U)


# ---- the loops ------------------------------------------------------------------------------------------------------------
def concat_loop(left, right, D):
    """PSMNet's build_concat_volume."""
    B, F, H, W = left.shape
    vol = left.new_zeros((B, 2 * F, D, H, W))
    for i in range(D):
        if i > 0:
            vol[:, :F, i, :, i:] = left[:, :, :, i:]
            vol[:, F:, i, :, i:] = right[:, :, :, :-i]
        else:
            vol[:, :F, i] = left
            vol[:, F:, i] = right
    return vol


def groupwise_correlation(fea1, fea2, G):
    B, F, H, W = fea1.shape
    return (fea1 * fea2).view(B, G, F // G, H, W).mean(dim=2)


def gwc_loop(left, right, D, G):
    """GwcNet's build_gwc_volume."""
    B, F, H, W = left.shape
    vol = left.new_zeros((B, G, D, H, W))
    for i in range(D):
        if i > 0:
            if i < W:
                vol[:, :, i, :, i:] = groupwise_correlation(left[:, :, :, i:], right[:, :, :, :-i], G)
        else:
            vol[:, :, i] = groupwise_correlation(left, right, G)
    return vol


# ---- the kernels' order ----------------------------------------------------------------------------------------------------
# Every torch op below rounds on its own (eager elementwise kernels fuse nothing), on the CPU and on the GPU alike.  A
# division by the Python number n could become a multiplication by 1/n, so n is divided as a tensor.
def _over(a, n):
    return a / torch.full_like(a, n)


def gwc_fwd_torch(left, right, D, G):
    """The group-wise correlation volume in the dtype and on the device of the inputs, in the kernels' order."""
    B, F, H, W = left.shape
    n = F // G
    out = left.new_zeros((B, G, D, H, W))
    for d in range(min(D, W)):
        Ls, Rs = left[..., d:], right[..., :W - d]
        acc = Ls[:, 0::n] * Rs[:, 0::n]                                  # channel c of every group: c, n + c, 2n + c, ...
        for c in range(1, n):
            acc = acc + Ls[:, c::n] * Rs[:, c::n]
        out[:, :, d, :, d:] = _over(acc, n)
    return out


def gwc_fwd_fp32(left, right, D, G):
    return gwc_fwd_torch(torch.from_numpy(np.asarray(left, np.float32)), torch.from_numpy(np.asarray(right, np.float32)),
                         D, G).numpy()


def concat_bwd_torch(g):
    """grad_left, grad_right of the concatenation volume from g (B, 2F, D, H, W), in g's dtype, in the kernels' order."""
    B, F2, D, H, W = g.shape
    F = F2 // 2
    gl, gr = g[:, :F, 0].clone(), g[:, F:, 0].clone()
    for d in range(1, min(D, W)):
        gl[..., d:] = gl[..., d:] + g[:, :F, d, :, d:]
        gr[..., :W - d] = gr[..., :W - d] + g[:, F:, d, :, d:]
    return gl, gr


def concat_bwd_fp32(g):
    gl, gr = concat_bwd_torch(torch.from_numpy(np.asarray(g, np.float32)))
    return gl.numpy(), gr.numpy()


def gwc_bwd_torch(left, right, g):
    """grad_left, grad_right of the group-wise correlation volume in the dtype of the inputs, in the kernels' order."""
    B, F, H, W = left.shape
    G, D = g.shape[1], g.shape[2]
    n = F // G
    t = _over(g, n).repeat_interleave(n, dim=1)                          # (B, F, D, H, W): t of channel c's group
    gl, gr = t[:, :, 0] * right, t[:, :, 0] * left
    for d in range(1, min(D, W)):
        gl[..., d:] = gl[..., d:] + t[:, :, d, :, d:] * right[..., :W - d]
        gr[..., :W - d] = gr[..., :W - d] + t[:, :, d, :, d:] * left[..., d:]
    return gl, gr


def gwc_bwd_fp32(left, right, g):
    with np.errstate(all='ignore'):
        gl, gr = gwc_bwd_torch(*(torch.from_numpy(np.asarray(a, np.float32)) for a in (left, right, g)))
    return gl.numpy(), gr.numpy()


# ---- a-priori bounds -------------------------------------------------------------------------------------------------------
def bound_gwc_fwd(left, right, D, G):
    n = left.shape[1] // G
    return gamma(n + 1) * gwc_loop(left.double().abs(), right.double().abs(), D, G)


def bound_concat_bwd(g):
    gl, gr = concat_bwd_torch(g.double().abs())
    b = gamma(max(g.shape[2] - 1, 0))
    return b * gl, b * gr


def bound_gwc_bwd(left, right, g):
    gl, gr = gwc_bwd_torch(left.double().abs(), right.double().abs(), g.double().abs())
    b = gamma(g.shape[2] + 1)
    return b * gl, b * gr


def max_ratio(got, want, bound):
    """max |got - want| / bound over the finite cells: <= 1 when got is within the bound (an exact match counts 0)."""
    err = (torch.as_tensor(got).double().cpu() - torch.as_tensor(want).double().cpu()).abs()
    bound = torch.as_tensor(bound).double().cpu()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


# ---- the tile plans of csrc/cost_volume.cu ----------------------------------------------------------------------------------
def smem_of(kind, tx, rp, D, n):
    if kind == 'concat_fwd':
        return CONCAT_CHUNK * (tx + rp) * 4
    if kind == 'gwc_fwd':
        return n * (tx + rp) * 4
    return (2 * D * tx + 2 * GWC_BWD_CHUNK * rp) * 4


def plan(kind, W, D, n=0):
    """(TX, RP, smem): TX the first power of two >= W up to 128, halved until the tile fits two CTAs per SM (a 1-column
    tile up to 227 KB); RP = min(TX + D - 1, W) the pitch of a staged shifted row.  smem 0: no tile fits."""
    tx = 1
    while tx < 128 and tx < W:
        tx *= 2
    while True:
        rp = min(tx + D - 1, W)
        s = smem_of(kind, tx, rp, D, n)
        if s <= SMEM_SOFT or (tx == 1 and s <= SMEM_HARD):
            return tx, rp, s
        if tx == 1:
            return 1, rp, 0
        tx //= 2


def staged(W, D, tx, x0):
    """The columns the kernels stage for the tile at x0: right rows [r_lo, x0 + nx) and, in the gwc backward, left rows
    [x0, x0 + nl)."""
    nx = min(tx, W - x0)
    r_lo = max(x0 - D + 1, 0)
    return (r_lo, x0 + nx), (x0, min(x0 + nx + D - 1, W))


def read_span(W, D, tx, x0):
    """The columns of right (x - d) and of left (x + d) that the tile at x0 reads, from the semantics: [lo, hi) each."""
    xs = range(x0, min(x0 + tx, W))
    rd = [x - d for x in xs for d in range(min(x, D - 1) + 1)]
    ld = [x + d for x in xs for d in range(min(W - 1 - x, D - 1) + 1)]
    return (min(rd), max(rd) + 1), (min(ld), max(ld) + 1)
