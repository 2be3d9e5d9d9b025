"""Two references of the non-local 2D propagation, propagate2d_nonlocal (DESIGN.md section 4.21), in any dtype and on any
device, with autograd:

- `propagate` is an explicit floor / gather restatement in stock torch ops.  Its sampling is one autograd.Function whose
  backward states torchvision's deform_conv2d backward per sample: grad_h scattered to the corners whose weight is not 0,
  and the coordinate weight (the right-sided derivative, no window test) for the positions.  In fp32 its forward rounds
  every product and sum on its own in the kernels' order.
- `propagate_torchvision` is the composition NLSPN runs: one torchvision.ops.deform_conv2d per step with the affinities as
  the mask and a weight of ones (torchvision is imported when it is called).

Neither is used by the library."""
import torch


def taps(K):
    """The base offsets (i - R, j - R) of the T = K*K - 1 taps, (i, j) in raster order without the centre."""
    R = (K - 1) // 2
    return [(i - R, j - R) for i in range(K) for j in range(K) if (i, j) != (R, R)]


def _geometry(y, x, H, W):
    """The four corners tl, tr, bl, br of positions y, x (B, H, W): flat indices, validity, and the weights' factors."""
    zero = (y <= -1) | (y >= H) | (x <= -1) | (x >= W)
    nan = ~zero & (torch.isnan(y) | torch.isnan(x))
    y0, x0 = torch.floor(y), torch.floor(x)            # no huge or non-finite coordinate becomes an integer
    ly, lx = y - y0, x - x0
    hy, hx = 1 - ly, 1 - lx
    idx, valid = [], []
    for yy in (y0, y0 + 1):
        for xx in (x0, x0 + 1):
            ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            idx.append((torch.where(ok, yy, 0) * W + torch.where(ok, xx, 0)).long())
            valid.append(ok)
    return zero, nan, (ly, lx, hy, hx), idx, valid


def _corners(h, idx, valid):
    B, C = h.shape[:2]
    flat = h.reshape(B, C, -1)
    return [torch.where(ok[:, None], torch.gather(flat, 2, i.reshape(B, 1, -1).expand(B, C, -1)).view_as(h), h.new_zeros(()))
            for i, ok in zip(idx, valid)]


def _weights(ly, lx, hy, hx):
    return hy * hx, hy * lx, ly * hx, ly * lx


class _Sample(torch.autograd.Function):
    """S(h, y, x), torchvision's bilinear_interpolate, for h (B, C, H, W) and positions y, x (B, H, W)."""

    @staticmethod
    def forward(ctx, h, y, x):
        H, W = h.shape[2:]
        zero, nan, f, idx, valid = _geometry(y, x, H, W)
        v = _corners(h, idx, valid)
        w = _weights(*f)
        S = w[0][:, None] * v[0]
        for r in range(1, 4):
            S = S + w[r][:, None] * v[r]
        S = torch.where(zero[:, None], h.new_zeros(()), S)
        S = torch.where(nan[:, None], h.new_full((), float('nan')), S)
        ctx.save_for_backward(h, y, x)
        return S

    @staticmethod
    def backward(ctx, g):
        h, y, x = ctx.saved_tensors
        B, C, H, W = h.shape
        zero, nan, (ly, lx, hy, hx), idx, valid = _geometry(y, x, H, W)
        gh = gy = gx = None
        if ctx.needs_input_grad[0]:
            # deformable col2im: the corners in the image within distance 1, so one of weight 0 takes no part
            live = ~zero & ~nan
            use = (live & valid[0], live & valid[1] & (lx > 0), live & valid[2] & (ly > 0), live & valid[3] & (ly > 0) & (lx > 0))
            gh = h.new_zeros(B, C, H * W)
            for r, wr in enumerate(_weights(ly, lx, hy, hx)):
                term = torch.where(use[r][:, None], g * wr[:, None], h.new_zeros(()))
                gh.scatter_add_(2, idx[r].reshape(B, 1, -1).expand(B, C, -1), term.reshape(B, C, -1))
            gh = gh.view_as(h)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            v = _corners(h, idx, valid)
            # torchvision's get_coordinate_weight: no window test, the corners at floor and floor + 1 that lie in the image
            cy = lx[:, None] * (v[3] - v[1]) + hx[:, None] * (v[2] - v[0])
            cx = ly[:, None] * (v[3] - v[2]) + hy[:, None] * (v[1] - v[0])
            gy, gx = (g * cy).sum(1), (g * cx).sum(1)
        return gh, gy, gx


def replace(h, sparse):
    """h~ = (1 - m) h + m sparse with m = 1[sparse > 0], computed as written; m is not differentiated."""
    m = (sparse > 0).to(h.dtype).detach()
    return (1 - m) * h + m * sparse


def step(h, offset, affinity, K):
    """One step: a_c S(h, p) + sum_k a_k S(h, p + base_k + delta_k), the tap sum from its first term, then the centre."""
    B, C, H, W = h.shape
    py = torch.arange(H, device=h.device, dtype=h.dtype).view(1, H, 1).expand(B, H, W)
    px = torch.arange(W, device=h.device, dtype=h.dtype).view(1, 1, W).expand(B, H, W)
    acc, s = None, None
    for k, (di, dj) in enumerate(taps(K)):
        a = affinity[:, k]
        s = a if s is None else s + a
        term = a[:, None] * _Sample.apply(h, (py + di) + offset[:, 2 * k], (px + dj) + offset[:, 2 * k + 1])
        acc = term if acc is None else acc + term
    ac = 1 - s
    return ac[:, None] * _Sample.apply(h, py, px) + acc


def propagate(feat, offset, affinity, sparse_depth=None, K=3, N=18):
    """The explicit restatement: N steps, the replacement before each when sparse_depth is given, h_N not replaced."""
    h = feat
    for _ in range(N):
        h = step(h if sparse_depth is None else replace(h, sparse_depth), offset, affinity, K)
    return h


def full_offset_mask(offset, affinity, K):
    """deform_conv2d's offset (B, 2K^2, H, W) and mask (B, K^2, H, W): a zero offset and a_c = 1 - sum_k a_k at the centre."""
    R, T = (K - 1) // 2, K * K - 1
    c = R * K + R
    s = affinity[:, 0]
    for k in range(1, T):
        s = s + affinity[:, k]
    off = torch.cat([offset[:, :2 * c], torch.zeros_like(offset[:, :2]), offset[:, 2 * c:]], 1)
    mask = torch.cat([affinity[:, :c], (1 - s)[:, None], affinity[:, c:]], 1)
    return off, mask


def propagate_torchvision(feat, offset, affinity, sparse_depth=None, K=3, N=18):
    """NLSPN's route: one deform_conv2d per step, groups = C, one offset group, a weight of ones, padding R."""
    from torchvision.ops import deform_conv2d
    C = feat.shape[1]
    off, mask = full_offset_mask(offset, affinity, K)
    weight = torch.ones(C, 1, K, K, dtype=feat.dtype, device=feat.device)
    h = feat
    for _ in range(N):
        h = deform_conv2d(h if sparse_depth is None else replace(h, sparse_depth), off, weight, padding=(K - 1) // 2, mask=mask)
    return h


def grads(fn, feat, offset, affinity, sparse_depth, K, N, grad_out, dtype=None):
    """(out, grad_feat, grad_offset, grad_affinity, grad_sparse or None) of fn through autograd, in `dtype` (default: the
    inputs')."""
    ins = [t if t is None else t.detach().to(dtype or t.dtype).requires_grad_(True) for t in (feat, offset, affinity, sparse_depth)]
    out = fn(*ins, K=K, N=N)
    out.backward(grad_out.to(out.dtype))
    return (out.detach(),) + tuple(None if t is None else t.grad for t in ins)


def normwise(a, b):
    """||a - b|| / ||b|| over the finite entries of b (0 when b is 0 there)."""
    a, b = a.double(), b.double()
    fin = torch.isfinite(b)
    num, den = (a[fin] - b[fin]).norm(), b[fin].norm()
    return float(num / den) if den > 0 else float(num)


def make_inputs(B, C, H, W, K, scale=2.0, seed=0, sparse=False, device='cpu'):
    """Random inputs: offsets uniform in +-scale pixels, affinities normalised NLSPN's way (sum |a| clamped to >= 1)."""
    g = torch.Generator().manual_seed(seed)
    T = K * K - 1
    feat = torch.randn(B, C, H, W, generator=g)
    offset = (torch.rand(B, 2 * T, H, W, generator=g) * 2 - 1) * scale
    raw = torch.randn(B, T, H, W, generator=g)
    affinity = raw / raw.abs().sum(1, keepdim=True).clamp_min(1.0)
    sp = None
    if sparse:
        sp = torch.rand(B, C, H, W, generator=g) * 5
        sp = torch.where(torch.rand(B, C, H, W, generator=g) < 0.2, sp, torch.zeros(()))
    return tuple(None if t is None else t.to(device) for t in (feat, offset, affinity, sp))
