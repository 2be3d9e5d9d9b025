"""Two restatements of propagate2d_dilated (PENet's DA-CSPN++ step, DESIGN.md section 4.22) in stock torch ops, and
PENet's refinement composed from it (INTEGRATION.md section 2g).

  composition  PENet's form: F.unfold(d_t, K, dilation=d, padding=d*R) with the centre row overwritten by d_0, an einsum
               with the weights, then the replacement d <- m*s + (1 - m)*u;
  explicit     a zero-padded shift-and-add, one shifted copy of d_t per tap.

Autograd of either gives the gradients the op defines.  `penet_refine` runs both refinement stages (d = 2 on nearest
upsampled half-resolution guides, then d = 1) with K = 3, 5 and 7 mixed by a softmax, on this module's composition or on
the library's op."""
import torch
import torch.nn.functional as F


def composition(kernel, blur, sparse=None, conf=None, K=3, dil=1, N=6):
    B, C, H, W = blur.shape
    R, KK = (K - 1) // 2, K * K
    c = KK // 2
    d = blur
    for _ in range(N):
        cols = F.unfold(d.reshape(B * C, 1, H, W), K, dilation=dil, padding=dil * R).view(B, C, KK, H, W)
        cols = torch.cat([cols[:, :, :c], blur.unsqueeze(2), cols[:, :, c + 1:]], 2)
        u = torch.einsum('bckhw,bkhw->bchw', cols, kernel)
        d = conf * sparse + (1 - conf) * u if sparse is not None else u
    return d


def explicit(kernel, blur, sparse=None, conf=None, K=3, dil=1, N=6):
    B, C, H, W = blur.shape
    R, KK = (K - 1) // 2, K * K
    c, h = KK // 2, dil * R
    d = blur
    for _ in range(N):
        dp = F.pad(d, (h, h, h, h))
        u = kernel[:, c:c + 1] * blur
        for j in range(KK):
            if j == c:
                continue
            i, l = divmod(j, K)
            y0, x0 = h + dil * (i - R), h + dil * (l - R)
            u = u + kernel[:, j:j + 1] * dp[:, :, y0:y0 + H, x0:x0 + W]
        d = conf * sparse + (1 - conf) * u if sparse is not None else u
    return d


def make_inputs(B, C, H, W, K, samples='soft', seed=0, device='cpu', scale=1.0):
    """kernel (B, K*K, H, W) of normalised-looking weights (|w| summing to about 1), blur, and (sparse, conf) for samples
    'soft' (sigmoid confidence on the valid pixels), 'hard' (0/1) or None."""
    g = torch.Generator().manual_seed(seed)
    kernel = torch.randn(B, K * K, H, W, generator=g)
    kernel = kernel / kernel.abs().sum(1, keepdim=True)
    blur = torch.randn(B, C, H, W, generator=g) * scale
    sparse = conf = None
    if samples:
        valid = (torch.rand(B, 1, H, W, generator=g) < 0.3).float()
        sparse = (torch.rand(B, 1, H, W, generator=g) * 4 + 0.5) * valid * scale
        conf = valid if samples == 'hard' else torch.sigmoid(torch.randn(B, 1, H, W, generator=g) * 2) * valid
    return [None if t is None else t.to(device) for t in (kernel, blur, sparse, conf)]


def grads(fn, kernel, blur, sparse, conf, K, dil, N, grad_out, dtype=None):
    """(out, grad_kernel, grad_blur, grad_sparse, grad_conf), the last two None without samples; dtype casts the inputs."""
    ins = [None if t is None else t.detach().to(dtype or t.dtype).requires_grad_(True) for t in (kernel, blur, sparse, conf)]
    out = fn(*ins, K, dil, N)
    live = [t for t in ins if t is not None]
    gs = torch.autograd.grad(out, live, grad_out.to(out.dtype).to(out.device), allow_unused=True)
    it = iter(gs)
    return [out.detach()] + [None if t is None else next(it) for t in ins]


def normwise(x, ref):
    x, ref = x.double().cpu(), ref.double().cpu()
    return float((x - ref).norm() / ref.norm().clamp_min(1e-30))


# ---- PENet's refinement (INTEGRATION.md section 2g) ------------------------------------------------------------------------
def normalise_guide(g):
    """(B, K*K - 1, h, w) raw guide -> (B, K*K, h, w) weights at the guide's own location: g / sum|g|, centre 1 - sum."""
    KK = g.shape[1] + 1
    c = KK // 2
    gh = g / g.abs().sum(1, keepdim=True)
    mid = 1 - gh.sum(1, keepdim=True)
    return torch.cat([gh[:, :c], mid, gh[:, c:]], 1)


def move_weights(w, K):
    """PENet's kernel_trans: the weight for tap j at p is w_{K*K-1-j}(p + o_j), o_j = (i - R, l - R) at w's resolution,
    zero outside; the centre stays at p."""
    B, KK, h, wd = w.shape
    R = (K - 1) // 2
    wp = F.pad(w, (R, R, R, R))
    out = []
    for j in range(KK):
        i, l = divmod(j, K)
        out.append(wp[:, KK - 1 - j:KK - j, i:i + h, l:l + wd])
    return torch.cat(out, 1)


def penet_refine(coarse, sparse, guides_half, guides_full, conf_logit, mix_half, mix_full, N=6, use_op=False):
    """Two stages of DA-CSPN++: d = 2 with the half-resolution guides (moved at half resolution, then nearest-upsampled x2),
    then d = 1 with the full-resolution guides.  guides_*: {K: (B, K*K - 1, ., .)}; mix_*: (B, 3, H, W) logits of the
    softmax over K = 3, 5, 7; the confidence is sigmoid(conf_logit) * 1[sparse > 0]."""
    conf = torch.sigmoid(conf_logit) * (sparse > 0).to(sparse.dtype)
    d = coarse
    for dil, guides, mix in ((2, guides_half, mix_half), (1, guides_full, mix_full)):
        wts = torch.softmax(mix, 1)
        outs = []
        for K in (3, 5, 7):
            w = move_weights(normalise_guide(guides[K]), K)
            if dil == 2:
                w = F.interpolate(w, scale_factor=2, mode='nearest')
            if use_op:
                import cspn_b200
                outs.append(cspn_b200.propagate2d_dilated(w, d, sparse, conf, K, dil, N))
            else:
                outs.append(composition(w, d, sparse, conf, K, dil, N))
        d = sum(wts[:, k:k + 1] * outs[k] for k in range(3))
    return d
