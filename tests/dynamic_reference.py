"""Two restatements of propagate2d_dynamic (DySPN's step, DESIGN.md section 4.23) in stock torch ops, and the DySPN head
of INTEGRATION.md section 2h composed from it.

  composition  a port's form: the per-step weights a_{t,ring(j)} * affinity_j, rho = 1 - their sum, F.unfold(d_t, K,
               padding=R) and an einsum with the weights, plus rho * d_0, then the replacement d <- m*s + (1 - m)*v;
  explicit     a zero-padded shift-and-add, one shifted copy of d_t per tap.

Autograd of either gives the gradients the op defines.  `dyspn_head` forms the affinity (a conv normalised by sum|.| at the
pixel), the attention (a conv and a sigmoid) and the confidence (a conv and a sigmoid on the valid samples) and
propagates, on this module's composition or on the library's op."""
import functools

import torch
import torch.nn.functional as F


@functools.lru_cache(maxsize=None)
def rings(K, device='cpu'):
    """ring(j) = max(|i - R|, |l - R|) of every tap j = i*K + l, as a LongTensor of K*K entries (cached per device, so
    that a CUDA graph can capture a call after a first eager one)."""
    R = (K - 1) // 2
    return torch.tensor([max(abs(j // K - R), abs(j % K - R)) for j in range(K * K)], device=device)


def steps(attention, K):
    return attention.shape[1] // ((K + 1) // 2)


def composition(affinity, attention, blur, sparse=None, conf=None, K=7):
    B, C, H, W = blur.shape
    R, KK, NR = (K - 1) // 2, K * K, (K + 1) // 2
    ring = rings(K, blur.device)
    d = blur
    for t in range(steps(attention, K)):
        w = attention[:, t * NR:(t + 1) * NR][:, ring] * affinity
        rho = 1 - w.sum(1, keepdim=True)
        cols = F.unfold(d.reshape(B * C, 1, H, W), K, padding=R).view(B, C, KK, H, W)
        v = rho * blur + torch.einsum('bckhw,bkhw->bchw', cols, w)
        d = conf * sparse + (1 - conf) * v if sparse is not None else v
    return d


def explicit(affinity, attention, blur, sparse=None, conf=None, K=7):
    B, C, H, W = blur.shape
    R, KK, NR = (K - 1) // 2, K * K, (K + 1) // 2
    ring = rings(K).tolist()
    d = blur
    for t in range(steps(attention, K)):
        a = attention[:, t * NR:(t + 1) * NR]
        ws = [a[:, ring[j]:ring[j] + 1] * affinity[:, j:j + 1] for j in range(KK)]
        S = ws[0]
        for j in range(1, KK):
            S = S + ws[j]
        v = (1 - S) * blur
        dp = F.pad(d, (R, R, R, R))
        for j in reversed(range(KK)):
            i, l = divmod(j, K)
            v = v + ws[j] * dp[:, :, i:i + H, l:l + W]
        d = conf * sparse + (1 - conf) * v if sparse is not None else v
    return d


def make_inputs(B, C, H, W, K, N, samples='soft', seed=0, device='cpu', scale=1.0):
    """affinity (B, K*K, H, W) normalised by sum|.| at the pixel, sigmoid attention (B, N*(K+1)//2, H, W), blur, and
    (sparse, conf) for samples 'soft' (sigmoid confidence on the valid pixels), 'hard' (0/1) or None."""
    g = torch.Generator().manual_seed(seed)
    affinity = torch.randn(B, K * K, H, W, generator=g)
    affinity = affinity / affinity.abs().sum(1, keepdim=True)
    attention = torch.sigmoid(torch.randn(B, N * ((K + 1) // 2), H, W, generator=g) * 2)
    blur = torch.randn(B, C, H, W, generator=g) * scale
    sparse = conf = None
    if samples:
        valid = (torch.rand(B, 1, H, W, generator=g) < 0.3).float()
        sparse = (torch.rand(B, 1, H, W, generator=g) * 4 + 0.5) * valid * scale
        conf = valid if samples == 'hard' else torch.sigmoid(torch.randn(B, 1, H, W, generator=g) * 2) * valid
    return [None if t is None else t.to(device) for t in (affinity, attention, blur, sparse, conf)]


def grads(fn, affinity, attention, blur, sparse, conf, K, grad_out, dtype=None):
    """(out, grad_affinity, grad_attention, grad_blur, grad_sparse, grad_conf), the last two None without samples; dtype
    casts the inputs."""
    ins = [None if t is None else t.detach().to(dtype or t.dtype).requires_grad_(True)
           for t in (affinity, attention, blur, sparse, conf)]
    out = fn(*ins, K)
    live = [t for t in ins if t is not None]
    gs = torch.autograd.grad(out, live, grad_out.to(out.dtype).to(out.device), allow_unused=True)
    it = iter(gs)
    return [out.detach()] + [None if t is None else next(it) for t in ins]


def normwise(x, ref):
    x, ref = x.double().cpu(), ref.double().cpu()
    return float((x - ref).norm() / ref.norm().clamp_min(1e-30))


# ---- the DySPN head (INTEGRATION.md section 2h) ----------------------------------------------------------------------------
def dyspn_head(feat, coarse, sparse, w_aff, w_att, w_conf, K=7, N=6, use_op=False):
    """feat (B, F, H, W) features; w_aff (K*K, F, 3, 3), w_att (N*(K+1)//2, F, 3, 3) and w_conf (1, F, 3, 3) the head's
    convolutions.  The affinity is the conv normalised by sum|.| at the pixel, the attention a sigmoid of its conv, and
    the confidence a sigmoid of its conv on the valid samples (sparse > 0); sparse=None propagates without replacement."""
    aff = F.conv2d(feat, w_aff, padding=1)
    aff = aff / aff.abs().sum(1, keepdim=True)
    att = torch.sigmoid(F.conv2d(feat, w_att, padding=1))
    conf = None
    if sparse is not None:
        conf = torch.sigmoid(F.conv2d(feat, w_conf, padding=1)) * (sparse > 0).to(sparse.dtype)
    if use_op:
        import cspn_b200
        return cspn_b200.propagate2d_dynamic(aff, att, coarse, sparse, conf, K)
    return composition(aff, att, coarse, sparse, conf, K)
