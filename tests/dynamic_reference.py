"""Three restatements of propagate2d_dynamic (DySPN's step, DESIGN.md section 4.23) in stock torch ops, and the DySPN
head of INTEGRATION.md section 2h composed from it.

  composition   a port's form: the per-step weights a_{t,ring(j)} * affinity_j, rho = 1 - their sum, F.unfold(d_t, K,
                padding=R) and an einsum with the weights, plus rho * d_0, then the replacement d <- m*s + (1 - m)*v;
  explicit      a zero-padded shift-and-add, one shifted copy of d_t per tap;
  kernel_order  the forward and an explicit backward in fp32, every product, sum and FMA in the order section 4.23 and
                cspn2d_dynamic.cu state, so on any input it gives the library's bits.

Autograd of the first two gives the gradients the op defines.  `dyspn_head` forms the affinity (a conv normalised by
sum|.| at the pixel), the attention (a conv and a sigmoid) and the confidence (a conv and a sigmoid on the valid samples)
and propagates, on this module's composition or on the library's op."""
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


# ---- the kernels' order -----------------------------------------------------------------------------------------------------
def fma(a, b, c):
    """fp32 fmaf(a, b, c), rounded once, on fp32 tensors (broadcast).  The product is exact in fp64 and TwoSum gives the
    sum's exact error e; an inexact sum is replaced by its round-to-odd value (truncated toward zero, lowest bit set) so
    that the cast to fp32 rounds correctly (53 >= 24 + 2 bits).  Rounding a*b + c in fp64 and then to fp32 instead is a
    double rounding, one ulp off when the fp64 sum lands on an fp32 midpoint.  Subnormals are kept; inf and NaN operands
    follow IEEE through the fp64 arithmetic."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    inexact = (e != 0) & torch.isfinite(s)
    over = inexact & ((e < 0) != (s < 0))              # |s| > |p + c|: truncation steps one ulp toward zero
    bits = (s.view(torch.int64) - over.long()) | inexact.long()
    return bits.view(torch.float64).float()


def _shift(x, dy, dx):
    """(x(y + dy, x + dx), inside): a +0.0 outside the image, and where the read is inside it."""
    H, W = x.shape[-2:]
    pad = max(abs(dy), abs(dx))
    xp = F.pad(x, (pad, pad, pad, pad))
    one = F.pad(torch.ones(1, 1, H, W, dtype=torch.bool, device=x.device), (pad, pad, pad, pad))
    win = (slice(pad + dy, pad + dy + H), slice(pad + dx, pad + dx + W))
    return xp[..., win[0], win[1]], one[..., win[0], win[1]]


def _blend(m, s, u):
    return m * s + (1 - m) * u


def kernel_order(affinity, attention, blur, sparse, conf, K, grad_out):
    """(out, grad_affinity, grad_attention, grad_blur, grad_sparse, grad_conf) as `grads` returns them, the last two None
    without samples, in fp32 with the kernels' operation order (section 4.23, the head of cspn2d_dynamic.cu).  Every
    product and sum is one fp32 torch op, every FMA `fma`; the signs of zeros follow the kernels: accumulators start from
    +0.0, a tap outside the image reads +0.0 (G1 adds mu * 0 there), the adjoint skips sources outside the image.  Runs
    on the inputs' device."""
    affinity, attention, blur, grad_out = (t.detach().float() for t in (affinity, attention, blur, grad_out))
    samp = sparse is not None
    if samp:
        sparse, conf = sparse.detach().float(), conf.detach().float()
    B, C, H, W = blur.shape
    R, KK, NR = (K - 1) // 2, K * K, (K + 1) // 2
    N = steps(attention, K)
    ring = rings(K).tolist()
    offs = [(j // K - R, j % K - R) for j in range(KK)]
    zero = torch.zeros((), device=blur.device)

    def att(t, r):
        return attention[:, t * NR + r:t * NR + r + 1]

    def weights(t):                                    # w_{t,j}, (B, 1, H, W) each
        return [att(t, ring[j]) * affinity[:, j:j + 1] for j in range(KK)]

    def rho(w):
        S = w[0]
        for j in range(1, KK):
            S = S + w[j]
        return 1 - S

    # forward: d_0 .. d_N and the pre-replacement v_0 .. v_{N-1}
    d, v_pre, ws = [blur], [], []
    for t in range(N):
        w = weights(t)
        ws.append(w)
        v = rho(w) * blur
        for j in reversed(range(KK)):
            v = fma(w[j], _shift(d[t], *offs[j])[0], v)
        v_pre.append(v)
        d.append(_blend(conf, sparse, v) if samp else v)

    # adjoint: lambda_N = grad_out, lambda_t(q) = sum over j descending of w_{t,j}(q - o_j) mu_t(q - o_j), inside only
    one_minus_m = 1 - conf if samp else None

    def mu(lam):
        return one_minus_m * lam if samp else lam

    lams = [None] * N + [grad_out]
    for t in reversed(range(N)):
        m_t = mu(lams[t + 1])
        acc = torch.zeros_like(blur)
        for j in reversed(range(KK)):
            dy, dx = offs[j]
            wq, inside = _shift(ws[t][j], -dy, -dx)
            mq, _ = _shift(m_t, -dy, -dx)
            acc = torch.where(inside, fma(wq, mq, acc), acc)
        lams[t] = acc

    g_aff = zero.expand(B, KK, H, W)
    g_att = torch.empty(attention.shape, device=blur.device)
    g_blur = lams[0]
    for t in range(N):
        m_t = mu(lams[t + 1])
        g_blur = fma(rho(ws[t]), m_t, g_blur)
        G0 = zero.expand(B, 1, H, W)
        for c in range(C):
            G0 = fma(m_t[:, c:c + 1], blur[:, c:c + 1], G0)
        taps = torch.stack([_shift(d[t], *o)[0] for o in offs], 2)          # (B, C, KK, H, W), +0.0 outside
        G1 = zero.expand(B, KK, H, W)
        for c in range(C):
            G1 = fma(m_t[:, c:c + 1], taps[:, c], G1)
        g = G1 - G0                                                        # g_{t,j} in channel j
        a_t = attention[:, t * NR:(t + 1) * NR][:, ring]
        g_aff = fma(a_t, g, g_aff)
        gr = [zero.expand(B, 1, H, W)] * NR
        for j in range(KK):
            gr[ring[j]] = fma(affinity[:, j:j + 1], g[:, j:j + 1], gr[ring[j]])
        g_att[:, t * NR:(t + 1) * NR] = torch.cat(gr, 1)
    g_sparse = g_conf = None
    if samp:
        gm = gs = zero.expand(B, 1, H, W)
        for t in range(N):
            A = Bs = zero.expand(B, 1, H, W)
            for c in range(C):
                l0 = lams[t + 1][:, c:c + 1]
                A = A + l0
                Bs = fma(l0, v_pre[t][:, c:c + 1], Bs)
            gm = gm + (A * sparse - Bs)
            gs = gs + conf * A
        g_sparse, g_conf = gs.contiguous(), gm.contiguous()
    return [d[N], g_aff.contiguous(), g_att, g_blur.contiguous(), g_sparse, g_conf]


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


def dyadic_inputs(B, C, H, W, K, N, samples, seed):
    """Affinities in {0, +-1/4, +-1/2}, attention in {0, 1/2, 1}, integer blur, samples and grad_out, confidences in {0,
    1/2, 1} (hard: 1 on the samples): every intermediate of the dyadic bit-for-bit cases (N = 3 at K = 3, N = 2 at K = 5
    and 7) is exact in fp32, so any order of operations gives fp64's values.  ([affinity, attention, blur, sparse,
    conf], grad_out) on the CPU."""
    g = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, 0.0, 0.0, 0.25, -0.25, 0.5, -0.5])
    affinity = vals[torch.randint(0, 7, (B, K * K, H, W), generator=g)]
    attention = torch.tensor([0.0, 0.5, 1.0, 1.0])[torch.randint(0, 4, (B, N * ((K + 1) // 2), H, W), generator=g)]
    blur = torch.randint(-4, 5, (B, C, H, W), generator=g).float()
    sparse = conf = None
    if samples:
        sparse = torch.randint(0, 5, (B, 1, H, W), generator=g).float()
        conf = torch.tensor([0.0, 0.5, 1.0])[torch.randint(0, 3, (B, 1, H, W), generator=g)]
        if samples == 'hard':
            conf = (sparse > 0).float()
    go = torch.randint(-2, 3, (B, C, H, W), generator=g).float()
    return [affinity, attention, blur, sparse, conf], go


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
