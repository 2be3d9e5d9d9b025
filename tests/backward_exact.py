"""Inputs on which the K x K (2D) and K x K x K (3D) propagation and both of its gradients are exact in fp32, the fp64
references they are checked against, and the case matrix of the exact GPU tests.  Shared by
tests/test_backward_exact_cpu.py (which checks the premises without a GPU) and tests/test_backward_exact_gpu.py.

Dyadic inputs.  With random gates a gradient is only checked to a tolerance, and an error confined to the pixels next to a
CTA tile edge can hide under it.  So the exact cases build inputs on which every intermediate value is a short dyadic
rational, and then any correct fp32 implementation, in any summation order, returns the bits of the fp64 reference:
  gathered norms  at each site p, m in {1, 2, 4} distinct taps k whose source p + off_k lies inside get g_k(p + off_k) = +-1;
                  the rest of the guidance is 0.  Each guidance value is read by exactly one site, so S = sum |a| = m and
                  w_k = +-1/m exactly;
  'paddle'        the same with the values at the site itself, g_k(p): any tap may be hot, also one that reads the padding;
  blur / feat and grad_out   integers in [-4, 4];   sparse   values in {-3, 0, 3}, so m = sign(sparse) takes all three values.
A step multiplies the denominators by at most 4, and the guidance gradient divides by S once more than the forward: every
value of N steps is a multiple of 4^-(N+1).  `check_exact` asserts that of a reference, and that it is far inside 24 bits.
"""
import itertools

import torch
import torch.nn.functional as F

from oracle.cspn_numpy_k import offsets_2d
from oracle.cspn_torch_port_3d_k import cspn3d_torch_k, offsets_3d


def shift(a, off, r):
    """b[..., p] = a[..., p + off] over the last len(off) dims, zero outside; every |off_i| <= r (also when r exceeds the
    extent: such a copy is all padding)."""
    nd = len(off)
    p = F.pad(a, (r,) * (2 * nd))
    lead = [slice(None)] * (a.dim() - nd)
    return p[tuple(lead + [slice(r + o, r + o + n) for o, n in zip(off, a.shape[-nd:])])]


def offsets(K, nd):
    return offsets_2d(K) if nd == 2 else offsets_3d(K)


def inside(shape, offs):
    """(taps, *shape) bool: the source p + off_k of site p lies inside the image / volume."""
    grids = torch.meshgrid(*[torch.arange(n) for n in shape], indexing='ij')
    return torch.stack([torch.stack([(g + o >= 0) & (g + o < n) for g, o, n in zip(grids, off, shape)]).all(0)
                        for off in offs])


# ---- the fp64 2D reference --------------------------------------------------------------------------------------------
def cspn2d_shift_ref(guidance, blur, sparse=None, prop_time=24, K=5, norm_type=None):
    """The K x K propagation restated on the unpadded grid with shifts, as oracle/cspn_torch_port_3d_k.py is.  The torch
    port (cspn2d_torch_k) normalises on the padded grid, where a margin position whose taps are all zero gives 0/0: the crop
    hides it in the forward, but autograd carries 0 * NaN into both gradients.  This form has no such positions, so it is the
    autograd reference wherever the guidance has zeros."""
    nt, r = K * K - 1, (K - 1) // 2
    norm_type = norm_type or f'{nt}sum'
    assert K in (3, 5, 7) and norm_type in (f'{nt}sum', f'{nt}sum_abs')
    offs = offsets_2d(K)
    g = guidance[:, :nt]
    if norm_type.endswith('_abs'):
        g = g.abs()
    a = torch.stack([shift(g[:, k], o, r) for k, o in enumerate(offs)], 1)
    w = a / a.abs().sum(1, keepdim=True)
    s = w.sum(1, keepdim=True)
    m = None if sparse is None else sparse.sign()
    result = blur
    for _ in range(prop_time):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + w[:, k:k + 1] * shift(result, o, r)
        result = (1.0 - s) * blur + acc
        if m is not None:
            result = (1 - m) * result + m * blur
    return result


def cspn3d_ref(guidance, feat, prop_time, K, norm_type):
    """cspn3d_torch_k, with per-channel gates (B, nt*C, ...) run as the B*C single-channel volumes they are."""
    nt = K ** 3 - 1
    B, C = feat.shape[:2]
    if guidance.shape[1] == nt * C and C > 1:
        out = cspn3d_torch_k(guidance.reshape(B * C, nt, *feat.shape[2:]), feat.reshape(B * C, 1, *feat.shape[2:]),
                             prop_time, K, norm_type)
        return out.reshape(feat.shape)
    return cspn3d_torch_k(guidance, feat, prop_time, K, norm_type)


# ---- dyadic inputs ----------------------------------------------------------------------------------------------------
def hot_taps(gen, n, valid, ms=(1, 2, 4)):
    """(n, taps, *S) bool: at each site m in `ms` (powers of two up to 4) distinct taps among the `valid` ones
    ((taps, *S) bool), m capped at the largest power of two the valid taps allow.  Random keys, -inf on invalid taps, the
    top m win."""
    taps, shape = valid.shape[0], valid.shape[1:]
    nvalid = valid.sum(0)
    assert nvalid.min() >= 1, 'a site without a valid tap'
    cap = torch.where(nvalid >= 4, 4, torch.where(nvalid >= 2, 2, 1))
    m = torch.minimum(torch.tensor(ms)[torch.randint(0, len(ms), (n, *shape), generator=gen)], cap)
    keys = torch.rand(n, taps, *shape, generator=gen).masked_fill(~valid, -float('inf'))
    top = keys.topk(4, dim=1).indices
    chosen = torch.arange(4).view(1, 4, *[1] * len(shape)) < m.unsqueeze(1)
    return torch.zeros(n, taps, *shape, dtype=torch.bool).scatter_(1, top, chosen)


def signs(gen, shape):
    return torch.randint(0, 2, shape, generator=gen).float() * 2 - 1


def small_ints(gen, shape):
    return torch.randint(-4, 5, shape, generator=gen).float()


def guidance_from_sites(val, K, gathered):
    """Guidance whose gates are `val` ((n, taps, *S), per site).  Gathered norms: g_k(p + off_k) = val_k(p) (the caller
    only sets taps whose source is inside); 'paddle': g_k(p) = val_k(p)."""
    if not gathered:
        return val.clone()
    nd = val.dim() - 2
    r = (K - 1) // 2
    return torch.stack([shift(val[:, k], tuple(-o for o in off), r) for k, off in enumerate(offsets(K, nd))], 1)


def dyadic_guidance(gen, n, shape, K, gathered, ms=(1, 2, 4)):
    nd = len(shape)
    offs = offsets(K, nd)
    valid = inside(shape, offs) if gathered else torch.ones(len(offs), *shape, dtype=torch.bool)
    val = hot_taps(gen, n, valid, ms).float() * signs(gen, (n, len(offs), *shape))
    return guidance_from_sites(val, K, gathered)


def sparse_values(gen, shape, sparse):
    if sparse is None:
        return None
    lo = -1 if sparse == 'signed' else 0        # 'bernoulli': {0, 3}; 'signed': {-3, 0, 3}
    return torch.randint(lo, 2, shape, generator=gen).float() * 3


def dyadic_2d(seed, B, C, H, W, K, sparse=None, gch=None):
    """(guidance (B, gch, H, W), blur, sparse (B, 1, H, W) or None, grad_out), fp32 on the CPU.  Channels >= K*K-1 hold
    small integers that the propagation never reads."""
    gen = torch.Generator().manual_seed(seed)
    nt = K * K - 1
    g = dyadic_guidance(gen, B, (H, W), K, True)
    if gch and gch > nt:
        g = torch.cat([g, small_ints(gen, (B, gch - nt, H, W))], 1)
    return g, small_ints(gen, (B, C, H, W)), sparse_values(gen, (B, 1, H, W), sparse), small_ints(gen, (B, C, H, W))


def dyadic_3d(seed, B, C, D, H, W, K, norm, per_channel=False):
    """(guidance (B, nt, D, H, W) or per-channel (B, nt*C, D, H, W), feat, grad_out), fp32 on the CPU."""
    gen = torch.Generator().manual_seed(seed)
    nt = K ** 3 - 1
    nv = B * C if per_channel else B
    g = dyadic_guidance(gen, nv, (D, H, W), K, norm != 'paddle').reshape(B, -1, D, H, W)
    assert g.shape[1] == (nt * C if per_channel else nt)
    return g, small_ints(gen, (B, C, D, H, W)), small_ints(gen, (B, C, D, H, W))


def fallback_taps(shape, K):
    """(taps, *shape) long: tap k, or where its source lies outside, the tap with the components of off_k that leave the
    image negated.  Every extent at least K makes that source inside, and the tap is never the centre."""
    nd = len(shape)
    r = (K - 1) // 2
    offs = offsets(K, nd)
    lut = torch.full((K ** nd,), -1, dtype=torch.long)
    for k, off in enumerate(offs):      # the window position of off, (r - o_0, r - o_1, ...) in raster order
        lut[sum((r - o) * K ** (nd - 1 - i) for i, o in enumerate(off))] = k
    grids = torch.meshgrid(*[torch.arange(n) for n in shape], indexing='ij')
    out = []
    for off in offs:
        pos = 0
        for i, (gi, o, n) in enumerate(zip(grids, off, shape)):
            oi = torch.where((gi + o >= 0) & (gi + o < n), o, -o)
            pos = pos + (r - oi) * K ** (nd - 1 - i)
        out.append(lut[pos])
    return torch.stack(out)


def one_tap_guidance(seed, shape, K, gathered):
    """A batch of one image / volume per tap: in item k every site has one hot tap (+-1): tap k, or for the gathered norms,
    where tap k's source lies outside, fallback_taps' reflection of it.  One tap per site: S = 1."""
    gen = torch.Generator().manual_seed(seed)
    nt = len(offsets(K, len(shape)))
    if gathered:
        assert min(shape) >= K
        taps = fallback_taps(shape, K)
    else:
        taps = torch.arange(nt).view(nt, *[1] * len(shape)).expand(nt, *shape)
    val = torch.zeros(nt, nt, *shape).scatter_(1, taps.unsqueeze(1), 1.0)
    return guidance_from_sites(val * signs(gen, val.shape), K, gathered)


# ---- exactness --------------------------------------------------------------------------------------------------------
def check_exact(t, N, what, unit=None):
    """The values of an exact case: finite multiples of `unit` (default 4^-(N+1)), and below 2^24 in those units."""
    unit = 4.0 ** -(N + 1) if unit is None else unit
    x = t.detach().double() / unit
    assert torch.isfinite(x).all(), what
    assert torch.equal(x, x.round()), f'{what}: not a multiple of {unit:g}'
    assert float(x.abs().max()) < 2.0 ** 24, f'{what}: {float(x.abs().max())} units of {unit:g}'


def autograd(ref, guidance, x, grad_out, dtype):
    """(out, grad_guidance, grad_x) of ref(guidance, x) in `dtype` on the CPU (new leaves: the inputs stay untouched)."""
    g = guidance.detach().to(dtype).requires_grad_(True)
    d = x.detach().to(dtype).requires_grad_(True)
    out = ref(g, d)
    out.backward(grad_out.to(dtype))
    return out.detach(), g.grad, d.grad


def exact_reference(ref, guidance, x, grad_out, N, fp32=True):
    """fp64 autograd of `ref`, checked to be an exact case: every tensor on the grid of check_exact, and (fp32) fp32 autograd
    of the same reference gives the same bits.  If this fails the input is not exact: fix the case, not the kernel."""
    r64 = autograd(ref, guidance, x, grad_out, torch.float64)
    r32 = autograd(ref, guidance, x, grad_out, torch.float32) if fp32 else r64
    for a, b, name in zip(r64, r32, ('out', 'grad_guidance', 'grad_x')):
        check_exact(a, N, name)
        assert torch.equal(a, b.double()), f'{name}: fp32 and fp64 autograd of the reference differ'
    return r64


# ---- the case matrix --------------------------------------------------------------------------------------------------
def pairwise(axes, allowed=lambda case: True):
    """A short list of cases (dicts over `axes`, name -> values) in which every pair of values of two axes that some allowed
    case holds appears together: greedy and deterministic, each pick the allowed case that covers most pairs still open."""
    names = list(axes)
    cases = [c for c in (dict(zip(names, v)) for v in itertools.product(*axes.values())) if allowed(c)]
    pairs = [frozenset((a, c[a], b, c[b]) for a, b in itertools.combinations(names, 2)) for c in cases]
    todo = set().union(*pairs)
    out = []
    while todo:
        i = max(range(len(cases)), key=lambda j: len(pairs[j] & todo))
        out.append(cases[i])
        todo -= pairs[i]
    return out


def norms_2d(K):
    return (f'{K * K - 1}sum', f'{K * K - 1}sum_abs')


def norms_3d(K):
    return (f'{K ** 3 - 1}sum', f'{K ** 3 - 1}sum_abs', 'paddle')


# 2D: 37 x 136 is 3 x 3 tiles of the 64 x 16 vectorised recompute and 5 x 5 of the 32 x 8 scalar kernels; 37 x 133 the same
# with an odd width; 5 x 5 is smaller than the 7 x 7 window.
AXES_2D = {
    'path': tuple((K, n) for K in (3, 5, 7) for n in norms_2d(K)),
    'hw': ((37, 136), (37, 133), (17, 65), (9, 33), (1, 100), (100, 1), (5, 5)),
    'bc': ((1, 1), (2, 3), (3, 2)),
    'N': (1, 2, 4),
    'sparse': (None, 'bernoulli', 'signed'),
    'misaligned': (False, True),
    'extra_channels': (False, True),
}
# 3D: 7 x 19 x 72 crosses 2 x 3 tiles of 64 x 16 and 3 x 3 of 32 x 8 in every z-plane
AXES_3D = {
    'path': tuple((K, n) for K in (3, 5) for n in norms_3d(K)),
    'dhw': ((7, 19, 72), (7, 19, 70), (5, 9, 33), (3, 1, 100)),
    'bc': ((1, 1), (2, 3), (3, 2)),
    'N': (1, 2, 4),
    'misaligned': (False, True),
    'per_channel': (False, True),
}


def _allowed_2d(c):
    return not (c['sparse'] == 'signed' and c['N'] > 3)     # with m = -1 the magnitudes double each step


def _allowed_3d(c):
    return not (c['per_channel'] and c['bc'][1] == 1)


def cases_2d():
    return pairwise(AXES_2D, _allowed_2d) + [
        # full NYU size at K = 5 and 7
        dict(path=(5, '24sum'), hw=(228, 304), bc=(1, 1), N=4, sparse='bernoulli', misaligned=False, extra_channels=False),
        dict(path=(7, '48sum_abs'), hw=(228, 304), bc=(1, 1), N=3, sparse='signed', misaligned=False, extra_channels=True),
    ]


def cases_3d():
    return pairwise(AXES_3D, _allowed_3d) + [
        dict(path=(5, '124sum_abs'), dhw=(8, 40, 136), bc=(1, 1), N=2, misaligned=False, per_channel=False),
    ]


def case_id(c):
    return '-'.join(f'{k}={"x".join(map(str, v)) if isinstance(v, tuple) else v}' for k, v in c.items())
