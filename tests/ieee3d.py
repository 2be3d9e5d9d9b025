"""The IEEE cases of the normalised 3D propagation (3x3x3 and 5x5x5, norms '{nt}sum', '{nt}sum_abs' and 'paddle'): input
families, their references and the case matrix.  Shared by tests/test_ieee3d_cpu.py (the premises, without a GPU) and
tests/test_ieee3d_gpu.py.

The contract (DESIGN.md sections 4.4 and 4.9): the weights are the quotients w_k = a_k / S, S = sum_k |a_k| in fp32, with
IEEE division -- 0 / 0 = NaN, exact quotients at a subnormal S, weights of 0 (and kappa = 1) where S overflows to inf --
and inf / NaN of feat travel as the oracle's products and sums have them.  Every kernel that divides once per voxel
instead (the raw-guidance steps) must fall back to the quotients wherever that would differ.

Three families:
  scaled dyadic    backward_exact.dyadic_3d's guidance (m in {1, 2, 4} hot taps of +-1 per site) times 2^e, with feat and
                   grad_out small integers times a companion scale.  Every value of the forward and of both gradients is
                   exact in fp32, so the kernels must return the bits of an fp64 reference in which S passes through a
                   rounding to fp32 (exact unless it overflows: a sum of at most 124 values +-2^e).  The exponents put the
                   sums on both sides of every threshold of the kernels: the smallest subnormal, deep subnormal sums,
                   2^-126 (cold_sum's FLT_MIN and the gather kernel's 1 / S > 8e37 at 2^-126 <= S < 2^-125), an
                   ordinary range, and 2^128 (sites with m >= 2 overflow, m = 1 does not, and sum_k |g_k| d of 'paddle'
                   overflows where |d| >= 2).
  special regions  random gates with a region scaled by 1e-42, a region set to +-3e37, one +inf and one -inf, one NaN, or an
                   all-zero block; region edges inside a quad of 4 voxels and across the 128-voxel row of a warp.
  non-finite feat  +inf, -inf or NaN at one voxel of each batch item: a corner, faces, the interior, and each lane of a quad.
The last two are checked against the fp32 oracle: equal NaN, +inf and -inf masks, and finite values to parity_ok(1e-4).
"""
import numpy as np
import torch

from oracle import cspn_numpy as onp
from oracle import cspn_numpy_3d_k as onk
from oracle.cspn_torch_port_3d_k import offsets_3d

import backward_exact as be

FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = 2.0 ** -126
GATHER_COLD = 8.0e37          # step3d_gather_vec4_kernel: 1 / S above this takes the quotients

# ---- scaled dyadic ------------------------------------------------------------------------------------------------------
EXPONENTS = (-149, -140, -128, -127, -126, -125, 0, 100, 127)


def companion(e):
    """log2 of the scale of feat and of grad_out at gate exponent e.  grad_guidance grows like grad_out * feat / S: the
    scales keep 2^24 of its units below 2^128, and every product 2^e * d of the forward on the grid of 2^-149."""
    return -22 if e <= -140 else (-13 if e <= -125 else 0)


def scaled_dyadic(seed, B, C, D, H, W, K, norm, e, per_channel=False):
    """(guidance, feat, grad_out), fp32 on the CPU: dyadic_3d's inputs with the gates times 2^e and feat, grad_out times
    2^companion(e)."""
    g, f, go = be.dyadic_3d(seed, B, C, D, H, W, K, norm, per_channel)
    c = 2.0 ** companion(e)
    return (g.double() * 2.0 ** e).float(), f * c, go * c


def units(e, N):
    """The grids of (out, grad_guidance, grad_feat) of a scaled case: backward_exact's 4^-(N+1) times the scales."""
    u, c = 4.0 ** -(N + 1), 2.0 ** companion(e)
    return u * c, u * c * c * 2.0 ** -e, u * c


class _RoundToF32(torch.autograd.Function):
    """S rounded to fp32 (to inf where it overflows), with the identity as its gradient."""

    @staticmethod
    def forward(ctx, s):
        return s.float().to(s.dtype)

    @staticmethod
    def backward(ctx, grad):
        return grad


def _cspn3d_f32_sum(guidance, feat, prop_time, K, norm_type, round_sum):
    """oracle/cspn_torch_port_3d_k.cspn3d_torch_k with S optionally rounded to fp32, for one gate shared by the channels."""
    nt, r = K ** 3 - 1, (K - 1) // 2
    offs = offsets_3d(K)
    g = guidance[:, :nt]
    if norm_type == 'paddle':
        a = g.abs()
        S = a.sum(1, keepdim=True)
    else:
        if 'abs' in norm_type:
            g = g.abs()
        a = torch.stack([be.shift(g[:, k], o, r) for k, o in enumerate(offs)], 1)
        S = a.abs().sum(1, keepdim=True)
    if round_sum:
        S = _RoundToF32.apply(S)
    gate = a / S
    gate_sum = gate.sum(1, keepdim=True)
    result = feat
    for _ in range(prop_time):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + gate[:, k:k + 1] * be.shift(result, o, r)
        result = acc if norm_type == 'paddle' else (1.0 - gate_sum) * feat + acc
    return result


def ieee_ref(guidance, feat, prop_time, K, norm_type, round_sum=True):
    """The fp64 reference of the scaled family (per-channel gates as B*C single-channel volumes, as be.cspn3d_ref)."""
    nt = K ** 3 - 1
    B, C = feat.shape[:2]
    if guidance.shape[1] == nt * C and C > 1:
        out = _cspn3d_f32_sum(guidance.reshape(B * C, nt, *feat.shape[2:]), feat.reshape(B * C, 1, *feat.shape[2:]),
                              prop_time, K, norm_type, round_sum)
        return out.reshape(feat.shape)
    return _cspn3d_f32_sum(guidance, feat, prop_time, K, norm_type, round_sum)


def sums(guidance, K, norm, C=1):
    """S of every site in fp64 (B', D, H, W), per-channel gates as B*C volumes: what the thresholds act on."""
    nt, r = K ** 3 - 1, (K - 1) // 2
    g = guidance.double().reshape(-1, nt, *guidance.shape[2:])
    if norm == 'paddle':
        return g.abs().sum(1)
    return torch.stack([be.shift(g[:, k].abs(), o, r) for k, o in enumerate(offsets_3d(K))], 1).sum(1)


def scaled_reference(g, f, go, N, K, norm, e, backward=True):
    """(out, grad_guidance, grad_feat) in fp64, each checked to lie on the case's grid (grads None without backward)."""
    ref = lambda gg, ff: ieee_ref(gg, ff, N, K, norm)
    if backward:
        r = be.autograd(ref, g, f, go, torch.float64)
    else:
        r = (ref(g.double(), f.double()), None, None)
    for t, u, name in zip(r, units(e, N), ('out', 'grad_guidance', 'grad_feat')):
        if t is not None:
            assert u >= 2.0 ** -149 and u * 2.0 ** 24 < 2.0 ** 128, (name, u)
            be.check_exact(t, N, f'{name} (e = {e})', unit=u)
    return r


# ---- special regions and non-finite feat ----------------------------------------------------------------------------------
SPECIAL = ('tiny', 'huge', 'inf', 'nan', 'zero')
NONFINITE = (float('inf'), -float('inf'), float('nan'))


def region(W):
    """(z, y, x) slices of the special region: x edges inside a quad (5 and W - 5), so across the 128-voxel row of a warp
    where W >= 136.  In volumes of 6 x 9 it holds whole 5 x 5 x 5 windows."""
    return slice(0, 5), slice(1, 8), slice(5, W - 5)


def special_gates(seed, B, C, D, H, W, K, kind, per_channel=False):
    """(guidance, feat), fp32 on the CPU: normal gates and feat in [-1, 3) (|d| > 1, so that 3e37 * d overflows), with
    the special `kind` applied to volume 0."""
    gen = torch.Generator().manual_seed(seed)
    nt = K ** 3 - 1
    g = torch.randn(B, nt * C if per_channel else nt, D, H, W, generator=gen)
    f = torch.rand(B, C, D, H, W, generator=gen) * 4 - 1
    z, y, x = region(W)
    if kind == 'tiny':
        g[0, :, z, y, x] *= 1e-42
    elif kind == 'huge':        # rows 1, 2: 8 taps of 3e37, a finite S whose sum |g| d overflows; below: S overflows
        keep = g[0, 8:, z, 1:3, x].clone()
        g[0, :, z, y, x] = torch.sign(g[0, :, z, y, x]) * 3e37
        g[0, 8:, z, 1:3, x] = keep
    elif kind == 'inf':
        g[0, 3, D // 2, H // 2, 6] = float('inf')
        g[0, nt - 5, D - 2, H - 3, W - 7] = -float('inf')
    elif kind == 'nan':
        g[0, nt // 2, D // 2, 1, W // 2 + 1] = float('nan')
    else:
        assert kind == 'zero'
        g[0, :, z, y, x] = 0.0
    return g, f


def nonfinite_sites(D, H, W):
    """One (z, y, x) per batch item: two corners, the six faces, the interior, and the four lanes of one quad."""
    zc, yc, xc = D // 2, H // 2, (W // 2) // 4 * 4
    return ([(0, 0, 0), (D - 1, H - 1, W - 1), (0, yc, xc), (D - 1, yc, xc + 1), (zc, 0, xc + 2), (zc, H - 1, xc + 3),
             (zc, yc, 0), (zc, yc, W - 1)] + [(zc, yc, 4 + j) for j in range(4)])


def nonfinite_feat(seed, C, D, H, W, K, value, per_channel=False):
    """(guidance, feat) with one `value` (inf, -inf or NaN) in feat per batch item, channel item % C."""
    sites = nonfinite_sites(D, H, W)
    gen = torch.Generator().manual_seed(seed)
    nt = K ** 3 - 1
    B = len(sites)
    g = torch.randn(B, nt * C if per_channel else nt, D, H, W, generator=gen)
    f = torch.rand(B, C, D, H, W, generator=gen) * 4 - 1
    for b, (z, y, x) in enumerate(sites):
        f[b, b % C, z, y, x] = value
    return g, f


def oracle(g, f, N, K, norm):
    """The fp32 oracle (numpy; at K = 3 the bits of cspn_numpy.cspn3d), per-channel gates channel by channel."""
    g, f = np.asarray(g, np.float32), np.asarray(f, np.float32)
    nt, C = K ** 3 - 1, f.shape[1]
    if g.shape[1] == nt * C and C > 1:
        return np.concatenate([onk.cspn3d_k(g[:, nt * c:nt * (c + 1)], f[:, c:c + 1], N, K, norm) for c in range(C)], 1)
    return onk.cspn3d_k(g, f, N, K, norm)


def masks(a):
    a = np.asarray(a)
    return np.isnan(a), a == np.inf, a == -np.inf


def check_masks_and_parity(out, ref, what):
    """NaN, +inf and -inf where the reference has them, and the finite values to parity_ok(1e-4)."""
    out, ref = np.asarray(out, np.float64), np.asarray(ref, np.float64)
    for m_out, m_ref, name in zip(masks(out), masks(ref), ('NaN', '+inf', '-inf')):
        bad = m_out != m_ref
        assert not bad.any(), (what, f'{name} mask: {int(bad.sum())} voxels differ, first at {tuple(np.argwhere(bad)[0])}',
                               int(m_ref.sum()))
    fin = np.isfinite(ref)
    ok, ratio, normwise = onp.parity_ok(out[fin], ref[fin], 1e-4)
    assert ok, (what, ratio, normwise)


# ---- the case matrix --------------------------------------------------------------------------------------------------------
# Routes of the forward.  K = 3 (generic3d_forward, cspn3d.cu): W = 136 with aligned pointers (the raw-guidance float4
# kernels), CSPN_B200_3D_PADDLE=planes (prep + float4 plane step), W = 135 (scalar plane step), a view 4 bytes off a 16-byte
# boundary (plane steps), CSPN_B200_MAX_WS3D_KB so that B = 3 runs as groups of 2 + 1 (W = 135: the plane route), and
# B * C * D > 65535 (gridDim.z: plane route, volume groups of 511 + 9).  K = 5 (cspn3d_wide.cu): the float4 and scalar steps.
ROUTES_3 = ('raw', 'planes', 'odd', 'misaligned', 'groups', 'bcd')
ROUTES_5 = ('vec', 'scalar')
W_OF = {'raw': 136, 'planes': 136, 'odd': 135, 'misaligned': 136, 'groups': 135, 'bcd': 4, 'vec': 136, 'scalar': 135}


def route_env(route, Bv, Cv, D, H, W, N):
    """The environment of a route: (CSPN_B200_3D_PADDLE, CSPN_B200_MAX_WS3D_KB), None for unset.  Bv, Cv: the volumes and
    channels the library sees (per-channel gates: B * C volumes of one channel).  'groups' caps the workspace at Bv - 1
    volumes of cspn3d.cu's group3d, so the last group is ragged."""
    if route == 'planes':
        return 'planes', None
    if route == 'groups':
        per_vol = 4 * (27 * D * H * W + (Cv * D * H * W if N > 1 else 0))
        return None, f'{(Bv - 0.5) * per_vol / 1024:.3f}'
    return None, None


def launches(route, K, norm, N):
    """The launches of a forward on `route`: one per step on the raw-guidance routes (and 'paddle' at K = 5), a prep more
    per volume group on the weight-plane routes, and two groups for 'groups' and 'bcd'."""
    if route == 'raw' or (K == 5 and norm == 'paddle'):
        return N
    return (2 if route in ('groups', 'bcd') else 1) * (1 + N)


def route_dims(route, D, H):
    """(B, D, H) of a case on `route` (B * C * D > 65535 for 'bcd' with C = 1, 3 volumes for 'groups')."""
    if route == 'bcd':
        return 520, 128, 1
    return (3 if route == 'groups' else 2), D, H


SCALED_AXES = {
    'path': tuple((3, n, r) for n in be.norms_3d(3) for r in ROUTES_3) + tuple((5, n, r) for n in be.norms_3d(5)
                                                                                for r in ROUTES_5),
    'e': EXPONENTS,
    'gates': ('C1', 'C2-shared', 'C2-per-channel'),
    'N': (1, 2, 3),
    'api': ('P3D-op', 'P3D-ctypes', 'P3DK-op', 'P3DK-ctypes'),
}


def _allowed(c):
    K, norm, route = c['path']
    if route == 'bcd' and c['gates'] != 'C1':
        return False
    return not (K == 5 and c['api'].startswith('P3D-'))   # Affinity_Propagate3D is the 3x3x3 module


def scaled_cases():
    return be.pairwise(SCALED_AXES, _allowed)


# backward: both autograd routes, the tile-crossing shapes of backward_exact.AXES_3D, the exponents
BACKWARD_AXES = {
    'path': tuple((K, n) for K in (3, 5) for n in be.norms_3d(K)),
    'e': EXPONENTS,
    'dhw': ((7, 19, 72), (7, 19, 70)),
    'gates': ('C1', 'C2-shared', 'C2-per-channel'),
    'N': (1, 2, 3),
}


def backward_cases():
    return be.pairwise(BACKWARD_AXES)


SPECIAL_AXES = {
    'path': SCALED_AXES['path'],
    'kind': SPECIAL + tuple(f'feat{v}' for v in NONFINITE),
    'gates': ('C1', 'C2-shared', 'C2-per-channel'),
    'N': (1, 2, 3),
    'api': SCALED_AXES['api'],
}


def _allowed_special(c):
    K, norm, route = c['path']
    if route == 'bcd':
        return False        # the gridDim.z route runs the scaled family; its volumes of 1 x 4 voxels have no interior
    return _allowed(c)


def special_cases():
    return be.pairwise(SPECIAL_AXES, _allowed_special)


def gates_shape(gates):
    """(C, per_channel) of the gates axis."""
    return {'C1': (1, False), 'C2-shared': (2, False), 'C2-per-channel': (2, True)}[gates]


def case_id(c):
    return '-'.join(f'{k}={"_".join(map(str, v)) if isinstance(v, tuple) else v}' for k, v in c.items())
