"""CPU tests of the dynamic propagation (DySPN's step, DESIGN.md section 4.23): the two autograd restatements of
tests/dynamic_reference.py against each other in fp64, forward and autograd; its fp32 FMA against exact rationals
(midpoints where rounding in fp64 and then fp32 is wrong, signed zeros, subnormals, inf and NaN) and its kernel-order
restatement against fp64; the ring map; attention 1 as a fixed-weight
step; the C ABI's workspace formulas and refusals without a device; the op schemas and fake kernels; the Python refusals;
no spills in the new translation unit; and the dilated propagation's machine code, unchanged by the shared tile helpers."""
import hashlib
import json
import os
import re
import shutil
import subprocess
from fractions import Fraction

import pytest
import torch

import dilated_reference as dr
import dynamic_reference as yr
from cspn_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
D = torch.float64
NAMES = ('out', 'affinity', 'attention', 'blur', 'sparse', 'conf')


def assert_same(r1, r2, tol=1e-12):
    for name, x, y in zip(NAMES, r1, r2):
        assert (x is None) == (y is None), name
        if x is not None:
            torch.testing.assert_close(x, y, rtol=tol, atol=tol, msg=name)


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
@pytest.mark.parametrize('shape,N', [((2, 1, 9, 11), 3), ((1, 3, 6, 7), 2), ((1, 1, 1, 13), 2), ((2, 2, 10, 1), 1), ((1, 1, 3, 4), 4)])
def test_restatements_agree_in_fp64(K, samples, shape, N):
    """Includes R >= H or W (every neighbour outside the image), 1 x W and H x 1 images, and C = 3."""
    B, C, H, W = shape
    ins = yr.make_inputs(B, C, H, W, K, N, samples, seed=K * 7 + N)
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(1))
    assert_same(yr.grads(yr.composition, *ins, K, go, dtype=D), yr.grads(yr.explicit, *ins, K, go, dtype=D))


@pytest.mark.parametrize('samples', [None, 'soft'])
def test_gradcheck(samples):
    ins = [None if t is None else t.double().requires_grad_(True) for t in yr.make_inputs(1, 2, 5, 6, 3, 2, samples, seed=3)]
    live = tuple(t for t in ins if t is not None)

    def f(*ts):
        it = iter(ts)
        return yr.explicit(*[None if t is None else next(it) for t in ins], 3)

    assert torch.autograd.gradcheck(f, live, eps=1e-6, atol=1e-5)


def test_ring_map():
    for K, counts in ((3, [1, 8]), (5, [1, 8, 16]), (7, [1, 8, 16, 24])):
        ring = yr.rings(K)
        assert ring.bincount().tolist() == counts
        assert ring[K * K // 2] == 0 and ring[0] == ring[K - 1] == ring[K * K - 1] == (K - 1) // 2
    # channel t*(R+1) + r is ring r at step t: zeroing it is zeroing ring r's affinity at step t
    aff, att, b, _, _ = [t.double() for t in yr.make_inputs(1, 1, 6, 7, 5, 2, None, seed=1)[:3]] + [None, None]
    for t in (0, 1):
        for r in (0, 1, 2):
            att2 = att.clone()
            att2[:, 3 * t + r] = 0
            aff2 = aff.clone()
            aff2[:, (yr.rings(5) == r).nonzero().flatten()] = 0
            steps = [(aff2 if s == t else aff, att[:, 3 * s:3 * s + 3]) for s in (0, 1)]
            want = b
            for s_aff, s_att in steps:                                  # one step at a time, d_0 the original blur
                B, C, H, W = b.shape
                w = s_att[:, yr.rings(5)] * s_aff
                cols = torch.nn.functional.unfold(want, 5, padding=2).view(B, C, 25, H, W)
                want = (1 - w.sum(1, keepdim=True)) * b + torch.einsum('bckhw,bkhw->bchw', cols, w)
            torch.testing.assert_close(yr.composition(aff, att2, b, K=5), want, rtol=1e-13, atol=1e-13)


def test_attention_one_is_a_fixed_weight_step():
    """attention 1 and a zero centre affinity: the dilated step at dilation 1 with rho = 1 - sum_j affinity_j as its centre
    weight, at every step."""
    for K in (3, 5, 7):
        aff, _, b, s, m = [None if t is None else t.double() for t in yr.make_inputs(2, 2, 8, 9, K, 1, 'soft', seed=K)]
        c = K * K // 2
        aff[:, c] = 0
        att = torch.ones(2, 4 * ((K + 1) // 2), 8, 9, dtype=D)
        kern = aff.clone()
        kern[:, c] = 1 - aff.sum(1)
        torch.testing.assert_close(yr.composition(aff, att, b, s, m, K), dr.composition(kern, b, s, m, K, 1, 4), rtol=1e-13, atol=1e-13)


def test_steps_follow_the_attention_channels():
    aff, att, b, _, _ = yr.make_inputs(1, 1, 5, 5, 3, 3, None, seed=2)
    assert yr.steps(att, 3) == 3
    one = yr.composition(aff, att[:, :2], b, K=3)
    assert one.shape == b.shape and not torch.equal(one, b)
    assert torch.equal(yr.composition(aff, att[:, :0], b, K=3), b)


# ---- the kernels' order of operations ------------------------------------------------------------------------------------
def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def exact_f32(q):
    """The Fraction q rounded to fp32, to nearest with ties to even, subnormals included, as a Python float."""
    if q == 0:
        return 0.0
    sign, q = (-1.0 if q < 0 else 1.0), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()        # 2^(e-1) <= q < 2^(e+1)
    e = max(e - 24, -149)                                             # 24 significant bits, or the subnormal quantum
    while q / Fraction(2) ** e >= 2 ** 24:
        e += 1
    m = round(q / Fraction(2) ** e)                                   # Fraction.__round__ ties to even
    v = m * Fraction(2) ** e
    if v >= Fraction(2) ** 128:
        return sign * float('inf')
    return sign * float(v)


def fma_exact(a, b, c):
    return exact_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def naive(a, b, c):
    """a*b + c rounded in fp64, then to fp32: the double rounding yr.fma avoids."""
    return (a.double() * b.double() + c.double()).float()


def f32_bits(x):
    return int(torch.tensor(x, dtype=torch.float32).view(torch.int32))


def test_fma_rounds_once_on_random_triples():
    """Exponents over the whole fp32 range, products near -c so that the sum cancels, and results in the subnormal
    range, against the exact value in Fractions rounded once."""
    g = torch.Generator().manual_seed(0)
    n = 3000
    a = torch.randn(n, generator=g) * torch.exp2(torch.randint(-60, 60, (n,), generator=g).float())
    b = torch.randn(n, generator=g) * torch.exp2(torch.randint(-60, 60, (n,), generator=g).float())
    c = torch.randn(n, generator=g) * torch.exp2(torch.randint(-120, 120, (n,), generator=g).float())
    near = torch.arange(n) % 3 == 1
    c = torch.where(near, -(a * b) * (1 + torch.randn(n, generator=g) * 2 ** -20), c)         # cancellation
    sub = torch.arange(n) % 3 == 2
    a = torch.where(sub, torch.randn(n, generator=g) * 2 ** -70, a)                          # subnormal results
    b = torch.where(sub, torch.randn(n, generator=g) * 2 ** -70, b)
    c = torch.where(sub, torch.randn(n, generator=g) * 2 ** -135, c)
    got = yr.fma(a, b, c)
    want = torch.tensor([fma_exact(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], dtype=torch.float32)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert int(((want != 0) & (want.abs() < 2 ** -126)).sum()) > 300                          # subnormals reached


def midpoint_cases():
    """(a, b, c) whose exact a*b + c lies within 2^-46 of an ulp of c from an fp32 midpoint, on the side the fp64 sum
    cannot see: a*b = 2^-24 (1 - 2^-46) = (1 + 2^-23) * 2^-24 (1 - 2^-23) just below half an ulp of c = 1 + k 2^-23, or
    2^-24 (1 + 4688 * 2^-46) = (1 + 2896 * 2^-23) * 2^-24 (1 - 2895 * 2^-23) just above it.  The fp64 sum rounds onto
    the midpoint, and the fp32 tie then goes to the even neighbour, which is wrong when the exact value lies on the odd
    side.  Scaled by powers of two and negated, so both signs and other binades are covered."""
    below = (1 + 2 ** -23, 2 ** -24 * (1 - 2 ** -23))
    above = (1 + 2896 * 2 ** -23, 2 ** -24 * (1 - 2895 * 2 ** -23))
    out = []
    for s in (1.0, -1.0):
        for e in (0, 40, -40, -100):
            sc = 2.0 ** e
            out.append((below[0] * s, below[1] * sc, (1 + 2 ** -23) * s * sc))   # c odd: the tie goes up, exact is below
            out.append((above[0] * s, above[1] * sc, (1 + 2 ** -22) * s * sc))   # c even: the tie stays, exact is above
    return out


def test_fma_is_right_where_the_fp64_then_fp32_rounding_is_wrong():
    for a, b, c in midpoint_cases():
        ta, tb, tc = f32([a]), f32([b]), f32([c])
        assert (float(ta), float(tb), float(tc)) == (a, b, c)                           # exact fp32 operands
        want = fma_exact(a, b, c)
        assert f32_bits(float(yr.fma(ta, tb, tc))) == f32_bits(want), (a, b, c)
        assert float(naive(ta, tb, tc)) != want, (a, b, c)                              # the double rounding's error
        assert abs(f32_bits(float(naive(ta, tb, tc))) - f32_bits(want)) == 1                # of one ulp


def test_fma_signed_zeros_and_special_operands():
    inf, nan, big, tiny = float('inf'), float('nan'), 3.4028234663852886e38, 2.0 ** -100
    cases = [  # (a, b, c, IEEE fmaf)
        (-0.0, 1.0, 0.0, 0.0), (-0.0, 1.0, -0.0, -0.0), (0.0, -1.0, -0.0, -0.0), (0.0, 1.0, -0.0, 0.0),
        (1.0, -1.0, 1.0, 0.0), (-1.0, 1.0, 1.0, 0.0),                          # exact cancellation: +0 to nearest
        (tiny, -tiny, 0.0, -0.0), (tiny, tiny, -0.0, 0.0), (tiny, -tiny, -0.0, -0.0),   # underflow keeps the sign
        (2.0 ** -75, 2.0 ** -75, 0.0, 2.0 ** -149 * 0),                        # 2^-150: a tie, to the even 0
        (2.0 ** -75, 1.5 * 2.0 ** -75, 0.0, 2.0 ** -149),                      # 1.5 * 2^-150 rounds up
        (2.0 ** -70, 2.0 ** -70, 2.0 ** -149, 2.0 ** -149 + 2.0 ** -140),      # subnormal sum, exact
        (inf, 0.0, 1.0, nan), (0.0, -inf, 1.0, nan), (inf, 2.0, -inf, nan), (inf, 2.0, 1.0, inf), (-inf, 2.0, 1.0, -inf),
        (2.0, 3.0, inf, inf), (2.0, 3.0, -inf, -inf), (nan, 0.0, 1.0, nan), (1.0, 1.0, nan, nan),
        (big, 2.0, -inf, -inf), (big, 2.0, 0.0, inf), (big, -2.0, 0.0, -inf), (big, 2.0, -big, big),   # no overflow
        (big, 1.0, big * 2.0 ** -24, inf), (big, 1.0, big * 2.0 ** -25, big),   # past max + half an ulp, and below it
    ]
    for a, b, c, want in cases:
        got = float(yr.fma(f32([a]), f32([b]), f32([c])))
        if want != want:
            assert got != got, (a, b, c)
        else:
            assert f32_bits(got) == f32_bits(want), (a, b, c, got, want)
            if abs(want) != inf and want != 0:                          # a Fraction has no signed zero
                assert f32_bits(got) == f32_bits(fma_exact(a, b, c)), (a, b, c)


def assert_within(got, ref, fwd_tol=1e-5, grad_tol=2e-3):
    """test_dynamic_gpu.py's `within`: element by element, relative to |ref| plus its mean."""
    for name, g, r in zip(NAMES, got, ref):
        assert (g is None) == (r is None), name
        if r is not None:
            tol = fwd_tol if name == 'out' else grad_tol
            bound = tol * (r.abs() + r.abs().mean())
            assert bool(((g.double() - r).abs() <= bound).all()), name


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
@pytest.mark.parametrize('shape,N', [((2, 3, 9, 11), 4), ((1, 1, 1, 13), 3), ((2, 2, 10, 1), 2), ((1, 2, 2, 3), 1)])
def test_kernel_order_within_tolerance_of_fp64(K, samples, shape, N):
    """Random inputs, the op's tolerance; 1 x W and H x 1 images and an image smaller than the halo included."""
    ins = yr.make_inputs(*shape, K, N, samples, seed=K * 3 + N)
    go = torch.randn(shape, generator=torch.Generator().manual_seed(2))
    got = yr.kernel_order(*ins, K, go)
    assert [None if g is None else tuple(g.shape) for g in got] == [None if t is None else tuple(t.shape) for t in
                                                                     [ins[2], ins[0], ins[1], ins[2], ins[3], ins[4]]]
    assert_within(got, yr.grads(yr.composition, *ins, K, go, dtype=D))


@pytest.mark.parametrize('K,N', [(3, 3), (5, 2), (7, 2)])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
def test_kernel_order_equals_fp64_on_dyadic_inputs(K, N, samples):
    ins, go = yr.dyadic_inputs(2, 2, 11, 13, K, N, samples, seed=K + N)
    ref = yr.grads(yr.composition, *ins, K, go, dtype=D)
    for name, g, r in zip(NAMES, yr.kernel_order(*ins, K, go), ref):
        assert (g is None) == (r is None), name
        assert g is None or torch.equal(g, r.float()), name


def test_kernel_order_follows_the_stated_order():
    """The restatement is not order-free: summing S with j descending, or swapping G1's channel order, changes bits
    on random inputs.  So a kernel that did either would fail the bit-for-bit checks the restatement serves."""
    K, N = 5, 3
    ins = yr.make_inputs(1, 3, 12, 14, K, N, 'soft', seed=9)
    go = torch.randn(1, 3, 12, 14, generator=torch.Generator().manual_seed(3))
    a, t, b, s, m = ins
    got = yr.kernel_order(*ins, K, go)
    # channel order: with the channels reversed, G1 and G0 add them in the other order
    rev = yr.kernel_order(a, t, b.flip(1), s, m, K, go.flip(1))
    assert torch.equal(rev[0], got[0].flip(1))                                       # the forward is per channel
    assert not torch.equal(rev[1], got[1]) and not torch.equal(rev[2], got[2])       # the channel sums are not
    # tap order of S: on these inputs 1 - S in another order differs in at least one pixel
    w = [t[:, yr.rings(K)[j]:yr.rings(K)[j] + 1] * a[:, j:j + 1] for j in range(K * K)]
    up, down = w[0], w[-1]
    for j in range(1, K * K):
        up, down = up + w[j], down + w[K * K - 1 - j]
    assert not torch.equal(up, down)


# ---- the library's surface without a device -----------------------------------------------------------------------------
def test_argtypes_cover_the_entry_points():
    for name in ('cspn2d_dyn_workspace_bytes', 'cspn2d_dyn_fwd_f32', 'cspn2d_dyn_bwd_workspace_bytes', 'cspn2d_dyn_bwd_f32'):
        assert name in _lib.SIGNATURES
    assert _lib.lib().cspn2d_dyn_fwd_f32.argtypes is not None
    assert len(_lib.lib().cspn2d_dyn_bwd_f32.argtypes) == 20


def test_workspace_formulas():
    L = _lib.lib()
    P = 2 * 3 * 7 * 9 * 4
    for N in (0, 1, 2, 3, 24):
        assert L.cspn2d_dyn_workspace_bytes(2, 3, 7, 9, 5, N) == (P if N >= 2 else 0)
        assert L.cspn2d_dyn_bwd_workspace_bytes(2, 3, 7, 9, 5, N) == max(2 * N - 1, 0) * P
    assert L.cspn2d_dyn_workspace_bytes(2, 3, 7, 9, 4, 2) == 0
    assert L.cspn2d_dyn_workspace_bytes(0, 3, 7, 9, 3, 2) == 0
    assert L.cspn2d_dyn_bwd_workspace_bytes(2, 3, 7, 9, 3, -1) == 0
    assert L.cspn2d_dyn_workspace_bytes(1, 1, 7, 9, 7, 2 ** 29) == 0    # 2^31 attention channels


INVALID, WORKSPACE, UNSUPPORTED = -1, -2, -4
P = 1 << 20          # fake, 4-byte aligned "device" addresses: every refusal comes before any device work


def fwd(a=P, t=9 * P, b=2 * P, s=None, m=None, out=4 * P, B=1, C=1, H=8, W=8, K=3, N=2, ws=5 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_dyn_fwd_f32(a, t, b, s, m, out, B, C, H, W, K, N, ws, wsb, None)


def bwd(s=None, m=None, ga=6 * P, gt=11 * P, gb=7 * P, gs=None, gm=None, t=9 * P, B=1, C=1, H=8, W=8, K=3, N=2, ws=12 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_dyn_bwd_f32(P, t, 2 * P, s, m, 3 * P, ga, gt, gb, gs, gm, B, C, H, W, K, N, ws, wsb, None)


def test_abi_refusals_without_a_device():
    assert fwd(a=None) == INVALID
    assert fwd(t=None) == INVALID                                  # no attention for N > 0
    assert fwd(b=None) == INVALID
    assert fwd(out=None) == INVALID
    assert fwd(s=8 * P) == INVALID                                 # sparse without confidence
    assert fwd(m=8 * P) == INVALID                                 # confidence without sparse
    assert fwd(b=2 * P + 2) == INVALID                             # misaligned
    assert fwd(t=9 * P + 1) == INVALID
    assert fwd(K=4) == INVALID
    assert fwd(K=9) == INVALID
    assert fwd(N=-1) == INVALID
    assert fwd(B=0) == INVALID
    assert fwd(H=0) == INVALID
    assert fwd(W=-3) == INVALID
    assert fwd(out=2 * P + 64) == INVALID                          # out overlaps blur
    assert b'overlaps' in _lib.lib().cspn_last_error()
    assert fwd(out=9 * P + 64) == INVALID                          # out overlaps the attention
    assert fwd(ws=4 * P + 16) == INVALID                           # the workspace overlaps out
    assert fwd(ws=None) == WORKSPACE
    assert fwd(wsb=4) == WORKSPACE
    assert b'dynamic propagation' in _lib.lib().cspn_last_error()
    assert fwd(B=65536, t=1 << 43, out=1 << 44, ws=1 << 45) == UNSUPPORTED    # B*C beyond gridDim.z
    assert fwd(B=300, C=300, t=1 << 43, out=1 << 44, ws=1 << 45) == UNSUPPORTED
    assert fwd(H=16 * 65536, out=1 << 44, t=1 << 45, ws=1 << 46) == UNSUPPORTED    # ceil(H/16) beyond gridDim.y
    assert bwd(gs=8 * P) == INVALID                                # grad_sparse without the samples
    assert bwd(gm=8 * P) == INVALID
    assert bwd(s=8 * P) == INVALID                                 # sparse without confidence
    assert bwd(t=None) == INVALID
    assert bwd(ga=P) == INVALID                                    # grad_affinity overlaps affinity
    assert bwd(gt=9 * P) == INVALID                                # grad_attention overlaps the attention
    assert bwd(gb=6 * P) == INVALID                                # two outputs overlap
    assert bwd(K=2) == INVALID
    assert bwd(N=-2) == INVALID
    assert bwd(wsb=16) == WORKSPACE
    assert bwd(B=65536, ga=1 << 44, gb=1 << 45, gt=1 << 46, ws=1 << 47, t=1 << 43) == UNSUPPORTED


def test_op_schemas_and_fake_kernels():
    from cspn_b200 import torch_op
    if not torch_op.available():
        pytest.skip('the torch op library is not built')
    torch_op.load()
    op = torch.ops.cspn_b200.propagate2d_dynamic.default
    assert str(op._schema) == ('cspn_b200::propagate2d_dynamic(Tensor affinity, Tensor attention, Tensor blur_depth, '
                               'Tensor? sparse_depth, Tensor? confidence, int kernel_size) -> Tensor')
    bop = torch.ops.cspn_b200.propagate2d_dynamic_backward.default
    assert 'bool need_confidence) -> (Tensor, Tensor, Tensor, Tensor, Tensor)' in str(bop._schema)
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        a, t, b, s = torch.empty(2, 25, 5, 7), torch.empty(2, 12, 5, 7), torch.empty(2, 3, 5, 7), torch.empty(2, 1, 5, 7)
        assert op(a, t, b, s, s, 5).shape == b.shape
        assert op(a, t, b, None, None, 5).shape == b.shape
        g = bop(a, t, b, s, s, b, 5, True, True, False, True, True)
        assert [tuple(x.shape) for x in g] == [(2, 25, 5, 7), (2, 12, 5, 7), (0,), (2, 1, 5, 7), (2, 1, 5, 7)]
        with pytest.raises(Exception):
            op(a, t[:, :11], b, None, None, 5)


def test_python_refusals():
    import cspn_b200
    a, t, b, s, m = yr.make_inputs(1, 2, 5, 6, 3, 2, 'soft')
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a[:, :8], t, b, s, m, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t[:, :3], b, s, m, 3)          # 3 channels are not a whole number of steps
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t[..., :5], b, s, m, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t, b, s, None, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t, b, None, m, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t, b, s.expand(1, 2, 5, 6), m, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dynamic(a, t, b, s, m, 4)
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateDynamic(3, 6)
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateDynamic(-1, 3)
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateDynamic(3, 3)(a, t, b, s, m)          # prop_time 3 needs 6 channels, got 4
    with pytest.raises(RuntimeError):
        cspn_b200.propagate2d_dynamic(a.double(), t, b, s, m, 3)
    with pytest.raises(_lib.CspnError):
        cspn_b200.propagate2d_dynamic(a, t, b, s, m, 3)                  # CPU tensors: no host entry point


def test_no_spills_in_the_new_translation_unit():
    log = os.path.join(ROOT, 'cspn_b200', '_build', 'ptxas.log')
    if not os.path.isfile(log):
        pytest.skip('the library is not built')
    part = open(log).read().split('== cspn2d_dynamic.cu')[1].split('\n== ')[0]
    assert 'dyn_step_kernel' in part and 'dyn_adjoint_kernel' in part and 'dyn_finalize_kernel' in part
    spills = [int(x) for x in re.findall(r'(\d+) bytes spill stores', part)]
    assert len(spills) == 27 and max(spills) == 0


# ---- the dilated propagation's machine code ------------------------------------------------------------------------------
def _anonymous(name):
    """The kernel's name with its anonymous namespace (a per-compile identifier) replaced by _GLOBAL__N_."""
    m = re.search(r'(\d+)_GLOBAL__N_', name)
    if not m:
        return name
    return name[:m.start(1)] + '_GLOBAL__N_' + name[m.end(1) + int(m.group(1)):]


def dilated_sass():
    """{kernel: SASS} of cspn2d_dilated.cu compiled as the build compiles it, and the nvcc release."""
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    if not os.path.isfile(cuobjdump):
        pytest.skip('cuobjdump not found')
    version = re.search(r'release (\S+),', subprocess.run([nvcc, '--version'], capture_output=True, text=True).stdout).group(1)
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, 'dilated.cubin')
        ccbin = ['-ccbin', shutil.which('g++')] if shutil.which('g++') else []
        r = subprocess.run([nvcc] + ccbin + build.NVCC_FLAGS + ['-cubin', '-o', cubin, os.path.join(build.CSRC, 'cspn2d_dilated.cu')],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines(keepends=True):
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            name = _anonymous(m.group(1))
            kernels[name] = ''
        elif name:
            kernels[name] += line
    return kernels, version


def test_dilated_kernels_keep_their_machine_code():
    """The dilated step, adjoint and finalize kernels read their tile helpers from cspn2d_stencil.cuh, shared with the
    dynamic propagation; their SASS is the SASS recorded before the move (tests/golden/cspn2d_dilated_sass_sm90a.json)."""
    golden = json.load(open(os.path.join(HERE, 'golden', 'cspn2d_dilated_sass_sm90a.json')))
    kernels, version = dilated_sass()
    if version != golden['nvcc']:
        pytest.skip(f'the recorded machine code is from nvcc {golden["nvcc"]}, this is {version}')
    assert sorted(kernels) == sorted(golden['kernels'])
    changed = [k for k, h in golden['kernels'].items() if hashlib.sha256(kernels[k].encode()).hexdigest() != h]
    assert not changed, changed
