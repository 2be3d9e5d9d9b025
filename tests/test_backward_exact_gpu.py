"""The backward of the K x K (2D, K = 3, 5, 7) and K x K x K (3D, K = 3, 5) propagation across CTA tiles.

Every backward kernel stages a tile plus an R-pixel halo in shared memory (32 x 8 per plane in the adjoint and gather
kernels, 64 x 16 in the vectorised recompute), so a gradient is only checked where a test makes one CTA read a halo that a
neighbouring tile owns.  These tests run at shapes that cross the tile boundaries of both tilings, with ragged last tiles,
odd widths and misaligned views, and check:
  - on dyadic inputs (tests/backward_exact.py) `out`, `grad_guidance` and `grad_blur` / `grad_feat` bit for bit against
    fp64 autograd of a reference, through the dispatcher op and the ctypes autograd.Function;
  - one hot tap at every site, tap by tap, also bit for bit;
  - random gates against fp64 autograd, to 2e-3 scale-relative at N = 24 and to 1e-4 with positive gates at N = 2;
  - that only one input requiring a gradient, and a non-contiguous grad_out, give the bits of the plain call.
"""
import pytest
import torch

import cspn_b200
from cspn_b200 import torch_op
from cspn_b200.synth import make_inputs

import backward_exact as be

pytestmark = pytest.mark.gpu

ROUTES = (False, True)          # the ctypes autograd.Function, then the dispatcher op


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary (a leaf: it can require grad)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def module(nd, N, K, norm, use_op):
    m = cspn_b200.Affinity_PropagateK(N, K, norm) if nd == 2 else cspn_b200.Affinity_Propagate3DK(N, K, norm)
    if use_op:
        torch_op.load()
    m._use_op = use_op
    return m


def run(m, g, x, go, s=None, misaligned=False, need=(True, True)):
    """(out, guidance.grad, x.grad) of module m on the GPU, grad_out = go."""
    dev = [None if t is None else t.cuda() for t in (g, x, s, go)]
    if misaligned:
        dev = [None if t is None else misaligned_copy(t) for t in dev]
    gc, xc, sc, goc = dev
    gc.requires_grad_(need[0])
    xc.requires_grad_(need[1])
    out = m(gc, xc, sc) if isinstance(m, cspn_b200.Affinity_PropagateK) else m(gc, xc)
    out.backward(goc)
    return out.detach(), gc.grad, xc.grad


def assert_bits(ours, ref, case):
    for a, b, name in zip(ours, ref, ('out', 'grad_guidance', 'grad_x')):
        a = a.double().cpu()
        bad = a != b
        assert not bad.any(), (case, name, f'{int(bad.sum())} of {bad.numel()} differ, first at '
                                            f'{tuple(bad.nonzero()[0].tolist())}', float((a - b).abs().max()))


# ---- 1. exact matrix ------------------------------------------------------------------------------------------------
CASES_2D = be.cases_2d()
CASES_3D = be.cases_3d()


@pytest.mark.parametrize('i', range(len(CASES_2D)), ids=[be.case_id(c) for c in CASES_2D])
def test_2d_backward_is_exact_on_dyadic_inputs(i):
    c = CASES_2D[i]
    (K, norm), (H, W), (B, C), N = c['path'], c['hw'], c['bc'], c['N']
    g, d, s, go = be.dyadic_2d(1000 + i, B, C, H, W, K, c['sparse'], K * K + 2 if c['extra_channels'] else None)
    ref = be.exact_reference(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, s, N, K, norm), g, d, go, N)
    for use_op in ROUTES:
        ours = run(module(2, N, K, norm, use_op), g, d, go, s, c['misaligned'])
        assert_bits(ours, ref, (be.case_id(c), use_op))
        if c['extra_channels']:
            assert torch.count_nonzero(ours[1][:, K * K - 1:]) == 0


@pytest.mark.parametrize('i', range(len(CASES_3D)), ids=[be.case_id(c) for c in CASES_3D])
def test_3d_backward_is_exact_on_dyadic_inputs(i):
    c = CASES_3D[i]
    (K, norm), (D, H, W), (B, C), N = c['path'], c['dhw'], c['bc'], c['N']
    g, f, go = be.dyadic_3d(2000 + i, B, C, D, H, W, K, norm, c['per_channel'])
    ref = be.exact_reference(lambda gg, ff: be.cspn3d_ref(gg, ff, N, K, norm), g, f, go, N)
    for use_op in ROUTES:
        assert_bits(run(module(3, N, K, norm, use_op), g, f, go, misaligned=c['misaligned']), ref, (be.case_id(c), use_op))


# ---- 2. one hot tap at every site, tap by tap ------------------------------------------------------------------------
# Item k of the batch has tap k hot at every site (reflected into the image where tap k would read the padding).  2D shapes
# of 2 x 2 tiles of 64 x 16 (W = 72: the vectorised recompute) or 3 x 3 of 32 x 8 (W = 70: the scalar one).
@pytest.mark.parametrize('K,norm', [(K, n) for K in (5, 7) for n in be.norms_2d(K)])
@pytest.mark.parametrize('W', [72, 70])
def test_2d_one_hot_tap_sweep_is_exact(K, norm, W):
    H, N, C = 20, 2, 2
    g = be.one_tap_guidance(K + W, (H, W), K, True)
    gen = torch.Generator().manual_seed(K * W)
    d, go = be.small_ints(gen, (g.shape[0], C, H, W)), be.small_ints(gen, (g.shape[0], C, H, W))
    ref = be.exact_reference(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, None, N, K, norm), g, d, go, N)
    for use_op in ROUTES:
        assert_bits(run(module(2, N, K, norm, use_op), g, d, go), ref, (K, norm, W, use_op))


@pytest.mark.parametrize('K,norm', [(3, n) for n in be.norms_3d(3)] + [(5, '124sum'), (5, '124sum_abs')])
def test_3d_one_hot_tap_sweep_is_exact(K, norm):
    """2 x 2 tiles of 32 x 8 in every z-plane.  One tap per site (S = 1) is exact by itself: the reference runs in fp64 only."""
    D, H, W, N, C = 5, 9, 36, 2, 1
    g = be.one_tap_guidance(K, (D, H, W), K, norm != 'paddle')
    gen = torch.Generator().manual_seed(K)
    f, go = be.small_ints(gen, (g.shape[0], C, D, H, W)), be.small_ints(gen, (g.shape[0], C, D, H, W))
    chunk = 32                    # the fp64 reference of 124 volumes at once needs several GB
    ref = [torch.cat(t) for t in zip(*[
        be.exact_reference(lambda gg, ff: be.cspn3d_ref(gg, ff, N, K, norm), g[i:i + chunk], f[i:i + chunk],
                           go[i:i + chunk], N, fp32=False) for i in range(0, g.shape[0], chunk)])]
    for use_op in ROUTES:
        assert_bits(run(module(3, N, K, norm, use_op), g, f, go), ref, (K, norm, use_op))


# ---- 3. random gates at tile-crossing shapes ---------------------------------------------------------------------------
def assert_close(ours, ref, tol, case):
    for a, b, name in zip(ours[1:], ref[1:], ('grad_guidance', 'grad_x')):
        a = a.double().cpu()
        err = (a - b).abs()
        assert (err <= tol * (b.abs() + b.abs().mean())).all(), (case, name, float(err.max()), float(b.abs().mean()))


TOL_2D = [(K, be.norms_2d(K)[j], hw, sparse) for K in (5, 7) for hw in ((37, 136), (37, 133))
          for j, sparse in enumerate((None, 'bernoulli'))]


@pytest.mark.parametrize('K,norm,hw,sparse', TOL_2D)
def test_2d_gradients_match_fp64_autograd_across_tiles(K, norm, hw, sparse):
    (H, W), N = hw, 24
    g, d, s = make_inputs(K * 7 + W, 1, 2, H, W, K * K - 1, sparse, 60)
    go = torch.randn(1, 2, H, W, generator=torch.Generator().manual_seed(W))
    s64 = None if s is None else s.double()
    ref = be.autograd(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, s64, N, K, norm), g, d, go, torch.float64)
    for use_op in ROUTES:
        assert_close(run(module(2, N, K, norm, use_op), g, d, go, s), ref, 2e-3, (K, norm, hw, sparse, use_op))


@pytest.mark.parametrize('K,norm', [(K, n) for K in (3, 5) for n in be.norms_3d(K)])
@pytest.mark.parametrize('W', [72, 70])
def test_3d_gradients_match_fp64_autograd_across_tiles(K, norm, W):
    D, H, N = 7, 19, 6
    gen = torch.Generator().manual_seed(K * 100 + W)
    g = torch.randn(1, K ** 3 - 1, D, H, W, generator=gen) if norm.endswith('sum') else torch.rand(1, K ** 3 - 1, D, H, W, generator=gen)
    g = g + 0.05 * torch.sign(g)                                 # keep |g| away from the kink of abs
    f, go = torch.rand(1, 2, D, H, W, generator=gen), torch.randn(1, 2, D, H, W, generator=gen)
    ref = be.autograd(lambda gg, ff: be.cspn3d_ref(gg, ff, N, K, norm), g, f, go, torch.float64)
    for use_op in ROUTES:
        assert_close(run(module(3, N, K, norm, use_op), g, f, go), ref, 2e-3, (K, norm, W, use_op))


@pytest.mark.parametrize('K,norm,W', [(5, '24sum', 136), (5, '24sum_abs', 133), (7, '48sum', 133), (7, '48sum_abs', 136)])
def test_2d_gradients_of_positive_gates_match_fp64_autograd_to_1e_4(K, norm, W):
    """Positive gates and two steps: well conditioned, so fp32 holds 1e-4 scale-relative."""
    H, N = 37, 2
    gen = torch.Generator().manual_seed(K + W)
    g = torch.rand(1, K * K - 1, H, W, generator=gen) + 0.05
    d, go = torch.rand(1, 2, H, W, generator=gen), torch.randn(1, 2, H, W, generator=gen)
    ref = be.autograd(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, None, N, K, norm), g, d, go, torch.float64)
    for use_op in ROUTES:
        assert_close(run(module(2, N, K, norm, use_op), g, d, go), ref, 1e-4, (K, norm, W, use_op))


# ---- 4. partial gradients and a strided grad_out ----------------------------------------------------------------------
# The four backward entry points: cspn2d_bwd_f32 (K = 3), cspn2d_k_bwd_f32, cspn3d_bwd_f32 (K = 3) and cspn3d_k_bwd_f32.
ENTRY = [(2, 3, '8sum_abs'), (2, 5, '24sum'), (2, 7, '48sum_abs'), (3, 3, '26sum'), (3, 5, '124sum_abs'), (3, 5, 'paddle')]


@pytest.mark.parametrize('nd,K,norm', ENTRY)
@pytest.mark.parametrize('use_op', ROUTES)
def test_one_gradient_alone_and_a_strided_grad_out_give_the_same_bits(nd, K, norm, use_op):
    N = 3
    if nd == 2:
        g, x, s = make_inputs(K, 2, 2, 37, 136, K * K - 1, 'signed', 60)
        shape = (2, 2, 37, 136)
    else:
        gen = torch.Generator().manual_seed(K)
        g, x, s = torch.rand(2, K ** 3 - 1, 7, 19, 72, generator=gen) - 0.3, torch.rand(2, 2, 7, 19, 72, generator=gen), None
        shape = x.shape
    go = torch.randn(*shape, generator=torch.Generator().manual_seed(nd + K))
    m = module(nd, N, K, norm, use_op)
    out, gg, gx = run(m, g, x, go, s)
    _, only_g, none_x = run(m, g, x, go, s, need=(True, False))
    _, none_g, only_x = run(m, g, x, go, s, need=(False, True))
    assert none_x is None and none_g is None
    assert torch.equal(only_g, gg) and torch.equal(only_x, gx)
    # the same grad_out in a transposed memory layout
    strided = go.cuda().transpose(-1, -2).contiguous().transpose(-1, -2)
    gc, xc = g.cuda().requires_grad_(True), x.cuda().requires_grad_(True)
    o = m(gc, xc, s.cuda()) if nd == 2 else m(gc, xc)
    seen = []
    o.register_hook(lambda grad: seen.append(grad.is_contiguous()))
    o.backward(strided)
    assert seen == [False]                                      # it reached the operator's backward as it was
    assert torch.equal(o.detach(), out) and torch.equal(gc.grad, gg) and torch.equal(xc.grad, gx)
