"""The premises of tests/test_backward_exact_gpu.py, checked without a GPU: the shift-based fp64 2D reference is the torch
port's operator, the dyadic inputs keep fp32 autograd of both references bit-identical to fp64, the input builders keep
their contract, and the case matrix is pairwise."""
import itertools

import pytest
import torch

from cspn_b200.synth import make_inputs
from oracle import cspn_torch_port as tp
from oracle import cspn_torch_port_k as tpk

import backward_exact as be


def grads(fn, g, d, go):
    g, d = g.double().requires_grad_(True), d.double().requires_grad_(True)
    out = fn(g, d)
    out.backward(go.double())
    return out.detach(), g.grad, d.grad


def assert_close_1e12(a, b, what):
    for x, y, name in zip(a, b, ('out', 'grad_guidance', 'grad_blur')):
        assert torch.isfinite(x).all() and torch.isfinite(y).all(), (what, name)
        err = float((x - y).abs().max())
        assert err <= 1e-12 * max(1.0, float(y.abs().max())), (what, name, err)


@pytest.mark.parametrize('K,abs_norm,sparse', [(K, a, s) for K in (3, 5, 7) for a in (False, True)
                                               for s in (None, 'bernoulli', 'signed')])
def test_the_shift_reference_is_the_torch_port(K, abs_norm, sparse):
    """Forward and both gradients on random inputs, C = 1 or 3, with guidance channels beyond K*K-1."""
    nt = K * K - 1
    norm = f'{nt}sum_abs' if abs_norm else f'{nt}sum'
    C = 3 if (K + abs_norm) % 2 else 1
    g, d, s = make_inputs(K * 10 + abs_norm, 2, C, 11, 14, nt + 2, sparse, 30)
    s = None if s is None else s.double()
    go = torch.randn(2, C, 11, 14, generator=torch.Generator().manual_seed(K), dtype=torch.float64)
    ours = grads(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, s, 6, K, norm), g, d, go)
    assert_close_1e12(ours, grads(lambda gg, dd: tpk.cspn2d_torch_k(gg, dd, s, 6, K, norm), g, d, go), (K, norm, sparse))
    if K == 3:
        assert_close_1e12(ours, grads(lambda gg, dd: tp.cspn2d_torch(gg, dd, s, 6, norm), g, d, go), (K, norm, sparse))
    assert torch.count_nonzero(ours[1][:, nt:]) == 0


@pytest.mark.parametrize('K,norm,sparse', [(K, n, s) for K in (3, 5, 7) for n in be.norms_2d(K)
                                           for s in (None, 'bernoulli', 'signed')])
def test_dyadic_2d_inputs_keep_fp32_autograd_exact(K, norm, sparse):
    N = 3 if sparse == 'signed' else 4
    g, d, s, go = be.dyadic_2d(K, 2, 2, 19, 37, K, sparse, K * K + 2)
    out, gg, gd = be.exact_reference(lambda a, b: be.cspn2d_shift_ref(a, b, s, N, K, norm), g, d, go, N)
    assert torch.count_nonzero(gg) and torch.count_nonzero(gd)
    if sparse is not None:
        assert set(s.unique().tolist()) == ({-3.0, 0.0, 3.0} if sparse == 'signed' else {0.0, 3.0})


@pytest.mark.parametrize('K,norm', [(K, n) for K in (3, 5) for n in be.norms_3d(K)])
@pytest.mark.parametrize('per_channel', [False, True])
def test_dyadic_3d_inputs_keep_fp32_autograd_exact(K, norm, per_channel):
    N = 4
    g, f, go = be.dyadic_3d(K, 2, 2, 6, 9, 13, K, norm, per_channel)
    out, gg, gf = be.exact_reference(lambda a, b: be.cspn3d_ref(a, b, N, K, norm), g, f, go, N)
    assert torch.count_nonzero(gg) and torch.count_nonzero(gf)


def gates_at_sites(g, K, gathered):
    """(n, taps, *S): the value of tap k that site p reads, g_k(p + off_k) (gathered) or g_k(p) ('paddle')."""
    nd = g.dim() - 2
    offs = be.offsets(K, nd)
    g = g[:, :len(offs)]
    if not gathered:
        return g
    return torch.stack([be.shift(g[:, k], o, (K - 1) // 2) for k, o in enumerate(offs)], 1)


@pytest.mark.parametrize('nd,K,shape,gathered', [
    (2, 3, (19, 37), True), (2, 5, (1, 100), True), (2, 7, (100, 1), True), (2, 7, (5, 5), True), (2, 7, (9, 33), True),
    (3, 3, (3, 1, 100), True), (3, 5, (6, 9, 13), True), (3, 5, (3, 1, 5), True), (3, 3, (5, 9, 33), False),
    (3, 5, (2, 3, 4), False)])
def test_dyadic_guidance_contract(nd, K, shape, gathered):
    """m in {1, 2, 4} hot taps at every site, every one +-1 and inside, every nonzero guidance value read by exactly one
    site (the site reading g_k(q) is q - off_k: so every nonzero value is read by one site when as many are read as set)."""
    n = 3
    g = be.dyadic_guidance(torch.Generator().manual_seed(K), n, shape, K, gathered)
    a = gates_at_sites(g, K, gathered)
    m = (a != 0).sum(1)
    assert set(m.unique().tolist()) <= {1, 2, 4}
    assert set(a.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert torch.count_nonzero(a) == torch.count_nonzero(g)
    if gathered:
        assert not (a != 0)[:, ~be.inside(shape, be.offsets(K, nd))].any()
    if min(shape) > 1 or not gathered:
        assert set(m.unique().tolist()) == {1, 2, 4}


@pytest.mark.parametrize('nd,K,shape,gathered', [(2, 5, (20, 70), True), (2, 7, (7, 9), True), (3, 3, (3, 4, 5), True),
                                                 (3, 5, (5, 6, 7), True), (3, 5, (2, 3, 4), False)])
def test_one_tap_guidance_contract(nd, K, shape, gathered):
    """Item k: exactly one hot tap per site, inside; tap k wherever its source is inside, else a tap whose offset differs
    from off_k only in the sign of the components that leave the image."""
    g = be.one_tap_guidance(K, shape, K, gathered)
    a = gates_at_sites(g, K, gathered)
    offs = be.offsets(K, nd)
    valid = be.inside(shape, offs)
    assert ((a != 0).sum(1) == 1).all() and set(a.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert torch.count_nonzero(a) == torch.count_nonzero(g)
    hot = (a != 0).float().argmax(1)                            # (item k, *shape): the hot tap
    for k, off in enumerate(offs):
        if not gathered:
            assert (hot[k] == k).all()
            continue
        assert (hot[k][valid[k]] == k).all()
        assert valid.gather(0, hot[k].unsqueeze(0)).all()
        for j in hot[k][~valid[k]].unique().tolist():
            assert all(abs(x) == abs(y) for x, y in zip(offs[j], off)), (k, j)


@pytest.mark.parametrize('axes,cases', [(be.AXES_2D, be.cases_2d()), (be.AXES_3D, be.cases_3d())], ids=['2d', '3d'])
def test_the_exact_matrix_is_pairwise(axes, cases):
    allowed = be._allowed_2d if 'hw' in axes else be._allowed_3d
    for a, b in itertools.combinations(axes, 2):
        for va, vb in itertools.product(axes[a], axes[b]):
            possible = any(allowed(dict(c, **{a: va, b: vb})) for c in cases)
            seen = any(c[a] == va and c[b] == vb for c in cases)
            assert seen or not possible, (a, va, b, vb)
