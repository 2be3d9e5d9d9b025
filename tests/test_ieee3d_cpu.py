"""The premises of tests/test_ieee3d_gpu.py, without a GPU: each case of tests/ieee3d.py reaches what it claims (sums of
|gates| on both sides of every threshold the case is meant to straddle, special values where they are meant to be), the
scaled dyadic references are finite and exact, and the matrix covers every route."""
import numpy as np
import pytest
import torch

import ieee3d as ie

be = ie.be
PATHS = [(K, n) for K in (3, 5) for n in be.norms_3d(K)]
SHAPE = (1, 2, 6, 9, 136)        # B, C, D, H, W of the forward cases


def site_sums(K, norm, e, per_channel=False, seed=1):
    B, C, D, H, W = SHAPE
    g, f, go = ie.scaled_dyadic(seed, B, C, D, H, W, K, norm, e, per_channel)
    return g, f, go, ie.sums(g, K, norm)


@pytest.mark.parametrize('K,norm', PATHS)
@pytest.mark.parametrize('e', ie.EXPONENTS)
def test_scaled_sums_fall_where_the_exponent_claims(K, norm, e):
    g, f, _, S = site_sums(K, norm, e)
    S32 = S.float().double()
    assert torch.equal(S32[torch.isfinite(S32)], S[torch.isfinite(S32)]), 'a finite S is not exact in fp32'
    assert set(torch.unique(S / 2.0 ** e).tolist()) == {1.0, 2.0, 4.0}, 'every m in {1, 2, 4} occurs'
    cold = ~((S32 >= ie.FLT_MIN) & (S32 <= ie.FLT_MAX))           # cold_sum of cspn3d_wide.cu / common.cuh
    gather_cold = (1.0 / S32).float().double() > ie.GATHER_COLD     # 1 / S of step3d_gather_vec4_kernel
    if e <= -140:
        assert cold.all() and gather_cold.all() and (S > 0).all()
    elif e == -128:      # cold_sum: m = 1, 2 subnormal, m = 4 exactly FLT_MIN; the gather kernel: every 1 / S >= 2^126
        assert cold.any() and (~cold).any() and gather_cold.all()
    elif e == -127:      # both thresholds straddled
        assert cold.any() and (~cold).any() and gather_cold.any() and (~gather_cold).any()
    elif e == -126:      # S >= FLT_MIN everywhere, 1 / S = 2^126 > 8e37 at m = 1 only
        assert not cold.any() and gather_cold.any() and (~gather_cold).any()
    elif e == 127:       # S = 2^128 overflows at m >= 2, not at m = 1
        assert torch.isinf(S32).any() and torch.isfinite(S32).any() and not gather_cold.any()
        # 'paddle' divides sum_k |g_k| d once: at a site of m = 1 that sum overflows where |d| >= 2 (first step)
        if norm == 'paddle':
            nt = K ** 3 - 1
            acc = sum(g[:, k:k + 1].double().abs() * be.shift(f.double(), o, (K - 1) // 2)
                      for k, o in enumerate(ie.offsets_3d(K)))
            one = (torch.isfinite(S32)).unsqueeze(1).expand_as(acc)
            assert (acc[one].abs() > ie.FLT_MAX).any() and (acc[one].abs() <= ie.FLT_MAX).any(), nt
    else:
        assert not cold.any() and not gather_cold.any()


@pytest.mark.parametrize('K,norm', PATHS)
@pytest.mark.parametrize('e', ie.EXPONENTS)
def test_scaled_references_are_exact_and_match_plain_fp64_autograd(K, norm, e):
    """The fp64 reference lies on the case's grid (scaled_reference checks it) and, where no S overflows, is plain fp64
    autograd of backward_exact.cspn3d_ref bit for bit.  Where S overflows, w = 0 and kappa = 1 there, and the site's
    guidance gradient is 0."""
    N, (B, C, D, H, W) = 2, (1, 2, 5, 7, 12)
    g, f, go = ie.scaled_dyadic(7 + e, B, C, D, H, W, K, norm, e)
    ref = ie.scaled_reference(g, f, go, N, K, norm, e)
    S32 = ie.sums(g, K, norm).float()
    if torch.isfinite(S32).all():
        plain = be.autograd(lambda gg, ff: be.cspn3d_ref(gg, ff, N, K, norm), g, f, go, torch.float64)
        for a, b in zip(ref, plain):
            assert torch.equal(a, b)
    else:
        assert e == 127
        one = ie.ieee_ref(g.double(), f.double(), 1, K, norm)
        over = torch.isinf(S32).unsqueeze(1).expand_as(f)
        want = torch.zeros_like(one) if norm == 'paddle' else f.double()
        assert torch.equal(one[over], want[over])
        if norm == 'paddle':     # the guidance of a site is its own: its gradient is 0 where its S overflowed
            assert (ref[1][torch.isinf(S32).unsqueeze(1).expand_as(g)] == 0).all()


def test_the_rounding_of_s_passes_the_gradient_unchanged():
    s = torch.tensor([2.0 ** 128, 3.0, 2.0 ** -149], dtype=torch.float64, requires_grad=True)
    r = ie._RoundToF32.apply(s)
    assert r[0] == float('inf') and r[1] == 3.0 and r[2] == 2.0 ** -149
    r.backward(torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64))
    assert torch.equal(s.grad, torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64))


@pytest.mark.parametrize('K', (3, 5))
@pytest.mark.parametrize('kind', ie.SPECIAL)
def test_special_regions_reach_what_they_claim(K, kind):
    B, C, D, H, W = 2, 1, 6, 9, 136
    g, f = ie.special_gates(11, B, C, D, H, W, K, kind)
    for norm in be.norms_3d(K):
        S = ie.sums(g, K, norm).float()[0]
        cold = ~((S >= ie.FLT_MIN) & (S <= ie.FLT_MAX))
        quad = cold[..., :W // 4 * 4].reshape(D, H, W // 4, 4)
        mixed = quad.any(-1) & ~quad.all(-1)         # one lane cold, its neighbours not
        if kind in ('tiny', 'huge', 'zero'):
            assert mixed.any(), (norm, 'no quad straddles the threshold')
            assert mixed[..., 1].any() and mixed[..., 32].any(), (norm, 'edges in quads 1 and 32: either side of a warp row')
        if kind == 'huge':
            assert torch.isinf(S).any() and ((S > 1e38) & torch.isfinite(S)).any()
        if kind == 'tiny':
            assert ((S > 0) & (S < ie.FLT_MIN)).any()
        if kind == 'huge' and norm == 'paddle':       # finite S whose sum |g| d overflows: the acc side of cold_paddle
            acc = sum(g[0, k].double().abs() * be.shift(f[0, 0].double(), o, (K - 1) // 2)
                      for k, o in enumerate(ie.offsets_3d(K)))
            assert ((acc.abs() > ie.FLT_MAX) & torch.isfinite(S)).any()
        if kind == 'zero':
            assert (S == 0).any()
        if kind == 'inf':
            assert torch.isinf(S).any()
        if kind == 'nan':
            assert torch.isnan(S).any()
    ref = ie.oracle(g.numpy(), f.numpy(), 2, K, be.norms_3d(K)[-1])
    assert not np.isfinite(ref).all() or kind in ('tiny', 'huge'), kind


@pytest.mark.parametrize('value', ie.NONFINITE)
def test_nonfinite_feat_sits_at_corners_faces_interior_and_every_lane(value):
    D, H, W = 6, 9, 136
    sites = ie.nonfinite_sites(D, H, W)
    g, f = ie.nonfinite_feat(3, 2, D, H, W, 3, value)
    assert f.shape[0] == len(sites)
    for b, (z, y, x) in enumerate(sites):
        bad = ~torch.isfinite(f[b])
        assert int(bad.sum()) == 1 and bool(bad[b % 2, z, y, x])
    zs, ys, xs = zip(*sites)
    assert {0, D - 1} <= set(zs) and {0, H - 1} <= set(ys) and {0, W - 1} <= set(xs)
    assert {x % 4 for z, y, x in sites if 0 < z < D - 1 and 0 < y < H - 1 and 0 < x < W - 1} == {0, 1, 2, 3}
    ref = ie.oracle(g.numpy(), f.numpy(), 1, 3, 'paddle')
    assert (~np.isfinite(ref)).any()


def test_the_matrix_covers_every_route_norm_exponent_and_gate_layout():
    for K, routes in ((3, ie.ROUTES_3), (5, ie.ROUTES_5)):
        for norm in be.norms_3d(K):
            for route in routes:
                seen = [c for c in ie.scaled_cases() if c['path'] == (K, norm, route)]
                assert {c['e'] for c in seen} == set(ie.EXPONENTS), (K, norm, route)
                if route != 'bcd':
                    assert {c['kind'] for c in ie.special_cases() if c['path'] == (K, norm, route)} == \
                        set(ie.SPECIAL_AXES['kind']), (K, norm, route)
    for axis in ('gates', 'N', 'api'):
        assert {c[axis] for c in ie.scaled_cases()} == set(ie.SCALED_AXES[axis])
    bwd = ie.backward_cases()
    for path in ie.BACKWARD_AXES['path']:
        assert {c['e'] for c in bwd if c['path'] == path} == set(ie.EXPONENTS)
        assert {c['dhw'] for c in bwd if c['path'] == path} == set(ie.BACKWARD_AXES['dhw'])


@pytest.mark.parametrize('route', ie.ROUTES_3)
def test_each_route_takes_its_branch_of_generic3d_forward(route):
    """The conditions of cspn3d.cu's generic3d_forward, restated: W % 4 and alignment pick the raw-guidance route, which
    also needs B * C * D <= 65535; group3d's cap makes 'groups' run in ragged groups."""
    B, D, H = ie.route_dims(route, 6, 9)
    W, C, N = ie.W_OF[route], 1, 2
    paddle_env, ws_env = ie.route_env(route, B, C, D, H, W, N)
    raw = W % 4 == 0 and route not in ('misaligned', 'planes') and B * C * D <= 65535
    assert raw == (route == 'raw')
    if route == 'bcd':
        assert B * C * D > 65535 and W % 4 == 0 and paddle_env is None and ws_env is None
        G = 65535 // (D * C)
        assert B > G and B % G != 0
    if route == 'groups':
        per_vol = 4 * (27 + C) * D * H * W
        G = int(float(ws_env) * 1024 // per_vol)
        assert 1 < G < B and B % G != 0
    if route == 'planes':
        assert paddle_env == 'planes'
