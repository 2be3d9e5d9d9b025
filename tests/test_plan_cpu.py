"""The cluster path's planner, checked on the CPU: geometry invariants of every plan, and a replay of the plan
(passes x bands x strips, each tile iterated in isolation with zero boundaries, useful region kept) on the numpy
oracle, which must reproduce the untiled result.  This is the halo argument of cspn2d_cluster.cu, executed."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import forced_plans as fpl
from conftest import load_golden
from cspn_b200 import _lib
from oracle import cspn_numpy as onp


def check_axis(tiles, L, T, halo, align, chained=False):
    """tiles = [[t0, u0, u1], ...] must partition [0, L) into useful ranges, each inside its tile minus the halo.
    Chained tiles get their left neighbour column handed over: their left edge is exact and starts the useful range."""
    assert tiles[0][1] == 0 and tiles[-1][2] == L
    for i, (t0, u0, u1) in enumerate(tiles):
        assert t0 % align == 0 and u0 % align == 0 and t0 >= 0
        assert u0 < u1
        if i:
            assert u0 == tiles[i - 1][2]                       # no gap, no overlap of stored ranges
        assert t0 <= u0 and u1 <= t0 + T                       # stored range inside the tile
        if chained:
            assert u0 == t0
        elif t0 > 0:
            assert u0 - t0 >= halo                             # a cut side keeps >= halo stale positions out
        if t0 + T < L:
            assert t0 + T - u1 >= halo


def check_plan(H, W, n, chained=False):
    info = _lib.plan_info(H, W, n, chained)
    if chained and not info['supported']:
        return info
    assert info['supported'], info
    assert info['chained'] == chained
    assert sum(p['count'] * p['iters'] for p in info['passes']) == n
    for p in info['passes']:
        assert 1 <= p['cs'] <= 16 and p['RB'] == p['PR'] * p['NW'] and p['TW'] == 128
        assert len(p['strips']) <= 128 and len(p['bands']) <= 64
        check_axis(p['strips'], W, p['TW'], p['iters'], 4, chained)
        check_axis(p['bands'], H, p['cs'] * p['RB'], p['iters'], 1)
        if chained:
            assert len(p['bands']) == 1 and len(p['strips']) >= 2 and p['iters'] <= 32 and p['NW'] == 8
    return info


@pytest.mark.parametrize('H,W,n', [(352, 1216, 24), (228, 304, 48), (228, 304, 4), (1080, 1920, 24), (24, 512, 70),
                                   (2000, 2000, 100), (3, 4, 2), (700, 64, 4), (1, 4, 1), (641, 128, 56), (40, 4096, 3000)])
def test_plan_geometry_for_named_shapes(H, W, n):
    check_plan(H, W, n)


@settings(max_examples=150, deadline=None)
@given(H=st.integers(1, 3000), W4=st.integers(1, 700), n=st.integers(1, 400))
def test_plan_geometry_for_random_shapes(H, W4, n):
    check_plan(H, 4 * W4, n)
    check_plan(H, 4 * W4, n, chained=True)


def test_headline_shape_chains_into_twelve_strips():
    info = check_plan(352, 1216, 24, chained=True)
    (p,) = info['passes']
    assert p['count'] == 1 and len(p['strips']) == 12 and p['strips'][1][0] == 104


def test_headline_shape_is_a_single_pass_single_band_plan():
    info = check_plan(352, 1216, 24)
    (p,) = info['passes']
    assert p['count'] == 1 and len(p['bands']) == 1 and p['cs'] * p['RB'] >= 352 and len(p['strips']) == 15


def replay_chained(info, guidance, blur, sparse, norm, lag=0):
    """Chained plan on the numpy oracle: strips left to right; a strip's column -1 is, at every step, what the strip to its
    left computed there (its history), so only the right edge goes stale.  `lag` > 0 hands the history over that many
    steps late (zeros before), a deliberately wrong plan for tests/test_cluster_exact_cpu.py."""
    f64 = np.float64
    gate_wb, gate_sum = onp.affinity_normalization_2d(guidance.astype(f64), norm)
    raw = blur.astype(f64)
    mask = None if sparse is None else onp.sparse_mask(sparse, f64)
    H, W = raw.shape[-2:]
    cur = raw
    for p in info['passes']:
        for _ in range(p['count']):
            nxt = np.full_like(cur, np.nan)
            hist = None                                          # [step] -> column (..., H, 1) left of the current strip
            for i, (tx0, ux0, ux1) in enumerate(p['strips']):
                xs = slice(tx0, min(tx0 + p['TW'], W))
                d, d0 = cur[..., xs], raw[..., xs]
                w, s = gate_wb[..., xs], gate_sum[..., xs]
                m = None if mask is None else mask[..., xs]
                rec = ux1 - 1 - tx0                              # tile column recorded for the next strip
                new_hist = []
                with np.errstate(invalid='ignore'):
                    for t in range(p['iters']):
                        new_hist.append(d[..., rec:rec + 1].copy())
                        left = hist[t - lag] if hist is not None and t >= lag else np.zeros_like(d[..., :1])
                        ext = np.concatenate([left, d], axis=-1)             # column -1 in front: exact, not zero
                        acc = np.zeros_like(d)
                        for k, (dy, dx) in enumerate(onp.OFFSETS_2D):
                            acc = acc + w[:, k:k + 1] * onp.shift2d(ext, dy, dx)[..., 1:]
                        d = (1.0 - s) * d0 + acc
                        if m is not None:
                            d = (1.0 - m) * d + m * d0
                nxt[..., ux0:ux1] = d[..., ux0 - tx0:ux1 - tx0]
                hist = new_hist
            cur = nxt
    return cur


def replay(info, guidance, blur, sparse, norm):
    """Runs the plan on the numpy oracle in float64, tile by tile."""
    f64 = np.float64
    gate_wb, gate_sum = onp.affinity_normalization_2d(guidance.astype(f64), norm)
    raw = blur.astype(f64)
    mask = None if sparse is None else onp.sparse_mask(sparse, f64)
    H, W = raw.shape[-2:]
    cur = raw
    for p in info['passes']:
        CH = p['cs'] * p['RB']
        for _ in range(p['count']):
            nxt = np.full_like(cur, np.nan)
            for by0, uy0, uy1 in p['bands']:
                for tx0, ux0, ux1 in p['strips']:
                    ys, xs = slice(by0, min(by0 + CH, H)), slice(tx0, min(tx0 + p['TW'], W))
                    d, d0 = cur[..., ys, xs], raw[..., ys, xs]
                    w, s = gate_wb[..., ys, xs], gate_sum[..., ys, xs]
                    m = None if mask is None else mask[..., ys, xs]
                    with np.errstate(invalid='ignore'):
                        for _ in range(p['iters']):            # zero outside the tile: shift2d pads with zeros
                            acc = np.zeros_like(d)
                            for k, (dy, dx) in enumerate(onp.OFFSETS_2D):
                                acc = acc + w[:, k:k + 1] * onp.shift2d(d, dy, dx)
                            d = (1.0 - s) * d0 + acc
                            if m is not None:
                                d = (1.0 - m) * d + m * d0
                    nxt[..., uy0:uy1, ux0:ux1] = d[..., uy0 - by0:uy1 - by0, ux0 - tx0:ux1 - tx0]
            cur = nxt
    return cur


@pytest.mark.parametrize('H,W,n,norm,with_sparse', [
    (50, 300, 10, '8sum', True),        # strips with halos, one band
    (60, 260, 45, '8sum_abs', False),   # several passes
    (700, 64, 6, '8sum', True),         # row bands
    (660, 260, 20, '8sum', True),       # bands x strips
    (33, 132, 131, '8sum', True),       # passes of unequal length
])
def test_replaying_the_plan_on_the_oracle_reproduces_the_untiled_result(H, W, n, norm, with_sparse):
    rng = np.random.default_rng(H * 31 + W + n)
    g = rng.standard_normal((1, 8, H, W))
    d = rng.uniform(0, 10, (1, 2, H, W))
    s = None
    if with_sparse:
        s = rng.uniform(-1, 10, (1, 1, H, W)) * (rng.uniform(size=(1, 1, H, W)) < 0.02)
    info = check_plan(H, W, n)
    ref = onp.cspn2d(g, d, s, n, norm, dtype=np.float64)
    out = replay(info, g, d, s, norm)
    assert not np.isnan(out).any()
    np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12)
    cinfo = check_plan(H, W, n, chained=True)
    if cinfo['supported']:
        out = replay_chained(cinfo, g, d, s, norm)
        assert not np.isnan(out).any()
        np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12)


# ---- the forced-plan matrix of tests/test_forced_plans_gpu.py (tests/forced_plans.py), checked without a GPU ----------

@pytest.mark.parametrize('index', range(len(fpl.CONFIGS) + 1))
def test_forced_configuration_index_gives_the_pinned_menu(index, monkeypatch):
    """configs() of cspn2d_cluster.cu is exactly the menu the forced-plan matrix covers: a configuration added there
    fails here until tests/forced_plans.py covers it."""
    monkeypatch.setenv('CSPN_B200_FORCE_CFG', str(index))
    info = _lib.plan_info(37, 260, 7)
    chained = _lib.plan_info(37, 260, 7, True)
    if index == len(fpl.CONFIGS):
        assert not info['supported'] and not chained['supported']
        return
    assert {(p['PR'], p['NW']) for p in info['passes']} == {fpl.CONFIGS[index]}
    assert chained['supported'] == (index in fpl.CHAINED)


@pytest.mark.parametrize('name', sorted(fpl.PROBLEMS))
def test_forced_matrix_is_honoured_and_replays_on_the_oracle(name, monkeypatch):
    """Every forced combination of the GPU matrix is a valid plan of the forced shape (the H100 can then only refuse it
    through its occupancy query), and replaying it tile by tile reproduces the untiled result."""
    pb = fpl.PROBLEMS[name]
    rng = np.random.default_rng(pb.H + pb.n)
    g = rng.standard_normal((1, 8, pb.H, pb.W))
    d = rng.uniform(0, 10, (1, 1, pb.H, pb.W))
    s = None
    if pb.sparse:
        s = rng.uniform(-1 if pb.sparse == 'signed' else 0, 10, (1, 1, pb.H, pb.W)) * (rng.uniform(size=d.shape) < 0.05)
    ref = onp.cspn2d(g, d, s, pb.n, pb.norm, dtype=np.float64)
    for plan in dict.fromkeys(pb.fwd + pb.bwd):
        fpl.force(monkeypatch, plan)
        info = check_plan(pb.H, pb.W, pb.n, fpl.chains(plan))
        fpl.check_honoured(plan, info)
        banded = any(len(p['bands']) > 1 for p in info['passes'])
        assert banded == (plan.cs * fpl.rows(plan.cfg) < pb.H), plan
        out = (replay_chained if fpl.chains(plan) else replay)(info, g, d, s, pb.norm)
        np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12, err_msg=str(plan))


def test_special_value_and_nan_patch_plans_are_honoured(monkeypatch):
    cases = []
    for name in fpl.SPECIAL:
        c = load_golden(name)
        H, W = c['blur'].shape[-2:]
        cases.append((H, W, c['prop_time'], fpl.special_plans(name, H)))
    cases += [(12, 16, n, fpl.NAN_PATCH_PLANS) for n in (1, 2, 3)]
    for H, W, n, plans in cases:
        for plan in plans:
            fpl.force(monkeypatch, plan)
            fpl.check_honoured(plan, check_plan(H, W, n))


def test_forced_matrix_reaches_every_configuration_in_every_mode(monkeypatch):
    """The axes every configuration must meet at least once (forward, chained, backward), read off the plans the planner
    makes for the matrix."""
    seen = {ci: set() for ci in range(len(fpl.CONFIGS))}
    for pb in fpl.PROBLEMS.values():
        for kind, plans in (('fwd', pb.fwd), ('bwd', pb.bwd)):
            for plan in plans:
                fpl.force(monkeypatch, plan)
                info = fpl.plan_info(plan, pb.H, pb.W, pb.n)
                n_pass = fpl.check_honoured(plan, info)
                banded = any(len(p['bands']) > 1 for p in info['passes'])
                unequal = len({p['iters'] for p in info['passes']}) > 1
                tags = {f'cs{plan.cs}' if plan.cs in (1, 16) else 'cs_mid'}
                tags |= {'banded'} if banded else ({'cs16_one_band'} if plan.cs == 16 else set())
                tags |= {f'{n_pass}_unequal_passes'} if unequal else set()
                tags |= {'bands_x_passes'} if banded and n_pass > 1 else set()
                tags |= {'general'} if banded or n_pass > 1 else {'plain'}
                tags |= {'strips'} if len(info['passes'][0]['strips']) > 1 else set()
                tags |= {pb.norm, f'sparse_{pb.sparse}', f'C{pb.C}', f'gch{pb.gch}'}
                if plan.chain:
                    tags = {f'chained_{t}' for t in tags} if fpl.chains(plan) else {'chain_falls_back'}
                seen[plan.cfg] |= {f'{kind}_{t}' for t in tags}
    axes = {'cs1', 'cs_mid', 'cs16', 'cs16_one_band', 'banded', '2_unequal_passes', '3_unequal_passes', 'bands_x_passes',
            'general', 'plain', 'strips', '8sum', '8sum_abs', 'sparse_signed', 'sparse_None', 'C2', 'gch9'}
    fwd = {f'fwd_{a}' for a in axes}
    bwd = {f'bwd_{a}' for a in ('cs1', 'cs_mid', 'cs16_one_band', 'banded', '3_unequal_passes', 'bands_x_passes', 'C2')}
    chained = {'fwd_chained_cs1', 'fwd_chained_cs16', 'fwd_chained_2_unequal_passes', 'fwd_chained_8sum', 'fwd_chained_8sum_abs'}
    for ci in seen:
        need = fwd | bwd | (chained if ci in fpl.CHAINED else {'fwd_chain_falls_back'})
        assert need <= seen[ci], (fpl.CONFIGS[ci], sorted(need - seen[ci]))
