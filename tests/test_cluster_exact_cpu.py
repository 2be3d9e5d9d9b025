"""The premises of tests/test_cluster_exact_gpu.py, checked without a GPU: the explicit fp64 reference is fp64 autograd,
every GPU case is exact, the blind spot those cases close is real, and the cases reach every part of the cluster plan."""
import copy

import numpy as np
import pytest
import torch

from cspn_b200 import _lib
from cspn_b200.synth import make_inputs
from oracle import cspn_numpy as onp, cspn_torch_port as tp

import backward_exact as be
import cluster_exact as ce
import forced_plans as fpl
from test_plan_cpu import replay, replay_chained


# ---- 1. the explicit reference is fp64 autograd ------------------------------------------------------------------------
@pytest.mark.parametrize('norm', fpl.NORMS)
@pytest.mark.parametrize('sparse', [None, 'bernoulli', 'signed'])
@pytest.mark.parametrize('inputs', ['random', 'dyadic'])
def test_explicit_reference_is_fp64_autograd(inputs, sparse, norm):
    N = 7
    if inputs == 'random':
        g, d, s = make_inputs(len(norm) + N, 2, 2, 13, 18, 9, sparse, 25)
        go = torch.randn(2, 2, 13, 18, generator=torch.Generator().manual_seed(3))
    else:
        g, d, s, go = be.dyadic_2d(11, 2, 2, 13, 18, 3, sparse, 9)
    s64 = None if s is None else s.double()
    ours = ce.reference(g.double(), d.double(), s64, N, norm, go.double())
    refs = [lambda a, b: be.cspn2d_shift_ref(a, b, s64, N, 3, norm)]
    if inputs == 'random':      # the torch port's padded grid gives 0/0 in autograd where the guidance has zeros
        refs.append(lambda a, b: tp.cspn2d_torch(a, b, s64, N, norm))
    for ref in refs:
        theirs = be.autograd(ref, g, d, go, torch.float64)
        for x, y, name in zip(ours, theirs, ('out', 'grad_guidance', 'grad_blur')):
            assert torch.isfinite(x).all(), name
            err = float((x - y).abs().max())
            assert err <= 1e-12 * max(1.0, float(y.abs().max())), (inputs, sparse, norm, name, err)


# ---- 2. every GPU case is exact --------------------------------------------------------------------------------------
def all_cases():
    return ce.FORCED + ce.LONG + ce.PERSISTENT + ce.CHAIN + ce.ROUTES


def persistent_batch(case, monkeypatch):
    """The batch test_later_rounds_of_persistent_clusters_are_exact picks, here from the planner's occupancy table."""
    (e,) = case.envs
    ce.apply(monkeypatch, e)
    B = ce.batch_for_rounds(_lib.plan_info(case.H, case.W, case.n), case.C)
    info = ce.plan_of(e, B, case.C, case.H, case.W, case.n)
    B = max(B, ce.batch_for_rounds(info, case.C))
    return B, ce.plan_of(e, B, case.C, case.H, case.W, case.n)


CASES = all_cases()


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c.name for c in CASES])
def test_every_gpu_case_is_exact(i, monkeypatch):
    """fp64 and fp32 runs of the reference give the same bits on the grid of ce.unit, inside 24 bits, with a nonzero
    output and, for a backward case, nonzero gradients in both inputs (guidance channels >= 8 are never read: zero)."""
    case = CASES[i]
    B = persistent_batch(case, monkeypatch)[0] if case.B is None else case.B
    g, d, s, go = ce.inputs(case, B)
    runs = []
    for dt in (torch.float64, torch.float32):
        cast = lambda t: None if t is None else t.to(dt)
        r = ce.reference(cast(g), cast(d), cast(s), case.n, case.norm, cast(go) if case.bwd else None)
        runs.append([t.double() for t in (r if case.bwd else (r,))])
    ce.check_exact(runs[0], case.family, case.n, case.name)
    for a, b, name in zip(*runs, ('out', 'grad_guidance', 'grad_blur')):
        assert torch.equal(a, b), f'{case.name} {name}: fp32 and fp64 runs of the reference differ'
    assert torch.count_nonzero(runs[0][0])
    if case.bwd:
        out, gg, gd = runs[0]
        assert torch.count_nonzero(gd), case.name
        assert torch.count_nonzero(gg[:, :8]) and not torch.count_nonzero(gg[:, 8:]), case.name


# ---- 3. the gap is real -----------------------------------------------------------------------------------------------
def one_short(info, axis):
    """The plan with every interior tile of `axis` ('strips' or 'bands') starting one position later: its halo on the
    cut side is one short, the useful ranges are unchanged."""
    bad = copy.deepcopy(info)
    for p in bad['passes']:
        p[axis] = [[t0 + 1 if t0 > 0 else t0, u0, u1] for t0, u0, u1 in p[axis]]
    return bad


def single_pass(monkeypatch, H, W, n, chained=False):
    monkeypatch.setenv('CSPN_B200_FORCE_PASSES', '1')
    for k in ('CSPN_B200_FORCE_CFG', 'CSPN_B200_FORCE_CS'):
        monkeypatch.delenv(k, raising=False)
    info = _lib.plan_info(H, W, n, chained)
    (p,) = info['passes']
    assert p['count'] == 1
    return info


GAPS = [('strip halo one column short', 40, 516, 'strips'), ('band one row short', 700, 132, 'bands'),
        ('chained history one step late', 40, 516, 'chain')]


@pytest.mark.parametrize('what,H,W,axis', GAPS, ids=[g[0] for g in GAPS])
def test_an_off_by_one_plan_passes_parity_on_random_gates_but_not_on_directed_taps(what, H, W, axis, monkeypatch):
    """A plan perturbed by one, replayed on the oracle at N = 24 in one pass: on random gates (cspn_b200.synth) it still
    passes parity_ok(1e-4), the bound of the tolerance tests; on directed taps it is wrong in at least one bit."""
    N, norm = 24, '8sum'
    info = single_pass(monkeypatch, H, W, N, axis == 'chain')
    if axis == 'chain':
        good = lambda *a: replay_chained(info, *a)
        bad = lambda *a: replay_chained(info, *a, lag=1)
    else:
        assert len(info['passes'][0][axis]) > 1, info
        good = lambda *a: replay(info, *a)
        bad = lambda *a: replay(one_short(info, axis), *a)
    g, d, s = make_inputs(H + W, 1, 1, H, W, 8, 'bernoulli', H * W // 20)
    g, d, s = g.numpy(), d.numpy(), s.numpy()
    ref = onp.cspn2d(g, d, s, N, norm, dtype=np.float64)
    out = bad(g, d, s, norm)
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (what, 'random gates: the perturbed plan already fails parity', ratio, normwise)
    g, d, s, _ = ce.directed(H * W, 8, 1, H, W, 8, 'bernoulli')
    g, d, s = g.numpy().astype(np.float64), d.numpy().astype(np.float64), s.numpy().astype(np.float64)
    ref = onp.cspn2d(g, d, s, N, norm, dtype=np.float64)
    assert np.array_equal(good(g, d, s, norm), ref), what
    assert not np.array_equal(bad(g, d, s, norm), ref), (what, 'directed taps do not see the perturbed plan')


# ---- 4. coverage ------------------------------------------------------------------------------------------------------
def plans_of_gpu_cases(monkeypatch):
    """(case, forward plan_info, B) of every forward call the GPU file makes, under the planner's occupancy table."""
    out = []
    for case in CASES:
        if case.envs is None:                                   # the forced-plan matrix
            for plan in fpl.PROBLEMS[case.problem].fwd:
                fpl.force(monkeypatch, plan)
                out.append((case, fpl.plan_info(plan, case.H, case.W, case.n), case.B))
            continue
        if case.B is None:
            B, info = persistent_batch(case, monkeypatch)
            out.append((case, info, B))
            continue
        for e in case.envs:
            ce.apply(monkeypatch, e)
            if case.W % 4:
                continue
            out.append((case, ce.plan_of(e, case.B, case.C, case.H, case.W, case.n), case.B))
    return out


def test_the_gpu_cases_reach_every_part_of_the_plan(monkeypatch):
    seen = set()
    for case, info, B in plans_of_gpu_cases(monkeypatch):
        assert info['supported'], (case.name, info)
        passes = sum(p['count'] for p in info['passes'])
        for p in info['passes']:
            ci = fpl.CONFIGS.index((p['PR'], p['NW']))
            seen |= {f'cfg{ci}', f'cs{p["cs"]}', 'passes1' if passes == 1 else ('passes3+' if passes >= 3 else 'passes2')}
            if len(p['bands']) > 1:
                seen.add('bands')
            if info['chained']:
                seen.add(f'chained_cfg{ci}')
        if min(ce.rounds(info, B, case.C)) >= 3:
            seen.add(f'rounds3+_{case.name}')
        if passes == 1 and case.n == 24 and case.family == 'directed':
            seen.add('single_pass_n24')
        if case.sparse == 'signed':
            seen.add(f'signed_{case.family}')
    need = {f'cfg{ci}' for ci in range(len(fpl.CONFIGS))} | {'cs1', 'cs16', 'passes1', 'passes3+', 'bands'}
    need |= {f'chained_cfg{ci}' for ci in fpl.CHAINED} | {f'rounds3+_{c.name}' for c in ce.PERSISTENT} | {'single_pass_n24'}
    need |= {f'signed_{f}' for f in ce.FAMILIES}
    assert need <= seen, sorted(need - seen)

