"""The 3x3 2D cluster kernel bit for bit against the explicit fp64 reference of tests/cluster_exact.py, under every plan:
the forced-plan matrix, long runs (N = 24, 48, 80) in 1, 2, 3 and an uneven number of passes, >= 3 rounds of the
persistent task loop, chained strips in every chain grouping, and every other route of the 3x3 operator.

On these inputs every value is a short dyadic rational, so the kernels must return the reference's bits: a halo one
column short, a useful range one column wide, a history handed over one step late or a staging buffer reused too early
is a wrong number at a pixel, not an error of 1e-11 under a tolerance.  Outputs and gradients of the C ABI calls sit in
sentinel-filled guarded buffers (tests/memory_contract.py).  A mismatch names the first differing pixel and where it lies
in the plan (strip, band, CTA, warp, patch row, lane, column, distance from the useful edges)."""
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op

import cluster_exact as ce
import forced_plans as fpl
from test_backward_exact_gpu import misaligned_copy

pytestmark = pytest.mark.gpu


def reference(case, g, d, s, go, bwd=True):
    """The fp64 reference, computed on the GPU and returned on the CPU, checked to be an exact case."""
    cu = lambda t: None if t is None else t.cuda().double()
    ref = ce.reference(cu(g), cu(d), cu(s), case.n, case.norm, cu(go) if bwd else None)
    ref = [t.cpu() for t in (ref if bwd else (ref,))]
    for t, name in zip(ref, ('out', 'grad_guidance', 'grad_blur')):
        ce.be.check_exact(t, case.n, f'{case.name} {name}', ce.unit(case.family, case.n))
    return ref


def run_backward(case, info, n_pass, g, d, s, go, ref, what):
    gg, gd, launches = fpl.backward(g, d, s, go, case.n, case.norm)
    assert launches == 2 * n_pass + 1, (what, launches, n_pass)      # forward steps + adjoint per pass, one gather
    ce.assert_exact(gg, ref[1], info, f'{what} grad_guidance')
    ce.assert_exact(gd, ref[2], info, f'{what} grad_blur')


def run_settings(case, e, g, d, s, go, ref, monkeypatch):
    """Forward (and backward) under planner settings `e`, through the C ABI.  Returns the plan_info of the forward."""
    ce.apply(monkeypatch, e)
    B = d.shape[0]
    info = ce.plan_of(e, B, case.C, case.H, case.W, case.n)
    assert info['supported'], (case.name, e, info)
    n_pass = sum(p['count'] for p in info['passes'])
    if e['CSPN_B200_FORCE_PASSES']:
        assert n_pass == int(e['CSPN_B200_FORCE_PASSES']), (case.name, e, info)
    what = f'{case.name} {ce.describe(e)}'
    if e['CSPN_B200_FORCE_CFG'] is not None and e['CSPN_B200_FORCE_CS'] is not None:
        plan = fpl.Plan(int(e['CSPN_B200_FORCE_CFG']), int(e['CSPN_B200_FORCE_CS']),
                        e['CSPN_B200_FORCE_PASSES'] and int(e['CSPN_B200_FORCE_PASSES']), e['CSPN_B200_CHAIN'] == '1')
        fpl.check_honoured(plan, info)          # the forced configuration and cluster size in every pass
    out, algo, launches, ws = fpl.forward(g, d, s, case.n, case.norm)
    assert _lib.ALGO_NAMES[algo] == 'cluster' and launches == n_pass, (what, algo, launches, n_pass)
    if info['chained']:
        assert (fpl.chain_flags(info, B, case.C, case.H, case.W, ws) == 1).all(), f'{what}: the chained kernel did not run'
    ce.assert_exact(out, ref[0], info, f'{what} out')
    if case.bwd:
        binfo = _lib.plan_info(case.H, case.W, case.n)            # the backward runs the unchained plan
        run_backward(case, binfo, sum(p['count'] for p in binfo['passes']), g, d, s, go, ref, what)
    return info


# ---- 1. the forced-plan matrix, exactly --------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(len(ce.FORCED)), ids=[c.name for c in ce.FORCED])
def test_forced_plans_are_exact(i, monkeypatch):
    """Every plan of the matrix (tests/forced_plans.py), GENERAL and chained kernels and banded plans whose band origins
    are not multiples of PR included: plan honoured, one launch per pass, chained flags set, device refusals warned.  Also
    two tall problems with 'signed' sparse (m = -1) at n = 3."""
    case = ce.FORCED[i]
    pb = fpl.PROBLEMS[case.problem]
    g, d, s, go = ce.inputs(case)
    ref = reference(case, g, d, s, go, case.bwd)
    for plan in pb.fwd:
        fpl.force(monkeypatch, plan)
        out, info = fpl.run_forced(plan, g, d, s, case.n, case.norm)
        if out is not None:
            ce.assert_exact(out, ref[0], info, f'{case.name} {plan} out')
    for plan in pb.bwd:
        fpl.force(monkeypatch, plan)
        info = fpl.plan_info(plan, case.H, case.W, case.n)
        if not info['supported']:
            fpl.refused(plan, (case.B, case.C, case.H, case.W, case.n))
            continue
        run_backward(case, info, fpl.check_honoured(plan, info), g, d, s, go, ref, f'{case.name} {plan}')


# ---- 2. long runs ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(len(ce.LONG)), ids=[c.name for c in ce.LONG])
def test_long_runs_are_exact_in_every_pass_split(i, monkeypatch):
    case = ce.LONG[i]
    g, d, s, go = ce.inputs(case)
    ref = reference(case, g, d, s, go)
    for e in case.envs:
        run_settings(case, e, g, d, s, go, ref, monkeypatch)


# ---- 3. persistent rounds ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(len(ce.PERSISTENT)), ids=[c.name for c in ce.PERSISTENT])
def test_later_rounds_of_persistent_clusters_are_exact(i, monkeypatch):
    """Enough images for every cluster to run >= 3 tasks: the prefetch, staging and mbarrier phases of later tasks."""
    case = ce.PERSISTENT[i]
    (e,) = case.envs
    ce.apply(monkeypatch, e)
    B = ce.batch_for_rounds(_lib.plan_info(case.H, case.W, case.n), case.C)
    info = ce.plan_of(e, B, case.C, case.H, case.W, case.n)
    B = max(B, ce.batch_for_rounds(info, case.C))
    info = ce.plan_of(e, B, case.C, case.H, case.W, case.n)
    r = ce.rounds(info, B, case.C)
    assert min(r) >= 3, (case.name, B, r, info)
    print(f"{case.name}: B = {B}, max_clusters {[p['max_clusters'] for p in info['passes']]}, "
          f"{min(r):.1f} tasks per cluster, {ce.describe(e)}{' (chained)' if info['chained'] else ''}")
    g, d, s, go = ce.inputs(case, B)
    ref = reference(case, g, d, s, go)
    run_settings(case, e, g, d, s, go, ref, monkeypatch)


# ---- 4. chained strips -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(len(ce.CHAIN)), ids=[c.name for c in ce.CHAIN])
def test_chained_strips_are_exact_in_every_grouping(i, monkeypatch):
    case = ce.CHAIN[i]
    g, d, s, go = ce.inputs(case)
    ref = reference(case, g, d, s, go, bwd=False)
    for e in case.envs:
        plan = fpl.Plan(int(e['CSPN_B200_FORCE_CFG']), int(e['CSPN_B200_FORCE_CS']), int(e['CSPN_B200_FORCE_PASSES']), True)
        fpl.force(monkeypatch, plan)
        ce.apply(monkeypatch, e)
        out, info = fpl.run_forced(plan, g, d, s, case.n, case.norm)
        if out is not None:
            ce.assert_exact(out, ref[0], info, f'{case.name} {plan} group {e["CSPN_B200_CHAIN_GROUP"]} out')


# ---- 5. every other route of the 3x3 operator -------------------------------------------------------------------------
def module_call(case, g, d, s, go, use_op, algo=_lib.ALGO_AUTO, misaligned=False):
    m = cspn_b200.Affinity_Propagate(case.n, 3, case.norm, algo)
    if use_op:
        torch_op.load()
    m._use_op = use_op
    dev = [None if t is None else t.cuda() for t in (g, d, s, go)]
    if misaligned:
        dev = [None if t is None else misaligned_copy(t) for t in dev]
    gc, dc, sc, goc = dev
    gc.requires_grad_(True)
    dc.requires_grad_(True)
    out = m(gc, dc, sc)
    out.backward(goc)
    return out.detach(), gc.grad, dc.grad


@pytest.mark.parametrize('i', range(len(ce.ROUTES)), ids=[c.name for c in ce.ROUTES])
def test_every_route_of_the_3x3_operator_is_exact(i, monkeypatch):
    case = ce.ROUTES[i]
    ce.apply(monkeypatch, case.envs[0])
    g, d, s, go = ce.inputs(case)
    ref = reference(case, g, d, s, go)
    info = _lib.plan_info(case.H, case.W, case.n) if case.W % 4 == 0 else None
    routes = [('ctypes', dict(use_op=False)), ('op', dict(use_op=True)),
              ('generic', dict(use_op=False, algo=_lib.ALGO_GENERIC)),
              ('misaligned ctypes', dict(use_op=False, misaligned=True)), ('misaligned op', dict(use_op=True, misaligned=True))]
    for name, kw in routes:
        for t, r, what in zip(module_call(case, g, d, s, go, **kw), ref, ('out', 'grad_guidance', 'grad_blur')):
            ce.assert_exact(t, r, None if 'generic' in name or 'misaligned' in name else info, f'{case.name} {name} {what}')
    monkeypatch.setenv('CSPN_B200_BWD', 'steps')               # the launch-per-step backward
    for t, r, what in zip(module_call(case, g, d, s, go, False), ref, ('out', 'grad_guidance', 'grad_blur')):
        ce.assert_exact(t, r, info, f'{case.name} BWD=steps {what}')
    monkeypatch.delenv('CSPN_B200_BWD')
    # the host-buffer entry: 1 MB chunks, one and three streams.  It reports the launches of all its chunks; a chunk of
    # these sizes launches what a one-image device call does (the plan does not depend on the batch, and these batches are
    # too small to chain), so the ratio is the chunk count: >= 4, so the stream slots are reused.
    cspn_b200.propagate2d(g[:1].cuda(), d[:1].cuda(), s[:1].cuda(), case.n, case.norm)
    per_chunk = _lib.lib().cspn_last_launches()
    assert per_chunk >= 1
    monkeypatch.setenv('CSPN_B200_HOST_CHUNK_MB', '1')
    for streams in (1, 3):
        monkeypatch.setenv('CSPN_B200_HOST_STREAMS', str(streams))
        out = cspn_b200.propagate2d(g, d, s, case.n, case.norm)
        assert not out.is_cuda
        launches = _lib.lib().cspn_last_launches()
        assert launches % per_chunk == 0 and launches // per_chunk >= 4, (case.name, streams, launches, per_chunk)
        ce.assert_exact(out, ref[0], info, f'{case.name} host entry, {streams} stream(s), {launches // per_chunk} chunks, out')
