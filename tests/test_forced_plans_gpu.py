"""Every kernel of the 2D cluster path, whatever plan the card would pick on its own: the forced-plan matrix of
tests/forced_plans.py run forward (plain, GENERAL, chained) and backward (kStoreSteps + kAdjoint + gather) against the
oracles, and bit for bit across plans that compute every pixel in the same order.

Each forced plan is checked to be the one that ran: plan_info shows the forced configuration, cluster size and pass
count, the call reports the cluster algorithm and one launch per pass (2 per pass + 1 for the backward), and a chained
call leaves its strips' "history complete" flags set in the workspace.  A combination the device cannot host must be
refused as unsupported; those refusals are reported as warnings."""
import numpy as np
import pytest
import torch

from cspn_b200.synth import make_inputs
from conftest import load_golden
from forced_plans import (NAN_PATCH_PLANS, NORMS, PROBLEMS, SPECIAL, backward, bit_group, check_honoured, force, plan_info,
                          refused, run_forced, special_plans)
from oracle import c_oracle, cspn_numpy as onp, cspn_torch_port as tp

pytestmark = pytest.mark.gpu


def inputs(pb, seed):
    """About one pixel in 20 sparse, so that masked pixels sit in every tile and halo."""
    return make_inputs(seed, pb.B, pb.C, pb.H, pb.W, pb.gch, pb.sparse, pb.H * pb.W // 20)


def same_bits(a, b):
    """Equal values at equal places, NaN included (torch.equal alone treats NaN as unequal to itself)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0), b.masked_fill(nb, 0))


def assert_bit_identical(results):
    """results: [(plan, key, tensors)]; within a key every plan's tensors equal the first plan's bit for bit."""
    first = {}
    for plan, key, ts in results:
        if key is None:
            continue
        if key not in first:
            first[key] = (plan, ts)
            continue
        p0, ts0 = first[key]
        for a, b in zip(ts, ts0):
            assert same_bits(a, b), f'{plan} differs from {p0}: max diff {float((a - b).abs().nan_to_num(0).max()):.3g}'


def grads_close(ours, theirs, name):
    """The scale-relative bound of test_cluster_backward_gpu.py, on the entries where fp64 autograd is finite; the NaN
    patterns must coincide."""
    assert torch.equal(torch.isnan(ours), torch.isnan(theirs)), (name, int(torch.isnan(ours).sum()), int(torch.isnan(theirs).sum()))
    fin = ~torch.isnan(theirs)
    o, t = ours[fin], theirs[fin]
    scale = t.abs().mean()
    err = (o - t).abs()
    assert (err <= 2e-3 * (t.abs() + scale)).all(), (name, float(err.max()), float(scale))


def autograd64(g, d, s, go, n, norm):
    g64 = g.double().requires_grad_(True)
    d64 = d.double().requires_grad_(True)
    tp.cspn2d_torch(g64, d64, None if s is None else s.double(), n, norm).backward(go.double())
    return g64.grad, d64.grad


@pytest.mark.parametrize('name', sorted(PROBLEMS))
def test_forced_forward_plans_match_oracle_and_each_other(name, monkeypatch):
    pb = PROBLEMS[name]
    g, d, s = inputs(pb, 100 + pb.H + pb.n)
    ref = c_oracle.cspn2d(g.numpy(), d.numpy(), None if s is None else s.numpy(), pb.n, pb.norm)
    results = []
    for plan in pb.fwd:
        force(monkeypatch, plan)
        out, info = run_forced(plan, g, d, s, pb.n, pb.norm)
        if out is None:
            continue
        ok, ratio, normwise = onp.parity_ok(out.numpy(), ref, 1e-4)
        assert ok and normwise <= 1e-5, (plan, ratio, normwise)
        results.append((plan, bit_group(plan, info), [out]))
    assert_bit_identical(results)


@pytest.mark.parametrize('name', sorted(k for k, pb in PROBLEMS.items() if pb.bwd))
def test_forced_backward_plans_match_autograd_and_each_other(name, monkeypatch):
    pb = PROBLEMS[name]
    g, d, s = inputs(pb, 200 + pb.H + pb.n)
    go = torch.randn(pb.B, pb.C, pb.H, pb.W, generator=torch.Generator().manual_seed(pb.H))
    ref_g, ref_d = autograd64(g, d, s, go, pb.n, pb.norm)
    results = []
    for plan in pb.bwd:
        force(monkeypatch, plan)
        info = plan_info(plan, pb.H, pb.W, pb.n)
        if not info['supported']:          # the forward test asserts the refusal; the backward would take launch-per-step
            refused(plan, (pb.B, pb.C, pb.H, pb.W, pb.n))
            continue
        n_pass = check_honoured(plan, info)
        gg, gd, launches = backward(g, d, s, go, pb.n, pb.norm)
        assert launches == 2 * n_pass + 1, (plan, launches, n_pass)      # forward steps + adjoint per pass, one gather
        grads_close(gg, ref_g, f'{plan} guidance')
        grads_close(gd, ref_d, f'{plan} blur')
        results.append((plan, bit_group(plan, info), [gg, gd]))
    assert_bit_identical(results)


@pytest.mark.parametrize('name', SPECIAL)
def test_special_value_goldens_under_every_configuration(name, monkeypatch):
    c = load_golden(name)
    g, d = torch.from_numpy(c['guidance']), torch.from_numpy(c['blur'])
    s = None if c['sparse_depth'] is None else torch.from_numpy(c['sparse_depth'])
    results = []
    for plan in special_plans(name, d.shape[-2]):
        force(monkeypatch, plan)
        out, info = run_forced(plan, g, d, s, c['prop_time'], c['norm_type'])
        if out is None:
            continue
        o = out.numpy()
        assert np.array_equal(np.isnan(o), np.isnan(c['out'])), plan
        assert np.array_equal(np.isinf(o), np.isinf(c['out'])), plan
        ok, ratio, normwise = onp.parity_ok(o, c['out'], 1e-4)
        assert ok, (plan, ratio, normwise)
        results.append((plan, bit_group(plan, info), [out]))
    assert_bit_identical(results)


@pytest.mark.parametrize('norm', NORMS)
@pytest.mark.parametrize('n', [1, 2, 3])
def test_backward_through_zero_affinity_patch_under_every_configuration(n, norm, monkeypatch):
    """0/0 affinities (the patch of test_cspn2d_gpu.py::test_nan_semantics_match_reference): the gradients carry NaN
    exactly where fp64 autograd's do, and agree elsewhere."""
    g, d, s = make_inputs(5, 1, 1, 12, 16, 8, 'bernoulli', 10)
    g[0, :, 3:8, 4:9] = 0
    go = torch.randn(1, 1, 12, 16, generator=torch.Generator().manual_seed(n))
    ref_g, ref_d = autograd64(g, d, s, go, n, norm)
    assert torch.isnan(ref_g).any() and torch.isnan(ref_d).any() and not torch.isnan(ref_d).all()
    results = []
    for plan in NAN_PATCH_PLANS:
        force(monkeypatch, plan)
        info = plan_info(plan, 12, 16, n)
        n_pass = check_honoured(plan, info)
        gg, gd, launches = backward(g, d, s, go, n, norm)
        # 2 per pass + 1 tells the cluster formulation from launch-per-step (2 n + 1) only for n > 1; at n = 1 it rests on
        # force() having cleared CSPN_B200_BWD and on the plan being supported (the cluster backward declines nothing else)
        assert launches == 2 * n_pass + 1, (plan, launches)
        grads_close(gg, ref_g, f'{plan} guidance')
        grads_close(gd, ref_d, f'{plan} blur')
        results.append((plan, bit_group(plan, info), [gg, gd]))
    assert_bit_identical(results)
