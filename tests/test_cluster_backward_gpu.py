"""The register-resident backward (cluster kernel in kStoreSteps / kAdjoint mode + one gather kernel, cspn2d_bwd.cu) against
fp64 autograd through the reference's op sequence, and against the launch-per-step formulation (CSPN_B200_BWD=steps)."""
import os

import pytest
import torch

import cspn_b200
from cspn_b200.synth import make_inputs
from forced_plans import backward as grads
from oracle import cspn_torch_port as tp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('norm', ['8sum', '8sum_abs'])
@pytest.mark.parametrize('shape,n,sparse', [
    ((2, 1, 12, 16), 5, 'signed'),       # one CTA, one strip
    ((1, 2, 48, 132), 6, 'bernoulli'),   # channels share the affinity; two strips
    ((1, 1, 100, 260), 24, 'bernoulli'),  # several CTAs per cluster: DSMEM partial rows
    ((1, 1, 40, 264), 40, None),         # multi-pass plan
    ((1, 1, 700, 64), 4, 'signed'),      # row bands
])
def test_cluster_backward_matches_reference_autograd(shape, n, sparse, norm, monkeypatch):
    B, C, H, W = shape
    g, d, s = make_inputs(31 + H, B, C, H, W, 9, sparse, 25)
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(1))
    g64 = g.double().requires_grad_(True)
    d64 = d.double().requires_grad_(True)
    tp.cspn2d_torch(g64, d64, None if s is None else s.double(), n, norm).backward(go.double())
    new_g, new_d, new_launches = grads(g, d, s, go, n, norm)          # default: the cluster formulation
    monkeypatch.setenv('CSPN_B200_BWD', 'steps')
    base_g, base_d, base_launches = grads(g, d, s, go, n, norm)
    assert new_launches < base_launches                      # it really took the cluster formulation
    for ours, theirs, name in ((new_g, g64.grad, 'guidance'), (new_d, d64.grad, 'blur')):
        scale = theirs.abs().mean()
        err = (ours - theirs).abs()
        assert (err <= 2e-3 * (theirs.abs() + scale)).all(), (name, float(err.max()), float(scale))
    # the two fp32 formulations sum in different orders: they agree to fp32 noise relative to the gradient's scale
    assert torch.allclose(new_g, base_g, rtol=2e-3, atol=2e-3 * float(base_g.abs().mean()))
    assert torch.allclose(new_d, base_d, rtol=2e-3, atol=2e-3 * float(base_d.abs().mean()))
