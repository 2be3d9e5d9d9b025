"""Model-level parity (SURVEY.md section 7.2's exit criterion) on the GPU, without the reference tree:
tests/golden/model/nyu_resnet50_tail.npz holds what the reference's OWN model code (resnet50 + Gudi UNet decoder,
torch_resnet_cspn_nyu.py, random seeded weights) handed to its post_process_layer (:372-375) and what that model
returned with the reference's own cspn.py as the layer -- generated where the reference tree exists by
tests/golden/make_golden_model.py.  Fed the same boundary tensors, the CUDA module must return the reference MODEL's output."""
import os

import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
from oracle import cspn_numpy as onp

pytestmark = pytest.mark.gpu
PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model', 'nyu_resnet50_tail.npz')


@pytest.mark.parametrize('route', ['module', 'ctypes_cluster', 'ctypes_generic'])
def test_module_reproduces_the_reference_models_output(route):
    z = np.load(PATH)
    g, d, s = [torch.from_numpy(z[k]).cuda() for k in ('guidance', 'blur', 'sparse_depth')]
    assert g.shape == (1, 8, 228, 304) and d.shape == (1, 1, 228, 304) and str(z['norm_type']) == '8sum'
    if route == 'module':
        layer = cspn_b200.Affinity_Propagate(int(z['prop_time']), 3, str(z['norm_type']))      # what _make_post_process_layer builds (:344-347)
        with torch.no_grad():
            out = layer(g, d, s)
    else:
        algo = _lib.ALGO_CLUSTER if route == 'ctypes_cluster' else _lib.ALGO_GENERIC
        out = cspn_b200.propagate2d(g, d, s, int(z['prop_time']), str(z['norm_type']), algo)
    ok, ratio, normwise = onp.parity_ok(out.cpu().numpy(), z['out'], 1e-4)
    assert ok, (route, ratio, normwise)
    assert normwise < 1e-5


def test_training_step_through_the_boundary_tensors_is_finite_and_consistent():
    """train.py:196-199: loss.backward() through the module with the model's own boundary tensors as leaves."""
    z = np.load(PATH)
    g = torch.from_numpy(z['guidance']).cuda().requires_grad_(True)
    d = torch.from_numpy(z['blur']).cuda().requires_grad_(True)
    s = torch.from_numpy(z['sparse_depth']).cuda()
    layer = cspn_b200.Affinity_Propagate(24, 3, '8sum')
    out = layer(g, d, s)
    target = torch.rand_like(out)
    mask = (target > 0.5).float()
    loss = ((out - target).abs() * mask).sum() / mask.sum()            # loss.py:16-23 (masked L1)
    loss.backward()
    assert torch.isfinite(g.grad).all() and torch.isfinite(d.grad).all()
    assert g.grad.abs().sum() > 0 and d.grad.abs().sum() > 0
