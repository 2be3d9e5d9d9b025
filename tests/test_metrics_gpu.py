"""Device-side metrics / loss (cspn_b200/metrics.py over csrc/metrics.cu) against goldens produced by the reference's OWN
utils.evaluate_error (utils.py:19-47) and Wighted_L1_Loss (loss.py:12-23) -- tests/golden/make_golden_metrics.py."""
import glob
import os

import numpy as np
import pytest
import torch

from cspn_b200 import metrics

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(HERE, 'golden', 'metrics', '*.npz')))


@pytest.mark.parametrize('name', CASES)
def test_evaluate_error_matches_reference(name):
    z = np.load(os.path.join(HERE, 'golden', 'metrics', name + '.npz'))
    gt, pred = torch.from_numpy(z['gt']).cuda(), torch.from_numpy(z['pred']).cuda()
    err = metrics.evaluate_error(gt_depth=gt, pred_depth=pred)
    assert set(err) == set(str(k) for k in z['keys']) | {'LG10'} and err['LG10'] == 0
    for k, ref in zip(z['keys'], z['metrics']):
        ours = err[str(k)]
        assert ours.is_cuda and ours.dim() == 0                       # stays on the device: no host round trip
        if str(k).startswith('DELTA'):
            n = float((gt > 0.0001).sum())
            assert abs(float(ours) - ref) * max(n, 1) < 0.5, (k, float(ours), ref)      # the COUNT is exact
        else:
            assert abs(float(ours) - ref) <= 2e-6 * abs(ref) + 1e-12, (k, float(ours), ref)


@pytest.mark.parametrize('name', [c for c in CASES if c != 'nothing_valid'])
def test_masked_l1_loss_and_gradient_match_reference(name):
    z = np.load(os.path.join(HERE, 'golden', 'metrics', name + '.npz'))
    gt = torch.from_numpy(z['gt']).cuda()
    pred = torch.from_numpy(z['pred']).cuda().requires_grad_(True)
    loss = metrics.Wighted_L1_Loss()(pred, gt)
    assert loss.is_cuda and loss.dim() == 0
    assert abs(float(loss) - float(z['loss'])) <= 2e-6 * abs(float(z['loss']))
    (3.0 * loss).backward()
    ref = 3.0 * torch.from_numpy(z['grad_pred']).cuda()
    assert torch.allclose(pred.grad, ref, rtol=1e-6, atol=1e-12)


def test_nothing_valid_is_all_zero_like_the_reference():
    gt = torch.zeros(1, 1, 8, 8, device='cuda')
    err = metrics.evaluate_error(gt, torch.rand(1, 1, 8, 8, device='cuda'))
    assert all(float(err[k]) == 0 for k in metrics.KEYS)


def test_training_tail_without_host_sync():
    """train.py:196-211 with the device-side tail: CSPN output -> loss -> backward -> metrics, nothing copied to the host."""
    import cspn_b200
    from cspn_b200.synth import make_inputs
    g, d, s = [t.cuda() for t in make_inputs(3, 2, 1, 64, 96)]
    g.requires_grad_(True)
    d.requires_grad_(True)
    # seeded: `ref` below averages over every pixel, so every target must be valid (an unseeded U(0, 10) draw of 12288
    # values has one at or below 1e-4 in about one run of eight)
    target = (torch.rand(2, 1, 64, 96, generator=torch.Generator().manual_seed(1)) * 10).cuda()
    assert (target > 0.0001).all()
    out = cspn_b200.Affinity_Propagate(8, 3)(g, d, s)
    loss = metrics.Wighted_L1_Loss()(out, target)
    loss.backward()
    err = metrics.evaluate_error(target, out.detach())
    ref = (out.detach() - target).abs().mean()
    assert torch.allclose(loss, ref, rtol=1e-5) and torch.allclose(err['MAE'], ref, rtol=1e-5)
    assert torch.isfinite(g.grad).all() and g.grad.abs().sum() > 0
