"""tests/metrics_reference.py, the restatement the exact GPU tests of the metrics / loss kernels compare against, tied to the
reference without a GPU: it reproduces every golden that the reference's own utils.evaluate_error and Wighted_L1_Loss
produced (tests/golden/make_golden_metrics.py), the special-value ones under golden/metrics/edges/ included, and its
gradient agrees with fp64 autograd."""
import glob
import os

import numpy as np
import pytest
import torch

import metrics_reference as mr

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden', 'metrics')


def names(sub=''):
    return sorted(os.path.join(sub, os.path.basename(f)[:-4]) for f in glob.glob(os.path.join(GOLDEN, sub, '*.npz')))


SEEDED, EDGES = names(), names('edges')


def load(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'))


def test_the_goldens_are_all_there():
    assert SEEDED == ['close_prediction', 'kitti_like', 'nothing_valid', 'nyu_like']
    assert len(EDGES) == 21 and 'edges/pred_nan' in EDGES and 'edges/gt_cut' in EDGES and 'edges/all_together' in EDGES


def test_constants_are_the_float32_ones():
    """The reference compares float32 tensors with Python scalars, which torch rounds to float32 first."""
    cut = torch.tensor([mr.VALID_CUT, np.nextafter(mr.VALID_CUT, np.float32(1))])
    assert (cut > 0.0001).tolist() == [False, True] and float(mr.VALID_CUT) < 0.0001
    for t, s in zip(mr.THRESHOLDS, (1.02, 1.05, 1.10, 1.25, 1.25 ** 2, 1.25 ** 3)):
        x = torch.tensor([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(4))])
        assert (x < s).tolist() == [True, False, False]
    assert float(mr.THRESHOLDS[0]) < 1.02 and float(mr.THRESHOLDS[4]) == 1.5625 and float(mr.THRESHOLDS[5]) == 1.953125


@pytest.mark.parametrize('name', SEEDED + EDGES)
def test_restatement_reproduces_the_reference_metrics(name):
    z = load(name)
    gt, pred = z['gt'], z['pred']
    n, deltas = mr.counts(gt, pred)
    assert n == int((torch.from_numpy(gt) > 0.0001).sum())
    if 'n_valid' in z:
        assert n == int(z['n_valid'])
    ours = dict(zip(mr.KEYS, mr.stats12(gt, pred)[1:11]))
    # The reference's RMSE is the root of its float MSE; the kernel's and the restatement's is the root of the fp64 mean,
    # which stays finite (and right) where MSE itself is beyond FLT_MAX: edges/pred_fltmax, 4.4e37 against inf.
    if name == 'edges/pred_fltmax':
        assert np.isinf(np.float32(ours['MSE'])) and 4e37 < ours['RMSE'] < 5e37
    with np.errstate(all='ignore'):
        ours['RMSE'] = float(np.sqrt(np.float32(ours['MSE'])))
    for k, ref in zip(z['keys'], z['metrics']):
        k, ref = str(k), float(ref)
        if k.startswith('DELTA'):           # the reference divides the count by float(n) in double: the same quotient
            assert ours[k] == ref, (k, ours[k] * max(n, 1), ref * max(n, 1))
        elif not np.isfinite(ref):          # the reference squares and sums in fp32: a mean it reports as inf is beyond FLT_MAX
            got = np.float32(ours[k])
            assert np.isnan(got) if np.isnan(ref) else got == ref, (k, ours[k], ref)
        else:                               # its fp32 sums carry rounding error, ours do not
            assert abs(ours[k] - ref) <= 2e-6 * abs(ref), (k, ours[k], ref)


@pytest.mark.parametrize('name', [c for c in SEEDED + EDGES if c != 'nothing_valid'])
def test_restatement_reproduces_the_reference_loss_and_gradient_bits(name):
    z = load(name)
    gt, pred = z['gt'], z['pred']
    loss, ref = mr.stats12(gt, pred)[3], float(z['loss'])
    if np.isfinite(ref):
        assert abs(loss - ref) <= 2e-6 * abs(ref)
    else:
        assert np.isnan(loss) if np.isnan(ref) else loss == ref
    grad = mr.masked_l1_grad(gt, pred)
    assert grad.shape == z['grad_pred'].shape and grad.dtype == np.float32
    assert not np.isnan(grad).any() and np.array_equal(grad, z['grad_pred']), name      # no NaN: equal values are equal bits


def test_edge_goldens_settle_the_special_values():
    """What the reference does with each special value, read off its own outputs: which are valid, which are counted under
    every threshold, which poison the sums."""
    def of(name):
        z = load('edges/' + name)
        return int(z['n_valid']), dict(zip([str(k) for k in z['keys']], z['metrics'])), z['grad_pred'][-1]
    base_n, base, _ = of('gt_zero')                       # the special element is not valid: the 60 ordinary pairs alone
    assert base_n == 60
    for name in ('gt_cut', 'gt_cut_below', 'gt_negative', 'gt_nan', 'gt_subnormal'):
        n, m, g = of(name)
        assert n == 60 and m == base and g == 0, name
    assert of('gt_cut_above')[0] == 61 and of('gt_posinf')[0] == 61
    counted = lambda name: round(of(name)[1]['DELTA1.02'] * 61) - round(base['DELTA1.02'] * 60)
    # a ratio of -0 or below is "within 2 %": pred -0, negative or -inf is counted under every threshold
    assert [counted(k) for k in ('pred_negzero', 'pred_negative', 'pred_neginf', 'gt_posinf_pred_negative', 'kink')] == [1] * 5
    assert [counted(k) for k in ('pred_zero', 'pred_posinf', 'pred_nan', 'pred_subnormal', 'pred_fltmax', 'gt_posinf',
                                 'both_posinf')] == [0] * 7
    assert np.isnan(of('pred_nan')[1]['MAE']) and np.isnan(of('both_posinf')[1]['MAE'])
    assert np.isinf(of('pred_posinf')[1]['MAE']) and np.isnan(of('gt_posinf')[1]['ABS_REL'])
    # the gradient of the special element: 0 at the kink and for a NaN difference, -1/n below, +1/n above
    s = np.float32(1) / np.float32(61)
    assert [of(k)[2] for k in ('kink', 'pred_nan', 'both_posinf')] == [0, 0, 0]
    assert [of(k)[2] for k in ('pred_zero', 'pred_neginf', 'gt_posinf', 'pred_posinf', 'pred_fltmax')] == [-s, -s, -s, s, s]


@pytest.mark.parametrize('seed,shape,p_valid', [(1, (2, 1, 37, 53), 0.3), (2, (5000,), 1.0), (3, (3, 2, 4, 5, 6), 0.05)])
@pytest.mark.parametrize('grad_loss', [1.0, -2.5, 0.0])
def test_restatement_agrees_with_fp64_autograd(seed, shape, p_valid, grad_loss):
    g = torch.Generator().manual_seed(seed)
    gt = (torch.rand(shape, generator=g) * 10 + 0.5) * (torch.rand(shape, generator=g) < p_valid)
    pred = torch.rand(shape, generator=g) * 10
    pred.view(-1)[::7] = gt.view(-1)[::7]                           # the kink: sign(0) = 0
    p64 = pred.double().requires_grad_(True)
    loss = mr.masked_l1_torch(p64, gt.double())
    (grad_loss * loss).backward()
    ours = mr.masked_l1_grad(gt, pred, grad_loss)
    assert ours.shape == tuple(shape)
    ref = p64.grad.numpy()
    assert ((ours == 0) == (ref == 0)).all() and (ref != 0).sum() == (0 if grad_loss == 0 else ((gt > 1e-4) & (pred != gt)).sum())
    assert np.abs(ours - ref).max() <= 2.0 ** -23 * np.abs(ref).max()
    assert abs(mr.stats12(gt, pred)[3] - loss.item()) <= 2.0 ** -23 * loss.item()      # each |pred - gt| is rounded to fp32


def test_restatement_of_nothing_valid_and_of_the_count_above_2_to_24():
    gt, pred = np.zeros(9, np.float32), np.ones(9, np.float32)
    assert not mr.stats12(gt, pred).any() and not mr.masked_l1_grad(gt, pred, 3.0).any()
    n = 2 ** 24 + 1                                                 # float32 holds 2^24 and 2^24 + 2
    assert mr.grad_scale(n) == np.float32(1.0 / n) and mr.grad_scale(n, count_dtype=np.float32) == np.float32(2.0 ** -24)
    assert mr.grad_scale(3, -2.5) == np.float32(np.float32(1) / np.float32(3)) * np.float32(-2.5)
