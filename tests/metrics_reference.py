"""Restatement of the depth metrics and the masked L1 loss (cspn_b200/csrc/metrics.cu, cspn_b200/metrics.py), from the
semantics of the reference's utils.evaluate_error (utils.py:19-47) and Wighted_L1_Loss (loss.py:16-23), in numpy.

Everything per element is fp32, as in the reference and in the kernel:
    valid      gt > 0.0001, the scalar rounded to float32 (a NaN gt is not valid, +inf is);
    diff       |gt - pred|;   rel = diff / gt;
    max_ratio  max(gt / pred, pred / gt), IEEE division, a NaN operand gives NaN (torch.max);
    deltas     max_ratio < t, strictly, t in {1.02, 1.05, 1.10, 1.25, 1.25^2, 1.25^3} rounded to float32.
What is summed is summed in fp64 (numpy's pairwise sum), and diff is squared in fp64 as the kernel squares it, so the means
are the exact ones to about 1e-15 and a correct kernel's float lies within one fp32 ulp of them.  Counts are integers.

The gradient of the loss is exact in fp32: sign(pred - gt) (0 at pred == gt and for a NaN difference, as torch.sign) times
fl(fl(1 / n_valid) * grad_loss) where gt is valid, 0 elsewhere.

Used by tests/test_metrics_cpu.py, which ties it to the goldens the reference's own functions produced, and by
tests/test_metrics_exact_gpu.py; the product never imports it."""
import numpy as np
import torch

VALID_CUT = np.float32(0.0001)
THRESHOLDS = np.array([1.02, 1.05, 1.10, 1.25, 1.25 ** 2, 1.25 ** 3], dtype=np.float32)
KEYS = ('MSE', 'RMSE', 'MAE', 'ABS_REL', 'DELTA1.02', 'DELTA1.05', 'DELTA1.10', 'DELTA1.25', 'DELTA1.25^2', 'DELTA1.25^3')


def _f32(t):
    if isinstance(t, torch.Tensor):
        t = t.detach().cpu().numpy()
    a = np.asarray(t)
    assert a.dtype == np.float32, a.dtype
    return a


def valid_mask(gt):
    return _f32(gt) > VALID_CUT


def max_ratio(g, p):
    """fp32 max(g / p, p / g) with NaN propagation, on float32 arrays."""
    with np.errstate(all='ignore'):
        return np.maximum(g / p, p / g)


def counts(gt, pred):
    """-> (n_valid, [six delta counts]) as Python ints."""
    gt, pred = _f32(gt), _f32(pred)
    v = gt > VALID_CUT
    ratio = max_ratio(gt[v], pred[v])
    return int(v.sum()), [int((ratio < t).sum()) for t in THRESHOLDS]


def sums(gt, pred):
    """-> (sum diff^2, sum diff, sum diff / gt) over the valid elements, accumulated in fp64."""
    gt, pred = _f32(gt), _f32(pred)
    v = gt > VALID_CUT
    g, p = gt[v], pred[v]
    with np.errstate(all='ignore'):
        diff = np.abs(g - p)
        rel = diff / g
        d64 = diff.astype(np.float64)
        return float((d64 * d64).sum()), float(d64.sum()), float(rel.astype(np.float64).sum())


def stats12(gt, pred):
    """The kernel's twelve numbers in fp64, before their rounding to float: n_valid, MSE, RMSE, MAE, ABS_REL, the six
    delta fractions, 0.  All zero when nothing is valid."""
    n, deltas = counts(gt, pred)
    out = np.zeros(12, np.float64)
    out[0] = n
    if n > 0:
        sq, ab, rel = sums(gt, pred)
        with np.errstate(all='ignore'):
            out[1:5] = sq / n, np.sqrt(sq / n), ab / n, rel / n
        out[5:11] = np.array(deltas, np.float64) / n
    return out


def grad_scale(n_valid, grad_loss=1.0, count_dtype=np.float64):
    """fl(fl(1 / n_valid) * grad_loss), 0 for n_valid == 0.  A float64 quotient of two integers below 2^53 rounded to
    float32 is the correctly rounded fp32 quotient (53 >= 2 * 24 + 2), so the default is fl(1 / n) for the exact count;
    count_dtype=np.float32 rounds the count to float32 first, which is what differs above 2^24."""
    if n_valid == 0:
        return np.float32(0) * np.float32(grad_loss)
    return np.float32(1.0 / float(count_dtype(n_valid))) * np.float32(grad_loss)


def masked_l1_grad(gt, pred, grad_loss=1.0, count_dtype=np.float64):
    """The exact fp32 gradient of the loss with respect to pred, shaped like pred."""
    gt, pred = _f32(gt), _f32(pred)
    v = gt > VALID_CUT
    with np.errstate(all='ignore'):
        d = pred - gt
        sign = (d > 0).astype(np.float32) - (d < 0).astype(np.float32)      # 0 for d == 0 and for NaN
        return np.where(v, grad_scale(int(v.sum()), grad_loss, count_dtype) * sign, np.float32(0)).astype(np.float32)


def masked_l1_torch(pred, gt):
    """The loss as torch ops, for autograd in any dtype: mean |pred - gt| over gt > 0.0001 (the cut is float32's)."""
    mask = gt > float(VALID_CUT)
    return (pred[mask] - gt[mask]).abs().sum() / int(mask.sum())


def ulp32(x):
    """The spacing of float32 at x (fp64 in, fp64 out)."""
    return float(np.spacing(np.abs(np.float32(x))))


def assert_stats(ours12, gt, pred, case=''):
    """ours12: the kernel's twelve floats.  n_valid and the six counts exactly; the four means NaN / inf where the
    restatement's are and within one fp32 ulp otherwise; slot 11 zero."""
    ours = np.asarray(ours12, dtype=np.float32)
    ref = stats12(gt, pred)
    n, deltas = counts(gt, pred)
    assert float(ours[0]) == float(np.float32(n)), (case, 'n_valid', float(ours[0]), n)
    for t in range(6):      # the kernel forms float(count / n) in fp64: the same quotient, the same rounding
        assert ours[5 + t] == np.float32(ref[5 + t]), (case, KEYS[4 + t], float(ours[5 + t]) * max(n, 1), deltas[t])
    for i in range(1, 5):
        with np.errstate(over='ignore'):
            r = np.float32(ref[i])      # a mean beyond FLT_MAX rounds to inf in the kernel's float as well
        if not np.isfinite(r):
            assert np.isnan(ours[i]) if np.isnan(r) else ours[i] == r, (case, KEYS[i - 1], float(ours[i]), ref[i])
        else:
            assert abs(float(ours[i]) - ref[i]) <= ulp32(ref[i]), (case, KEYS[i - 1], float(ours[i]), ref[i])
    assert ours[11] == 0, case
