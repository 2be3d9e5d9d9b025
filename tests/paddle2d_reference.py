"""References of the 2D propagation with the Paddle module's own-location gates (CSPN.cspn with dim_num = 2,
cspn_paddle/demo.py:20-54), K in {3, 5, 7}.  TEST INFRASTRUCTURE ONLY: shared by tests/test_cspn2d_paddle_cpu.py,
tests/test_cspn2d_paddle_gpu.py and tools/time_2d_paddle.py; the product package never imports it.

Both restate the rule of oracle/cspn_numpy_3d_k.py's 'paddle' with the depth axis removed, over the taps of
oracle/cspn_numpy_k.py::offsets_2d:
    w_k(p) = |g_k(p)| / sum_j |g_j(p)|   (own location, j over all K*K-1 channels)
    d_{t+1}(p) = sum_k w_k(p) d_t(p + off_k)   (zero padding, no centre term, no sparse replacement)
guidance (B, K*K-1, H, W) is shared by the C channels of feat (B, C, H, W); (B, (K*K-1)*C, H, W) with C > 1 gives
channel c guide channels [nt*c, nt*c+nt) (demo.py:28-45), which is B*C single-channel images.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.cspn_numpy_k import offsets_2d, shift2d_k
from oracle.cspn_torch_port_k import pads_2d


def _per_channel(guidance, feat, nt):
    B, C, H, W = feat.shape
    if C > 1 and guidance.shape[1] == nt * C:
        return guidance.reshape(B * C, nt, H, W), feat.reshape(B * C, 1, H, W)
    assert guidance.shape == (B, nt, H, W), (guidance.shape, feat.shape)
    return None


def cspn2d_paddle(guidance, feat, prop_time=24, K=3, dtype=np.float32):
    """numpy, op for op in `dtype`.  The sum of |g| runs over the channels in order, as the kernels' does, so the weights
    carry the kernels' bits; the steps differ from the kernels' FMAs by rounding only."""
    nt = K * K - 1
    guidance = np.asarray(guidance, dtype=dtype)
    feat = np.asarray(feat, dtype=dtype)
    views = _per_channel(guidance, feat, nt)
    if views is not None:
        return cspn2d_paddle(*views, prop_time, K, dtype).reshape(feat.shape)
    with np.errstate(divide='ignore', invalid='ignore'):
        g = np.abs(guidance)
        normalizer = np.zeros_like(g[:, 0])
        for k in range(nt):
            normalizer = normalizer + g[:, k]
        gate = g / normalizer[:, None]
        result = feat
        for _ in range(prop_time):
            acc = np.zeros_like(result)
            for k, (dy, dx) in enumerate(offsets_2d(K)):
                acc = acc + gate[:, k:k + 1] * shift2d_k(result, dy, dx)
            result = acc
    return result.astype(dtype, copy=False)


def cspn2d_torch_paddle(guidance, feat, prop_time=24, K=3):
    """torch ops: K*K-1 ZeroPad2d copies of d_t per step (the pad tuples of oracle/cspn_torch_port_k.py::pads_2d, then the
    crop [r:r+H, r:r+W]), weighted and summed.  In fp64 the autograd reference of the 2D 'paddle' path."""
    nt, r = K * K - 1, (K - 1) // 2
    assert K in (3, 5, 7)
    views = _per_channel(guidance, feat, nt)
    if views is not None:
        return cspn2d_torch_paddle(*views, prop_time, K).reshape(feat.shape)
    H, W = feat.shape[-2:]
    a = guidance.abs()
    gate = a / a.sum(1, keepdim=True)
    result = feat
    for _ in range(prop_time):
        acc = 0
        for k, p in enumerate(pads_2d(K)):
            acc = acc + gate[:, k:k + 1] * F.pad(result, p)[..., r:r + H, r:r + W]
        result = acc
    return result
