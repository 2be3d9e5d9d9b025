"""Reference of the propagation with caller-supplied gates (fluid.layers.affinity_propagate(input, gate_weight, kernel_size)
run prop_step times, cspn_paddle/demo.py:41-43, 51-52), 2D and 3D.  TEST INFRASTRUCTURE ONLY: shared by
tests/test_gates_cpu.py, tests/test_gates_gpu.py and tools/time_gates.py; the product package never imports it.

    d_{t+1}(p) = sum_k g_k(p) d_t(p + off_k),   d_0 = input,
over the taps of offsets_2d(K) / offsets_3d(K), with the gates used exactly as given (no |.|, no normalisation, no centre
term), zero padding and the taps summed in order.  Built on backward_exact.shift, so in fp64 it is the autograd reference of
both gradients.  gate_weight (B, K**d-1, ...) is shared by the C channels of input; (B, (K**d-1)*C, ...) with C > 1 gives
channel c gate channels [nt*c, nt*c+nt) (demo.py:28-45), which is B*C single-channel images.
"""
import torch

import backward_exact as be


def affinity_propagate_ref(input, gate_weight, K=3, prop_step=1):
    nd = input.dim() - 2
    nt, r = K ** nd - 1, (K - 1) // 2
    B, C = input.shape[:2]
    if C > 1 and gate_weight.shape[1] == nt * C:
        return affinity_propagate_ref(input.reshape(B * C, 1, *input.shape[2:]),
                                      gate_weight.reshape(B * C, nt, *input.shape[2:]), K, prop_step).reshape(input.shape)
    assert gate_weight.shape == (B, nt) + tuple(input.shape[2:]), (gate_weight.shape, input.shape)
    offs = be.offsets(K, nd)
    d = input
    for _ in range(prop_step):
        acc = 0
        for k, o in enumerate(offs):
            acc = acc + gate_weight[:, k:k + 1] * be.shift(d, o, r)
        d = acc
    return d


def paddle_gates(guidance, nt):
    """demo.py's normalisation, |g| / sum_j |g_j| over the nt channels of each gate (per-channel guidance (B, nt*C, ...) is
    normalised block by block), with the sum taken channel by channel in order, as the 'paddle' kernels take it, in the
    dtype of `guidance`."""
    g = guidance.reshape(-1, nt, *guidance.shape[2:])
    a = g.abs()
    S = a[:, 0]
    for k in range(1, nt):
        S = S + a[:, k]
    return (a / S.unsqueeze(1)).reshape(guidance.shape)
