"""Array-level model of the staged cluster backward (cspn2d_bwd.cu::bwd2d_cluster): the plane bookkeeping of
cluster2d_forward_steps / cluster2d_adjoint_steps (which plane every pass reads, writes and continues from) and the
arithmetic of bwd_gather_finalize_kernel, restated in numpy and compared with fp64 autograd through the reference's op
sequence.  Catches off-by-one errors in the orchestration without a GPU."""
import numpy as np
import pytest
import torch

from cspn_b200 import _lib
from oracle import cspn_numpy as onp, cspn_torch_port as tp


def folded(guidance, sparse, norm):
    gate_wb, gate_sum = onp.affinity_normalization_2d(guidance, norm)          # w_k, s
    m = np.zeros_like(gate_sum) if sparse is None else onp.sparse_mask(sparse, sparse.dtype)
    return (1 - m) * gate_wb, (1 - m) * (1 - gate_sum) + m, m                  # w', kappa, m


def fwd_step(w, c, d):
    return c + sum(w[:, k:k + 1] * onp.shift2d(d, dy, dx) for k, (dy, dx) in enumerate(onp.OFFSETS_2D))


def adj_step(w, lam):
    return sum(onp.shift2d(w[:, k:k + 1] * lam, -dy, -dx) for k, (dy, dx) in enumerate(onp.OFFSETS_2D))


def staged_backward(guidance, blur, sparse, grad_out, passes, norm):
    """passes: step counts of the plan's launches.  Mirrors the pointer arithmetic of the C++ drivers with plane indices."""
    N = sum(passes)
    w, kappa, m = folded(guidance[:, :8], sparse, norm)
    c = kappa * blur
    steps = [None] * N          # steps[t] = d_{t+1}
    done = 0
    for iters in passes:        # cluster2d_forward_steps
        d = steps[done - 1] if done else blur                   # init / blur
        out_idx, iter_base = done + iters - 1, done
        for s in range(iters):
            d = fwd_step(w, c, d)
            steps[iter_base + s if s < iters - 1 else out_idx] = d
        done += iters
    lam = [None] * N            # lam[t] = lambda_t
    done = 0
    for iters in passes:        # cluster2d_adjoint_steps
        l = lam[N - done] if done else grad_out                 # `start`
        out_idx, iter_base = N - done - iters, N - done - 1
        for s in range(iters):
            l = adj_step(w, l)
            lam[iter_base - s if s < iters - 1 else out_idx] = l
        done += iters
    assert all(x is not None for x in steps) and all(x is not None for x in lam)
    # bwd_gather_finalize_kernel
    B, C, H, W = blur.shape
    gw = np.zeros((B, 8, H, W))
    gc = np.zeros_like(blur)
    for t in range(N):
        lp = grad_out if t == N - 1 else lam[t + 1]
        dt = blur if t == 0 else steps[t - 1]
        gc += lp
        for k, (dy, dx) in enumerate(onp.OFFSETS_2D):
            gw[:, k] += (lp * onp.shift2d(dt, dy, dx)).sum(axis=1)
    grad_blur = kappa * gc + lam[0]
    gkappa = (gc * blur).sum(axis=1, keepdims=True)
    g = guidance[:, :8]
    sg = np.sign(g) if 'abs' in norm else np.ones_like(g)
    a = np.stack([onp.shift2d((np.abs(g) if 'abs' in norm else g)[:, k], dy, dx) for k, (dy, dx) in enumerate(onp.OFFSETS_2D)], 1)
    S = np.abs(a).sum(axis=1, keepdims=True)
    Hk = (1 - m) * (gw - gkappa)
    T = (Hk * a / S).sum(axis=1, keepdims=True)
    ga = (Hk - np.sign(a) * T) / S                               # dL/da_k at p; g_k(p + off_k) is its only source
    grad_g = np.zeros_like(guidance)
    for k, (dy, dx) in enumerate(onp.OFFSETS_2D):
        grad_g[:, k] = onp.shift2d(ga[:, k], -dy, -dx) * sg[:, k]
    return grad_g, grad_blur


@pytest.mark.parametrize('norm', ['8sum', '8sum_abs'])
@pytest.mark.parametrize('passes', [[5], [3, 3, 2], [1, 1], [4, 3]])
def test_staged_backward_bookkeeping_and_arithmetic_match_autograd(passes, norm):
    rng = np.random.default_rng(sum(passes))
    B, C, H, W, n = 2, 2, 7, 9, sum(passes)
    g = rng.standard_normal((B, 9, H, W))
    d = rng.uniform(0, 10, (B, C, H, W))
    s = rng.uniform(-1, 5, (B, 1, H, W)) * (rng.uniform(size=(B, 1, H, W)) < 0.2)
    go = rng.standard_normal((B, C, H, W))
    gt = torch.tensor(g, requires_grad=True)
    dt = torch.tensor(d, requires_grad=True)
    tp.cspn2d_torch(gt, dt, torch.tensor(s), n, norm).backward(torch.tensor(go))
    grad_g, grad_d = staged_backward(g, d, s, go, passes, norm)
    np.testing.assert_allclose(grad_d, dt.grad.numpy(), rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(grad_g, gt.grad.numpy(), rtol=1e-8, atol=1e-9)


def test_the_planner_supplies_such_pass_lists():
    info = _lib.plan_info(40, 264, 40)
    passes = [p['iters'] for p in info['passes'] for _ in range(p['count'])]
    assert sum(passes) == 40 and len(passes) > 1
