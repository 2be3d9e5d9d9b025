"""GPU tests of the K x K 2D propagation (K = 5, 7 in cspn2d_wide.cu; K = 3 delegated to the 3x3 kernels): forward
against the numpy oracle, IEEE special values, batch independence across launch groups, backward against fp64 autograd
through the torch port, and torch.compile / CUDA-graph capture / a training step through the module."""
import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
from cspn_b200.synth import make_inputs
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_k as onk
from oracle import cspn_torch_port as tp
from oracle import cspn_torch_port_k as tpk

pytestmark = pytest.mark.gpu


def norm_name(K, abs_norm):
    return f'{K * K - 1}sum_abs' if abs_norm else f'{K * K - 1}sum'


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


# pairwise over K x norm x sparse x C x shape x N (every pair of values of two axes appears in some case)
FWD = [
    # K, abs, sparse, C, (B, H, W), N, misaligned
    (5, False, None, 1, (1, 1, 1), 1, False),
    (7, True, 'bernoulli', 3, (1, 1, 1), 2, False),
    (5, True, 'signed', 3, (1, 1, 40), 24, False),
    (7, False, None, 1, (1, 1, 37), 48, False),
    (5, False, 'bernoulli', 3, (1, 3, 4), 2, False),
    (7, True, 'signed', 1, (2, 5, 6), 24, False),
    (5, True, None, 3, (1, 20, 37), 48, False),
    (7, False, 'bernoulli', 1, (2, 21, 45), 1, False),
    (5, False, 'signed', 3, (1, 24, 64), 2, True),
    (7, True, None, 1, (2, 19, 32), 24, True),
    (5, True, 'bernoulli', 1, (2, 228, 304), 24, False),
    (7, False, 'signed', 1, (2, 228, 304), 48, False),
    (5, False, None, 1, (1, 352, 1216), 24, False),
    (7, True, 'bernoulli', 3, (1, 352, 1216), 2, False),
    (5, True, 'signed', 1, (1, 7, 9), 1, True),
    (7, False, 'signed', 3, (1, 9, 5), 48, False),
]


@pytest.mark.parametrize('K,abs_norm,sparse,C,bhw,N,misaligned', FWD,
                         ids=[f'K{c[0]}-{"abs" if c[1] else "sgn"}-{c[2]}-C{c[3]}-{"x".join(map(str, c[4]))}-N{c[5]}'
                              f'{"-misaligned" if c[6] else ""}' for c in FWD])
def test_forward_matches_the_oracle(K, abs_norm, sparse, C, bhw, N, misaligned):
    B, H, W = bhw
    norm = norm_name(K, abs_norm)
    g, d, s = make_inputs(K * 1000 + H + W + N, B, C, H, W, K * K - 1 + (2 if C == 3 else 0), sparse, 30)
    ref = onk.cspn2d_k(g.numpy(), d.numpy(), None if s is None else s.numpy(), N, K, norm)
    gc, dc, sc = g.cuda(), d.cuda(), None if s is None else s.cuda()
    if misaligned:
        gc, dc = misaligned_copy(gc), misaligned_copy(dc)
        sc = None if sc is None else misaligned_copy(sc)
    out = cspn_b200.propagate2d_k(gc, dc, sc, K, N, norm)
    torch.cuda.synchronize()
    assert _lib.lib().cspn_last_launches() == 1 + N      # one launch group for the batch: prep + N steps
    out = out.cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (ratio, normwise)


def _check_special(g, d, s, N, K, norm):
    ref = onk.cspn2d_k(g, d, s, N, K, norm)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = cspn_b200.propagate2d_k(t(g), t(d), t(s), K, N, norm).cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref)), (K, norm, N)
    assert np.array_equal(np.isinf(out), np.isinf(ref)), (K, norm, N)
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (K, norm, N, ratio, normwise)
    return ref


@pytest.mark.parametrize('K', [5, 7])
@pytest.mark.parametrize('corner', [False, True])
def test_zero_guidance_patch_nan_front_moves_r_pixels_per_step(K, corner):
    r = (K - 1) // 2
    g, d, s = [None if a is None else a.numpy() for a in make_inputs(K, 1, 1, 40, 64, K * K - 1, 'bernoulli', 20)]
    y0, x0 = (0, 0) if corner else (14, 24)
    g[:, :, y0:y0 + 12, x0:x0 + 12] = 0.0          # 0/0 -> NaN wherever the whole K x K window is zero
    extents = []
    for N in (1, 2, 3):
        for abs_norm in (False, True):
            ref = _check_special(g, d, s, N, K, norm_name(K, abs_norm))
        ys, xs = np.nonzero(np.isnan(ref[0, 0]))
        assert ys.size
        extents.append((ys.max() - ys.min(), xs.max() - xs.min()))
    if not corner:
        for a, b in zip(extents, extents[1:]):
            assert b[0] - a[0] == 2 * r and b[1] - a[1] == 2 * r, extents


@pytest.mark.parametrize('K', [5, 7])
@pytest.mark.parametrize('case', ['subnormal', 'overflow', 'inf'])
def test_special_affinity_sums_follow_ieee_division(K, case):
    """Subnormal sum_k |a_k| divides exactly, an overflowing sum gives weights of 0, +-inf guidance gives NaN where inf/inf."""
    g, d, s = [None if a is None else a.numpy() for a in make_inputs(K + 7, 1, 2, 24, 36, K * K - 1, 'signed', 10)]
    if case == 'subnormal':
        g[:, :, 6:16, 8:20] *= np.float32(1e-42)
    elif case == 'overflow':
        g[:, :, 6:16, 8:20] = np.sign(g[:, :, 6:16, 8:20]) * np.float32(3e37)
    else:
        g[0, 3, 10, 12] = np.inf
        g[0, 7, 15, 20] = -np.inf
    for abs_norm in (False, True):
        for N in (1, 3):
            _check_special(g, d, s, N, K, norm_name(K, abs_norm))


@pytest.mark.parametrize('abs_norm', [False, True])
def test_k3_is_the_3x3_operator_bit_for_bit(abs_norm):
    norm = '8sum_abs' if abs_norm else '8sum'
    g, d, s = [t.cuda() for t in make_inputs(3, 2, 2, 64, 96, 8, 'signed', 40)]
    ref = cspn_b200.Affinity_Propagate(12, 3, norm)(g, d, s)
    assert torch.equal(cspn_b200.Affinity_PropagateK(12, 3, norm)(g, d, s), ref)
    assert torch.equal(cspn_b200.propagate2d_k(g, d, s, 3, 12, norm), ref)
    L = _lib.lib()
    out = torch.empty_like(d)
    ws_bytes = L.cspn2d_k_workspace_bytes(2, 2, 64, 96, 3, 12)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    rc = L.cspn2d_k_fwd_f32(g.data_ptr(), d.data_ptr(), s.data_ptr(), out.data_ptr(), 2, 2, 64, 96, 8, 3, 12, int(abs_norm),
                            ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert L.cspn_last_algo() == _lib.ALGO_CLUSTER and torch.equal(out, ref)
    # and the backward through both modules
    gs = [g.clone().requires_grad_(True) for _ in range(2)]
    ds = [d.clone().requires_grad_(True) for _ in range(2)]
    go = torch.randn_like(d)
    cspn_b200.Affinity_Propagate(5, 3, norm)(gs[0], ds[0], s).backward(go)
    cspn_b200.Affinity_PropagateK(5, 3, norm)(gs[1], ds[1], s).backward(go)
    assert torch.equal(gs[0].grad, gs[1].grad) and torch.equal(ds[0].grad, ds[1].grad)


@pytest.mark.parametrize('K', [5, 7])
def test_an_image_gives_the_same_bits_alone_and_in_a_batch_of_launch_groups(K, monkeypatch):
    B, C, H, W, N = 8, 1, 48, 64, 6
    g, d, s = [t.cuda() for t in make_inputs(K + 70, B, C, H, W, K * K - 1, 'signed', 30)]
    alone = [cspn_b200.propagate2d_k(g[i:i + 1], d[i:i + 1], s[i:i + 1], K, N) for i in range(B)]
    one_group = cspn_b200.propagate2d_k(g, d, s, K, N)
    torch.cuda.synchronize()
    assert _lib.lib().cspn_last_launches() == 1 + N          # the whole batch is one launch group
    monkeypatch.setenv('CSPN_B200_KXK_GROUP', '3')            # groups of 3, 3, 2 images
    grouped = cspn_b200.propagate2d_k(g, d, s, K, N)
    torch.cuda.synchronize()
    assert _lib.lib().cspn_last_launches() == 3 * (1 + N)
    for i in range(B):
        assert torch.equal(alone[i], one_group[i:i + 1]) and torch.equal(alone[i], grouped[i:i + 1]), i
    gg = [None, None]
    for j, group in enumerate((None, '3')):
        if group is None:
            monkeypatch.delenv('CSPN_B200_KXK_GROUP')
        else:
            monkeypatch.setenv('CSPN_B200_KXK_GROUP', group)
        gc, dc = g.clone().requires_grad_(True), d.clone().requires_grad_(True)
        cspn_b200.Affinity_PropagateK(N, K)(gc, dc, s).sum().backward()
        gg[j] = (gc.grad, dc.grad)
    assert torch.equal(gg[0][0], gg[1][0]) and torch.equal(gg[0][1], gg[1][1])


BWD = [(K, abs_norm, shape, N) for K in (5, 7) for abs_norm in (False, True)
       for shape, N in (((2, 2, 12, 17), 5), ((1, 2, 10, 16), 24), ((1, 2, 9, 13), 1))]


@pytest.mark.parametrize('K,abs_norm,shape,N', BWD)
def test_gradients_match_fp64_autograd_of_the_torch_port(K, abs_norm, shape, N):
    B, C, H, W = shape
    norm = norm_name(K, abs_norm)
    nt = K * K - 1
    g, d, s = make_inputs(K * 31 + H + N, B, C, H, W, nt + 3, 'signed', 12)
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(K + N))
    g64, d64 = g.double().requires_grad_(True), d.double().requires_grad_(True)
    tpk.cspn2d_torch_k(g64, d64, s.double(), N, K, norm).backward(go.double())
    for use_op in (True, False):
        gc, dc = g.cuda().requires_grad_(True), d.cuda().requires_grad_(True)
        m = cspn_b200.Affinity_PropagateK(N, K, norm)
        m._use_op = use_op                                      # dispatcher op and ctypes autograd.Function
        out = m(gc, dc, s.cuda())
        out.backward(go.cuda())
        for ours, theirs, name in ((gc.grad, g64.grad, 'guidance'), (dc.grad, d64.grad, 'blur')):
            ours = ours.double().cpu()
            scale = theirs.abs().mean()
            err = (ours - theirs).abs()
            assert (err <= 2e-3 * (theirs.abs() + scale)).all(), (name, use_op, float(err.max()), float(scale))
        assert torch.count_nonzero(gc.grad[:, nt:]) == 0      # channels >= K*K-1 get zero gradient


@pytest.mark.parametrize('K', [5, 7])
def test_torch_compile_fullgraph_forward_and_backward(K):
    m = cspn_b200.Affinity_PropagateK(6, K, norm_name(K, True))
    g, d, s = [t.cuda() for t in make_inputs(K + 5, 2, 1, 24, 32, K * K - 1, 'bernoulli', 20)]

    def f(g, d, s):
        return m(g, d, s)

    cf = torch.compile(f, fullgraph=True)
    outs, grads = [], []
    for fn in (f, cf):
        gc, dc = g.clone().requires_grad_(True), d.clone().requires_grad_(True)
        out = fn(gc, dc, s)
        out.square().sum().backward()
        outs.append(out.detach())
        grads.append((gc.grad, dc.grad))
    assert torch.equal(outs[0], outs[1])
    assert torch.allclose(grads[0][0], grads[1][0], rtol=1e-5, atol=1e-6)
    assert torch.allclose(grads[0][1], grads[1][1], rtol=1e-5, atol=1e-6)


def test_cuda_graph_capture_of_the_forward():
    m = cspn_b200.Affinity_PropagateK(8, 5)
    g, d, s = [t.cuda() for t in make_inputs(55, 2, 1, 40, 64, 24, 'bernoulli', 20)]
    ref = m(g, d, s)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(g, d, s)                                              # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(g, d, s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    d.mul_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.allclose(out, m(g, d, s), rtol=0, atol=0)


@pytest.mark.parametrize('K', [5, 7])
def test_training_step_through_the_module(K):
    """conv -> K x K CSPN -> L1 -> SGD changes the producer's weights."""
    torch.manual_seed(0)
    nt = K * K - 1
    net = torch.nn.Conv2d(4, nt + 1, 3, padding=1).cuda()
    post = cspn_b200.Affinity_PropagateK(6, K, f'{nt}sum_abs')
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    x = torch.rand(2, 4, 20, 24, device='cuda')
    target = torch.rand(2, 1, 20, 24, device='cuda')
    w0 = net.weight.detach().clone()
    losses = []
    for _ in range(3):
        y = net(x)
        out = post(y[:, :nt], y[:, nt:], x[:, 3:4].clone())
        loss = (out - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert not torch.equal(net.weight, w0) and all(l == l for l in losses)
