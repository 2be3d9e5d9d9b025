"""GPU tests of the aggregation of the 2D steps (propagate2d_aggregate, cspn2d_agg_*_f32; DESIGN.md section 4.20): the
anchors bit for bit (one step with weight 1 is the K x K propagation forward and backward; random steps and weights are
the restatement built from separate propagations; dyadic cases are fp64), the bounds against fp64 autograd, the IEEE
masks, the launch counts, the memory contract, equal bits across batch splits, streams, runs, CUDA graphs and both Python
routes, and the dispatcher op under opcheck, torch.compile and a training step."""
import ctypes
import math

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _propagate2d_keep, norm_code_2d_k
from oracle import cspn_numpy as onp

import aggregate_reference as ar
import backward_exact as be
import memory_contract as mc

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def inputs(seed, B, C, H, W, K, T, gch=None, device='cuda'):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, gch or K * K - 1, H, W, generator=gen)
    d = torch.rand(B, C, H, W, generator=gen)
    s = (torch.rand(B, 1, H, W, generator=gen) < 0.3).float() * torch.rand(B, 1, H, W, generator=gen)
    s[:, :, :2] *= -1                                   # some negative samples: sign() and 1[> 0] differ there
    sw = torch.randn(B, T, H, W, generator=gen)
    go = torch.randn(B, C, H, W, generator=gen)
    return [t.to(device) for t in (g, d, s, sw, go)]


def iterate(g, d, s, K, n, norm, keep):
    """d_n from the library's own propagation: the K x K template's bits at every K (K = 3 on its generic route)."""
    code = norm_code_2d_k(K, norm)
    if keep:
        return _propagate2d_keep(g, d, s, K, n, code, _lib.ALGO_GENERIC)
    if K == 3:
        return cspn_b200.propagate2d(g, d, s, n, ('8sum', '8sum_abs')[code], _lib.ALGO_GENERIC)
    return cspn_b200.propagate2d_k(g, d, s, K, n, norm)


def run(g, d, s, sw, go, steps, K, norm=None, keep=False, use_op=True, monkeypatch=None):
    """(out, grad_guidance, grad_blur, grad_sparse, grad_step_weight) through the public function."""
    if monkeypatch is not None:
        monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', '0' if use_op else '1')
    leaves = [t.clone().requires_grad_(True) for t in (g, d, s, sw)]
    out = cspn_b200.propagate2d_aggregate(leaves[0], leaves[1], leaves[3], leaves[2], K, norm, keep, steps)
    out.backward(go)
    return [out.detach()] + [t.grad for t in leaves]


def autograd64(g, d, s, sw, go, steps, K, norm, keep):
    leaves = [t.detach().double().cpu().requires_grad_(True) for t in (g, d, s, sw)]
    out = ar.composition(*leaves, steps, K, norm, keep)
    out.backward(go.double().cpu())
    return [out.detach()] + [t.grad for t in leaves]


def bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- 1. anchors, bit for bit ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [5, 7])
@pytest.mark.parametrize('keep', [False, True])
@pytest.mark.parametrize('W,N', [(64, 6), (37, 3)])
def test_one_step_with_unit_weight_is_the_kxk_propagation(K, keep, W, N):
    """steps=(N,), weight 1: the forward of propagate2d_k and the gradients of Affinity_PropagateK's backward."""
    g, d, s, _, go = inputs(K * 10 + W + keep, 2, 2, 21, W, K, 1)
    sw = torch.ones(2, 1, 21, W, device='cuda')
    out, gg, gd, gs, gw = run(g, d, s, sw, go, (N,), K, keep=keep)
    gc, dc, sc = [t.clone().requires_grad_(True) for t in (g, d, s)]
    ref = cspn_b200.Affinity_PropagateK(N, K, keep_sparse=keep)(gc, dc, sc)
    ref.backward(go)
    assert bits(out, ref.detach())
    assert bits(gg, gc.grad) and bits(gd, dc.grad)
    if keep:
        assert bits(gs, sc.grad)
    else:
        assert gs is None
    assert bits(gw, ar.grad_step_weight(go, [ref.detach()]))


@pytest.mark.parametrize('keep', [False, True])
def test_one_step_with_unit_weight_at_k3_is_the_generic_route(keep, monkeypatch):
    """K = 3: the forward of propagate2d(algo=ALGO_GENERIC) and the backward that CSPN_B200_BWD=steps selects."""
    g, d, s, _, go = inputs(33 + keep, 2, 2, 19, 40, 3, 1)
    sw = torch.ones(2, 1, 19, 40, device='cuda')
    out, gg, gd, gs, gw = run(g, d, s, sw, go, (7,), 3, keep=keep)
    assert bits(out, iterate(g, d, s, 3, 7, None, keep))
    monkeypatch.setenv('CSPN_B200_BWD', 'steps')
    gc, dc, sc = [t.clone().requires_grad_(True) for t in (g, d, s)]
    ref = cspn_b200.Affinity_PropagateK(7, 3, keep_sparse=keep)(gc, dc, sc)
    ref.backward(go)
    assert bits(gg, gc.grad) and bits(gd, dc.grad)
    if keep:
        assert bits(gs, sc.grad)


RANDOM = [(3, '8sum', False, (1, 2, 5, 6), 64), (3, '8sum_abs', True, (3, 4), 41), (5, '24sum', True, (1, 2, 3, 4, 5, 6, 7, 8), 64),
          (5, '24sum_abs', False, (2, 9), 30), (7, '48sum', False, (4, 5, 11), 36), (7, '48sum_abs', True, (1, 12), 64)]


@pytest.mark.parametrize('K,norm,keep,steps,W', RANDOM)
def test_random_steps_and_weights_are_the_restatement(K, norm, keep, steps, W):
    """out and grad_step_weight have the bits of the kernels' sums over separate propagations d_{s_j}."""
    g, d, s, sw, go = inputs(K * 7 + len(steps) + W, 2, 3, 18, W, K, len(steps), gch=K * K + 2)
    out, _, _, _, gw = run(g, d, s, sw, go, steps, K, norm, keep)
    ds = [iterate(g, d, s, K, n, norm, keep) for n in steps]
    assert bits(out, ar.aggregate(ds, sw))
    assert bits(gw, ar.grad_step_weight(go, ds))


@pytest.mark.parametrize('K,sparse,keep', [(3, 'signed', False), (5, 'bernoulli', True), (7, None, False), (5, 'signed', True)])
def test_dyadic_cases_equal_fp64(K, sparse, keep):
    steps = (1, 3, 4)
    g, d, s, go = be.dyadic_2d(K * 5 + keep, 2, 2, 13, 20, K, sparse)
    s = torch.zeros(2, 1, 13, 20) if s is None else s
    sw = ar.dyadic_weights(torch.Generator().manual_seed(K + 1), (2, len(steps), 13, 20))
    ref = autograd64(g, d, s, sw, go, steps, K, None, keep)
    got = run(*[t.cuda() for t in (g, d, s, sw, go)], steps, K, keep=keep)
    for a, b, name in zip(got, ref, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse', 'grad_step_weight')):
        if b is None or (name == 'grad_sparse' and not keep):
            continue
        assert torch.equal(a.double().cpu(), b), name


# ---- 2. bounds and IEEE ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K,norm,keep,steps', [(3, '8sum', False, (1, 2, 3, 4, 5)), (5, '24sum_abs', True, (2, 6, 9)),
                                               (7, '48sum', True, (1, 4)), (5, '24sum', False, tuple(range(1, 13)))])
@pytest.mark.parametrize('use_op', [True, False])
def test_gradients_within_the_kxk_tolerance_of_fp64_autograd(K, norm, keep, steps, use_op, monkeypatch):
    g, d, s, sw, go = inputs(K + len(steps), 2, 2, 12, 17, K, len(steps))
    got = run(g, d, s, sw, go, steps, K, norm, keep, use_op, monkeypatch)
    ref = autograd64(g, d, s, sw, go, steps, K, norm, keep)
    for a, b, name in zip(got, ref, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse', 'grad_step_weight')):
        if name == 'grad_sparse' and not keep:
            assert a is None
            continue
        ok, err, scale = ar.within(a, b)
        assert ok, (name, err, scale)


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('where', ['guidance', 'blur', 'weight'])
def test_ieee_masks_equal_the_fp64_composition(K, where):
    g, d, s, sw, go = inputs(K + 50, 1, 2, 14, 20, K, 3)
    steps = (1, 3, 4)
    if where == 'guidance':
        g[0, 2, 5, 6] = float('nan')
        g[0, 0, 9, 12] = float('inf')
    elif where == 'blur':
        d[0, 1, 7, 3] = float('inf')
        d[0, 0, 2, 15] = float('nan')
    else:
        sw[0, 1, 4, 4] = float('nan')
        sw[0, 0, 10, 10] = float('inf')
        sw[0, 2, 3, 3] = 0.0
    out, _, _, _, gw = run(g, d, s, sw, go, steps, K, keep=True)
    ref = autograd64(g, d, s, sw, go, steps, K, None, True)
    for a, b, name in ((out, ref[0], 'out'), (gw, ref[4], 'grad_step_weight')):
        a = a.double().cpu()
        assert torch.equal(torch.isnan(a), torch.isnan(b)), name
        assert torch.equal(torch.isinf(a), torch.isinf(b)) and torch.equal(a[torch.isinf(a)], b[torch.isinf(b)]), name
        fin = torch.isfinite(b)
        assert ar.within(a[fin], b[fin])[0], name


# ---- 3. behaviour -----------------------------------------------------------------------------------------------------------
def c_fwd(g, d, s, sw, steps, K, keep, out=None, ws=None):
    L = _lib.lib()
    B, C, H, W = d.shape
    st = (ctypes.c_int * len(steps))(*steps)
    out = torch.empty_like(d) if out is None else out
    if ws is None:
        n = L.cspn2d_agg_workspace_bytes(B, C, H, W, K, st, len(steps), int(keep))
        ws = mc.workspace(n)
    rc = L.cspn2d_agg_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(sw), _ptr(out), B, C, H, W, g.shape[1], K, st, len(steps), 0,
                              int(keep), ws.ptr(), ws.nbytes, _stream())
    _lib.check(rc, 'cspn2d_agg_fwd_f32')
    return out, L.cspn_last_launches()


def c_bwd(g, d, s, sw, go, steps, K, keep, outs, ws):
    L = _lib.lib()
    B, C, H, W = d.shape
    st = (ctypes.c_int * len(steps))(*steps)
    rc = L.cspn2d_agg_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(sw), _ptr(go), *[None if o is None else o.ptr() for o in outs],
                              B, C, H, W, g.shape[1], K, st, len(steps), 0, int(keep), ws.ptr(), ws.nbytes, _stream())
    _lib.check(rc, 'cspn2d_agg_bwd_f32')
    return L.cspn_last_launches()


@pytest.mark.parametrize('K', [3, 5, 7])
def test_launch_counts(K):
    g, d, s, sw, go = inputs(K, 2, 1, 16, 32, K, 70)
    steps = tuple(range(1, 71))
    assert c_fwd(g, d, s, sw, steps, K, True)[1] == 1 + 70
    L = _lib.lib()
    st = (ctypes.c_int * 70)(*steps)
    ws = mc.workspace(L.cspn2d_agg_bwd_workspace_bytes(2, 1, 16, 32, K, st, 70, 1))
    outs = [mc.guarded(t.shape) for t in (g, d, s, sw)]
    assert c_bwd(g, d, s, sw, go, steps, K, True, outs, ws) == 2 + 2 * 70 + math.ceil(70 / 64)
    assert c_fwd(g, d, s, sw[:, :3].contiguous(), (2, 5, 9), K, False)[1] == 1 + 9


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('offset', [0, 4])
@pytest.mark.parametrize('keep', [False, True])
def test_memory_contract(K, offset, keep):
    """Outputs written exactly (guarded, every element), inputs untouched, and no workspace word read before it is
    written: sentinel- and zero-filled workspaces give the same bits.  Offset 4 takes the one-pixel-per-thread kernels."""
    g, d, s, sw, go = inputs(K + offset, 2, 2, 20, 32, K, 3, gch=K * K + 1)
    steps = (2, 3, 5)
    ins = [g, d, s, sw, go]
    before = mc.snapshot(ins)
    L = _lib.lib()
    st = (ctypes.c_int * 3)(*steps)
    fw = []
    for fill in ('sentinel', 'zero'):
        o = mc.guarded(d.shape, offset)
        ws = mc.workspace(L.cspn2d_agg_workspace_bytes(2, 2, 20, 32, K, st, 3, int(keep)), offset, fill)
        c_fwd(g, d, s, sw, steps, K, keep, o.t, ws)
        torch.cuda.synchronize()
        mc.assert_written(o, 'out')
        assert ws.guards_intact()
        fw.append(o.t.clone())
    assert mc.same_bits(*fw)
    bw = []
    for fill in ('sentinel', 'zero'):
        outs = [mc.guarded(t.shape, offset) for t in (g, d, s, sw)]
        ws = mc.workspace(L.cspn2d_agg_bwd_workspace_bytes(2, 2, 20, 32, K, st, 3, int(keep)), offset, fill)
        c_bwd(g, d, s, sw, go, steps, K, keep, outs, ws)
        torch.cuda.synchronize()
        for o, name in zip(outs, ('grad_guidance', 'grad_blur', 'grad_sparse', 'grad_step_weight')):
            mc.assert_written(o, name)
        assert ws.guards_intact()
        bw.append([o.t.clone() for o in outs])
    for a, b in zip(*bw):
        assert mc.same_bits(a, b)
    assert mc.unchanged(before, ins)


def test_equal_bits_across_batch_splits_streams_runs_and_routes(monkeypatch):
    g, d, s, sw, go = inputs(91, 5, 2, 24, 48, 5, 4)
    steps = (1, 2, 6, 7)
    ref = run(g, d, s, sw, go, steps, 5, keep=True)
    for group in ('1', '2', '3'):
        monkeypatch.setenv('CSPN_B200_KXK_GROUP', group)
        assert all(bits(a, b) for a, b in zip(run(g, d, s, sw, go, steps, 5, keep=True), ref)), group
    monkeypatch.delenv('CSPN_B200_KXK_GROUP')
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = run(g, d, s, sw, go, steps, 5, keep=True)
    torch.cuda.current_stream().wait_stream(side)
    assert all(bits(a, b) for a, b in zip(other, ref))
    assert all(bits(a, b) for a, b in zip(run(g, d, s, sw, go, steps, 5, keep=True), ref))
    for use_op in (True, False):
        assert all(bits(a, b) for a, b in zip(run(g, d, s, sw, go, steps, 5, None, True, use_op, monkeypatch), ref)), use_op


def test_cuda_graph_capture_forward_and_backward():
    g, d, s, sw, go = inputs(17, 2, 1, 40, 64, 7, 5)
    steps = (1, 2, 3, 4, 8)
    ref = run(g, d, s, sw, go, steps, 7, keep=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(g, d, s, sw, go, steps, 7, keep=True)                 # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    leaves = [t.clone().requires_grad_(True) for t in (g, d, s, sw)]
    with torch.cuda.graph(graph):
        out = cspn_b200.propagate2d_aggregate(leaves[0], leaves[1], leaves[3], leaves[2], 7, None, True, steps)
        grads = torch.autograd.grad(out, leaves, go)
    graph.replay()
    torch.cuda.synchronize()
    assert bits(out, ref[0]) and all(bits(a, b) for a, b in zip(grads, ref[1:]))


def test_opcheck():
    torch_op.load()
    g, d, s, sw, _ = inputs(7, 1, 1, 12, 16, 5, 2)
    for t in (g, d, s, sw):
        t.requires_grad_(True)
    for keep in (False, True):
        torch.library.opcheck(torch.ops.cspn_b200.propagate2d_aggregate.default, (g, d, s, sw, [1, 3], 5, 0, keep),
                              test_utils=('test_schema', 'test_faketensor', 'test_autograd_registration',
                                          'test_aot_dispatch_dynamic'))


def test_torch_compile_fullgraph():
    g, d, s, sw, go = inputs(8, 2, 1, 24, 32, 5, 3)
    steps = (1, 2, 4)

    def f(g, d, s, sw):
        return cspn_b200.propagate2d_aggregate(g, d, sw, s, 5, None, True, steps)

    cf = torch.compile(f, fullgraph=True)
    res = []
    for fn in (f, cf):
        leaves = [t.clone().requires_grad_(True) for t in (g, d, s, sw)]
        out = fn(*leaves)
        out.backward(go)
        res.append([out.detach()] + [t.grad for t in leaves])
    assert all(bits(a, b) for a, b in zip(*res))


def test_training_tail_against_fp64_autograd():
    """CSPN++'s composition: three kernel sizes on guidance slices of 8 / 24 / 48 channels, softmax'd step weights per
    size and a softmax'd kernel weight mixing them; the gradients of the producing convolution match fp64 autograd."""
    torch.manual_seed(0)
    N = 6
    net = torch.nn.Conv2d(4, 8 + 24 + 48 + 3 * N + 3, 3, padding=1).cuda()
    x = torch.rand(2, 4, 16, 20, device='cuda')
    blur, sparse = torch.rand(2, 1, 16, 20, device='cuda'), (torch.rand(2, 1, 16, 20, device='cuda') > 0.8).float()

    def tail(y, fn):
        gs = (y[:, :8], y[:, 8:32], y[:, 32:80])
        lam = [torch.softmax(y[:, 80 + N * i:80 + N * (i + 1)], 1) for i in range(3)]
        kw = torch.softmax(y[:, 80 + 3 * N:], 1)
        outs = [fn(gs[i], lam[i], K) for i, K in enumerate((3, 5, 7))]
        return sum(kw[:, i:i + 1] * outs[i] for i in range(3))

    y = net(x)
    ours = tail(y, lambda g, lam, K: cspn_b200.propagate2d_aggregate(g, blur, lam, sparse, K, keep_sparse=True))
    (gw,) = torch.autograd.grad(ours.square().mean(), net.weight)
    w64 = net.weight.detach().double().requires_grad_(True)
    y64 = torch.nn.functional.conv2d(x.double(), w64, net.bias.detach().double(), padding=1)
    ref = tail(y64, lambda g, lam, K: ar.composition(g, blur.double(), sparse.double(), lam, None, K, None, True))
    (gw64,) = torch.autograd.grad(ref.square().mean(), w64)
    assert ar.within(ours.detach(), ref.detach(), 1e-5)[0]
    ok, err, scale = ar.within(gw, gw64)
    assert ok, (err, scale)


def test_smoke_parity_with_the_oracle_at_k5():
    """The op at steps=(N,), weight 1, against the numpy oracle's K x K propagation (the oracle's parity bound)."""
    from oracle import cspn_numpy_k as onk
    g, d, s, _, _ = inputs(5, 2, 1, 30, 44, 5, 1)
    out = cspn_b200.propagate2d_aggregate(g, d, torch.ones(2, 1, 30, 44, device='cuda'), s, 5, steps=(6,))
    ref = onk.cspn2d_k(g.cpu().numpy(), d.cpu().numpy(), s.cpu().numpy(), 6, 5, '24sum')
    assert onp.parity_ok(out.cpu().numpy(), ref, 1e-4)[0]
