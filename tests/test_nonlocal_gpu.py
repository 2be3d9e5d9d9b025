"""GPU tests of propagate2d_nonlocal (NLSPN's non-local propagation, DESIGN.md section 4.21): the forward and every
gradient against the fp64 explicit restatement of tests/nonlocal_reference.py, bit for bit on exact cases, the IEEE masks,
determinism across calls, streams, CUDA graphs, routes and batch splits, and the memory contract."""

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
import memory_contract as mc
import nonlocal_reference as nr

pytestmark = pytest.mark.gpu


def kernel(feat, offset, affinity, sparse, K, N, grad_out):
    """(out, grad_feat, grad_offset, grad_affinity, grad_sparse or None) through the library."""
    return nr.grads(lambda f, o, a, s, K, N: cspn_b200.propagate2d_nonlocal(f, o, a, s, K, N), feat, offset, affinity, sparse, K, N,
                    grad_out)


def to(dev, *ts):
    return [None if t is None else t.to(dev) for t in ts]


def bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def check_tolerance(feat, offset, affinity, sparse, K, N, seed=0):
    """Normwise distance to the fp64 restatement at most 4x that of the eager-fp32 restatement, output and every gradient."""
    gen = torch.Generator().manual_seed(seed)
    go = torch.randn(feat.shape, generator=gen).cuda()
    got = kernel(feat, offset, affinity, sparse, K, N, go)
    e32 = nr.grads(nr.propagate, feat, offset, affinity, sparse, K, N, go)
    ref = nr.grads(nr.propagate, feat, offset, affinity, sparse, K, N, go, dtype=torch.float64)
    for name, g, e, r in zip(('out', 'feat', 'offset', 'affinity', 'sparse'), got, e32, ref):
        if r is None:
            assert g is None
            continue
        dk, de = nr.normwise(g, r), nr.normwise(e, r)
        assert dk <= 4 * de + 1e-7, (name, dk, de)


@pytest.mark.parametrize('K,N', [(3, 18), (5, 6), (7, 4)])
@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('sparse', [False, True])
@pytest.mark.parametrize('scale', [2.5, 50.0])
def test_forward_and_gradients_within_tolerance_of_fp64(K, N, C, sparse, scale):
    ins = nr.make_inputs(2, C, 21, 37, K, scale=scale, seed=K * 10 + C, sparse=sparse, device='cuda')
    check_tolerance(*ins, K, N)


@pytest.mark.parametrize('shape', [(1, 1, 1, 9), (2, 2, 7, 1), (1, 1, 1, 1), (3, 1, 5, 33)])
def test_degenerate_and_odd_shapes(shape):
    B, C, H, W = shape
    check_tolerance(*nr.make_inputs(B, C, H, W, 3, scale=1.5, seed=H * W, sparse=True, device='cuda'), 3, 5)


def test_non_contiguous_views():
    f, o, a, s = nr.make_inputs(2, 6, 16, 40, 5, scale=3.0, seed=3, sparse=True, device='cuda')
    fv, sv = f[:, ::2], s[:, 1::2]                   # channel-strided views of feat and sparse_depth
    ov = torch.cat([o, o], 3)[..., :40]              # a view with a row stride of 80
    av = a.transpose(2, 3).contiguous().transpose(2, 3)
    assert not fv.is_contiguous() and not ov.is_contiguous() and not av.is_contiguous()
    check_tolerance(fv, ov, av, sv, 5, 3)


def exact_inputs(K, seed, quarter):
    g = torch.Generator().manual_seed(seed)
    B, C, H, W, T = 2, 2, 9, 11, K * K - 1
    feat = torch.randint(-8, 9, (B, C, H, W), generator=g).float()
    step = 0.25 if quarter else 1.0
    offset = torch.randint(-12, 13, (B, 2 * T, H, W), generator=g).float() * step
    affinity = torch.tensor([0.0, 0.25, -0.25, 0.5, -0.5])[torch.randint(0, 5, (B, T, H, W), generator=g)]
    sparse = torch.where(torch.rand(B, C, H, W, generator=g) < 0.3, torch.randint(1, 9, (B, C, H, W), generator=g).float(),
                         torch.zeros(()))
    go = torch.randint(-4, 5, (B, C, H, W), generator=g).float()
    return feat, offset, affinity / (1 if not quarter else 2), sparse, go


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('quarter,N', [(False, 1), (False, 2), (False, 4), (True, 1), (True, 2)])
@pytest.mark.parametrize('sparse', [False, True])
def test_exact_cases_equal_fp64(K, quarter, N, sparse):
    """Integer offsets with affinities in {0, +-1/4, +-1/2} up to N = 4, quarter-pixel offsets at N <= 2: every value is
    exact in fp32, so the kernels must give fp64's bits."""
    f, o, a, s, go = exact_inputs(K, K * 7 + N, quarter)
    s = s if sparse else None
    got = kernel(*to('cuda', f, o, a, s), K, N, go.cuda())
    ref = nr.grads(nr.propagate, f, o, a, s, K, N, go, dtype=torch.float64)
    for name, g, r in zip(('out', 'feat', 'offset', 'affinity', 'sparse'), got, ref):
        assert (g is None) == (r is None), name
        if r is not None:
            assert torch.equal(g.cpu(), r.float()), name


SPECIALS = {'nan': float('nan'), 'inf': float('inf'), '-inf': float('-inf'), 'huge': 1e30}


@pytest.mark.parametrize('where', ['feat', 'offset', 'affinity', 'sparse', 'grad_out'])
@pytest.mark.parametrize('value', list(SPECIALS))
def test_ieee_masks_equal_the_reference(where, value):
    f, o, a, s = nr.make_inputs(1, 2, 10, 12, 3, scale=2.0, seed=5, sparse=True)
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(1))
    tgt = {'feat': f, 'offset': o, 'affinity': a, 'sparse': s, 'grad_out': go}[where]
    tgt.view(-1)[[3, 57, tgt.numel() // 2]] = SPECIALS[value]
    if where == 'offset':
        o[0, 4, 2, 3] = -1.0 - 0.0     # a position exactly at -1 next to the special ones
    got = kernel(*to('cuda', f, o, a, s), 3, 3, go.cuda())
    # the restatement in fp32 and the kernels' order: a huge value overflows where fp64 would not
    ref = nr.grads(nr.propagate, f, o, a, s, 3, 3, go)
    for name, g, r in zip(('out', 'feat', 'offset', 'affinity', 'sparse'), got, ref):
        g = g.cpu()
        assert torch.equal(torch.isnan(g), torch.isnan(r)), (name, int((torch.isnan(g) != torch.isnan(r)).sum()))
        assert torch.equal(torch.isposinf(g), torch.isposinf(r)), name
        assert torch.equal(torch.isneginf(g), torch.isneginf(r)), name


def test_infinite_zero_weight_corner():
    """An integer position next to an infinite pixel: the zero-weight corner gives NaN in the forward (0 * inf), as
    torchvision does, and takes no part in grad_feat."""
    f = torch.zeros(1, 1, 4, 5)
    f[0, 0, 2, 3] = float('inf')
    o = torch.zeros(1, 16, 4, 5)
    a = torch.full((1, 8, 4, 5), 0.125)
    go = torch.ones(1, 1, 4, 5)
    got = kernel(*to('cuda', f, o, a, None), 3, 1, go.cuda())
    ref = nr.grads(nr.propagate, f, o, a, None, 3, 1, go, dtype=torch.float64)
    for g, r in zip(got, ref):
        if r is not None:
            assert torch.equal(torch.isnan(g.cpu()), torch.isnan(r.float()))
            fin = torch.isfinite(r)
            assert torch.equal(g.cpu()[fin], r.float()[fin])


def run_both(f, o, a, s, go, K=3, N=5):
    return kernel(f, o, a, s, K, N, go)


def test_determinism_calls_streams_graphs_routes_and_batch_split(monkeypatch):
    f, o, a, s = nr.make_inputs(3, 2, 24, 40, 3, scale=8.0, seed=11, sparse=True, device='cuda')
    go = torch.randn(f.shape, device='cuda')
    ref = run_both(f, o, a, s, go)
    assert all(bits(x, y) for x, y in zip(run_both(f, o, a, s, go), ref))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = run_both(f, o, a, s, go)
    torch.cuda.current_stream().wait_stream(side)
    assert all(bits(x, y) for x, y in zip(other, ref))
    for route in ('1', '0'):
        monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', route)
        assert all(bits(x, y) for x, y in zip(run_both(f, o, a, s, go), ref)), route
    monkeypatch.delenv('CSPN_B200_NO_TORCH_OP')
    for b in range(3):
        one = run_both(f[b:b + 1], o[b:b + 1], a[b:b + 1], s[b:b + 1], go[b:b + 1])
        assert all(bits(x, y[b:b + 1]) for x, y in zip(one, ref)), b


def test_cuda_graph_capture_and_replay_on_new_values():
    f, o, a, s = nr.make_inputs(2, 1, 20, 36, 3, scale=4.0, seed=21, sparse=True, device='cuda')
    go = torch.randn(f.shape, device='cuda')
    leaves = [t.clone().requires_grad_(True) for t in (f, o, a, s)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = cspn_b200.propagate2d_nonlocal(*leaves, 3, 6)       # warm-up on the side stream
        torch.autograd.grad(out, leaves, go)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = cspn_b200.propagate2d_nonlocal(*leaves, 3, 6)
        grads = torch.autograd.grad(out, leaves, go)
    f2, o2, a2, s2 = nr.make_inputs(2, 1, 20, 36, 3, scale=4.0, seed=22, sparse=True, device='cuda')
    with torch.no_grad():
        for leaf, new in zip(leaves, (f2, o2, a2, s2)):
            leaf.copy_(new)
    graph.replay()
    torch.cuda.synchronize()
    want = kernel(f2, o2, a2, s2, 3, 6, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


def test_requested_gradients_only_and_prop_time_zero():
    f, o, a, s = nr.make_inputs(2, 2, 12, 20, 5, scale=3.0, seed=4, sparse=True, device='cuda')
    go = torch.randn(f.shape, device='cuda')
    full = kernel(f, o, a, s, 5, 4, go)
    for i in range(4):
        leaves = [t.clone().requires_grad_(j == i) for j, t in enumerate((f, o, a, s))]
        out = cspn_b200.propagate2d_nonlocal(*leaves, 5, 4)
        (g,) = torch.autograd.grad(out, [leaves[i]], go)
        assert bits(g, full[1 + i]), i
    assert cspn_b200.propagate2d_nonlocal(f, o, a, s, 5, 0) is f
    m = cspn_b200.Affinity_PropagateNonLocal(4, 5)
    assert bits(m(f, o, a, s), full[0])


def c_call_fwd(f, o, a, s, out, K, N, ws):
    L = _lib.lib()
    B, C, H, W = f.shape
    rc = L.cspn2d_nl_fwd_f32(f.data_ptr(), o.data_ptr(), a.data_ptr(), None if s is None else s.data_ptr(), out.data_ptr(), B, C, H,
                             W, K, N, None if ws is None else ws.t.data_ptr(), 0 if ws is None else ws.nbytes,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


def c_call_bwd(f, o, a, s, go, outs, K, N, ws):
    L = _lib.lib()
    B, C, H, W = f.shape
    rc = L.cspn2d_nl_bwd_f32(f.data_ptr(), o.data_ptr(), a.data_ptr(), s.data_ptr(), go.data_ptr(), *[x.t.data_ptr() for x in outs],
                             B, C, H, W, K, N, ws.t.data_ptr(), ws.nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


@pytest.mark.parametrize('K', [3, 7])
@pytest.mark.parametrize('offset', [0, 4])
def test_memory_contract(K, offset):
    """Outputs written exactly (guarded, every element), inputs untouched, and no workspace word read before it is
    written: sentinel- and zero-filled workspaces give the same bits."""
    f, o, a, s = nr.make_inputs(2, 3, 13, 19, K, scale=6.0, seed=K + offset, sparse=True, device='cuda')
    go = torch.randn(f.shape, device='cuda')
    ins = [f, o, a, s, go]
    before = mc.snapshot(ins)
    L = _lib.lib()
    N = 4
    fw, bw = [], []
    for fill in ('sentinel', 'zero'):
        out = mc.guarded(f.shape, offset)
        ws = mc.workspace(L.cspn2d_nl_workspace_bytes(2, 3, 13, 19, K, N), offset, fill)
        c_call_fwd(f, o, a, s, out.t, K, N, ws)
        torch.cuda.synchronize()
        mc.assert_written(out, 'out')
        assert ws.guards_intact()
        fw.append(out.t.clone())
        outs = [mc.guarded(t.shape, offset) for t in (f, o, a, s)]
        ws = mc.workspace(L.cspn2d_nl_bwd_workspace_bytes(2, 3, 13, 19, K, N), offset, fill)
        c_call_bwd(f, o, a, s, go, outs, K, N, ws)
        torch.cuda.synchronize()
        for x, name in zip(outs, ('grad_feat', 'grad_offset', 'grad_affinity', 'grad_sparse')):
            mc.assert_written(x, name)
        assert ws.guards_intact()
        bw.append([x.t.clone() for x in outs])
    assert mc.same_bits(*fw)
    for x, y in zip(*bw):
        assert mc.same_bits(x, y)
    assert mc.unchanged(before, ins)
    want = kernel(f, o, a, s, K, N, go)
    assert bits(fw[0], want[0]) and all(bits(x, y) for x, y in zip(bw[0], want[1:]))


def test_refuses_overlapping_device_buffers():
    f, o, a, s = nr.make_inputs(1, 1, 8, 8, 3, device='cuda')
    L = _lib.lib()
    rc = L.cspn2d_nl_fwd_f32(f.data_ptr(), o.data_ptr(), a.data_ptr(), None, o.data_ptr(), 1, 1, 8, 8, 3, 1, None, 0,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == -1                                  # CSPN_ERR_INVALID_ARGUMENT
    assert b'overlaps' in L.cspn_last_error()


def test_opcheck():
    from cspn_b200 import torch_op
    torch_op.load()
    f, o, a, s = nr.make_inputs(1, 2, 6, 9, 3, seed=2, sparse=True, device='cuda')
    for t in (f, o, a, s):
        t.requires_grad_(True)
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_nonlocal.default, (f, o, a, s, 3, 2))
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_nonlocal.default, (f, o, a, None, 3, 1))
