"""GPU tests of propagate2d_dynamic (DySPN's step, DESIGN.md section 4.23): the forward and every gradient against the fp64
composition of tests/dynamic_reference.py and bit for bit against its kernel_order, bit for bit on dyadic cases across CTA
tile seams, the 4-pixel and 1-pixel
paths, the anchor to propagate2d_dilated, the IEEE masks, determinism, the requested gradients and launch counts, the
memory contract, the DySPN head end to end (INTEGRATION.md section 2h), torch.compile and opcheck."""
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
import dilated_reference as dr
import dynamic_reference as yr
import memory_contract as mc

pytestmark = pytest.mark.gpu
NAMES = ('out', 'affinity', 'attention', 'blur', 'sparse', 'conf')


def op(a, t, b, s, m, K):
    return cspn_b200.propagate2d_dynamic(a, t, b, s, m, K)


def run(ins, K, go):
    """(out, grad_affinity, grad_attention, grad_blur, grad_sparse, grad_conf) through the library."""
    return yr.grads(op, *ins, K, go)


def cuda(ts):
    return [None if t is None else t.cuda() for t in ts]


def bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def within(got, ref, fwd_tol=1e-5, grad_tol=2e-3):
    for name, g, r in zip(NAMES, got, ref):
        assert (g is None) == (r is None), name
        if r is None:
            continue
        tol = fwd_tol if name == 'out' else grad_tol
        g, r = g.double(), r.to(g.device)
        bound = tol * (r.abs() + r.abs().mean())
        assert bool(((g - r).abs() <= bound).all()), (name, float(((g - r).abs() / bound).max()))


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('N', [1, 6, 24])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
def test_forward_and_gradients_within_tolerance_of_fp64(K, N, samples):
    # C and W % 4 vary with the case, so every value of each meets every K, N and sample mode
    case = K + N + (0 if samples is None else len(samples))
    C = (1, 3)[case % 2]
    W = (48, 45)[(case // 2) % 2]
    ins = yr.make_inputs(2, C, 29, W, K, N, samples, seed=case * 31 + N, device='cuda')
    go = torch.randn(2, C, 29, W, device='cuda')
    got = run(ins, K, go)
    within(got, yr.grads(yr.composition, *ins, K, go, dtype=torch.float64))
    # and the bits of the kernels' stated order of operations
    for name, g, r in zip(NAMES, got, yr.kernel_order(*ins, K, go)):
        assert bits(g, r), name


@pytest.mark.parametrize('K', [3, 7])
def test_misaligned_and_strided_views(K):
    a, t, b, s, m = yr.make_inputs(2, 2, 20, 40, K, 6, 'soft', seed=K, device='cuda')
    av = torch.cat([a, a], 3)[..., 1:41]                             # misaligned start, row stride 80
    tv = torch.cat([t, t], 1)[:, ::2]
    bv = torch.cat([b, b], 1)[:, 1::2]
    ins = (av, tv, bv, s, m)
    assert not av.is_contiguous() and not tv.is_contiguous() and not bv.is_contiguous()
    go = torch.randn(2, 2, 20, 40, device='cuda')
    within(run(ins, K, go), yr.grads(yr.composition, *ins, K, go, dtype=torch.float64))


@pytest.mark.parametrize('K', [3, 5, 7])
def test_vector_and_scalar_paths_give_the_same_bits(K):
    """W % 4 == 0 from an aligned base runs 4 pixels per thread; the same values 4 bytes into a buffer run the 1-pixel
    path; each pixel's arithmetic is the same."""
    ins = yr.make_inputs(2, 3, 17, 64, K, 6, 'soft', seed=4, device='cuda')
    go = torch.randn(2, 3, 17, 64, device='cuda')
    ref = run(ins, K, go)

    def shifted(t):
        buf = torch.empty(t.numel() + 1, device='cuda')
        v = buf[1:].view(t.shape)
        v.copy_(t)
        return v

    got = run([shifted(t) for t in ins], K, go)
    assert all(bits(x, y) for x, y in zip(got, ref))


@pytest.mark.parametrize('K,N', [(3, 3), (5, 2), (7, 2)])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
@pytest.mark.parametrize('shape', [(2, 2, 13, 20), (1, 2, 37, 260), (1, 1, 45, 261)])
def test_dyadic_cases_equal_fp64_bit_for_bit(K, N, samples, shape):
    """(37, 260) crosses three 128 x 16 tiles of the 4-pixel step in x and y, with partial last tiles; (45, 261) runs
    the 1-pixel step across nine 32-wide tiles."""
    ins, go = yr.dyadic_inputs(*shape, K, N, samples, seed=K * 10 + N + shape[2])
    ref = yr.grads(yr.composition, *ins, K, go, dtype=torch.float64)
    # the premise: every intermediate is exact, so fp32 in any order gives fp64's values
    r32 = yr.grads(yr.explicit, *ins, K, go)
    assert all(x is None or torch.equal(x, y.float()) for x, y in zip(r32, ref))
    got = run(cuda(ins), K, go.cuda())
    for name, g, r in zip(NAMES, got, ref):
        assert (g is None) == (r is None), name
        if r is not None:
            assert torch.equal(g.cpu(), r.float()), name


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [40, 37])
@pytest.mark.parametrize('samples', [None, 'soft'])
def test_anchor_to_propagate2d_dilated(K, W, samples):
    """Attention 1 and a zero centre affinity: propagate2d_dilated at dilation 1 with rho = 1 - sum_j affinity_j, summed in
    fp32 with j ascending, as its centre weight.  The output and the blur gradient are bit for bit."""
    N = 6
    a, _, b, s, m = yr.make_inputs(2, 2, 23, W, K, N, samples, seed=K + W, device='cuda')
    c = K * K // 2
    a[:, c] = 0
    t = torch.ones(2, N * ((K + 1) // 2), 23, W, device='cuda')
    S = a[:, 0]
    for j in range(1, K * K):
        S = S + a[:, j]
    kern = a.clone()
    kern[:, c] = 1 - S
    go = torch.randn(2, 2, 23, W, device='cuda')
    got = run((a, t, b, s, m), K, go)
    want = dr.grads(lambda k, x, s_, m_, K, d, n: cspn_b200.propagate2d_dilated(k, x, s_, m_, K, d, n), kern, b, s, m, K, 1, N, go)
    assert bits(got[0], want[0]) and bits(got[3], want[2])


SPECIALS = {'nan': float('nan'), 'inf': float('inf'), '-inf': float('-inf')}


@pytest.mark.parametrize('where', ['affinity', 'attention', 'blur', 'sparse', 'conf', 'grad_out'])
@pytest.mark.parametrize('value', list(SPECIALS))
def test_ieee_masks_equal_fp64(where, value):
    a, t, b, s, m = yr.make_inputs(1, 2, 10, 12, 3, 3, 'soft', seed=5)
    go = torch.randn(b.shape, generator=torch.Generator().manual_seed(1))
    tgt = {'affinity': a, 'attention': t, 'blur': b, 'sparse': s, 'conf': m, 'grad_out': go}[where]
    tgt.view(-1)[[3, 57, tgt.numel() // 2 + 5]] = SPECIALS[value]
    got = run(cuda((a, t, b, s, m)), 3, go.cuda())
    ref = yr.grads(yr.composition, a, t, b, s, m, 3, go, dtype=torch.float64)
    for name, g, r in zip(NAMES, got, ref):
        g = g.cpu()
        assert torch.equal(torch.isnan(g), torch.isnan(r)), (name, int((torch.isnan(g) != torch.isnan(r)).sum()))
        assert torch.equal(torch.isposinf(g), torch.isposinf(r)), name
        assert torch.equal(torch.isneginf(g), torch.isneginf(r)), name


def test_determinism_calls_streams_routes_and_batch_split(monkeypatch):
    ins = yr.make_inputs(3, 2, 24, 40, 5, 6, 'soft', seed=11, device='cuda')
    go = torch.randn(3, 2, 24, 40, device='cuda')
    ref = run(ins, 5, go)
    assert all(bits(x, y) for x, y in zip(run(ins, 5, go), ref))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = run(ins, 5, go)
    torch.cuda.current_stream().wait_stream(side)
    assert all(bits(x, y) for x, y in zip(other, ref))
    for route in ('1', '0'):
        monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', route)
        assert all(bits(x, y) for x, y in zip(run(ins, 5, go), ref)), route
    monkeypatch.delenv('CSPN_B200_NO_TORCH_OP')
    for b in range(3):
        one = run([t[b:b + 1] for t in ins], 5, go[b:b + 1])
        assert all(bits(x, y[b:b + 1]) for x, y in zip(one, ref)), b


def test_cuda_graph_capture_and_replay_on_new_values():
    ins = yr.make_inputs(2, 1, 20, 36, 7, 4, 'soft', seed=21, device='cuda')
    go = torch.randn(2, 1, 20, 36, device='cuda')
    leaves = [t.clone().requires_grad_(True) for t in ins]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = op(*leaves, 7)
        torch.autograd.grad(out, leaves, go)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = op(*leaves, 7)
        grads = torch.autograd.grad(out, leaves, go)
    new = yr.make_inputs(2, 1, 20, 36, 7, 4, 'soft', seed=22, device='cuda')
    with torch.no_grad():
        for leaf, t in zip(leaves, new):
            leaf.copy_(t)
    graph.replay()
    torch.cuda.synchronize()
    want = run(new, 7, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


def test_requested_gradients_only_and_no_steps():
    ins = yr.make_inputs(2, 2, 12, 20, 7, 4, 'soft', seed=4, device='cuda')
    go = torch.randn(2, 2, 12, 20, device='cuda')
    full = run(ins, 7, go)
    for i in range(5):
        leaves = [t.clone().requires_grad_(j == i) for j, t in enumerate(ins)]
        (g,) = torch.autograd.grad(op(*leaves, 7), [leaves[i]], go)
        assert bits(g, full[1 + i]), i
    a, t, b, s, m = ins
    assert op(a, t[:, :0], b, s, m, 7) is b
    assert bits(cspn_b200.Affinity_PropagateDynamic(4, 7)(*ins), full[0])
    leaves = [x.clone().requires_grad_(True) for x in (a, b, s, m)]
    t0 = t[:, :0].clone().requires_grad_(True)
    out = torch.ops.cspn_b200.propagate2d_dynamic(leaves[0], t0, *leaves[1:], 7)       # N = 0 through the op
    g = torch.autograd.grad(out, leaves + [t0], go)
    assert bits(out, b) and bits(g[1], go) and all(bool((x == 0).all()) for x in (g[0], g[2], g[3])) and g[4].numel() == 0


def launches_of_backward(ins, need):
    """The C backward's launch count with the gradients `need` (affinity, attention, blur, sparse, conf) requested, N = 5."""
    a, t, b, s, m = ins
    outs = [torch.empty_like(x) if n else None for x, n in zip(ins, need)]
    ws = torch.empty(_lib.lib().cspn2d_dyn_bwd_workspace_bytes(1, 1, 16, 16, 3, 5), dtype=torch.uint8, device='cuda')
    rc = _lib.lib().cspn2d_dyn_bwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), torch.ones_like(b).data_ptr(),
                                       *[None if o is None else o.data_ptr() for o in outs], 1, 1, 16, 16, 3, 5, ws.data_ptr(),
                                       ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    return _lib.lib().cspn_last_launches()


def test_partial_backward_runs_no_recomputed_steps():
    ins = yr.make_inputs(1, 1, 16, 16, 3, 5, 'soft', seed=1, device='cuda')
    assert launches_of_backward(ins, (True, True, True, True, True)) == 4 + 5 + 1
    assert launches_of_backward(ins, (False, True, False, False, False)) == 4 + 4 + 1   # the attention needs the iterates
    assert launches_of_backward(ins, (True, False, False, False, False)) == 4 + 4 + 1
    assert launches_of_backward(ins, (False, False, False, False, True)) == 4 + 4 + 1
    assert launches_of_backward(ins, (False, False, True, True, False)) == 5 + 1
    assert launches_of_backward(ins, (False, False, False, True, False)) == 4 + 1


def c_fwd(a, t, b, s, m, out, K, N, ws):
    B, C, H, W = b.shape
    rc = _lib.lib().cspn2d_dyn_fwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), out.data_ptr(), B, C, H, W,
                                       K, N, ws.t.data_ptr() if ws.nbytes else None, ws.nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


def c_bwd(a, t, b, s, m, go, outs, K, N, ws):
    B, C, H, W = b.shape
    ptrs = [None if x is None else x.t.data_ptr() for x in outs]
    rc = _lib.lib().cspn2d_dyn_bwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), go.data_ptr(), *ptrs, B, C,
                                       H, W, K, N, ws.t.data_ptr() if ws.nbytes else None, ws.nbytes,
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


@pytest.mark.parametrize('K', [3, 7])
@pytest.mark.parametrize('offset', [0, 4])
@pytest.mark.parametrize('which', ['all', 'blur_only', 'attention_conf'])
@pytest.mark.parametrize('shape', [(2, 3, 13, 20), (1, 1, 17, 132)])
def test_memory_contract(K, offset, which, shape):
    """Outputs written exactly (guarded, every element), NULL outputs skipped, inputs untouched, and no workspace word
    read before it is written: sentinel- and zero-filled workspaces give the same bits.  (17, 132) crosses a 4-pixel
    tile seam in x and a 16-row seam in y."""
    B, C, H, W = shape
    N = 4
    a, t, b, s, m = yr.make_inputs(B, C, H, W, K, N, 'soft', seed=K + offset, device='cuda')
    go = torch.randn(B, C, H, W, device='cuda')
    ins = [a, t, b, s, m, go]
    before = mc.snapshot(ins)
    L = _lib.lib()
    want_out = {'all': (1, 1, 1, 1, 1), 'blur_only': (0, 0, 1, 0, 0), 'attention_conf': (0, 1, 0, 0, 1)}[which]
    fw, bw = [], []
    for fill in ('sentinel', 'zero'):
        out = mc.guarded(b.shape, offset)
        ws = mc.workspace(L.cspn2d_dyn_workspace_bytes(B, C, H, W, K, N), offset, fill)
        c_fwd(a, t, b, s, m, out.t, K, N, ws)
        torch.cuda.synchronize()
        mc.assert_written(out, 'out')
        assert ws.guards_intact()
        fw.append(out.t.clone())
        outs = [mc.guarded(x.shape, offset) if w else None for x, w in zip((a, t, b, s, m), want_out)]
        ws = mc.workspace(L.cspn2d_dyn_bwd_workspace_bytes(B, C, H, W, K, N), offset, fill)
        c_bwd(a, t, b, s, m, go, outs, K, N, ws)
        torch.cuda.synchronize()
        for x, name in zip(outs, NAMES[1:]):
            if x is not None:
                mc.assert_written(x, name)
        assert ws.guards_intact()
        bw.append([None if x is None else x.t.clone() for x in outs])
    assert mc.same_bits(*fw)
    for x, y in zip(*bw):
        assert x is None or mc.same_bits(x, y)
    assert mc.unchanged(before, ins)
    want = run((a, t, b, s, m), K, go)
    assert bits(fw[0], want[0])
    assert all(x is None or bits(x, y) for x, y in zip(bw[0], want[1:]))


def test_refuses_overlapping_device_buffers():
    a, t, b, s, m = yr.make_inputs(1, 1, 8, 8, 3, 1, 'soft', device='cuda')
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    rc = L.cspn2d_dyn_fwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), t.data_ptr(), 1, 1, 8, 8, 3, 1, None,
                              0, st)
    assert rc == -1 and b'overlaps' in L.cspn_last_error()
    g = torch.empty(1, 9, 8, 8, device='cuda')
    rc = L.cspn2d_dyn_bwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), b.data_ptr(), g.data_ptr(), g.data_ptr(),
                              None, None, None, 1, 1, 8, 8, 3, 1, None, 0, st)
    assert rc == -1 and b'overlaps' in L.cspn_last_error()


def head_inputs(B, F, H, W, K, N, seed, device):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, F, H, W, generator=g)
    coarse = torch.rand(B, 1, H, W, generator=g) * 5 + 1
    sparse = torch.where(torch.rand(B, 1, H, W, generator=g) < 0.2, torch.rand(B, 1, H, W, generator=g) * 5 + 1, torch.zeros(()))
    w_aff = torch.randn(K * K, F, 3, 3, generator=g) * 0.3
    w_att = torch.randn(N * ((K + 1) // 2), F, 3, 3, generator=g) * 0.3
    w_conf = torch.randn(1, F, 3, 3, generator=g) * 0.3
    return [t.to(device) for t in (feat, coarse, sparse, w_aff, w_att, w_conf)]


def head_grads(leaves, use_op, dtype, go, K, N, samples):
    ls = [t.detach().to(dtype).requires_grad_(True) for t in leaves]
    feat, coarse, sparse, wa, wt, wc = ls
    out = yr.dyspn_head(feat, coarse, sparse if samples else None, wa, wt, wc, K, N, use_op=use_op)
    used = [feat, coarse, wa, wt] + ([wc] if samples else [])
    return [out.detach()] + list(torch.autograd.grad(out, used, go.to(dtype)))


@pytest.mark.parametrize('samples', [True, False])
def test_dyspn_head_end_to_end(samples):
    """INTEGRATION.md section 2h: the affinity conv normalised by sum|.|, the attention conv with a sigmoid, N = 6, K = 7 and
    the optional confidence replacement, against an fp64 model built from stock torch ops: the forward and the gradient
    of the features, the coarse depth and every convolution weight."""
    B, F, H, W, K, N = 2, 8, 24, 36, 7, 6
    leaves = head_inputs(B, F, H, W, K, N, 0, 'cuda')
    go = torch.randn(B, 1, H, W, device='cuda')
    got = head_grads(leaves, True, torch.float32, go, K, N, samples)
    ref = head_grads(leaves, False, torch.float64, go, K, N, samples)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert yr.normwise(g, r) < (1e-5 if i == 0 else 2e-4), (i, yr.normwise(g, r))


def test_torch_compile_is_one_node():
    ins = yr.make_inputs(2, 1, 16, 24, 5, 4, 'soft', seed=3, device='cuda')
    go = torch.randn(2, 1, 16, 24, device='cuda')

    def f(a, t, b, s, m):
        return cspn_b200.propagate2d_dynamic(a, t, b, s, m, 5) * 2

    torch._dynamo.reset()
    explain = torch._dynamo.explain(f)(*ins)
    assert explain.graph_break_count == 0 and explain.graph_count == 1
    cf = torch.compile(f, fullgraph=True)
    res = []
    for fn in (f, cf):
        leaves = [t.clone().requires_grad_(True) for t in ins]
        out = fn(*leaves)
        out.backward(go)
        res.append([out.detach()] + [t.grad for t in leaves])
    assert all(bits(a, b) for a, b in zip(*res))


def test_opcheck():
    from cspn_b200 import torch_op
    torch_op.load()
    a, t, b, s, m = yr.make_inputs(1, 2, 6, 9, 3, 2, 'soft', seed=2, device='cuda')
    for x in (a, t, b, s, m):
        x.requires_grad_(True)
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_dynamic.default, (a, t, b, s, m, 3))
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_dynamic.default, (a, t, b, None, None, 3))
