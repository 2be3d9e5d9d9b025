"""GPU tests of propagate2d_dilated (PENet's DA-CSPN++ step, DESIGN.md section 4.22): the forward and every gradient
against the fp64 composition of tests/dilated_reference.py, bit for bit on dyadic cases and against the polyphase
dilation-1 runs, the anchor to affinity_propagate, the IEEE masks, determinism, the memory contract, PENet's refinement
end to end (INTEGRATION.md section 2g) and torch.compile."""
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
import dilated_reference as dr
import memory_contract as mc

pytestmark = pytest.mark.gpu
NAMES = ('out', 'kernel', 'blur', 'sparse', 'conf')


def op(k, b, s, m, K, dil, N):
    return cspn_b200.propagate2d_dilated(k, b, s, m, K, dil, N)


def run(ins, K, dil, N, go):
    """(out, grad_kernel, grad_blur, grad_sparse, grad_conf) through the library."""
    return dr.grads(op, *ins, K, dil, N, go)


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
@pytest.mark.parametrize('dil', [1, 2, 3, 4])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
def test_forward_and_gradients_within_tolerance_of_fp64(K, dil, samples):
    # C, W % 4 and N vary with the case, so every value of each meets every K, d and sample mode
    case = K + dil + (0 if samples is None else len(samples))
    C = (1, 3)[case % 2]
    W = (48, 45)[(case // 2) % 2]
    N = (1, 6, 24)[(K + 2 * dil) % 3]
    ins = dr.make_inputs(2, C, 29, W, K, samples, seed=case * 31 + dil, device='cuda')
    go = torch.randn(2, C, 29, W, device='cuda')
    within(run(ins, K, dil, N, go), dr.grads(dr.composition, *ins, K, dil, N, go, dtype=torch.float64))


@pytest.mark.parametrize('K,dil', [(3, 2), (7, 1), (5, 4)])
def test_misaligned_and_strided_views(K, dil):
    k, b, s, m = dr.make_inputs(2, 2, 20, 40, K, 'soft', seed=K, device='cuda')
    kv = torch.cat([k, k], 3)[..., 1:41]                             # misaligned start, row stride 80
    bv = torch.cat([b, b], 1)[:, 1::2]
    ins = (kv, bv, s, m)
    assert not kv.is_contiguous() and not bv.is_contiguous()
    go = torch.randn(2, 2, 20, 40, device='cuda')
    within(run(ins, K, dil, 6, go), dr.grads(dr.composition, *ins, K, dil, 6, go, dtype=torch.float64))


def test_vector_and_scalar_paths_give_the_same_bits():
    """W % 4 == 0 from an aligned base runs 4 pixels per thread; the same values 4 bytes into a buffer run the scalar
    path; each pixel's arithmetic is the same."""
    k, b, s, m = dr.make_inputs(2, 3, 17, 64, 5, 'soft', seed=4, device='cuda')
    go = torch.randn(2, 3, 17, 64, device='cuda')
    ref = run((k, b, s, m), 5, 2, 6, go)

    def shifted(t):
        buf = torch.empty(t.numel() + 1, device='cuda')
        v = buf[1:].view(t.shape)
        v.copy_(t)
        return v

    got = run([shifted(t) for t in (k, b, s, m)], 5, 2, 6, go)
    assert all(bits(x, y) for x, y in zip(got, ref))


def dyadic_inputs(B, C, H, W, K, samples, seed):
    g = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, 0.0, 0.0, 0.25, -0.25, 0.5, -0.5, 1.0, -1.0])
    kernel = vals[torch.randint(0, 9, (B, K * K, H, W), generator=g)]
    blur = torch.randint(-4, 5, (B, C, H, W), generator=g).float()
    sparse = conf = None
    if samples:
        sparse = torch.randint(0, 5, (B, 1, H, W), generator=g).float()
        conf = torch.tensor([0.0, 0.5, 1.0])[torch.randint(0, 3, (B, 1, H, W), generator=g)]
        if samples == 'hard':
            conf = (sparse > 0).float()
    go = torch.randint(-2, 3, (B, C, H, W), generator=g).float()
    return [kernel, blur, sparse, conf], go


@pytest.mark.parametrize('K,N', [(3, 3), (5, 2), (7, 2)])
@pytest.mark.parametrize('dil', [1, 2, 4])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
def test_dyadic_cases_equal_fp64_bit_for_bit(K, N, dil, samples):
    ins, go = dyadic_inputs(2, 2, 13, 20, K, samples, seed=K * 10 + N + dil)
    ref = dr.grads(dr.composition, *ins, K, dil, N, go, dtype=torch.float64)
    # the premise: every intermediate is exact, so fp32 in any order gives fp64's values
    r32 = dr.grads(dr.explicit, *ins, K, dil, N, go)
    assert all(x is None or torch.equal(x, y.float()) for x, y in zip(r32, ref))
    got = run(cuda(ins), K, dil, N, go.cuda())
    for name, g, r in zip(NAMES, got, ref):
        assert (g is None) == (r is None), name
        if r is not None:
            assert torch.equal(g.cpu(), r.float()), name


def polyphase_grads(ins, K, dil, N, go):
    res = [torch.empty_like(t) if t is not None else None for t in [ins[1]] + list(ins)]
    H, W = ins[1].shape[2:]
    for a in range(min(dil, H)):
        for b in range(min(dil, W)):
            sub = [None if t is None else t[..., a::dil, b::dil].contiguous() for t in ins]
            got = run(sub, K, 1, N, go[..., a::dil, b::dil].contiguous())
            for r, g in zip(res, got):
                if r is not None:
                    r[..., a::dil, b::dil] = g
    return res


@pytest.mark.parametrize('K,dil', [(3, 2), (5, 2), (7, 3), (3, 4), (7, 4)])
@pytest.mark.parametrize('samples', [None, 'soft'])
def test_polyphase_identity_bit_for_bit(K, dil, samples):
    ins = dr.make_inputs(2, 2, 27, 52, K, samples, seed=dil * 5 + K, device='cuda')
    go = torch.randn(2, 2, 27, 52, device='cuda')
    got = run(ins, K, dil, 6, go)
    want = polyphase_grads(ins, K, dil, 6, go)
    for name, g, w in zip(NAMES, got, want):
        assert bits(g, w), name


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [40, 37])
@pytest.mark.parametrize('C', [1, 2])
def test_anchor_to_affinity_propagate(K, W, C):
    """d = 1, no samples, zero centre weight: the K x K gates path with the gates in reversed tap order.  The output and
    the blur gradient are bit for bit; the kernel gradient too at C = 1, and within the tolerance of fp64 at C = 2,
    where the K x K gather sums the channels before the steps and this op the steps before the channels."""
    k, b, _, _ = dr.make_inputs(2, C, 23, W, K, None, seed=K + W, device='cuda')
    c = K * K // 2
    k[:, c] = 0
    gates = torch.cat([k[:, :c], k[:, c + 1:]], 1).flip(1).contiguous()
    go = torch.randn(2, C, 23, W, device='cuda')
    got = run((k, b, None, None), K, 1, 6, go)
    want = dr.grads(lambda g, x, s, m, K, dil, N: cspn_b200.affinity_propagate(x, g, K, N), gates, b, None, None, K, 1, 6, go)
    assert torch.equal(got[0], want[0]) and torch.equal(got[2], want[2])
    gk = got[1]
    moved = torch.cat([gk[:, :c], gk[:, c + 1:]], 1).flip(1)
    if C == 1:
        assert torch.equal(moved, want[1])
    else:
        ref = dr.grads(dr.composition, k, b, None, None, K, 1, 6, go, dtype=torch.float64)
        within(got, ref)


SPECIALS = {'nan': float('nan'), 'inf': float('inf'), '-inf': float('-inf')}


@pytest.mark.parametrize('where', ['kernel', 'blur', 'sparse', 'conf', 'grad_out'])
@pytest.mark.parametrize('value', list(SPECIALS))
@pytest.mark.parametrize('dil', [1, 2])
def test_ieee_masks_equal_fp64(where, value, dil):
    k, b, s, m = dr.make_inputs(1, 2, 10, 12, 3, 'soft', seed=5)
    go = torch.randn(b.shape, generator=torch.Generator().manual_seed(1))
    tgt = {'kernel': k, 'blur': b, 'sparse': s, 'conf': m, 'grad_out': go}[where]
    tgt.view(-1)[[3, 57, tgt.numel() // 2 + 5]] = SPECIALS[value]
    got = run(cuda((k, b, s, m)), 3, dil, 3, go.cuda())
    ref = dr.grads(dr.composition, k, b, s, m, 3, dil, 3, go, dtype=torch.float64)
    for name, g, r in zip(NAMES, got, ref):
        g = g.cpu()
        assert torch.equal(torch.isnan(g), torch.isnan(r)), (name, int((torch.isnan(g) != torch.isnan(r)).sum()))
        assert torch.equal(torch.isposinf(g), torch.isposinf(r)), name
        assert torch.equal(torch.isneginf(g), torch.isneginf(r)), name


def test_determinism_calls_streams_graphs_routes_and_batch_split(monkeypatch):
    ins = dr.make_inputs(3, 2, 24, 40, 5, 'soft', seed=11, device='cuda')
    go = torch.randn(3, 2, 24, 40, device='cuda')
    ref = run(ins, 5, 2, 6, go)
    assert all(bits(x, y) for x, y in zip(run(ins, 5, 2, 6, go), ref))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = run(ins, 5, 2, 6, go)
    torch.cuda.current_stream().wait_stream(side)
    assert all(bits(x, y) for x, y in zip(other, ref))
    for route in ('1', '0'):
        monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', route)
        assert all(bits(x, y) for x, y in zip(run(ins, 5, 2, 6, go), ref)), route
    monkeypatch.delenv('CSPN_B200_NO_TORCH_OP')
    for b in range(3):
        one = run([t[b:b + 1] for t in ins], 5, 2, 6, go[b:b + 1])
        assert all(bits(x, y[b:b + 1]) for x, y in zip(one, ref)), b


def test_cuda_graph_capture_and_replay_on_new_values():
    ins = dr.make_inputs(2, 1, 20, 36, 3, 'soft', seed=21, device='cuda')
    go = torch.randn(2, 1, 20, 36, device='cuda')
    leaves = [t.clone().requires_grad_(True) for t in ins]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = op(*leaves, 3, 2, 6)
        torch.autograd.grad(out, leaves, go)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = op(*leaves, 3, 2, 6)
        grads = torch.autograd.grad(out, leaves, go)
    new = dr.make_inputs(2, 1, 20, 36, 3, 'soft', seed=22, device='cuda')
    with torch.no_grad():
        for leaf, t in zip(leaves, new):
            leaf.copy_(t)
    graph.replay()
    torch.cuda.synchronize()
    want = run(new, 3, 2, 6, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


def test_requested_gradients_only_and_prop_time_zero():
    ins = dr.make_inputs(2, 2, 12, 20, 7, 'soft', seed=4, device='cuda')
    go = torch.randn(2, 2, 12, 20, device='cuda')
    full = run(ins, 7, 2, 4, go)
    for i in range(4):
        leaves = [t.clone().requires_grad_(j == i) for j, t in enumerate(ins)]
        (g,) = torch.autograd.grad(op(*leaves, 7, 2, 4), [leaves[i]], go)
        assert bits(g, full[1 + i]), i
    assert op(*ins, 7, 2, 0) is ins[1]
    assert bits(cspn_b200.Affinity_PropagateDilated(4, 7, 2)(*ins), full[0])


def launches_of_backward(ins, need):
    """The C backward's launch count with the gradients `need` (kernel, blur, sparse, conf) requested, N = 5."""
    k, b, s, m = ins
    outs = [torch.empty_like(t) if n else None for t, n in zip(ins, need)]
    ws = torch.empty(_lib.lib().cspn2d_dil_bwd_workspace_bytes(1, 1, 16, 16, 3, 1, 5), dtype=torch.uint8, device='cuda')
    rc = _lib.lib().cspn2d_dil_bwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), torch.ones_like(b).data_ptr(),
                                       *[None if o is None else o.data_ptr() for o in outs], 1, 1, 16, 16, 3, 1, 5, ws.data_ptr(),
                                       ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    return _lib.lib().cspn_last_launches()


def test_partial_backward_runs_no_recomputed_steps():
    ins = dr.make_inputs(1, 1, 16, 16, 3, 'soft', seed=1, device='cuda')
    assert launches_of_backward(ins, (True, True, True, True)) == 4 + 5 + 1
    assert launches_of_backward(ins, (False, False, False, True)) == 4 + 4 + 1    # the confidence needs the iterates, not lambda_0
    assert launches_of_backward(ins, (False, True, True, False)) == 5 + 1
    assert launches_of_backward(ins, (False, False, True, False)) == 4 + 1


def c_fwd(k, b, s, m, out, K, dil, N, ws):
    B, C, H, W = b.shape
    rc = _lib.lib().cspn2d_dil_fwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), out.data_ptr(), B, C, H, W, K, dil, N,
                                       ws.t.data_ptr() if ws.nbytes else None, ws.nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


def c_bwd(k, b, s, m, go, outs, K, dil, N, ws):
    B, C, H, W = b.shape
    ptrs = [None if x is None else x.t.data_ptr() for x in outs]
    rc = _lib.lib().cspn2d_dil_bwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), go.data_ptr(), *ptrs, B, C, H, W, K,
                                       dil, N, ws.t.data_ptr() if ws.nbytes else None, ws.nbytes,
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.lib().cspn_last_error()


@pytest.mark.parametrize('K,dil', [(3, 2), (7, 1)])
@pytest.mark.parametrize('offset', [0, 4])
@pytest.mark.parametrize('which', ['all', 'blur_only', 'kernel_conf'])
def test_memory_contract(K, dil, offset, which):
    """Outputs written exactly (guarded, every element), NULL outputs skipped, inputs untouched, and no workspace word
    read before it is written: sentinel- and zero-filled workspaces give the same bits."""
    B, C, H, W, N = 2, 3, 13, 20, 4
    k, b, s, m = dr.make_inputs(B, C, H, W, K, 'soft', seed=K + offset, device='cuda')
    go = torch.randn(B, C, H, W, device='cuda')
    ins = [k, b, s, m, go]
    before = mc.snapshot(ins)
    L = _lib.lib()
    want_out = {'all': (1, 1, 1, 1), 'blur_only': (0, 1, 0, 0), 'kernel_conf': (1, 0, 0, 1)}[which]
    fw, bw = [], []
    for fill in ('sentinel', 'zero'):
        out = mc.guarded(b.shape, offset)
        ws = mc.workspace(L.cspn2d_dil_workspace_bytes(B, C, H, W, K, dil, N), offset, fill)
        c_fwd(k, b, s, m, out.t, K, dil, N, ws)
        torch.cuda.synchronize()
        mc.assert_written(out, 'out')
        assert ws.guards_intact()
        fw.append(out.t.clone())
        outs = [mc.guarded(t.shape, offset) if w else None for t, w in zip((k, b, s, m), want_out)]
        ws = mc.workspace(L.cspn2d_dil_bwd_workspace_bytes(B, C, H, W, K, dil, N), offset, fill)
        c_bwd(k, b, s, m, go, outs, K, dil, N, ws)
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
    want = run((k, b, s, m), K, dil, N, go)
    assert bits(fw[0], want[0])
    assert all(x is None or bits(x, y) for x, y in zip(bw[0], want[1:]))


def test_refuses_overlapping_device_buffers():
    k, b, s, m = dr.make_inputs(1, 1, 8, 8, 3, 'soft', device='cuda')
    rc = _lib.lib().cspn2d_dil_fwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), k.data_ptr(), 1, 1, 8, 8, 3, 1, 1, None,
                                       0, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b'overlaps' in _lib.lib().cspn_last_error()


def penet_inputs(B, H, W, seed, device):
    g = torch.Generator().manual_seed(seed)
    sparse = torch.where(torch.rand(B, 1, H, W, generator=g) < 0.2, torch.rand(B, 1, H, W, generator=g) * 5 + 1, torch.zeros(()))
    coarse = torch.rand(B, 1, H, W, generator=g) * 5 + 1
    half = {K: torch.randn(B, K * K - 1, H // 2, W // 2, generator=g) for K in (3, 5, 7)}
    full = {K: torch.randn(B, K * K - 1, H, W, generator=g) for K in (3, 5, 7)}
    conf = torch.randn(B, 1, H, W, generator=g)
    mh, mf = torch.randn(B, 3, H, W, generator=g), torch.randn(B, 3, H, W, generator=g)
    leaves = [coarse, sparse, half[3], half[5], half[7], full[3], full[5], full[7], conf, mh, mf]
    return [t.to(device) for t in leaves]


def penet_grads(leaves, use_op, dtype, go):
    ls = [t.detach().to(dtype).requires_grad_(True) for t in leaves]
    c, s, h3, h5, h7, f3, f5, f7, cf, mh, mf = ls
    out = dr.penet_refine(c, s, {3: h3, 5: h5, 7: h7}, {3: f3, 5: f5, 7: f7}, cf, mh, mf, N=6, use_op=use_op)
    return [out.detach()] + list(torch.autograd.grad(out, ls, go.to(dtype)))


def test_penet_refinement_end_to_end():
    """Both stages (d = 2 on nearest-upsampled half-resolution guides, then d = 1), K = 3, 5 and 7 with 6 steps each and
    softmax mixing, against an fp64 model built from stock torch ops: forward and the gradient of every input."""
    B, H, W = 2, 24, 36
    leaves = penet_inputs(B, H, W, 0, 'cuda')
    go = torch.randn(B, 1, H, W, device='cuda')
    got = penet_grads(leaves, True, torch.float32, go)
    ref = penet_grads(leaves, False, torch.float64, go)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert dr.normwise(g, r) < (1e-5 if i == 0 else 2e-4), (i, dr.normwise(g, r))


def test_torch_compile_is_one_node():
    ins = dr.make_inputs(2, 1, 16, 24, 5, 'soft', seed=3, device='cuda')
    go = torch.randn(2, 1, 16, 24, device='cuda')

    def f(k, b, s, m):
        return cspn_b200.propagate2d_dilated(k, b, s, m, 5, 2, 4) * 2

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
    k, b, s, m = dr.make_inputs(1, 2, 6, 9, 3, 'soft', seed=2, device='cuda')
    for t in (k, b, s, m):
        t.requires_grad_(True)
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_dilated.default, (k, b, s, m, 3, 2, 2))
    torch.library.opcheck(torch.ops.cspn_b200.propagate2d_dilated.default, (k, b, None, None, 3, 1, 1))
