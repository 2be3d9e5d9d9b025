"""GPU tests of propagate2d_linear (SPN's three-way scans, DESIGN.md section 4.24), forward and backward, on both routes (the
dispatcher op and the ctypes seam): the fp64 composition of tests/linear_reference.py within tolerance and its
kernel-order restatement bit for bit, over every single direction, a two-direction subset and all four, shared and
per-channel gates, C in {1, 3}, H and W in {1, 2, odd}, every plan the shape selector picks, and 8x1x352x1216; the flip
and transpose identities on the kernel; the anchors (zero gates, a broadcast first column, the stability bound); every
requested-gradient subset; the tie rule; determinism; the memory contract of the C entry points; an SPN head end to end
against an fp64 model; torch.compile and opcheck.

Tolerance: normwise error against fp64 below 64 u (u = 2^-24) times sqrt(S / 8) for scans of S steps.  Largest ratios
of error to that bound observed on an H100 over the sweep and 8x1x352x1216: output 0.024, grad_feat 0.024, grad_gate
0.035."""
import math

import pytest
import torch

import linear_reference as R
import memory_contract as mc
from cspn_b200 import _lib
from test_linear_cpu import PLAN_SHAPES

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SUBSETS = [('l2r',), ('r2l',), ('t2b',), ('b2t',), ('l2r', 'b2t'), R.DIRECTIONS]
SHAPES = [(1, 1), (1, 6), (2, 2), (7, 1), (5, 13), (12, 9)]


def op(feat, gate, dirs, route):
    import cspn_b200
    if route == 'ctypes':
        import os
        old = os.environ.get('CSPN_B200_NO_TORCH_OP')
        os.environ['CSPN_B200_NO_TORCH_OP'] = '1'
        try:
            return cspn_b200.propagate2d_linear(feat, gate, dirs)
        finally:
            if old is None:
                del os.environ['CSPN_B200_NO_TORCH_OP']
            else:
                os.environ['CSPN_B200_NO_TORCH_OP'] = old
    return cspn_b200.propagate2d_linear(feat, gate, dirs)


def run(feat, gate, dirs, go, route='op', need=(True, True)):
    """(out, grad_feat, grad_gate) of the library, a gradient not asked for None."""
    f = feat.detach().clone().requires_grad_(need[0])
    g = gate.detach().clone().requires_grad_(need[1])
    out = op(f, g, dirs, route)
    wanted = [t for t, n in zip((f, g), need) if n]
    got = list(torch.autograd.grad(out, wanted, go))
    return out.detach(), (got.pop(0) if need[0] else None), (got.pop(0) if need[1] else None)


def bound(S):
    return 64 * U * math.sqrt(max(S, 8) / 8)


def check(feat, gate, dirs, route='op', seed=0, fp64=True):
    B, C, H, W = feat.shape
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(seed)).cuda()
    out, gf, gg = run(feat, gate, dirs, go, route)
    ko, _, kgf, kgg = R.kernel_order(feat, gate, dirs, go)
    assert mc.same_bits(out, ko), 'forward bits'
    assert mc.same_bits(gf, kgf), 'grad_feat bits'
    assert mc.same_bits(gg, kgg), 'grad_gate bits'
    if fp64:
        ro, rgf, rgg = R.grads(R.composition, feat, gate, dirs, go)
        S = max(H, W)
        for x, ref, what in ((out, ro, 'out'), (gf, rgf, 'grad_feat'), (gg, rgg, 'grad_gate')):
            assert R.normwise(x, ref) < bound(S), (what, R.normwise(x, ref) / bound(S))


@pytest.mark.parametrize('dirs', SUBSETS, ids=lambda d: '+'.join(d))
@pytest.mark.parametrize('C,per_channel', [(1, False), (3, False), (3, True)])
def test_sweep_against_fp64_and_kernel_order(dirs, C, per_channel):
    for i, (H, W) in enumerate(SHAPES):
        f, g = R.random_inputs(2, C, H, W, dirs, per_channel, seed=i, device='cuda')
        check(f, g, dirs, 'op' if i % 2 == 0 else 'ctypes', seed=i)


@pytest.mark.parametrize('dirs', SUBSETS, ids=lambda d: '+'.join(d))
def test_dyadic_inputs_equal_fp64(dirs):
    f, g = R.dyadic_inputs(2, 3, 6, 7, dirs, True, seed=4, device='cuda')
    go = torch.randint(-4, 5, (2, 3, 6, 7), generator=torch.Generator().manual_seed(2)).float().cuda() / 4
    out, gf, gg = run(f, g, dirs, go)
    ro, rgf, rgg = R.grads(R.composition, f, g, dirs, go)
    assert torch.equal(out.double(), ro) and torch.equal(gf.double(), rgf) and torch.equal(gg.double(), rgg)


@pytest.mark.parametrize('B,C,H,W,dirs', PLAN_SHAPES, ids=lambda v: '+'.join(v) if isinstance(v, tuple) else str(v))
def test_every_plan(B, C, H, W, dirs):
    """Every cluster size and segment seam the plan reaches, shared and per-channel gates, on both routes."""
    f, g = R.random_inputs(B, C, H, W, dirs, C > 1, seed=H + W, device='cuda')
    check(f, g, dirs, fp64=max(H, W) < 400 and B * C < 8)
    f, g = R.random_inputs(B, C, H, W, dirs, False, seed=H * W, device='cuda')
    check(f, g, dirs, route='ctypes', fp64=False)


def test_kitti_shape():
    f, g = R.random_inputs(8, 1, 352, 1216, R.DIRECTIONS, False, seed=11, device='cuda')
    check(f, g, R.DIRECTIONS, seed=3)


def test_identities_on_the_kernel():
    import cspn_b200
    f, g4 = R.random_inputs(2, 3, 9, 14, R.DIRECTIONS, True, seed=5, device='cuda')
    blocks = g4.reshape(2, 4, 9, 9, 14)
    g = blocks[:, 0]
    l2r = lambda x, gt: cspn_b200.propagate2d_linear(x.contiguous(), gt.contiguous(), ('l2r',))
    fW, fH, T = (lambda t: t.flip(-1)), (lambda t: t.flip(-2)), (lambda t: t.transpose(-1, -2))
    assert torch.equal(cspn_b200.propagate2d_linear(f, g, ('r2l',)), fW(l2r(fW(f), fW(g))))
    assert torch.equal(cspn_b200.propagate2d_linear(f, g, ('t2b',)), T(l2r(T(f), T(g))))
    assert torch.equal(cspn_b200.propagate2d_linear(f, g, ('b2t',)), fH(T(l2r(T(fH(f)), T(fH(g))))))
    # each block of a four-direction call is the one-direction call
    hs = [cspn_b200.propagate2d_linear(f, blocks[:, k].contiguous(), (d,)) for k, d in enumerate(R.DIRECTIONS)]
    _, planes = torch.ops.cspn_b200.propagate2d_linear(f, g4, 15)
    for k in range(4):
        assert torch.equal(planes[k], hs[k])
    assert torch.equal(cspn_b200.propagate2d_linear(f, g4), torch.stack(hs).max(0).values)


def test_anchors():
    import cspn_b200
    f, _ = R.random_inputs(2, 3, 11, 17, R.DIRECTIONS, seed=8, device='cuda')
    assert torch.equal(cspn_b200.propagate2d_linear(f, torch.zeros(2, 12, 11, 17, device='cuda')), f)     # zero gates give x
    g = torch.zeros(2, 3, 11, 17, device='cuda')
    g[:, 1, :, 1:] = 1                                                  # g1 = 1 after a zero first column
    assert torch.equal(cspn_b200.propagate2d_linear(f, g, ('l2r',)), f[..., :1].expand_as(f))
    gb = torch.zeros(2, 3, 11, 17, device='cuda')
    gb[:, 1, :-1, :] = 1                                                # b2t: the last row broadcast upwards
    assert torch.equal(cspn_b200.propagate2d_linear(f, gb, ('b2t',)), f[..., -1:, :].expand_as(f))
    f, g = R.random_inputs(4, 2, 40, 60, R.DIRECTIONS, True, seed=9, device='cuda')
    out = cspn_b200.propagate2d_linear(f, g.abs())                      # g >= 0, sum g <= 1: each node a convex combination
    assert out.abs().max() <= f.abs().max() * (1 + 1e-5)


def test_every_requested_gradient_subset():
    f, g = R.random_inputs(2, 3, 7, 10, R.DIRECTIONS, False, seed=12, device='cuda')
    go = torch.randn(2, 3, 7, 10, generator=torch.Generator().manual_seed(0)).cuda()
    _, _, kgf, kgg = R.kernel_order(f, g, R.DIRECTIONS, go)
    for route in ('op', 'ctypes'):
        for need in ((True, False), (False, True), (True, True)):
            _, gf, gg = run(f, g, R.DIRECTIONS, go, route, need)
            assert (gf is None) != need[0] and (gg is None) != need[1]
            if need[0]:
                assert mc.same_bits(gf, kgf)
            if need[1]:
                assert mc.same_bits(gg, kgg)


def test_ties_route_the_gradient_to_the_first_direction():
    f = torch.randn(2, 1, 6, 9).cuda()
    g = torch.zeros(2, 6, 6, 9).cuda()                                  # both directions give x: a tie everywhere
    go = torch.randn(2, 1, 6, 9).cuda()
    out, gf, gg = run(f, g, ('t2b', 'b2t'), go)
    assert torch.equal(out, f) and torch.equal(gf, go)
    assert torch.equal(gg[:, 3:], torch.zeros_like(gg[:, 3:]))
    assert torch.equal(gg[:, 1], go[:, 0] * ((torch.cat([torch.zeros_like(f[:, :, :1]), f[:, :, :-1]], 2) - f)[:, 0]))


def test_determinism():
    f, g = R.random_inputs(2, 3, 33, 70, R.DIRECTIONS, False, seed=13, device='cuda')
    go = torch.randn(2, 3, 33, 70, generator=torch.Generator().manual_seed(1)).cuda()
    a = run(f, g, R.DIRECTIONS, go)
    b = run(f, g, R.DIRECTIONS, go)
    assert all(torch.equal(mc.words(x), mc.words(y)) for x, y in zip(a, b))


# ---- the memory contract of the C entry points -----------------------------------------------------------------------------
@pytest.mark.parametrize('offset', [0, 4])
@pytest.mark.parametrize('dirs,mode', [(R.DIRECTIONS, 0), (('r2l',), 1), (('l2r', 't2b'), 1), (R.DIRECTIONS, 1)],
                         ids=['four-shared', 'r2l-per-channel', 'two-per-channel', 'four-per-channel'])
def test_memory_contract(offset, dirs, mode):
    L = _lib.lib()
    B, C, H, W = 2, 3, 13, 21
    mask = sum(1 << R.DIRECTIONS.index(d) for d in dirs)
    nd = len(dirs)
    f, g = R.random_inputs(B, C, H, W, dirs, mode == 1, seed=offset, device='cuda')
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    ko, kplanes, kgf, kgg = R.kernel_order(f, g, dirs, go)
    stream = torch.cuda.current_stream().cuda_stream
    before = mc.snapshot([f, g, go])
    # forward: planes in the workspace, then in a caller buffer
    for caller_planes in ((False, True) if nd > 1 else (False,)):
        out = mc.guarded((B, C, H, W), offset)
        planes = mc.guarded((nd, B, C, H, W), offset) if caller_planes else None
        need = 0 if caller_planes else L.cspn2d_lin_workspace_bytes(B, C, H, W, mask, mode)
        ws = mc.workspace(need, offset) if need else None
        rc = L.cspn2d_lin_fwd_f32(f.data_ptr(), g.data_ptr(), out.ptr(), planes.ptr() if planes else None, B, C, H, W, mask, mode,
                                  ws.ptr() if ws else None, need, stream)
        assert rc == 0, L.cspn_last_error()
        torch.cuda.synchronize()
        mc.assert_written(out, 'out')
        assert mc.same_bits(out.t, ko)
        if planes:
            mc.assert_written(planes, 'planes')
            assert mc.same_bits(planes.t, kplanes)
        if ws:
            assert ws.guards_intact()
    # backward, with a sentinel and then a zero workspace: the same bits
    saved = kplanes.contiguous() if nd > 1 else ko.contiguous()
    need = L.cspn2d_lin_bwd_workspace_bytes(B, C, H, W, mask, mode)
    results = []
    for fill in ('sentinel', 'zero'):
        gx, gg = mc.guarded((B, C, H, W), offset), mc.guarded(tuple(g.shape), offset)
        ws = mc.workspace(need, offset, fill) if need else None
        rc = L.cspn2d_lin_bwd_f32(f.data_ptr(), g.data_ptr(), saved.data_ptr(), go.data_ptr(), gx.ptr(), gg.ptr(), B, C, H, W, mask,
                                  mode, ws.ptr() if ws else None, need, stream)
        assert rc == 0, L.cspn_last_error()
        torch.cuda.synchronize()
        mc.assert_written(gx, 'grad_feat')
        mc.assert_written(gg, 'grad_gate')
        assert mc.same_bits(gx.t, kgf) and mc.same_bits(gg.t, kgg)
        if ws:
            assert ws.guards_intact()
        results.append((gx.t.clone(), gg.t.clone()))
    # one gradient at a time writes only that one
    for which in (0, 1):
        gx = mc.guarded((B, C, H, W), offset)
        gg = mc.guarded(tuple(g.shape), offset)
        ws = mc.workspace(need, offset) if need else None
        rc = L.cspn2d_lin_bwd_f32(f.data_ptr(), g.data_ptr(), saved.data_ptr(), go.data_ptr(), gx.ptr() if which == 0 else None,
                                  gg.ptr() if which == 1 else None, B, C, H, W, mask, mode, ws.ptr() if ws else None, need, stream)
        assert rc == 0, L.cspn_last_error()
        torch.cuda.synchronize()
        if which == 0:
            mc.assert_written(gx, 'grad_feat')
            assert gg.untouched() and mc.same_bits(gx.t, kgf)
        else:
            mc.assert_written(gg, 'grad_gate')
            assert gx.untouched() and mc.same_bits(gg.t, kgg)
    assert all(torch.equal(mc.words(a), mc.words(b)) for a, b in zip(*results))
    assert mc.unchanged(before, [f, g, go])


# ---- integration ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('per_channel', [False, True])
def test_spn_head_end_to_end(per_channel):
    gen = torch.Generator().manual_seed(21)
    B, Cin, C, H, W = 2, 5, 3, 24, 40
    guide = torch.randn(B, Cin, H, W, generator=gen, dtype=torch.float64)
    feat = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64)
    Gc = 12 * (C if per_channel else 1)
    weight = torch.randn(Gc, Cin, 3, 3, generator=gen, dtype=torch.float64) * 0.3
    bias = torch.randn(Gc, generator=gen, dtype=torch.float64) * 0.1
    torch.backends.cudnn.allow_tf32, tf32 = False, torch.backends.cudnn.allow_tf32     # the guidance conv in fp32, not TF32
    ins64 = [t.cuda().requires_grad_(True) for t in (guide, feat, weight, bias)]
    ins32 = [t.cuda().float().requires_grad_(True) for t in (guide, feat, weight, bias)]
    ref = R.spn_head(*ins64)
    out = R.spn_head(*ins32, use_op=True)
    go = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64).cuda()
    g64 = torch.autograd.grad(ref, ins64, go)
    g32 = torch.autograd.grad(out, ins32, go.float())
    torch.backends.cudnn.allow_tf32 = tf32
    assert R.normwise(out, ref) < bound(W)
    for a, b in zip(g32, g64):
        assert R.normwise(a, b) < 4 * bound(W)


def test_torch_compile_and_opcheck():
    import cspn_b200
    from cspn_b200 import torch_op
    if not torch_op.available():
        pytest.skip('the torch op library is not built')
    torch_op.load()
    f, g = R.random_inputs(2, 3, 9, 12, R.DIRECTIONS, True, seed=30, device='cuda')
    mod = cspn_b200.Affinity_PropagateLinear()
    compiled = torch.compile(mod, fullgraph=True)
    fr, gr = f.clone().requires_grad_(True), g.clone().requires_grad_(True)
    out = compiled(fr, gr)
    out.sum().backward()
    ko, _, kgf, kgg = R.kernel_order(f, g, R.DIRECTIONS, torch.ones_like(f))
    assert mc.same_bits(out.detach(), ko) and mc.same_bits(fr.grad, kgf) and mc.same_bits(gr.grad, kgg)
    for mask, gate in ((15, g), (1, g[:, :9].contiguous()), (10, g[:, :18].contiguous())):
        torch.library.opcheck(torch.ops.cspn_b200.propagate2d_linear.default, (f, gate.requires_grad_(True), mask))
