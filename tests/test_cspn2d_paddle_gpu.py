"""GPU tests of the 2D propagation with the Paddle module's own-location gates (cspn2d_wide.cu, K in {3, 5, 7}): forward
against the numpy oracle over a pairwise case matrix, against the 3D 'paddle' operators at D = 1, IEEE special values, batch
and channel independence, the backward bit for bit on dyadic inputs and to a tolerance on random gates, where the entry
points write and what they read, and torch.compile / CUDA-graph capture / a training step through the module."""
import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_3d_k as on3

import backward_exact as be
import memory_contract as mc
import paddle2d_reference as pr

pytestmark = pytest.mark.gpu

ROUTES = (False, True)          # the ctypes autograd.Function, then the dispatcher op


def inputs(seed, B, C, H, W, K, per_channel=False, signed=False):
    gen = torch.Generator().manual_seed(seed)
    nt = K * K - 1
    shape = (B, nt * C if per_channel else nt, H, W)
    g = torch.randn(*shape, generator=gen) if signed else torch.rand(*shape, generator=gen)
    return g, torch.rand(B, C, H, W, generator=gen)


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary (a leaf: it can require grad)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def strided_copy(t):
    """The same values in a non-contiguous view (W and H strides swapped)."""
    v = t.transpose(-1, -2).contiguous().transpose(-1, -2)
    assert not v.is_contiguous() or min(t.shape[-2:]) == 1
    return v


def launches():
    torch.cuda.synchronize()
    return _lib.lib().cspn_last_launches()


def module(N, K, use_op):
    m = cspn_b200.Affinity_Propagate2DPaddle(N, K)
    if use_op:
        torch_op.load()
    m._use_op = use_op
    return m


def check_oracle(out, ref, what):
    out = out.detach().cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref)), what
    assert np.array_equal(np.isinf(out), np.isinf(ref)), what
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (what, ratio, normwise)


# ---- 1. forward against the oracle: pairwise over K, shape, B x C, gate layout, N and memory layout ------------------
BIG = ((228, 304), (352, 1216))
AXES = {
    'K': (3, 5, 7),
    'hw': ((37, 136), (37, 133), (17, 65), (1, 100), (100, 1), (5, 5)) + BIG,
    'bc': ((1, 1), (1, 3), (3, 1), (3, 3)),
    'gates': ('shared', 'per_channel'),
    'N': (1, 2, 24, 48),
    'layout': ('contiguous', 'misaligned', 'strided'),
}


def _allowed(c):
    if c['gates'] == 'per_channel' and c['bc'][1] == 1:
        return False                                   # one channel: per-channel gates are the shared ones
    if c['hw'] in BIG and (c['N'] > 2 or c['bc'] == (3, 3)):
        return False                                   # keeps the numpy oracle's time in bounds
    return True


FWD = be.pairwise(AXES, _allowed)


@pytest.mark.parametrize('i', range(len(FWD)), ids=[be.case_id(c) for c in FWD])
def test_forward_matches_the_oracle(i):
    c = FWD[i]
    K, (H, W), (B, C), N = c['K'], c['hw'], c['bc'], c['N']
    g, f = inputs(100 + i, B, C, H, W, K, c['gates'] == 'per_channel', signed=bool(i % 2))
    ref = pr.cspn2d_paddle(g.numpy(), f.numpy(), N, K)
    gc, fc = g.cuda(), f.cuda()
    if c['layout'] == 'misaligned':
        gc, fc = misaligned_copy(gc), misaligned_copy(fc)
    elif c['layout'] == 'strided':
        gc, fc = strided_copy(gc), strided_copy(fc)
    out = cspn_b200.propagate2d_paddle(gc, fc, K, N)
    assert launches() == 1 + N                          # one prep, then one launch per step
    check_oracle(out, ref, be.case_id(c))
    m = cspn_b200.Affinity_Propagate2DPaddle(N, K)
    assert torch.equal(m(gc, fc), out)                  # the dispatcher op gives the same bits


# ---- 2. against the 3D 'paddle' operators at D = 1 --------------------------------------------------------------------
def in_plane(K):
    return [k for k, (dz, _, _) in enumerate(on3.offsets_3d(K)) if dz == 0]


@pytest.mark.parametrize('K', [3, 5])
@pytest.mark.parametrize('W', [136, 133])
def test_it_is_the_3d_paddle_operator_at_depth_one(K, W):
    """The 2D gates in the in-plane channels of a K x K x K gate, the others zero, D = 1: Affinity_Propagate3D (K = 3) and
    Affinity_Propagate3DK give this operator's result to 1e-5.  Bits: at K = 3 with an odd width (every kernel on its
    one-pixel path) all of them agree, and the test holds that.  Elsewhere about 30-40 % agree: the 3D 'paddle' steps
    that read the raw guidance divide sum_k |g_k| d(p + off_k) by sum |g| once per voxel, where this path multiplies
    by stored quotients."""
    B, C, H, N = 2, 2, 37, 12
    g, f = inputs(K * W, B, C, H, W, K)
    g3 = torch.zeros(B, K ** 3 - 1, 1, H, W)
    g3[:, in_plane(K), 0] = g
    g, f, g3 = g.cuda(), f.cuda(), g3.cuda()
    a = cspn_b200.Affinity_Propagate2DPaddle(N, K)(g, f)
    mods = [cspn_b200.Affinity_Propagate3DK(N, K, 'paddle')] + ([cspn_b200.Affinity_Propagate3D(N, 3, 'paddle')] if K == 3 else [])
    for m in mods:
        b = m(g3, f[:, :, None])[:, :, 0]
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), (type(m).__name__, float((a - b).abs().max()))
        if K == 3 and W % 2:
            assert torch.equal(a, b), type(m).__name__


# ---- 3. IEEE special values -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('where', ['interior', 'tile_edge', 'corner'])
@pytest.mark.parametrize('W', [136, 133])
def test_zero_gates_nan_front_moves_r_per_step(K, where, W):
    """0 / 0 = NaN where every gate of a pixel is zero, then the NaN front moves r pixels per step on every side.  The
    tile-edge block straddles a 64 x 16 tile corner of the vectorised step (W = 136) and a 32 x 8 one of the scalar step."""
    r, H = (K - 1) // 2, 40
    g, f = inputs(K + W, 1, 2, H, W, K, signed=True)
    y, x = {'interior': (20, 70), 'tile_edge': (14, 62) if W == 136 else (6, 30), 'corner': (0, 0)}[where]
    g[:, :, y:y + 4, x:x + 4] = 0.0
    extents = []
    for N in (1, 2, 3):
        ref = pr.cspn2d_paddle(g.numpy(), f.numpy(), N, K)
        check_oracle(cspn_b200.propagate2d_paddle(g.cuda(), f.cuda(), K, N), ref, (K, where, W, N))
        idx = np.nonzero(np.isnan(ref[0, 0]))
        extents.append(tuple(int(i.max() - i.min()) for i in idx))
    if where != 'corner':
        assert extents == [(3, 3), (3 + 2 * r, 3 + 2 * r), (3 + 4 * r, 3 + 4 * r)], extents


@pytest.mark.parametrize('case', ['subnormal', 'overflow', 'inf'])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [24, 23])
def test_special_gate_sums_follow_ieee_division(case, K, W):
    """A subnormal sum of |gates| divides exactly, an overflowing one gives weights of 0, +-inf guidance gives NaN."""
    g, f = inputs(60 + K + W, 1, 2, 14, W, K, signed=True)
    g = g.numpy()
    if case == 'subnormal':
        g[:, :, 3:11, 5:17] *= np.float32(1e-42)
    elif case == 'overflow':
        g[:, :, 3:11, 5:17] = np.sign(g[:, :, 3:11, 5:17]) * np.float32(2e38)
    else:
        g[0, 1, 6, 7] = np.inf
        g[0, K * K - 2, 9, 12] = -np.inf
    for N in (1, 3):
        ref = pr.cspn2d_paddle(g, f.numpy(), N, K)
        check_oracle(cspn_b200.propagate2d_paddle(torch.from_numpy(g).cuda(), f.cuda(), K, N), ref, (case, K, W, N))


# ---- 4. batch and channel independence --------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
def test_an_image_gives_the_same_bits_alone_and_in_a_batch(K, monkeypatch):
    B, C, H, W, N = 5, 2, 20, 72, 4
    monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
    g, f = [t.cuda() for t in inputs(K, B, C, H, W, K)]
    alone = [cspn_b200.propagate2d_paddle(g[i:i + 1], f[i:i + 1], K, N) for i in range(B)]
    whole = cspn_b200.propagate2d_paddle(g, f, K, N)
    assert launches() == 1 + N
    monkeypatch.setenv('CSPN_B200_KXK_GROUP', '2')                 # groups 2, 2, 1
    grouped = cspn_b200.propagate2d_paddle(g, f, K, N)
    assert launches() == 3 * (1 + N)
    for i in range(B):
        assert torch.equal(alone[i], whole[i:i + 1]) and torch.equal(alone[i], grouped[i:i + 1]), i
    grads = []
    for group in (None, '2'):
        if group is None:
            monkeypatch.delenv('CSPN_B200_KXK_GROUP')
        else:
            monkeypatch.setenv('CSPN_B200_KXK_GROUP', group)
        gc, fc = g.clone().requires_grad_(True), f.clone().requires_grad_(True)
        cspn_b200.Affinity_Propagate2DPaddle(N, K)(gc, fc).square().sum().backward()
        grads.append((gc.grad, fc.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    gc, fc = g[2:3].clone().requires_grad_(True), f[2:3].clone().requires_grad_(True)
    cspn_b200.Affinity_Propagate2DPaddle(N, K)(gc, fc).square().sum().backward()
    assert torch.equal(gc.grad, grads[0][0][2:3]) and torch.equal(fc.grad, grads[0][1][2:3])


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('use_op', ROUTES)
def test_per_channel_gates_are_a_loop_over_channels(K, use_op):
    """guidance (B, nt*C, H, W): channel c with guide channels [nt*c, nt*c+nt), forward and both gradients, bit for bit
    against shared-gate calls channel by channel (demo.py:28-45)."""
    B, C, H, W, N = 2, 3, 19, 40, 5
    nt = K * K - 1
    g, f = inputs(K + 7, B, C, H, W, K, per_channel=True)
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(K)).cuda()
    m = module(N, K, use_op)
    gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
    out = m(gc, fc)
    out.backward(go)
    for c in range(C):
        g1 = g[:, nt * c:nt * (c + 1)].contiguous().cuda().requires_grad_(True)
        f1 = f[:, c:c + 1].contiguous().cuda().requires_grad_(True)
        o1 = m(g1, f1)
        o1.backward(go[:, c:c + 1].contiguous())
        assert torch.equal(o1.detach(), out.detach()[:, c:c + 1]), c
        assert torch.equal(g1.grad, gc.grad[:, nt * c:nt * (c + 1)]) and torch.equal(f1.grad, fc.grad[:, c:c + 1]), c


# ---- 5. backward, exact on dyadic inputs ------------------------------------------------------------------------------
def paddle_ref(N, K):
    return lambda g, x: pr.cspn2d_torch_paddle(g, x, N, K)


def dyadic(seed, B, C, H, W, K, per_channel):
    """Own-location dyadic gates (tests/backward_exact.py): m in {1, 2, 4} hot taps of +-1 per pixel, any tap, also one
    that reads the padding; feat and grad_out small integers."""
    gen = torch.Generator().manual_seed(seed)
    g = be.dyadic_guidance(gen, B * C if per_channel else B, (H, W), K, False).reshape(B, -1, H, W)
    return g, be.small_ints(gen, (B, C, H, W)), be.small_ints(gen, (B, C, H, W))


def run(m, g, x, go, layout='contiguous', need=(True, True)):
    """(out, guidance.grad, x.grad) of module m on the GPU, grad_out = go."""
    dev = [t.cuda() for t in (g, x, go)]
    if layout == 'misaligned':
        dev = [misaligned_copy(t) for t in dev]
    gc, xc, goc = dev
    gc.requires_grad_(need[0])
    xc.requires_grad_(need[1])
    out = m(gc, xc)
    out.backward(goc)
    return out.detach(), gc.grad, xc.grad


def assert_bits(ours, ref, case):
    for a, b, name in zip(ours, ref, ('out', 'grad_guidance', 'grad_feat')):
        a = a.double().cpu()
        bad = a != b
        assert not bad.any(), (case, name, f'{int(bad.sum())} of {bad.numel()} differ, first at '
                                            f'{tuple(bad.nonzero()[0].tolist())}', float((a - b).abs().max()))


BWD_AXES = {
    'K': (3, 5, 7),
    'hw': ((37, 136), (37, 133), (17, 65), (1, 100), (100, 1), (5, 5)),
    'bc': ((1, 1), (2, 3), (3, 2)),
    'N': (1, 2, 4),
    'misaligned': (False, True),
    'per_channel': (False, True),
}
EXACT = be.pairwise(BWD_AXES, lambda c: not (c['per_channel'] and c['bc'][1] == 1)) + [
    dict(K=5, hw=(228, 304), bc=(1, 1), N=4, misaligned=False, per_channel=False),
    dict(K=7, hw=(228, 304), bc=(1, 2), N=3, misaligned=False, per_channel=True),
]


@pytest.mark.parametrize('i', range(len(EXACT)), ids=[be.case_id(c) for c in EXACT])
def test_backward_is_exact_on_dyadic_inputs(i):
    c = EXACT[i]
    K, (H, W), (B, C), N = c['K'], c['hw'], c['bc'], c['N']
    g, f, go = dyadic(3000 + i, B, C, H, W, K, c['per_channel'])
    ref = be.exact_reference(paddle_ref(N, K), g, f, go, N)
    for use_op in ROUTES:
        ours = run(module(N, K, use_op), g, f, go, 'misaligned' if c['misaligned'] else 'contiguous')
        assert_bits(ours, ref, (be.case_id(c), use_op))


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [72, 70])
def test_one_hot_tap_sweep_is_exact(K, W):
    """Item k of the batch has tap k hot at every pixel, also where it reads the padding (own-location gates may).  2 x 2
    tiles of 64 x 16 (W = 72, vectorised recompute) or 3 x 3 of 32 x 8 (W = 70, scalar)."""
    H, N, C = 20, 2, 2
    g = be.one_tap_guidance(K + W, (H, W), K, False)
    gen = torch.Generator().manual_seed(K * W)
    f, go = be.small_ints(gen, (g.shape[0], C, H, W)), be.small_ints(gen, (g.shape[0], C, H, W))
    ref = be.exact_reference(paddle_ref(N, K), g, f, go, N)
    for use_op in ROUTES:
        assert_bits(run(module(N, K, use_op), g, f, go), ref, (K, W, use_op))


# ---- 6. backward, random gates, partial gradients ---------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [136, 133])
def test_gradients_match_fp64_autograd_at_24_steps(K, W):
    H, N = 37, 24
    g, f = inputs(K * 7 + W, 1, 2, H, W, K, signed=bool(W % 2))
    g = g + 0.05 * torch.sign(g) if W % 2 else g + 0.05             # keep |g| away from the kink of abs
    go = torch.randn(1, 2, H, W, generator=torch.Generator().manual_seed(W))
    ref = be.autograd(paddle_ref(N, K), g, f, go, torch.float64)
    for use_op in ROUTES:
        ours = run(module(N, K, use_op), g, f, go)
        for a, b, name in zip(ours[1:], ref[1:], ('grad_guidance', 'grad_feat')):
            err = (a.double().cpu() - b).abs()
            assert (err <= 2e-3 * (b.abs() + b.abs().mean())).all(), (K, W, use_op, name, float(err.max()))


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('use_op', ROUTES)
def test_one_gradient_alone_and_a_strided_grad_out_give_the_same_bits(K, use_op):
    N = 3
    g, f = inputs(K, 2, 2, 37, 136, K, signed=True)
    go = torch.randn(2, 2, 37, 136, generator=torch.Generator().manual_seed(K))
    m = module(N, K, use_op)
    out, gg, gf = run(m, g, f, go)
    _, only_g, none_f = run(m, g, f, go, need=(True, False))
    _, none_g, only_f = run(m, g, f, go, need=(False, True))
    assert none_f is None and none_g is None
    assert torch.equal(only_g, gg) and torch.equal(only_f, gf)
    strided = go.cuda().transpose(-1, -2).contiguous().transpose(-1, -2)
    gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
    o = m(gc, fc)
    seen = []
    o.register_hook(lambda grad: seen.append(grad.is_contiguous()))
    o.backward(strided)
    assert seen == [False]                                      # it reached the operator's backward as it was
    assert torch.equal(o.detach(), out) and torch.equal(gc.grad, gg) and torch.equal(fc.grad, gf)


# ---- 7. where the entry points write and what they read (tests/memory_contract.py) ------------------------------------
def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def run_contract(call, inputs, out_shapes, ws_bytes, what):
    """call(outs, ws_ptr) on a workspace of exactly ws_bytes at offsets 0 and 4 bytes, filled with the sentinel and with
    zeros: every output fully written inside its guards, nothing stored past the workspace, inputs unchanged, and all four
    runs give the same bits.  Returns the outputs of the first run (CPU)."""
    first = None
    for off in (0, 4):
        for fill in ('sentinel', 'zero'):
            tag = f'{what}, workspace +{off} B filled with {fill}'
            outs = [mc.guarded(s) for s in out_shapes]
            ws = mc.workspace(ws_bytes, off, fill)
            before = mc.snapshot(inputs)
            _lib.check(call([o.t for o in outs], ws.ptr()), what)
            torch.cuda.synchronize()
            for j, o in enumerate(outs):
                mc.assert_written(o, f'{tag}: output {j}')
            assert ws.guards_intact(), f'{tag}: a store landed outside the workspace'
            assert mc.unchanged(before, inputs), f'{tag}: an input changed'
            res = [o.t.cpu() for o in outs]
            first = first or res
            for j, (a, b) in enumerate(zip(res, first)):
                assert mc.same_bits(a, b), f'{tag}: output {j} differs from the first run'
    return first


def assert_values(ours, refs, what):
    for j, (a, b) in enumerate(zip(ours, refs)):
        bad = a.double() != b
        assert not bad.any(), (what, j, f'{int(bad.sum())} of {bad.numel()} differ')


# (K, H, W, B, C, N, per_channel)
CONTRACT = [
    (3, 37, 136, 2, 3, 4, False),
    (3, 37, 133, 1, 2, 2, True),
    (5, 37, 136, 2, 2, 3, True),
    (5, 37, 133, 3, 1, 2, False),
    (7, 37, 136, 1, 1, 2, False),
    (7, 37, 133, 2, 3, 3, False),
    (5, 37, 136, 1, 2, 0, False),
    (7, 17, 65, 1, 1, 1, False),
]


@pytest.mark.parametrize('K,H,W,B,C,N,per_channel', CONTRACT)
def test_forward_writes_exactly_out(K, H, W, B, C, N, per_channel):
    g, f, _ = dyadic(H * W + N + K, B, C, H, W, K, per_channel)
    ref = pr.cspn2d_torch_paddle(g.double(), f.double(), N, K)
    be.check_exact(ref, N, 'out')
    gc, fc = g.cuda(), f.cuda()
    Bi, Ci = (B * C, 1) if per_channel else (B, C)
    L = _lib.lib()
    ws_bytes = L.cspn2d_paddle_workspace_bytes(Bi, Ci, H, W, K, N)
    call = lambda o, ws: L.cspn2d_paddle_fwd_f32(ptr(gc), ptr(fc), ptr(o[0]), Bi, Ci, H, W, K, N, ws, ws_bytes, stream())
    out = run_contract(call, [gc, fc], [(B, C, H, W)], ws_bytes, f'K={K} paddle forward')
    assert_values(out, [ref], (K, H, W, N))


@pytest.mark.parametrize('K,H,W,B,C,N,per_channel', CONTRACT)
def test_backward_writes_exactly_its_gradients(K, H, W, B, C, N, per_channel):
    g, f, go = dyadic(H * W + 7 * N + K, B, C, H, W, K, per_channel)
    if N == 0:
        ref_g, ref_f = torch.zeros(g.shape, dtype=torch.float64), go.double()
    else:
        ref_g, ref_f = be.exact_reference(paddle_ref(N, K), g, f, go, N)[1:]
    gc, fc, goc = g.cuda(), f.cuda(), go.cuda()
    Bi, Ci = (B * C, 1) if per_channel else (B, C)
    L = _lib.lib()
    ws_bytes = L.cspn2d_paddle_bwd_workspace_bytes(Bi, Ci, H, W, K, N)
    call = lambda o, ws: L.cspn2d_paddle_bwd_f32(ptr(gc), ptr(fc), ptr(goc), ptr(o[0]), ptr(o[1]), Bi, Ci, H, W, K, N, ws,
                                                 ws_bytes, stream())
    shapes = [tuple(g.shape), (B, C, H, W)]
    inputs = [gc, fc, goc]
    full = run_contract(call, inputs, shapes, ws_bytes, f'K={K} paddle backward')
    assert_values(full, [ref_g, ref_f], (K, H, W, N))
    for drop in range(2):                                       # either gradient NULL: the other keeps its bits
        outs = [None if j == drop else mc.guarded(s) for j, s in enumerate(shapes)]
        ws = mc.workspace(ws_bytes)
        before = mc.snapshot(inputs)
        _lib.check(call([None if o is None else o.t for o in outs], ws.ptr()), 'paddle backward')
        torch.cuda.synchronize()
        keep = outs[1 - drop]
        mc.assert_written(keep, f'gradient {drop} NULL')
        assert mc.same_bits(keep.t.cpu(), full[1 - drop]) and ws.guards_intact() and mc.unchanged(before, inputs), drop


# ---- 8. integration ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 7])
def test_torch_compile_fullgraph_forward_and_backward(K):
    m = cspn_b200.Affinity_Propagate2DPaddle(5, K)
    g, f = [t.cuda() for t in inputs(5, 2, 2, 24, 40, K)]

    def fn(g, f):
        return m(g, f)

    cf = torch.compile(fn, fullgraph=True)
    outs, grads = [], []
    for call in (fn, cf):
        gc, fc = g.clone().requires_grad_(True), f.clone().requires_grad_(True)
        out = call(gc, fc)
        out.square().sum().backward()
        outs.append(out.detach())
        grads.append((gc.grad, fc.grad))
    assert torch.equal(outs[0], outs[1])
    assert torch.allclose(grads[0][0], grads[1][0], rtol=1e-5, atol=1e-6)
    assert torch.allclose(grads[0][1], grads[1][1], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('K', [3, 5])
def test_cuda_graph_capture_and_replay(K):
    m = cspn_b200.Affinity_Propagate2DPaddle(6, K)
    g, f = [t.cuda() for t in inputs(55, 2, 1, 32, 64, K)]
    ref = m(g, f)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(g, f)                                                    # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(g, f)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    f.mul_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, m(g, f))


@pytest.mark.parametrize('K', [3, 5])
def test_training_step_through_the_module(K):
    """Conv2d -> 2D 'paddle' CSPN -> L1 -> SGD changes the producer's weights (demo.py:60-75 with dimNum = 2)."""
    torch.manual_seed(0)
    nt = K * K - 1
    net = torch.nn.Conv2d(3, nt + 1, 3, padding=1).cuda()
    post = cspn_b200.Affinity_Propagate2DPaddle(4, K)
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    x = torch.rand(2, 3, 24, 32, device='cuda')
    target = torch.rand(2, 1, 24, 32, device='cuda')
    w0 = net.weight.detach().clone()
    losses = []
    for _ in range(3):
        y = net(x)
        out = post(y[:, :nt], y[:, nt:])
        loss = (out - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert not torch.equal(net.weight, w0) and all(l == l for l in losses)
