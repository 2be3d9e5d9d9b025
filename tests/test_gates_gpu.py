"""GPU tests of the propagation with caller-supplied gates (fluid.layers.affinity_propagate: cspn2d_wide.cu, K in {3, 5, 7};
cspn3d_wide.cu, K in {3, 5}), through both the dispatcher op and the ctypes route: bit for bit against the fp64 restatement
on dyadic inputs over a pairwise case matrix and a one-hot-tap sweep, the bits of propagate2d_paddle (and the 3D 'paddle'
operator to tolerance) when the gates are demo.py's, softmax gates at many steps and a training step through a softmax, IEEE
special values, batch and channel independence, partial gradients, launch counts, where the entry points write and what they
read, and opcheck / torch.compile / CUDA-graph capture."""
import contextlib
import os

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op

import backward_exact as be
import gates_reference as gr
import memory_contract as mc

pytestmark = pytest.mark.gpu

ROUTES = ('ctypes', 'op')


@contextlib.contextmanager
def route(name):
    """affinity_propagate through the ctypes autograd.Function or through the dispatcher op."""
    old = os.environ.get('CSPN_B200_NO_TORCH_OP')
    if name == 'ctypes':
        os.environ['CSPN_B200_NO_TORCH_OP'] = '1'
    else:
        os.environ.pop('CSPN_B200_NO_TORCH_OP', None)
        torch_op.load()
    try:
        yield
    finally:
        if old is None:
            os.environ.pop('CSPN_B200_NO_TORCH_OP', None)
        else:
            os.environ['CSPN_B200_NO_TORCH_OP'] = old


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary (a leaf: it can require grad)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def launches():
    torch.cuda.synchronize()
    return _lib.lib().cspn_last_launches()


def ref_fn(K, N):
    return lambda g, x: gr.affinity_propagate_ref(x, g, K, N)


def run(name, K, N, g, x, go, misaligned=False, need=(True, True)):
    """(out, input.grad, gate.grad) of affinity_propagate on the GPU through route `name`."""
    dev = [t.detach().cuda().clone() for t in (g, x, go)]      # fresh leaves, also for CUDA arguments
    if misaligned:
        dev = [misaligned_copy(t) for t in dev]
    gc, xc, goc = dev
    gc.requires_grad_(need[1])
    xc.requires_grad_(need[0])
    with route(name):
        out = cspn_b200.affinity_propagate(xc, gc, K, N)
        out.backward(goc)
    return out.detach(), xc.grad, gc.grad


def assert_bits(ours, ref, case):
    """ours = (out, grad_input, grad_gate); ref = (out, grad_gate, grad_input) of be.autograd."""
    for a, b, name in zip(ours, (ref[0], ref[2], ref[1]), ('out', 'grad_input', 'grad_gate')):
        a = a.double().cpu()
        bad = a != b
        assert not bad.any(), (case, name, f'{int(bad.sum())} of {bad.numel()} differ, first at '
                                            f'{tuple(bad.nonzero()[0].tolist())}', float((a - b).abs().max()))


def dyadic_gates(gen, n, shape, K):
    """At each site m in {1, 2, 4} taps of +-1/m (any tap, also one that reads the padding), the rest 0."""
    g = be.dyadic_guidance(gen, n, shape, K, False)
    return g / g.abs().sum(1, keepdim=True)


def dyadic(seed, B, C, spatial, K, per_channel):
    gen = torch.Generator().manual_seed(seed)
    g = dyadic_gates(gen, B * C if per_channel else B, spatial, K).reshape(B, -1, *spatial)
    return g, be.small_ints(gen, (B, C, *spatial)), be.small_ints(gen, (B, C, *spatial))


# ---- 1. bit for bit on dyadic inputs: pairwise over K, shape, B x C, gate layout, N and memory layout ----------------
AXES = {
    'Ksp': tuple((K, hw) for K in (3, 5, 7) for hw in ((37, 136), (37, 133), (17, 65), (1, 100), (100, 1))) +
           tuple((K, dhw) for K in (3, 5) for dhw in ((7, 19, 72), (7, 19, 70), (3, 1, 100))),
    'bc': ((1, 1), (2, 3), (3, 2)),
    'N': (1, 2, 4),
    'misaligned': (False, True),
    'per_channel': (False, True),
}
EXACT = be.pairwise(AXES, lambda c: not (c['per_channel'] and c['bc'][1] == 1)) + [
    dict(Ksp=(3, (228, 304)), bc=(1, 1), N=4, misaligned=False, per_channel=False),
    dict(Ksp=(5, (228, 304)), bc=(2, 1), N=2, misaligned=False, per_channel=False),
    dict(Ksp=(7, (228, 304)), bc=(1, 2), N=3, misaligned=False, per_channel=True),
]


@pytest.mark.parametrize('i', range(len(EXACT)), ids=[be.case_id(c) for c in EXACT])
def test_exact_on_dyadic_inputs(i):
    c = EXACT[i]
    (K, sp), (B, C), N = c['Ksp'], c['bc'], c['N']
    g, x, go = dyadic(4000 + i, B, C, sp, K, c['per_channel'])
    ref = be.exact_reference(ref_fn(K, N), g, x, go, N)
    for name in ROUTES:
        assert_bits(run(name, K, N, g, x, go, c['misaligned']), ref, (be.case_id(c), name))


@pytest.mark.parametrize('K,sp', [(3, (20, 72)), (5, (20, 70)), (7, (20, 72)), (7, (20, 70)), (3, (3, 19, 72)),
                                  (3, (3, 19, 70)), (5, (3, 19, 72))])
def test_one_hot_tap_sweep_is_exact(K, sp):
    """Item k of the batch has gate k = +-1 at every site, also where the tap reads the padding: the result is shift_k^N,
    forward and gradients.  W = 72 crosses 64 x 16 tiles of the vectorised step, W = 70 32 x 8 tiles of the scalar one."""
    N, C = 2, 2
    g = be.one_tap_guidance(K * sp[-1], sp, K, False)
    gen = torch.Generator().manual_seed(K * sp[-1])
    x, go = be.small_ints(gen, (g.shape[0], C, *sp)), be.small_ints(gen, (g.shape[0], C, *sp))
    ref = be.exact_reference(ref_fn(K, N), g, x, go, N)
    for name in ROUTES:
        assert_bits(run(name, K, N, g, x, go), ref, (K, sp, name))


# ---- 2. anchored to the existing operators ----------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('W', [136, 133])
@pytest.mark.parametrize('per_channel', [False, True])
def test_paddle_gates_give_the_bits_of_propagate2d_paddle(K, W, per_channel):
    B, C, H, N = 2, 3, 37, 12
    nt = K * K - 1
    gen = torch.Generator().manual_seed(K * W)
    g = torch.randn(B, nt * C if per_channel else nt, H, W, generator=gen).cuda()
    x = torch.rand(B, C, H, W, generator=gen).cuda()
    want = cspn_b200.propagate2d_paddle(g, x, K, N)
    for name in ROUTES:
        with route(name):
            got = cspn_b200.affinity_propagate(x, gr.paddle_gates(g, nt), K, N)
        assert torch.equal(got, want), (name, float((got - want).abs().max()))


@pytest.mark.parametrize('K', [3, 5])
@pytest.mark.parametrize('W', [72, 70])
def test_paddle_gates_agree_with_the_3d_paddle_operator(K, W):
    B, C, D, H, N = 2, 2, 5, 19, 6
    nt = K ** 3 - 1
    gen = torch.Generator().manual_seed(K * W)
    g = torch.randn(B, nt, D, H, W, generator=gen).cuda()
    x = torch.rand(B, C, D, H, W, generator=gen).cuda()
    b = cspn_b200.propagate3d_k(g, x, K, N, 'paddle')
    for name in ROUTES:
        with route(name):
            a = cspn_b200.affinity_propagate(x, gr.paddle_gates(g, nt), K, N)
        assert ((a - b).abs() <= 1e-4 * (b.abs() + b.abs().mean())).all(), (name, float((a - b).abs().max()))


# ---- 3. random gates: softmax-normalised at many steps, and a training step through the softmax ------------------------
def softmax_case(seed, B, C, sp, K):
    gen = torch.Generator().manual_seed(seed)
    nt = K ** len(sp) - 1
    logits = 2 * torch.randn(B, nt, *sp, generator=gen)
    return logits, torch.rand(B, C, *sp, generator=gen), torch.randn(B, C, *sp, generator=gen)


def close(a, b, what):
    a = a.double().cpu()
    err = (a - b).abs()
    assert (err <= 2e-3 * (b.abs() + b.abs().mean())).all(), (what, float(err.max()))


@pytest.mark.parametrize('K,sp,N', [(3, (37, 136), 24), (5, (37, 133), 24), (7, (37, 136), 24), (3, (7, 19, 72), 12),
                                    (5, (7, 19, 70), 12)])
def test_softmax_gates_match_fp64_in_both_directions(K, sp, N):
    logits, x, go = softmax_case(K * sp[-1], 1, 2, sp, K)
    g = torch.softmax(logits, 1)
    ref = be.autograd(ref_fn(K, N), g, x, go, torch.float64)
    for name in ROUTES:
        out, gx, gg = run(name, K, N, g, x, go)
        for a, b, what in ((out, ref[0], 'out'), (gx, ref[2], 'grad_input'), (gg, ref[1], 'grad_gate')):
            close(a, b, (K, sp, name, what))


@pytest.mark.parametrize('K,sp', [(3, (24, 40)), (5, (4, 12, 20))])
def test_training_step_through_a_softmax(K, sp):
    """The gates are a softmax of logits in torch: the logits' and the input's gradients match fp64 autograd through the
    same softmax."""
    N = 4
    logits, x, go = softmax_case(7 * K, 2, 1, sp, K)

    def ref(lg, xx):
        return gr.affinity_propagate_ref(xx, torch.softmax(lg, 1), K, N)

    want = be.autograd(ref, logits, x, go, torch.float64)
    for name in ROUTES:
        lg, xc = logits.cuda().requires_grad_(True), x.cuda().requires_grad_(True)
        with route(name):
            out = cspn_b200.affinity_propagate(xc, torch.softmax(lg, 1), K, N)
        out.backward(go.cuda())
        close(out.detach(), want[0], (name, 'out'))
        close(lg.grad, want[1], (name, 'grad_logits'))
        close(xc.grad, want[2], (name, 'grad_input'))


# ---- 4. IEEE special values, N = 0, independence, partial gradients ---------------------------------------------------
@pytest.mark.parametrize('sp', [(14, 24), (14, 23), (3, 10, 24), (3, 10, 23)])
def test_nan_and_inf_gates_match_the_restatement(sp):
    """W = 24 runs the vectorised steps, W = 23 the scalar ones.  An infinite gate on a tap that reads the padding gives NaN
    (inf * 0); elsewhere +-inf spreads; a NaN gate poisons its pixel and then its neighbours."""
    K, N = 3, 2
    nd = len(sp)
    nt = K ** nd - 1
    gen = torch.Generator().manual_seed(sum(sp))
    g = torch.randn(1, nt, *sp, generator=gen) / nt
    x = torch.rand(1, 2, *sp, generator=gen) + 0.5
    lead = (0,) * (nd - 2)
    H, W = sp[-2:]
    g[(0, 0) + lead + (2, 5)] = float('nan')
    g[(0, 1) + lead + (4, 12)] = float('inf')               # reads (+1, 0) / (+1, +1, 0): inside
    g[(0, nt - 1) + lead + (0, 3)] = float('-inf')          # reads (-1, -1) / (-1, -1, -1): the padding
    g[(0, 2) + lead + (H - 1, W - 1)] = float('inf')        # reads (+1, -1) / (+1, +1, -1) from row H - 1: the padding
    with torch.no_grad():
        ref = gr.affinity_propagate_ref(x, g, K, N)
    assert torch.isnan(ref).any() and torch.isinf(ref).any()
    for name in ROUTES:
        with route(name):
            out = cspn_b200.affinity_propagate(x.cuda(), g.cuda(), K, N).cpu()
        assert torch.equal(torch.isnan(out), torch.isnan(ref)), name
        assert torch.equal(torch.isinf(out) & (out > 0), torch.isinf(ref) & (ref > 0)), name
        assert torch.equal(torch.isinf(out) & (out < 0), torch.isinf(ref) & (ref < 0)), name
        fin = torch.isfinite(ref)
        assert torch.allclose(out[fin], ref[fin], rtol=1e-5, atol=1e-6), name


def test_zero_steps_return_the_input_itself():
    for x, g, K in ((torch.rand(1, 2, 8, 8), torch.rand(1, 48, 8, 8), 7), (torch.rand(1, 2, 3, 8, 8), torch.rand(1, 124, 3, 8, 8), 5)):
        xc, gc = x.cuda().requires_grad_(True), g.cuda().requires_grad_(True)
        for name in ROUTES:
            with route(name):
                assert cspn_b200.affinity_propagate(xc, gc, K, 0) is xc


@pytest.mark.parametrize('K,sp', [(3, (20, 72)), (7, (20, 70)), (3, (4, 9, 40)), (5, (4, 9, 39))])
def test_an_image_gives_the_same_bits_alone_and_in_a_batch(K, sp, monkeypatch):
    B, C, N = 4, 2, 3
    gen = torch.Generator().manual_seed(K)
    g = (torch.randn(B, K ** len(sp) - 1, *sp, generator=gen) / 8).cuda()
    x, go = torch.rand(B, C, *sp, generator=gen).cuda(), torch.randn(B, C, *sp, generator=gen).cuda()
    results = []
    for group in (None, '3'):
        if group is None:
            monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
            monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
        else:                                            # launch groups of 3 and 1 images / 1 volume and the rest
            monkeypatch.setenv('CSPN_B200_KXK_GROUP', group)
            monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str(C * x[0, 0].numel() * 4 / 1024))
        results.append(run('ctypes', K, N, g, x, go))
    for b in range(B):
        alone = run('op', K, N, g[b:b + 1], x[b:b + 1], go[b:b + 1])
        for whole in results:
            for a, w in zip(alone, whole):
                assert torch.equal(a, w[b:b + 1]), b
    for c in range(C):                                   # a channel alone with the shared gate
        alone = run('op', K, N, g, x[:, c:c + 1].contiguous(), go[:, c:c + 1].contiguous(), need=(True, False))
        assert torch.equal(alone[0], results[0][0][:, c:c + 1]) and torch.equal(alone[1], results[0][1][:, c:c + 1]), c


@pytest.mark.parametrize('K,sp', [(5, (19, 40)), (3, (3, 9, 40))])
@pytest.mark.parametrize('name', ROUTES)
def test_per_channel_gates_are_a_loop_over_channels(K, sp, name):
    B, C, N = 2, 3, 3
    nt = K ** len(sp) - 1
    gen = torch.Generator().manual_seed(K)
    g = torch.randn(B, nt * C, *sp, generator=gen) / nt
    x, go = torch.rand(B, C, *sp, generator=gen), torch.randn(B, C, *sp, generator=gen)
    whole = run(name, K, N, g, x, go)
    for c in range(C):
        one = run(name, K, N, g[:, nt * c:nt * (c + 1)].contiguous(), x[:, c:c + 1].contiguous(), go[:, c:c + 1].contiguous())
        assert torch.equal(one[0], whole[0][:, c:c + 1]) and torch.equal(one[1], whole[1][:, c:c + 1]), c
        assert torch.equal(one[2], whole[2][:, nt * c:nt * (c + 1)]), c


@pytest.mark.parametrize('K,sp', [(7, (37, 136)), (3, (37, 133)), (5, (5, 19, 72)), (3, (5, 19, 70))])
@pytest.mark.parametrize('name', ROUTES)
def test_one_gradient_alone_gives_the_same_bits(K, sp, name):
    N = 3
    gen = torch.Generator().manual_seed(K)
    g = torch.randn(2, K ** len(sp) - 1, *sp, generator=gen) / 8
    x, go = torch.rand(2, 2, *sp, generator=gen), torch.randn(2, 2, *sp, generator=gen)
    out, gx, gg = run(name, K, N, g, x, go)
    _, only_x, no_g = run(name, K, N, g, x, go, need=(True, False))
    _, no_x, only_g = run(name, K, N, g, x, go, need=(False, True))
    assert no_g is None and no_x is None
    assert torch.equal(only_x, gx) and torch.equal(only_g, gg)


# ---- 5. launch counts: no prep ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
def test_2d_launches(K):
    L = _lib.lib()
    B, C, H, W, N = 2, 2, 20, 40, 5
    g, x, go = [torch.rand(*s).cuda() for s in ((B, K * K - 1, H, W), (B, C, H, W), (B, C, H, W))]
    ptr = lambda t: None if t is None else t.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty_like(x)
    ws = torch.empty(max(1, L.cspn2d_gates_workspace_bytes(B, C, H, W, K, N)), dtype=torch.uint8, device='cuda')
    _lib.check(L.cspn2d_gates_fwd_f32(ptr(g), ptr(x), ptr(out), B, C, H, W, K, N, ptr(ws), ws.numel(), st), 'fwd')
    assert launches() == N                                 # one launch per step
    wsb = torch.empty(L.cspn2d_gates_bwd_workspace_bytes(B, C, H, W, K, N), dtype=torch.uint8, device='cuda')
    gg, gx = torch.empty_like(g), torch.empty_like(x)
    for pg, px, want in ((gg, gx, (N - 1) + N + 1),      # forward steps, adjoint steps, one gather
                         (None, gx, N),                      # the input gradient alone: the adjoint steps
                         (gg, None, (N - 1) + (N - 1) + 1)):  # the gate gradient alone: no lambda_0
        _lib.check(L.cspn2d_gates_bwd_f32(ptr(g), ptr(x), ptr(go), ptr(pg), ptr(px), B, C, H, W, K, N, ptr(wsb), wsb.numel(), st),
                   'bwd')
        assert launches() == want, (pg is None, px is None)


@pytest.mark.parametrize('K', [3, 5])
def test_3d_launches(K):
    L = _lib.lib()
    B, C, D, H, W, N = 2, 2, 3, 9, 40, 4
    g, x, go = [torch.rand(*s).cuda() for s in ((B, K ** 3 - 1, D, H, W), (B, C, D, H, W), (B, C, D, H, W))]
    ptr = lambda t: None if t is None else t.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty_like(x)
    ws = torch.empty(L.cspn3d_gates_workspace_bytes(B, C, D, H, W, K, N), dtype=torch.uint8, device='cuda')
    _lib.check(L.cspn3d_gates_fwd_f32(ptr(g), ptr(x), ptr(out), B, C, D, H, W, K, N, ptr(ws), ws.numel(), st), 'fwd')
    assert launches() == N
    wsb = torch.empty(L.cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, K, N), dtype=torch.uint8, device='cuda')
    gg, gx = torch.empty_like(g), torch.empty_like(x)
    for pg, px, want in ((gg, gx, B * ((N - 1) + N + K)),   # per volume: forward steps, adjoint steps, K gathers
                         (None, gx, B * N),
                         (gg, None, B * ((N - 1) + (N - 1) + K))):
        _lib.check(L.cspn3d_gates_bwd_f32(ptr(g), ptr(x), ptr(go), ptr(pg), ptr(px), B, C, D, H, W, K, N, ptr(wsb), wsb.numel(),
                                          st), 'bwd')
        assert launches() == want, (pg is None, px is None)


# ---- 6. where the entry points write and what they read (tests/memory_contract.py) ------------------------------------
def ptr(t):
    return None if t is None else t.data_ptr()


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


# (K, spatial, B, C, N, per_channel)
CONTRACT = [
    (3, (37, 136), 2, 3, 4, False),
    (3, (37, 133), 1, 2, 2, True),
    (5, (37, 136), 2, 2, 3, True),
    (7, (37, 133), 2, 1, 1, False),
    (7, (17, 65), 1, 1, 0, False),
    (3, (5, 19, 72), 2, 2, 3, False),
    (3, (5, 19, 70), 1, 1, 1, False),
    (5, (3, 19, 72), 1, 2, 2, True),
    (5, (3, 9, 33), 2, 1, 0, False),
]


def abi(nd):
    L = _lib.lib()
    return (getattr(L, f'cspn{nd}d_gates_workspace_bytes'), getattr(L, f'cspn{nd}d_gates_fwd_f32'),
            getattr(L, f'cspn{nd}d_gates_bwd_workspace_bytes'), getattr(L, f'cspn{nd}d_gates_bwd_f32'))


@pytest.mark.parametrize('K,sp,B,C,N,per_channel', CONTRACT)
def test_forward_writes_exactly_out(K, sp, B, C, N, per_channel):
    g, x, _ = dyadic(sum(sp) + N + K, B, C, sp, K, per_channel)
    ref = gr.affinity_propagate_ref(x.double(), g.double(), K, N)
    gc, xc = g.cuda(), x.cuda()
    Bi, Ci = (B * C, 1) if per_channel else (B, C)
    wsq, fwd, _, _ = abi(len(sp))
    ws_bytes = wsq(Bi, Ci, *sp, K, N)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda o, ws: fwd(ptr(gc), ptr(xc), ptr(o[0]), Bi, Ci, *sp, K, N, ws, ws_bytes, st)
    out = run_contract(call, [gc, xc], [(B, C, *sp)], ws_bytes, f'K={K} {len(sp)}D gates forward')
    assert torch.equal(out[0].double(), ref)


@pytest.mark.parametrize('K,sp,B,C,N,per_channel', CONTRACT)
def test_backward_writes_exactly_its_gradients(K, sp, B, C, N, per_channel):
    g, x, go = dyadic(sum(sp) + 7 * N + K, B, C, sp, K, per_channel)
    if N == 0:
        ref_g, ref_x = torch.zeros(g.shape, dtype=torch.float64), go.double()
    else:
        ref_g, ref_x = be.exact_reference(ref_fn(K, N), g, x, go, N)[1:]
    gc, xc, goc = g.cuda(), x.cuda(), go.cuda()
    Bi, Ci = (B * C, 1) if per_channel else (B, C)
    _, _, wsq, bwd = abi(len(sp))
    ws_bytes = wsq(Bi, Ci, *sp, K, N)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda o, ws: bwd(ptr(gc), ptr(xc), ptr(goc), ptr(o[0]), ptr(o[1]), Bi, Ci, *sp, K, N, ws, ws_bytes, st)
    shapes = [tuple(g.shape), (B, C, *sp)]
    inputs = [gc, xc, goc]
    full = run_contract(call, inputs, shapes, ws_bytes, f'K={K} {len(sp)}D gates backward')
    assert torch.equal(full[0].double(), ref_g) and torch.equal(full[1].double(), ref_x)
    for drop in range(2):                                       # either gradient NULL: the other keeps its bits
        outs = [None if j == drop else mc.guarded(s) for j, s in enumerate(shapes)]
        ws = mc.workspace(ws_bytes)
        before = mc.snapshot(inputs)
        _lib.check(call([None if o is None else o.t for o in outs], ws.ptr()), 'gates backward')
        torch.cuda.synchronize()
        keep = outs[1 - drop]
        mc.assert_written(keep, f'gradient {drop} NULL')
        assert mc.same_bits(keep.t.cpu(), full[1 - drop]) and ws.guards_intact() and mc.unchanged(before, inputs), drop


# ---- 7. tracing -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('nd,K', [(2, 3), (2, 5), (3, 3), (3, 5)])
def test_opcheck(nd, K):
    torch_op.load()
    sp = (12, 20) if nd == 2 else (3, 6, 20)
    gen = torch.Generator().manual_seed(K)
    op = getattr(torch.ops.cspn_b200, f'affinity_propagate{nd}d')
    for C, per_channel in ((1, False), (2, False), (2, True)):
        g = (torch.randn(1, (K ** nd - 1) * (C if per_channel else 1), *sp, generator=gen) / 8).cuda().requires_grad_(True)
        x = torch.rand(1, C, *sp, generator=gen).cuda().requires_grad_(True)
        torch.library.opcheck(op, (x, g, K, 3))


@pytest.mark.parametrize('nd,K', [(2, 7), (3, 5)])
def test_torch_compile_fullgraph_is_one_node(nd, K):
    torch_op.load()
    sp = (24, 40) if nd == 2 else (3, 8, 24)
    gen = torch.Generator().manual_seed(K)
    g = (torch.randn(2, K ** nd - 1, *sp, generator=gen) / 8).cuda()
    x = torch.rand(2, 2, *sp, generator=gen).cuda()
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm

    def fn(x, g):
        return cspn_b200.affinity_propagate(x, g, K, 5)

    cf = torch.compile(fn, fullgraph=True, backend=backend)
    outs, grads = [], []
    for call in (fn, cf):
        xc, gc = x.clone().requires_grad_(True), g.clone().requires_grad_(True)
        out = call(xc, gc)
        out.square().sum().backward()
        outs.append(out.detach())
        grads.append((xc.grad, gc.grad))
    name = f'cspn_b200.affinity_propagate{nd}d'
    calls = [n for gm in graphs for n in gm.graph.nodes if n.op == 'call_function']
    assert len(graphs) == 1 and sum(name in str(n.target) for n in calls) == 1, [str(n.target) for n in calls]
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


@pytest.mark.parametrize('nd,K', [(2, 3), (3, 3)])
def test_cuda_graph_capture_and_replay(nd, K):
    sp = (32, 64) if nd == 2 else (3, 16, 64)
    gen = torch.Generator().manual_seed(K)
    g = (torch.randn(2, K ** nd - 1, *sp, generator=gen) / 8).cuda()
    x = torch.rand(2, 1, *sp, generator=gen).cuda()
    for name in ROUTES:
        with route(name):
            f = lambda: cspn_b200.affinity_propagate(x, g, K, 6)
            ref = f()
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                f()                                            # warm-up on the side stream
            torch.cuda.current_stream().wait_stream(st)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = f()
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref), name
            x.mul_(0.5)
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, f()), name
