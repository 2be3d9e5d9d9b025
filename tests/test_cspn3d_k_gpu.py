"""GPU tests of the K x K x K 3D propagation (K = 5 in cspn3d_wide.cu; K = 3 delegated to the 3x3x3 kernels): forward against
the numpy oracle, an embedding cross-check against the 3x3x3 operator, IEEE special values, per-channel gates, batch
independence across volume groups, backward against fp64 autograd through the torch port, properties at demo.py's volume,
and torch.compile / CUDA-graph capture / a training step through the module."""
import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_3d_k as onk
from oracle import cspn_torch_port_3d_k as tpk

pytestmark = pytest.mark.gpu

NT = 124


def inputs_3d(seed, B, C, D, H, W, K=5, signed=True, gch=None):
    gen = torch.Generator().manual_seed(seed)
    gch = gch or K ** 3 - 1
    g = torch.randn(B, gch, D, H, W, generator=gen) if signed else torch.rand(B, gch, D, H, W, generator=gen)
    return g, torch.rand(B, C, D, H, W, generator=gen)


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def launches():
    torch.cuda.synchronize()
    return _lib.lib().cspn_last_launches()


# pairwise over norm x C x shape x N x alignment (every pair of values of two axes appears in some case)
FWD = [
    # norm, C, (B, D, H, W), N, misaligned
    ('paddle', 1, (1, 1, 1, 1), 1, False),
    ('124sum', 3, (1, 1, 1, 1), 2, False),
    ('124sum_abs', 1, (2, 1, 7, 9), 12, False),
    ('paddle', 3, (2, 1, 7, 9), 24, True),
    ('124sum', 1, (1, 4, 1, 13), 24, False),
    ('124sum_abs', 3, (1, 4, 1, 13), 1, True),
    ('paddle', 1, (1, 3, 3, 3), 2, False),
    ('124sum', 3, (1, 3, 3, 3), 12, True),
    ('124sum_abs', 1, (1, 6, 5, 3), 2, True),
    ('paddle', 3, (1, 6, 5, 3), 12, False),
    ('124sum', 1, (2, 7, 9, 17), 1, True),
    ('124sum_abs', 3, (1, 7, 9, 17), 24, False),
    ('paddle', 1, (2, 8, 12, 64), 24, False),
    ('124sum', 1, (1, 8, 12, 64), 2, True),
    ('124sum_abs', 1, (2, 5, 16, 36), 12, False),
    ('paddle', 3, (1, 5, 16, 36), 1, False),
    ('124sum', 3, (1, 9, 20, 40), 24, False),
    ('124sum_abs', 1, (1, 9, 20, 40), 12, True),
    ('paddle', 1, (1, 12, 18, 4), 12, True),
    ('paddle', 1, (1, 12, 18, 4), 2, False),
]


@pytest.mark.parametrize('norm,C,bdhw,N,misaligned', FWD,
                         ids=[f'{c[0]}-C{c[1]}-{"x".join(map(str, c[2]))}-N{c[3]}{"-misaligned" if c[4] else ""}' for c in FWD])
def test_forward_matches_the_oracle(norm, C, bdhw, N, misaligned):
    B, D, H, W = bdhw
    g, f = inputs_3d(1000 + D * 31 + H * 7 + W + N, B, C, D, H, W, signed=(norm == '124sum'))
    ref = onk.cspn3d_k(g.numpy(), f.numpy(), N, 5, norm)
    gc, fc = g.cuda(), f.cuda()
    if misaligned:
        gc, fc = misaligned_copy(gc), misaligned_copy(fc)
    out = cspn_b200.propagate3d_k(gc, fc, 5, N, norm)
    # one volume group: N step launches for 'paddle' (no prep), 1 + N for the gathered norms
    assert launches() == (N if norm == 'paddle' else 1 + N)
    out = out.cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (ratio, normwise)


CENTRE = [k for k, (dz, dy, dx) in enumerate(onk.offsets_3d(5)) if max(abs(dz), abs(dy), abs(dx)) <= 1]


@pytest.mark.parametrize('norm3,norm5', [('26sum', '124sum'), ('26sum_abs', '124sum_abs'), ('paddle', 'paddle')])
@pytest.mark.parametrize('W', [24, 13])
def test_a_5x5x5_kernel_zero_outside_the_central_3x3x3_is_the_3x3x3_operator(norm3, norm5, W):
    """Checks the tap mapping without the oracle: the central 26 taps of the 5x5x5 window, in order, are the 26 of 3x3x3."""
    assert len(CENTRE) == 26 and [onk.offsets_3d(5)[k] for k in CENTRE] == list(onp.OFFSETS_3D)
    g3, f = inputs_3d(77 + W, 2, 2, 7, 11, W, K=3, signed=(norm3 == '26sum'))
    g5 = torch.zeros(2, NT, 7, 11, W)
    g5[:, CENTRE] = g3
    for N in (1, 6):
        a = cspn_b200.propagate3d(g3.cuda(), f.cuda(), N, norm3)
        b = cspn_b200.propagate3d_k(g5.cuda(), f.cuda(), 5, N, norm5)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-5), (N, float((a - b).abs().max()))


@pytest.mark.parametrize('norm', ['26sum', '26sum_abs', 'paddle'])
def test_k3_is_the_3x3x3_operator_bit_for_bit(norm):
    g, f = [t.cuda() for t in inputs_3d(3, 2, 2, 6, 10, 16, K=3, signed=(norm == '26sum'))]
    ref = cspn_b200.Affinity_Propagate3D(7, 3, norm)(g, f)
    assert torch.equal(cspn_b200.Affinity_Propagate3DK(7, 3, norm)(g, f), ref)
    assert torch.equal(cspn_b200.propagate3d_k(g, f, 3, 7, norm), ref)
    L = _lib.lib()
    out = torch.empty_like(f)
    ws_bytes = L.cspn3d_k_workspace_bytes(2, 2, 6, 10, 16, 3, 7)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    rc = L.cspn3d_k_fwd_f32(g.data_ptr(), f.data_ptr(), out.data_ptr(), 2, 2, 6, 10, 16, 3, 7, _lib.NORM3D[norm], ws.data_ptr(),
                            ws_bytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    go = torch.randn_like(f)
    for use_op in (True, False):          # the backward through both modules, dispatcher op and ctypes autograd.Function
        gs = [g.clone().requires_grad_(True) for _ in range(2)]
        fs = [f.clone().requires_grad_(True) for _ in range(2)]
        m3, mk = cspn_b200.Affinity_Propagate3D(5, 3, norm), cspn_b200.Affinity_Propagate3DK(5, 3, norm)
        m3._use_op = mk._use_op = use_op
        m3(gs[0], fs[0]).backward(go)
        mk(gs[1], fs[1]).backward(go)
        assert torch.equal(gs[0].grad, gs[1].grad) and torch.equal(fs[0].grad, fs[1].grad), use_op


def _check_special(g, f, N, norm):
    ref = onk.cspn3d_k(g, f, N, 5, norm)
    out = cspn_b200.propagate3d_k(torch.from_numpy(g).cuda(), torch.from_numpy(f).cuda(), 5, N, norm).cpu().numpy()
    assert np.array_equal(np.isnan(out), np.isnan(ref)), (norm, N)
    assert np.array_equal(np.isinf(out), np.isinf(ref)), (norm, N)
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (norm, N, ratio, normwise)
    return ref


@pytest.mark.parametrize('corner', [False, True])
@pytest.mark.parametrize('W', [32, 31])
def test_zero_guidance_block_nan_front_grows_2r_per_step(corner, W):
    """0 / 0 = NaN where every gate of a voxel is zero; the NaN front then moves r = 2 voxels per step on every side."""
    g, f = [t.numpy() for t in inputs_3d(40 + W, 1, 1, 24, 24, W, signed=True)]
    o = (0, 0, 0) if corner else (7, 7, 11)
    g[:, :, o[0]:o[0] + 10, o[1]:o[1] + 10, o[2]:o[2] + 10] = 0.0
    for norm in ('124sum', '124sum_abs', 'paddle'):
        extents = []
        for N in (1, 2, 3):
            ref = _check_special(g, f, N, norm)
            idx = np.nonzero(np.isnan(ref[0, 0]))
            assert idx[0].size, (norm, N)
            extents.append(tuple(int(i.max() - i.min()) for i in idx))
        if not corner:
            for a, b in zip(extents, extents[1:]):
                assert all(y - x == 4 for x, y in zip(a, b)), (norm, extents)


@pytest.mark.parametrize('case', ['subnormal', 'overflow', 'inf'])
@pytest.mark.parametrize('W', [24, 23])
def test_special_gate_sums_follow_ieee_division(case, W):
    """A subnormal sum of |gates| divides exactly, an overflowing sum gives weights of 0, +-inf guidance gives NaN."""
    g, f = [t.numpy() for t in inputs_3d(60 + W, 1, 2, 12, 14, W, signed=True)]
    if case == 'subnormal':
        g[:, :, 2:9, 3:11, 5:17] *= np.float32(1e-42)
    elif case == 'overflow':
        g[:, :, 2:9, 3:11, 5:17] = np.sign(g[:, :, 2:9, 3:11, 5:17]) * np.float32(3e37)
    else:
        g[0, 3, 5, 6, 7] = np.inf
        g[0, 70, 8, 9, 12] = -np.inf
    for norm in ('124sum', '124sum_abs', 'paddle'):
        for N in (1, 3):
            _check_special(g, f, N, norm)


@pytest.mark.parametrize('norm', ['124sum', '124sum_abs', 'paddle'])
def test_per_channel_gates_forward_and_backward(norm):
    """guidance (B, 124*C, ...): channel c of feat is propagated with guide channels [124c, 124c+124), forward and backward
    checked against the same work done channel by channel with shared-gate calls."""
    B, C, D, H, W, n = 2, 3, 5, 8, 12, 4
    gen = torch.Generator().manual_seed(11)
    guide = torch.randn(B, NT * C, D, H, W, generator=gen) if norm == '124sum' else torch.rand(B, NT * C, D, H, W, generator=gen)
    feat = torch.rand(B, C, D, H, W, generator=gen)
    layer = cspn_b200.Affinity_Propagate3DK(n, 5, norm)
    gc, fc = guide.cuda().requires_grad_(True), feat.cuda().requires_grad_(True)
    out = layer(gc, fc)
    assert out.shape == feat.shape
    ref = np.stack([onk.cspn3d_k(guide[:, NT * c:NT * (c + 1)].numpy(), feat[:, c:c + 1].numpy(), n, 5, norm)[:, 0]
                    for c in range(C)], 1)
    ok, ratio, normwise = onp.parity_ok(out.detach().cpu().numpy(), ref, 1e-4)
    assert ok, (ratio, normwise)
    out.sum().backward()
    gg, gf = torch.zeros_like(guide), torch.zeros_like(feat)
    for c in range(C):
        g1 = guide[:, NT * c:NT * (c + 1)].contiguous().cuda().requires_grad_(True)
        f1 = feat[:, c:c + 1].contiguous().cuda().requires_grad_(True)
        o1 = layer(g1, f1)
        assert torch.equal(o1.detach().cpu()[:, 0], out.detach().cpu()[:, c])
        o1.sum().backward()
        gg[:, NT * c:NT * (c + 1)] = g1.grad.cpu()
        gf[:, c:c + 1] = f1.grad.cpu()
    assert torch.allclose(gc.grad.cpu(), gg, rtol=1e-5, atol=1e-7) and torch.allclose(fc.grad.cpu(), gf, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize('norm', ['124sum_abs', 'paddle'])
def test_a_volume_gives_the_same_bits_alone_and_in_ragged_volume_groups(norm, monkeypatch):
    B, C, D, H, W, N = 5, 1, 6, 10, 16, 4
    g, f = [t.cuda() for t in inputs_3d(8, B, C, D, H, W, signed=False)]
    per_launch = N if norm == 'paddle' else 1 + N
    alone = [cspn_b200.propagate3d_k(g[i:i + 1], f[i:i + 1], 5, N, norm) for i in range(B)]
    whole = cspn_b200.propagate3d_k(g, f, 5, N, norm)
    assert launches() == per_launch
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', '1000')          # one volume needs 126 * 960 * 4 B = 473 KB: groups 2, 2, 1
    grouped = cspn_b200.propagate3d_k(g, f, 5, N, norm)
    assert launches() == 3 * per_launch
    for i in range(B):
        assert torch.equal(alone[i], whole[i:i + 1]) and torch.equal(alone[i], grouped[i:i + 1]), i
    grads = []
    for cap in (None, '1000'):
        if cap is None:
            monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB')
        else:
            monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', cap)
        gc, fc = g.clone().requires_grad_(True), f.clone().requires_grad_(True)
        cspn_b200.Affinity_Propagate3DK(N, 5, norm)(gc, fc).sum().backward()
        grads.append((gc.grad, fc.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    gc, fc = g[2:3].clone().requires_grad_(True), f[2:3].clone().requires_grad_(True)
    cspn_b200.Affinity_Propagate3DK(N, 5, norm)(gc, fc).sum().backward()
    assert torch.equal(gc.grad, grads[0][0][2:3]) and torch.equal(fc.grad, grads[0][1][2:3])


BWD = [(norm, shape, N) for norm in ('124sum', '124sum_abs', 'paddle')
       for shape, N in (((2, 1, 4, 6, 8), 3), ((1, 2, 5, 5, 11), 4), ((1, 1, 6, 7, 16), 5), ((1, 1, 3, 3, 4), 1))]


@pytest.mark.parametrize('norm,shape,N', BWD)
def test_gradients_match_fp64_autograd_of_the_torch_port(norm, shape, N):
    B, C, D, H, W = shape
    g, f = inputs_3d(31 + D + W + N, B, C, D, H, W, signed=(norm != 'paddle'))
    g = g + 0.05 * torch.sign(g)                                   # keep |g| away from the kink of abs
    go = torch.randn(B, C, D, H, W, generator=torch.Generator().manual_seed(N))
    g64, f64 = g.double().requires_grad_(True), f.double().requires_grad_(True)
    tpk.cspn3d_torch_k(g64, f64, N, 5, norm).backward(go.double())
    for use_op in (True, False):
        gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
        m = cspn_b200.Affinity_Propagate3DK(N, 5, norm)
        m._use_op = use_op                                         # dispatcher op and ctypes autograd.Function
        m(gc, fc).backward(go.cuda())
        for ours, theirs, name in ((gc.grad, g64.grad, 'guidance'), (fc.grad, f64.grad, 'feat')):
            ours = ours.double().cpu()
            scale = theirs.abs().mean()
            err = (ours - theirs).abs()
            assert (err <= 2e-3 * (theirs.abs() + scale)).all(), (name, use_op, float(err.max()), float(scale))


def test_properties_at_the_demo_volume():
    """demo.py's volume (3 x 1 x 48 x 64 x 128), N = 24: linear in feat; the gathered norms preserve a constant everywhere;
    'paddle' preserves it where no tap of the last N steps reaches the zero padding (N = 6, 12 voxels from every face)."""
    B, C, D, H, W, N = 3, 1, 48, 64, 128, 24
    g, f = [t.cuda() for t in inputs_3d(12, B, C, D, H, W, signed=False)]
    f2 = torch.rand_like(f)
    const = torch.full_like(f, 1.25)
    for norm in ('124sum', '124sum_abs', 'paddle'):
        gn = g - 0.5 if norm == '124sum' else g
        m = cspn_b200.Affinity_Propagate3DK(N, 5, norm)
        out = m(gn, f)
        assert torch.isfinite(out).all()
        assert torch.allclose(m(gn, 0.5 * f + 3 * f2), 0.5 * out + 3 * m(gn, f2), rtol=1e-4, atol=1e-4), norm
        if norm != 'paddle':
            assert torch.allclose(m(gn, const), const, rtol=1e-4), norm
    inner = (slice(None), slice(None), slice(12, -12), slice(12, -12), slice(12, -12))
    out = cspn_b200.Affinity_Propagate3DK(6, 5, 'paddle')(g, const)
    assert torch.allclose(out[inner], const[inner], rtol=1e-5)
    assert not torch.allclose(out, const, rtol=1e-5)               # and not at the faces


@pytest.mark.parametrize('norm', ['124sum_abs', 'paddle'])
def test_torch_compile_fullgraph_forward_and_backward(norm):
    m = cspn_b200.Affinity_Propagate3DK(5, 5, norm)
    g, f = [t.cuda() for t in inputs_3d(5, 2, 1, 6, 12, 16, signed=False)]

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


@pytest.mark.parametrize('norm', ['124sum', 'paddle'])
def test_cuda_graph_capture_and_replay(norm):
    m = cspn_b200.Affinity_Propagate3DK(6, 5, norm)
    g, f = [t.cuda() for t in inputs_3d(55, 2, 1, 8, 12, 32)]
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


@pytest.mark.parametrize('norm', ['124sum_abs', 'paddle'])
def test_training_step_through_the_module(norm):
    """Conv3d -> 5x5x5 CSPN -> L1 -> SGD changes the producer's weights."""
    torch.manual_seed(0)
    net = torch.nn.Conv3d(2, NT + 1, 3, padding=1).cuda()
    post = cspn_b200.Affinity_Propagate3DK(4, 5, norm)
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    x = torch.rand(2, 2, 6, 10, 12, device='cuda')
    target = torch.rand(2, 1, 6, 10, 12, device='cuda')
    w0 = net.weight.detach().clone()
    losses = []
    for _ in range(3):
        y = net(x)
        out = post(y[:, :NT], y[:, NT:])
        loss = (out - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert not torch.equal(net.weight, w0) and all(l == l for l in losses)


@pytest.mark.parametrize('k', [0, 61, 62, 123])
@pytest.mark.parametrize('W', [16, 13])
def test_one_hot_gates_are_exact_shifts_forward_and_backward(k, W):
    """A gate that is 1 on tap k and 0 elsewhere makes every step a shift by off_k: no rounding anywhere, so the forward equals
    the oracle bit for bit (for the gathered norm too, with its NaN where the tap reads the padding) and the 'paddle'
    gradient of feat equals fp64 autograd bit for bit.  This pins each tap's place in the forward and the adjoint."""
    B, C, D, H, N = 1, 2, 9, 10, 2                                 # N * r < D, H: part of every volume stays inside
    g = torch.zeros(B, NT, D, H, W)
    g[:, k] = 1.0
    f = torch.rand(B, C, D, H, W, generator=torch.Generator().manual_seed(k + W))
    go = torch.randn(B, C, D, H, W, generator=torch.Generator().manual_seed(2 * k + W))
    for norm in ('paddle', '124sum_abs'):
        ref = onk.cspn3d_k(g.numpy(), f.numpy(), N, 5, norm)
        out = cspn_b200.propagate3d_k(g.cuda(), f.cuda(), 5, N, norm).cpu().numpy()
        assert np.array_equal(out, ref, equal_nan=True), norm
        assert np.count_nonzero(np.nan_to_num(ref)) > ref.size // 8, norm      # not all padding
    f64 = f.double().requires_grad_(True)
    tpk.cspn3d_torch_k(g.double(), f64, N, 5, 'paddle').backward(go.double())
    for use_op in (True, False):
        gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
        m = cspn_b200.Affinity_Propagate3DK(N, 5, 'paddle')
        m._use_op = use_op
        m(gc, fc).backward(go.cuda())
        assert torch.equal(fc.grad.cpu().double(), f64.grad), use_op
        assert torch.count_nonzero(gc.grad) == 0                  # d|g|/dg = sign(g) = 0 on the zero taps; 0 on the hot one


@pytest.mark.parametrize('norm', ['124sum', '124sum_abs', 'paddle'])
@pytest.mark.parametrize('shape', [(1, 1, 5, 6, 8), (1, 2, 4, 5, 7)])
def test_gradients_of_positive_gates_match_fp64_autograd_to_1e_4(norm, shape):
    """With positive gates and two steps the gradient is well conditioned, so fp32 holds 1e-4 scale-relative: tight enough
    that a 2^-10 error on one of the 124 taps' gradients does not pass."""
    B, C, D, H, W = shape
    g, f = inputs_3d(90 + W, B, C, D, H, W, signed=False)
    g = g + 0.05
    go = torch.randn(B, C, D, H, W, generator=torch.Generator().manual_seed(W))
    g64, f64 = g.double().requires_grad_(True), f.double().requires_grad_(True)
    tpk.cspn3d_torch_k(g64, f64, 2, 5, norm).backward(go.double())
    for use_op in (True, False):
        gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
        m = cspn_b200.Affinity_Propagate3DK(2, 5, norm)
        m._use_op = use_op                                         # dispatcher op and ctypes autograd.Function
        m(gc, fc).backward(go.cuda())
        for ours, theirs, name in ((gc.grad, g64.grad, 'guidance'), (fc.grad, f64.grad, 'feat')):
            err = (ours.double().cpu() - theirs).abs()
            assert (err <= 1e-4 * (theirs.abs() + theirs.abs().mean())).all(), (name, use_op, float(err.max()))
