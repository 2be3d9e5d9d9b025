"""GPU tests of resize_trilinear (cspn_b200/csrc/resize_trilinear.cu; DESIGN.md section 4.14): the forward and the gather
backward bit for bit against the fp32 restatement of tests/resize_reference.py in all three modes, within a-priori bounds of
fp64 at the timing shapes and exactly at power-of-two ratios, determinism across streams, under
use_deterministic_algorithms and in CUDA graphs, the IEEE footprint, the memory contract, the torch integration, and one
training tail through the Paddle 3D propagation."""
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _resize_bwd, _resize_fwd, _ResizeTrilinearFn
from oracle import cspn_torch_port as tp

import memory_contract as mc
import resize_reference as rr

pytestmark = pytest.mark.gpu
MODES = [(True, 1), (False, 0), (False, 1)]

# (B, C, in_size, out_size): odd sizes, up on some axes and down on others, Wo a multiple of 4 and not
SHAPES = [
    (1, 1, (4, 5, 6), (7, 9, 13)),
    (2, 3, (7, 3, 9), (3, 8, 4)),
    (3, 2, (5, 6, 7), (9, 4, 16)),
    (1, 2, (1, 5, 1), (3, 1, 6)),
    (2, 1, (6, 1, 11), (1, 2, 5)),
    (1, 3, (9, 10, 33), (17, 7, 64)),
    (2, 2, (3, 4, 5), (3, 4, 5)),
    (1, 1, (2, 3, 130), (5, 6, 9)),
    (1, 1, (3, 2, 4), (6, 4, 33)),
]


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def bits_equal(a, b):
    return mc.same_bits(a.contiguous(), b.contiguous())


def fwd(x, out_size, ac, am):
    return cspn_b200.resize_trilinear(x, out_size, align_corners=ac, align_mode=am)


# ---- the forward and the backward against the fp32 restatement, bit for bit ---------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('B,C,in_size,out_size', SHAPES)
def test_forward_is_the_fp32_restatement_bit_for_bit(B, C, in_size, out_size, align_corners, align_mode):
    x = rand(B * 7 + C, B, C, *in_size)
    got = fwd(x.cuda(), out_size, align_corners, align_mode)
    want = torch.from_numpy(rr.forward_fp32(x.numpy(), out_size, align_corners, align_mode))
    assert got.shape == (B, C, *out_size) and bits_equal(got.cpu(), want)


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_forward_of_a_non_contiguous_input(align_corners, align_mode):
    base = rand(3, 2, 9, 4, 6, 5).cuda()
    x = base.permute(1, 0, 2, 3, 4)[:, :, :, :, ::2]              # (9, 2, 4, 6, 3), strided
    assert not x.is_contiguous()
    got = fwd(x, (5, 11, 8), align_corners, align_mode)
    want = torch.from_numpy(rr.forward_fp32(x.contiguous().cpu().numpy(), (5, 11, 8), align_corners, align_mode))
    assert bits_equal(got.cpu(), want)


@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('B,C,in_size,out_size', SHAPES)
def test_backward_is_the_fp32_restatement_bit_for_bit(B, C, in_size, out_size, align_corners, align_mode):
    x = rand(1, B, C, *in_size).cuda().requires_grad_(True)
    g = rand(2, B, C, *out_size)
    fwd(x, out_size, align_corners, align_mode).backward(g.cuda())
    want = torch.from_numpy(rr.backward_fp32(g.numpy(), in_size, align_corners, align_mode))
    assert bits_equal(x.grad.cpu(), want)


# ---- accuracy against fp64 at the timing shapes, and exactness at power-of-two ratios -------------------------------------
TIMING = [(3, 1, (48, 64, 128), (96, 128, 256)), (4, 1, (48, 64, 128), (192, 256, 512))]


@pytest.mark.parametrize('B,C,in_size,out_size', TIMING)
def test_timing_shapes_within_the_a_priori_bounds_of_fp64(B, C, in_size, out_size):
    gen = torch.Generator('cuda').manual_seed(4)
    x = torch.randn(B, C, *in_size, device='cuda', generator=gen)
    g = torch.randn(B, C, *out_size, device='cuda', generator=gen)
    for ac, am in MODES:
        out = fwd(x, out_size, ac, am)
        ref = rr.resize_torch(x.double(), out_size, ac, am)
        assert ((out.double() - ref).abs() <= rr.bound_fwd(rr.resize_torch(x.double().abs(), out_size, ac, am))).all()
        del out, ref
        gx = _resize_bwd(g, in_size, ac, am)
        ref = rr.adjoint_torch(g.double(), in_size, ac, am)
        k = rr.bound_bwd(in_size, out_size, ac, am)
        err = (gx.double() - ref).abs()
        assert (err <= k * rr.adjoint_torch(g.double().abs(), in_size, ac, am)).all(), float(err.max())
        assert float(err.norm() / ref.norm()) < 1e-6
        del gx, ref, err


@pytest.mark.parametrize('in_size,out_size,modes', [
    ((4, 6, 8), (8, 12, 16), [(False, 1), (False, 0)]),  # r = 1/2 without align_corners: weights 0, 1/2 (mode 1), 1/4, 3/4 (mode 0)
    ((5, 3, 9), (9, 5, 17), [(True, 1)]),             # r = 1/2 with align_corners
    ((9, 5, 17), (5, 3, 9), [(True, 1)]),             # r = 2
    ((8, 4, 16), (2, 1, 4), [(False, 1), (False, 0)]),   # r = 4, 4 (mode 1: s = 4o; mode 0: s = 4o + 1.5)
])
def test_power_of_two_ratios_on_small_integers_are_exact(in_size, out_size, modes):
    x = torch.randint(-8, 9, (2, 2, *in_size), generator=torch.Generator().manual_seed(5)).float()
    g = torch.randint(-8, 9, (2, 2, *out_size), generator=torch.Generator().manual_seed(6)).float()
    for ac, am in modes:
        assert torch.equal(fwd(x.cuda(), out_size, ac, am).cpu().double(), rr.resize_torch(x.double(), out_size, ac, am))
        gx = _resize_bwd(g.cuda(), in_size, ac, am).cpu().double()
        assert torch.equal(gx, rr.adjoint_torch(g.double(), in_size, ac, am))


# ---- determinism -------------------------------------------------------------------------------------------------------
def test_backward_bits_do_not_depend_on_the_stream_or_the_run():
    g = torch.randn(3, 2, 37, 41, 90, device='cuda')
    ref = _resize_bwd(g, (13, 20, 45), True, 1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = _resize_bwd(g, (13, 20, 45), True, 1)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(ref, again) and torch.equal(ref, _resize_bwd(g, (13, 20, 45), True, 1))
    # an image's bits do not depend on the rest of the batch
    assert torch.equal(_resize_bwd(g[1:2].contiguous(), (13, 20, 45), True, 1), ref[1:2])


def test_runs_under_deterministic_algorithms():
    x = torch.randn(2, 1, 6, 7, 8, device='cuda', requires_grad=True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = fwd(x, (12, 14, 16), True, 1)
        out.square().sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    want = rr.backward_fp32((2 * out.detach()).cpu().numpy(), (6, 7, 8), True, 1)
    assert bits_equal(x.grad.cpu(), torch.from_numpy(want))


def test_cuda_graph_capture_and_replay():
    x = torch.randn(2, 3, 12, 16, 32, device='cuda', requires_grad=True)
    g = torch.randn(2, 3, 24, 32, 64, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            fwd(x, (24, 32, 64), False, 1).backward(g)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        out = fwd(x, (24, 32, 64), False, 1)
        out.backward(g)
    with torch.no_grad():
        x.copy_(torch.randn_like(x))
    g.copy_(torch.randn_like(g))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, _resize_fwd(x.detach(), 24, 32, 64, False, 1))
    assert torch.equal(x.grad, _resize_bwd(g, (12, 16, 32), False, 1))


# ---- IEEE ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_a_non_finite_input_spreads_as_in_the_restatement(align_corners, align_mode, value):
    for (d, h, w) in [(0, 0, 0), (4, 5, 6), (2, 3, 3), (4, 0, 6)]:
        x = rand(8, 1, 2, 5, 6, 7)
        x[0, 1, d, h, w] = value
        for out_size in [(9, 11, 13), (3, 4, 5), (10, 12, 14)]:
            got = fwd(x.cuda(), out_size, align_corners, align_mode).cpu()
            want = torch.from_numpy(rr.forward_fp32(x.numpy(), out_size, align_corners, align_mode))
            assert bits_equal(got, want) and not torch.isfinite(got).all()


# ---- launches and the memory contract ----------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,in_size,out_size', [(2, 3, (5, 6, 7), (9, 11, 16)), (1, 2, (7, 9, 11), (3, 4, 5)),
                                                  (3, 1, (4, 4, 4), (8, 8, 13))])
def test_launch_counts_and_memory_contract(B, C, in_size, out_size):
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    x = torch.randn(B, C, *in_size, device='cuda')
    g = torch.randn(B, C, *out_size, device='cuda')
    before = mc.snapshot([x, g])
    for ac, am in MODES:
        for offset in (0, 4):                                   # a 16-byte aligned out (float4 stores when Wo % 4 == 0) and not
            out = mc.guarded((B, C, *out_size), offset)
            assert L.cspn_resize_trilinear_fwd_f32(x.data_ptr(), out.ptr(), B, C, *in_size, *out_size, int(ac), am, st) == 0
            assert L.cspn_last_launches() == 1
            torch.cuda.synchronize()
            mc.assert_written(out, 'out')
            assert torch.equal(out.t, _resize_fwd(x, *out_size, ac, am))
        nbytes = L.cspn_resize_trilinear_bwd_workspace_bytes(*in_size, *out_size)
        results = []
        for fill in ('sentinel', 'zero'):
            gx = mc.guarded((B, C, *in_size), 4)
            ws = mc.workspace(nbytes, 8, fill)
            assert L.cspn_resize_trilinear_bwd_f32(g.data_ptr(), gx.ptr(), B, C, *in_size, *out_size, int(ac), am, ws.ptr(),
                                                   nbytes, st) == 0
            assert L.cspn_last_launches() == 2
            torch.cuda.synchronize()
            mc.assert_written(gx, 'grad_x')
            assert ws.guards_intact()
            results.append(gx.t.clone())
        assert mc.same_bits(results[0], results[1]) and torch.equal(results[0], _resize_bwd(g, in_size, ac, am))
    assert mc.unchanged(before, [x, g])


def test_c_abi_refuses_overlapping_device_buffers():
    L = _lib.lib()
    buf = torch.zeros(1 << 12, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    assert L.cspn_resize_trilinear_fwd_f32(p, p + 4 * 100, 1, 1, 4, 5, 6, 8, 10, 12, 1, 1, st) == -1
    ws = torch.empty(1024, dtype=torch.uint8, device='cuda')
    assert L.cspn_resize_trilinear_bwd_f32(p, p + 4 * 100, 1, 1, 4, 5, 6, 8, 10, 12, 1, 1, ws.data_ptr(), 1024, st) == -1
    assert L.cspn_last_launches() == 0 and not buf.any()


# ---- torch integration -------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    x = torch.randn(2, 3, 7, 9, 11, device='cuda')
    g = torch.randn(2, 3, 13, 5, 20, device='cuda')
    for ac, am in MODES:
        res = []
        for route in ('op', 'fn'):
            xr = x.clone().requires_grad_(True)
            out = (torch.ops.cspn_b200.resize_trilinear(xr, 13, 5, 20, ac, am) if route == 'op'
                   else _ResizeTrilinearFn.apply(xr, 13, 5, 20, ac, am))
            out.backward(g)
            res.append((out.detach(), xr.grad))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_opcheck():
    torch_op.load()
    x = torch.randn(2, 3, 4, 5, 6, device='cuda', requires_grad=True)
    for ac, am in MODES:
        torch.library.opcheck(torch.ops.cspn_b200.resize_trilinear.default, (x, 7, 3, 9, ac, am))
        g = torch.randn(2, 3, 7, 3, 9, device='cuda')
        torch.library.opcheck(torch.ops.cspn_b200.resize_trilinear_backward.default, (g, 4, 5, 6, ac, am))


def test_torch_compile_fullgraph_forward_and_backward():
    x = torch.randn(2, 2, 6, 8, 10, device='cuda')

    def fn(t):
        return cspn_b200.resize_trilinear(t, scale=2.0, align_corners=False, align_mode=0).square().sum()

    res = []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        xc = x.clone().requires_grad_(True)
        loss = call(xc)
        loss.backward()
        res.append((loss.detach(), xc.grad))
    assert torch.equal(res[0][1], res[1][1]) and torch.allclose(res[0][0], res[1][0], rtol=1e-6)


def test_python_surface_on_the_device():
    x = torch.randn(1, 2, 5, 6, 7, device='cuda')
    assert cspn_b200.resize_trilinear(x, scale=1.5).shape == (1, 2, 7, 9, 10)
    assert torch.equal(cspn_b200.resize_trilinear(x, (7, 9, 10)), cspn_b200.resize_trilinear(x, scale=1.5))
    assert cspn_b200.resize_trilinear(x[:0], scale=2.0).shape == (0, 2, 10, 12, 14)
    with pytest.raises(ValueError):
        cspn_b200.resize_trilinear(x, (7, 9, 10), align_mode=3)
    # sizes the C ABI's ints cannot hold are refused before any allocation, on both routes
    torch_op.load()
    for size in [(2 ** 32 + 1, 1, 1), (1 << 11, 1 << 10, 1 << 10)]:
        with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
            cspn_b200.resize_trilinear(x, size)
        with pytest.raises(RuntimeError, match='2\\^31'):
            torch.ops.cspn_b200.resize_trilinear(x, *size, True, 1)
        with pytest.raises(RuntimeError, match='2\\^31'):
            torch.ops.cspn_b200.resize_trilinear_backward(torch.zeros(1, 2, 2, 2, 2, device='cuda'), *size, True, 1)


# ---- one training tail: resample a low-resolution guide and feature volume, propagate, mean, backward ---------------------
def test_training_tail_through_the_paddle_3d_propagation_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(9)
    guide = torch.randn(2, 26, 4, 6, 8, generator=gen)
    feat = torch.rand(2, 1, 4, 6, 8, generator=gen)
    size, steps = (8, 12, 16), 6
    gc, fc = guide.cuda().requires_grad_(True), feat.cuda().requires_grad_(True)
    g_up = cspn_b200.resize_trilinear(gc, size, align_corners=False, align_mode=1)
    f_up = cspn_b200.resize_trilinear(fc, size, align_corners=True)
    loss = cspn_b200.Affinity_Propagate3D(steps, 3, 'paddle')(g_up, f_up).mean()
    loss.backward()
    gd, fd = guide.double().requires_grad_(True), feat.double().requires_grad_(True)
    ref = tp.cspn3d_torch(rr.resize_torch(gd, size, False, 1), rr.resize_torch(fd, size, True, 1), steps, 'paddle').mean()
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    for got, want in ((gc.grad, gd.grad), (fc.grad, fd.grad)):
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
