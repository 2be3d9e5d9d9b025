"""GPU tests of disparity_regression (cspn_b200/csrc/disparity_regression.cu; DESIGN.md section 4.15): the softmax stage
against fp64 on resize_trilinear's own fp32 output, the whole op within the a-priori bounds of the fp64 composition
resize -> softmax -> expectation at odd shapes and at both timing shapes, exact results on sharp columns, determinism,
the IEEE footprint, the memory contract, peak memory, the torch integration, and one training tail through the Paddle 3D
propagation."""
import pytest
import torch
import torch.nn.functional as F

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _disparity_bwd, _disparity_fwd, _DisparityRegressionFn
from oracle import cspn_torch_port as tp

import disparity_reference as dr
import memory_contract as mc

pytestmark = pytest.mark.gpu
MODES = [(True, 1), (False, 0), (False, 1)]

# (B, C, in_size, out_size): up on some axes and down on others, Wo a multiple of 4 and not, identity, size-1 axes
SHAPES = [
    (1, 1, (5, 4, 6), (17, 13, 21)),
    (2, 3, (7, 3, 9), (4, 8, 5)),
    (3, 2, (6, 9, 7), (24, 5, 16)),
    (1, 2, (1, 5, 1), (3, 1, 6)),
    (2, 1, (6, 1, 11), (1, 2, 5)),
    (1, 3, (9, 10, 33), (17, 37, 64)),
    (2, 2, (4, 5, 6), (4, 5, 6)),
    (1, 1, (12, 16, 30), (48, 64, 121)),
]
TIMING = [(4, 1, (48, 64, 128), (192, 256, 512)), (1, 1, (48, 96, 312), (192, 384, 1248))]


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def fwd(cost, out_size, ac, am):
    return cspn_b200.disparity_regression(cost, out_size, align_corners=ac, align_mode=am)


# ---- the softmax stage alone, on resize_trilinear's fp32 output -----------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('B,C,in_size,out_size', SHAPES)
def test_softmax_stage_within_its_bound(B, C, in_size, out_size, align_corners, align_mode):
    cost = (rand(B * 7 + C, B, C, *in_size) * 3).cuda()
    u32 = cspn_b200.resize_trilinear(cost, out_size, align_corners=align_corners, align_mode=align_mode)
    got = fwd(cost, out_size, align_corners, align_mode)
    assert got.shape == (B, C, *out_size[1:])
    assert dr.max_ratio(got, dr.regress_torch(u32.double()), dr.bound_softmax(u32)) <= 1.0


# ---- the whole op within the a-priori bounds of the fp64 composition -------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('B,C,in_size,out_size', SHAPES)
def test_whole_op_within_the_bounds_of_fp64(B, C, in_size, out_size, align_corners, align_mode):
    cost = (rand(B * 5 + C, B, C, *in_size) * 3).cuda()
    g = rand(3, B, C, *out_size[1:]).cuda()
    y = fwd(cost, out_size, align_corners, align_mode)
    assert dr.max_ratio(y, dr.forward_torch(cost, out_size, align_corners, align_mode),
                        dr.bound_fwd(cost, out_size, align_corners, align_mode)) <= 1.0
    gc = _disparity_bwd(cost, g, *out_size, align_corners, align_mode)
    assert dr.max_ratio(gc, dr.grad_torch(cost, g, out_size, align_corners, align_mode),
                        dr.bound_bwd(cost, g, out_size, align_corners, align_mode)) <= 1.0


# the backward's fallback tiles of one cell by two and one by one (a deep cost volume upsampled 6-8x in H and W), in every
# mode: (align_corners, align_mode, tile) -> (in_size, out_size), tile as tests/disparity_reference.bwd_plan picks it
SMALL_TILES = [
    (True, 1, (1, 2), (28, 4, 5), (28, 32, 40)),
    (True, 1, (1, 1), (40, 4, 5), (40, 32, 40)),
    (False, 0, (1, 2), (32, 4, 5), (32, 32, 40)),
    (False, 0, (1, 1), (44, 4, 5), (44, 32, 40)),
    (False, 1, (1, 2), (40, 4, 5), (40, 32, 40)),
    (False, 1, (1, 1), (60, 4, 5), (60, 32, 40)),
]


@pytest.mark.parametrize('align_corners,align_mode,tile,in_size,out_size', SMALL_TILES)
def test_small_backward_tiles_within_the_bounds_of_fp64(align_corners, align_mode, tile, in_size, out_size):
    assert dr.bwd_plan(in_size, out_size, align_corners, align_mode)[0] == tile
    cost = (rand(sum(in_size), 2, 1, *in_size) * 3).cuda()
    g = rand(5, 2, 1, *out_size[1:]).cuda()
    y = fwd(cost, out_size, align_corners, align_mode)
    assert dr.max_ratio(y, dr.forward_torch(cost, out_size, align_corners, align_mode),
                        dr.bound_fwd(cost, out_size, align_corners, align_mode)) <= 1.0
    gc = _disparity_bwd(cost, g, *out_size, align_corners, align_mode)
    assert dr.max_ratio(gc, dr.grad_torch(cost, g, out_size, align_corners, align_mode),
                        dr.bound_bwd(cost, g, out_size, align_corners, align_mode)) <= 1.0
    # the bits do not depend on the tile: one image at a time gives the same
    assert torch.equal(_disparity_bwd(cost[1:], g[1:], *out_size, align_corners, align_mode), gc[1:])


# ---- the upsampled values are resize_trilinear's bits ----------------------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('B,C,in_size,out_size', SHAPES[:3] + SHAPES[5:])
def test_forward_is_the_softmax_stage_of_resize_trilinear_bit_for_bit(B, C, in_size, out_size, align_corners, align_mode):
    """The softmax stage restated in torch fp32 on resize_trilinear's own output gives the kernel's bits: a blend in any
    other order would move U by an ulp and y with it somewhere."""
    cost = (rand(B * 3 + C, B, C, *in_size) * 3).cuda()
    u32 = cspn_b200.resize_trilinear(cost, out_size, align_corners=align_corners, align_mode=align_mode)
    assert mc.same_bits(fwd(cost, out_size, align_corners, align_mode), dr.softmax_stage_torch(u32))


@pytest.mark.parametrize('B,C,in_size,out_size', TIMING)
def test_timing_shapes_within_the_bounds_of_fp64(B, C, in_size, out_size):
    gen = torch.Generator('cuda').manual_seed(4)
    cost = torch.randn(B, C, *in_size, device='cuda', generator=gen) * 3
    g = torch.randn(B, C, *out_size[1:], device='cuda', generator=gen)
    for ac, am in MODES:
        y = fwd(cost, out_size, ac, am)
        ref = dr.forward_torch(cost, out_size, ac, am)
        ratio = dr.max_ratio(y, ref, dr.bound_fwd(cost, out_size, ac, am))
        err = dr.normwise(y, ref)
        del ref
        gc = _disparity_bwd(cost, g, *out_size, ac, am)
        ref = dr.grad_torch(cost, g, out_size, ac, am)
        gratio = dr.max_ratio(gc, ref, dr.bound_bwd(cost, g, out_size, ac, am))
        gerr = dr.normwise(gc, ref)
        del ref
        torch.cuda.empty_cache()
        print(f'{(B, C, *in_size)} -> {out_size} mode {(ac, am)}: y normwise {err:.2e} (bound ratio {ratio:.2e}), '
              f'grad_cost normwise {gerr:.2e} (bound ratio {gratio:.2e})')
        assert ratio <= 1.0 and gratio <= 1.0 and err < 1e-6 and gerr < 1e-5


# ---- exact cases -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W,Ho,Wo', [(4, 6, 7, 11), (3, 5, 12, 20), (6, 4, 3, 9)])
def test_sharp_columns_give_exact_results(H, W, Ho, Wo):
    """A spike of 1000 at d = k: with (D, Do) = (5, 17) and align_corners (r = 1/4), U at o = 4k is the spike row's blend
    exactly and every other o is >= 234 below it, so exp underflows to 0 there: y = 4k and grad_cost = 0 exactly."""
    cost, k = dr.sharp_cost(2, 3, H, W, seed=H * W)
    cost = cost.cuda().requires_grad_(True)
    y = fwd(cost, (17, Ho, Wo), True, 1)
    assert torch.equal(y, (4 * k).float().cuda()[:, :, None, None].expand_as(y))
    y.backward(torch.randn_like(y))
    assert torch.equal(cost.grad, torch.zeros_like(cost))


# ---- determinism -----------------------------------------------------------------------------------------------------------
def test_bits_do_not_depend_on_the_stream_the_run_or_the_batch():
    cost = torch.randn(4, 2, 13, 20, 45, device='cuda')
    g = torch.randn(4, 2, 77, 173, device='cuda')
    size = (51, 77, 173)
    ref = (_disparity_fwd(cost, *size, True, 1), _disparity_bwd(cost, g, *size, True, 1))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = (_disparity_fwd(cost, *size, True, 1), _disparity_bwd(cost, g, *size, True, 1))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(ref, again, (_disparity_fwd(cost, *size, True, 1), _disparity_bwd(cost, g, *size, True, 1))):
        assert torch.equal(a, b) and torch.equal(a, c)
    for half in (slice(0, 2), slice(2, 4)):
        assert torch.equal(_disparity_fwd(cost[half], *size, True, 1), ref[0][half])
        assert torch.equal(_disparity_bwd(cost[half], g[half], *size, True, 1), ref[1][half])


def test_runs_under_deterministic_algorithms():
    cost = torch.randn(2, 1, 6, 7, 8, device='cuda', requires_grad=True)
    g = torch.randn(2, 1, 28, 32, device='cuda')
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        y = fwd(cost, (24, 28, 32), False, 1)
        y.backward(g)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(y, _disparity_fwd(cost.detach(), 24, 28, 32, False, 1))
    assert torch.equal(cost.grad, _disparity_bwd(cost.detach(), g, 24, 28, 32, False, 1))


def test_cuda_graph_capture_and_replay():
    cost = torch.randn(2, 3, 12, 16, 32, device='cuda', requires_grad=True)
    g = torch.randn(2, 3, 64, 128, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            cost.grad = None
            fwd(cost, (48, 64, 128), True, 1).backward(g)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    cost.grad = None
    with torch.cuda.graph(graph):
        y = fwd(cost, (48, 64, 128), True, 1)
        y.backward(g)
    with torch.no_grad():
        cost.copy_(torch.randn_like(cost))
    g.copy_(torch.randn_like(g))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, _disparity_fwd(cost.detach(), 48, 64, 128, True, 1))
    assert torch.equal(cost.grad, _disparity_bwd(cost.detach(), g, 48, 64, 128, True, 1))


# ---- IEEE -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_nan_masks_are_the_fp64_compositions(align_corners, align_mode, value):
    for where in [(0, 0, 0), (4, 5, 6), (2, 3, 3), (4, 0, 6)]:
        cost = rand(8, 1, 2, 5, 6, 7)
        cost[0, 1][where] = value
        if value == float('-inf'):                 # a whole column of -inf too
            cost[0, 0, :, 2, 2] = value
        g = rand(9, 1, 2, 13, 15)
        for out_size in [(9, 13, 15), (3, 13, 15), (17, 13, 15)]:
            gs = g[:, :, :out_size[1], :out_size[2]].contiguous()
            y = fwd(cost.cuda(), out_size, align_corners, align_mode).cpu()
            want = torch.isnan(dr.forward_torch(cost, out_size, align_corners, align_mode))
            assert torch.equal(torch.isnan(y), want) and want.any()
            gc = _disparity_bwd(cost.cuda(), gs.cuda(), *out_size, align_corners, align_mode).cpu()
            assert torch.equal(torch.isnan(gc), torch.isnan(dr.grad_torch(cost, gs, out_size, align_corners, align_mode)))


# ---- launches and the memory contract ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,in_size,out_size', [(2, 3, (5, 6, 7), (9, 11, 16)), (1, 2, (7, 9, 11), (3, 4, 5)),
                                                  (3, 1, (4, 4, 4), (16, 16, 13))])
def test_launch_counts_and_memory_contract(B, C, in_size, out_size):
    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    cost = torch.randn(B, C, *in_size, device='cuda')
    g = torch.randn(B, C, *out_size[1:], device='cuda')
    before = mc.snapshot([cost, g])
    for ac, am in MODES:
        y = mc.guarded((B, C, *out_size[1:]), 4)
        assert L.cspn_disparity_regression_fwd_f32(cost.data_ptr(), y.ptr(), B, C, *in_size, *out_size, int(ac), am, st) == 0
        assert L.cspn_last_launches() == 1
        torch.cuda.synchronize()
        mc.assert_written(y, 'out')
        assert torch.equal(y.t, _disparity_fwd(cost, *out_size, ac, am))
        nbytes = L.cspn_disparity_regression_bwd_workspace_bytes(*in_size, *out_size)
        results = []
        for fill in ('sentinel', 'zero'):
            gc = mc.guarded((B, C, *in_size), 4)
            ws = mc.workspace(nbytes, 8, fill)
            assert L.cspn_disparity_regression_bwd_f32(cost.data_ptr(), g.data_ptr(), gc.ptr(), B, C, *in_size, *out_size,
                                                       int(ac), am, ws.ptr(), nbytes, st) == 0
            assert L.cspn_last_launches() == 2
            torch.cuda.synchronize()
            mc.assert_written(gc, 'grad_cost')
            assert ws.guards_intact()
            results.append(gc.t.clone())
        assert mc.same_bits(results[0], results[1]) and torch.equal(results[0], _disparity_bwd(cost, g, *out_size, ac, am))
    assert mc.unchanged(before, [cost, g])


def test_c_abi_refuses_overlapping_device_buffers():
    L = _lib.lib()
    buf = torch.zeros(1 << 12, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    assert L.cspn_disparity_regression_fwd_f32(p, p + 4 * 100, 1, 1, 4, 5, 6, 8, 10, 12, 1, 1, st) == -1
    ws = torch.empty(1024, dtype=torch.uint8, device='cuda')
    assert L.cspn_disparity_regression_bwd_f32(p, p + 4 * 2048, p + 4 * 100, 1, 1, 4, 5, 6, 8, 10, 12, 1, 1, ws.data_ptr(),
                                               1024, st) == -1
    assert L.cspn_disparity_regression_bwd_f32(p, p + 4 * 2048, p + 4 * 1000, 1, 1, 4, 5, 6, 8, 10, 12, 1, 1, p + 4 * 1100,
                                               1024, st) == -1
    assert L.cspn_last_launches() == 0 and not buf.any()


# ---- peak memory -------------------------------------------------------------------------------------------------------------
def test_forward_and_backward_never_hold_the_upsampled_volume():
    B, C, in_size, out_size = TIMING[0]
    volume = 4 * B * C * out_size[0] * out_size[1] * out_size[2]          # 402.65 MB
    assert volume >= 200e6
    cost = torch.randn(B, C, *in_size, device='cuda', requires_grad=True)
    g = torch.randn(B, C, *out_size[1:], device='cuda')
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fwd(cost, out_size, True, 1).backward(g)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    print(f'peak above the inputs: {extra / 1e6:.2f} MB for a {volume / 1e6:.2f} MB upsampled volume')
    assert extra < volume / 8


# ---- torch integration -------------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    cost = torch.randn(2, 3, 7, 9, 11, device='cuda')
    g = torch.randn(2, 3, 5, 20, device='cuda')
    for ac, am in MODES:
        res = []
        for route in ('op', 'fn'):
            cr = cost.clone().requires_grad_(True)
            y = (torch.ops.cspn_b200.disparity_regression(cr, 13, 5, 20, ac, am) if route == 'op'
                 else _DisparityRegressionFn.apply(cr, 13, 5, 20, ac, am))
            y.backward(g)
            res.append((y.detach(), cr.grad))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_opcheck():
    torch_op.load()
    cost = torch.randn(2, 3, 4, 5, 6, device='cuda', requires_grad=True)
    for ac, am in MODES:
        torch.library.opcheck(torch.ops.cspn_b200.disparity_regression.default, (cost, 7, 3, 9, ac, am))
        g = torch.randn(2, 3, 3, 9, device='cuda')
        torch.library.opcheck(torch.ops.cspn_b200.disparity_regression_backward.default, (cost.detach(), g, 7, 3, 9, ac, am))


def test_torch_compile_fullgraph_forward_and_backward():
    cost = torch.randn(2, 1, 6, 8, 10, device='cuda')

    def fn(t):
        return cspn_b200.disparity_regression(t, scale=4.0).square().sum()

    res = []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        cc = cost.clone().requires_grad_(True)
        loss = call(cc)
        loss.backward()
        res.append((loss.detach(), cc.grad))
    assert torch.equal(res[0][1], res[1][1]) and torch.allclose(res[0][0], res[1][0], rtol=1e-6)


def test_python_surface_on_the_device():
    cost = torch.randn(1, 2, 5, 6, 7, device='cuda')
    assert cspn_b200.disparity_regression(cost, scale=4).shape == (1, 2, 24, 28)
    assert torch.equal(cspn_b200.disparity_regression(cost, (20, 24, 28)), cspn_b200.disparity_regression(cost, scale=4))
    assert cspn_b200.disparity_regression(cost[:0], scale=2.0).shape == (0, 2, 12, 14)
    torch_op.load()
    with pytest.raises(RuntimeError, match='2\\^31'):
        torch.ops.cspn_b200.disparity_regression(cost, 1 << 11, 1 << 10, 1 << 10, True, 1)
    with pytest.raises(RuntimeError, match='shared memory'):
        torch.ops.cspn_b200.disparity_regression(torch.zeros(1, 1, 20000, 1, 1, device='cuda'), 20000, 1, 1, True, 1)


# ---- one training tail: propagate a low-resolution cost volume, regress disparity x4, masked smooth L1, backward ----------
def test_training_tail_through_the_paddle_3d_propagation_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(9)
    guide = torch.randn(2, 26, 6, 8, 10, generator=gen)
    cost = torch.randn(2, 1, 6, 8, 10, generator=gen) * 2
    size, steps = (24, 32, 40), 6
    target = torch.rand(2, 1, 32, 40, generator=gen) * 24
    mask = target > 2

    def loss_of(y):
        m = mask.to(y.device)
        return F.smooth_l1_loss(y[m], target.to(y)[m])

    gc, cc = guide.cuda().requires_grad_(True), cost.cuda().requires_grad_(True)
    y = cspn_b200.disparity_regression(cspn_b200.Affinity_Propagate3D(steps, 3, 'paddle')(gc, cc), size)
    loss = loss_of(y)
    loss.backward()
    gd, cd = guide.double().requires_grad_(True), cost.double().requires_grad_(True)
    ref = loss_of(dr.forward_torch(tp.cspn3d_torch(gd, cd, steps, 'paddle'), size))
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    for got, want in ((gc.grad, gd.grad), (cc.grad, cd.grad)):
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
