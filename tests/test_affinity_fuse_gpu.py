"""GPU tests of affinity fusion (cspn_b200/csrc/affinity_fuse.cu; DESIGN.md section 4.18): the forward and both gradients
bit for bit against the fp32 order restatement and within the a-priori bounds of fp64 autograd, at odd shapes, with
repeated, full-resolution and downsampling levels, under all three alignment rules and at the three timing shapes; the
four anchors, the IEEE masks, the memory contract, determinism, both routes, the torch integration and one training
tail."""
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _AffinityFuseFn, _fuse_bwd, _fuse_fwd, _level_args

import affinity_fuse_reference as fr
import memory_contract as mc

pytestmark = pytest.mark.gpu

ALIGN = [(True, 1), (True, 0), (False, 0)]          # Paddle's default, F.interpolate(align_corners=True), and =False
# (B, C, H, W, level sizes): odd sizes, 1 x 1 and 1 x 2 levels, a full-resolution level, downsampling levels, L = 1 and
# L = 8, C past a forward channel chunk and not a multiple of it, W % 4 == 0 (the float4 store) and not
SHAPES = [
    (2, 3, 13, 19, ((1, 1), (2, 3), (4, 5))),
    (1, 5, 7, 8, ((7, 8), (2, 2))),
    (2, 6, 11, 30, ((20, 45), (3, 7), (1, 2), (11, 30))),
    (1, 2, 9, 10, tuple((1 + k % 5, 1 + (3 * k) % 11) for k in range(8))),
    (3, 17, 33, 47, ((4, 6), (8, 12), (17, 24))),
    (1, 1, 6, 5, ((3, 2),)),
    (2, 9, 64, 1, ((1, 1), (16, 1))),
]
# (name, B, H, W): C = 32, p = (64, 32, 16, 8), PSMNet's quarter-resolution feature map, align_corners=False, align_mode=0
TIMING = [('training crop', 4, 64, 128), ('KITTI inference', 1, 96, 312), ('SceneFlow test', 1, 136, 240)]
PS = (64, 32, 16, 8)


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, device='cuda', generator=torch.Generator('cuda').manual_seed(seed)) * scale


def inputs(seed, B, C, H, W, hws):
    levels = [rnd(seed + l, B, C, h, w) for l, (h, w) in enumerate(hws)]
    return levels, rnd(seed + 20, B, len(hws), H, W), rnd(seed + 21, B, C, H, W)


def kernel(levels, gate, grad_out, ac, am):
    """out, grad_levels, grad_gate through the C ABI (the ctypes route, no autograd)."""
    out = _fuse_fwd(levels, gate, ac, am)
    gl, gg = _fuse_bwd(levels, gate, out, grad_out, ac, am)
    return out, gl, gg


def autograd64(levels, gate, grad_out, ac, am):
    xs = [x.detach().double().requires_grad_(True) for x in levels]
    g = gate.detach().double().requires_grad_(True)
    out = fr.compose(xs, g, ac, am)
    out.backward(grad_out.double())
    return out.detach(), [x.grad for x in xs], g.grad


def check_all(levels, gate, go, ac, am):
    out, gl, gg = kernel(levels, gate, go, ac, am)
    want = fr.fwd_torch(levels, gate, ac, am)
    assert mc.same_bits(out, want)
    wl, wg = fr.bwd_torch(levels, gate, want, go, ac, am)
    assert mc.same_bits(gg, wg)
    assert all(mc.same_bits(a, b) for a, b in zip(gl, wl))
    o64, gl64, gg64 = autograd64(levels, gate, go, ac, am)
    assert fr.max_ratio(out, o64, fr.bound_fwd(levels, gate, ac, am)) <= 1.0
    lb, gb = fr.bound_bwd(levels, gate, go, ac, am)
    assert fr.max_ratio(gg, gg64, gb) <= 1.0
    for got, w, bound in zip(gl, gl64, lb):
        assert fr.max_ratio(got, w, bound) <= 1.0


# ---- exactness ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ac,am', ALIGN)
@pytest.mark.parametrize('B,C,H,W,hws', SHAPES)
def test_odd_shapes_bit_for_bit_and_within_the_bounds(B, C, H, W, hws, ac, am):
    check_all(*inputs(B * 7 + W, B, C, H, W, hws), ac, am)


@pytest.mark.parametrize('name,B,H,W', TIMING)
def test_timing_shapes(name, B, H, W):
    check_all(*inputs(11, B, 32, H, W, [(H // p, W // p) for p in PS]), False, 0)
    torch.cuda.empty_cache()


def test_a_repeated_level_gets_the_sum_of_its_gradients():
    levels, gate, go = inputs(3, 2, 4, 12, 17, ((3, 4), (6, 9)))
    x, y = (t.clone().requires_grad_(True) for t in levels)
    g = gate[:, :2].clone()
    g3 = torch.cat([g, rnd(40, 2, 1, 12, 17)], 1).requires_grad_(True)
    out = cspn_b200.affinity_fuse2d([x, y, x], g3, False, 0)
    out.backward(go)
    want, gl, gg = kernel([x.detach(), y.detach(), x.detach()], g3.detach(), go, False, 0)
    assert torch.equal(mc.words(out), mc.words(want))
    assert torch.equal(mc.words(x.grad), mc.words(gl[0] + gl[2])) and torch.equal(mc.words(y.grad), mc.words(gl[1]))
    assert torch.equal(mc.words(g3.grad), mc.words(gg))


# ---- the anchors ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ac,am', ALIGN)
def test_one_level_is_resize_trilinear(ac, am):
    x = rnd(1, 2, 5, 7, 9)
    gate = rnd(2, 2, 1, 20, 31)
    gate[gate == 0] = 1.0
    got = cspn_b200.affinity_fuse2d([x], gate, ac, am)
    want = cspn_b200.resize_trilinear(x[:, :, None], (1, 20, 31), align_corners=ac, align_mode=am)[:, :, 0]
    assert torch.equal(mc.words(got), mc.words(want))


def test_a_one_hot_gate_is_that_levels_upsampling():
    levels, _, _ = inputs(4, 2, 6, 21, 26, ((2, 3), (5, 7), (11, 13)))
    pick = torch.randint(0, 3, (2, 21, 26), device='cuda', generator=torch.Generator('cuda').manual_seed(5))
    gate = F.one_hot(pick, 3).permute(0, 3, 1, 2).float() * -2.5
    for ac, am in ALIGN:
        got = cspn_b200.affinity_fuse2d(levels, gate, ac, am)
        ups = torch.stack([cspn_b200.resize_trilinear(x[:, :, None], (1, 21, 26), align_corners=ac, align_mode=am)[:, :, 0]
                           for x in levels])
        want = torch.gather(ups, 0, pick[None, :, None].expand(1, 2, 6, 21, 26))[0]
        assert torch.equal(got, want)                       # equal values: -0.0 may come back as +0.0


def test_a_constant_gate_is_the_mean_of_the_interpolated_levels():
    levels, _, _ = inputs(6, 2, 5, 29, 35, ((1, 2), (3, 4), (7, 8), (14, 17)))
    gate = torch.full((2, 4, 29, 35), 0.3, device='cuda')
    for ac in (True, False):
        got = cspn_b200.affinity_fuse2d(levels, gate, ac, 0)
        want = sum(F.interpolate(x, size=(29, 35), mode='bilinear', align_corners=ac).double() for x in levels) / 4
        assert fr.max_ratio(got, want, fr.bound_fwd(levels, gate, ac, 0)) <= 2.0   # two fp32 evaluations of one blend


def test_a_full_resolution_level_under_a_one_hot_gate_is_itself():
    levels, _, _ = inputs(7, 2, 3, 19, 24, ((4, 5), (19, 24)))
    gate = torch.zeros(2, 2, 19, 24, device='cuda')
    gate[:, 1] = rnd(8, 2, 19, 24).abs() + 0.01
    for ac, am in ALIGN:
        assert torch.equal(mc.words(cspn_b200.affinity_fuse2d(levels, gate, ac, am)), mc.words(levels[1]))


# ---- IEEE --------------------------------------------------------------------------------------------------------------------
GATE_CASES = ['zero_pixel', 'neg_zero_pixel', 'inf_gate', 'neg_inf_gate', 'nan_gate', 'zero_gates', 'subnormal_gates']
LEVEL_CASES = ['nan_level', 'inf_level', 'zero_weight_inf']


def masks_equal(got, want):
    return (torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(torch.isinf(got), torch.isinf(want))
            and torch.equal(got[torch.isinf(got)], want[torch.isinf(want)].float()))


@pytest.mark.parametrize('case', GATE_CASES + LEVEL_CASES)
def test_ieee_masks(case):
    B, C, H, W, hws = 1, 4, 13, 18, ((2, 3), (5, 6), (13, 18))
    levels, gate, go = inputs(3, B, C, H, W, hws)
    if case == 'zero_pixel':
        gate[0, :, 4, 8] = 0.0
    elif case == 'neg_zero_pixel':
        gate[0, :, 7:9, 2] = -0.0
    elif case == 'inf_gate':
        gate[0, 1, 5, 7] = float('inf')
    elif case == 'neg_inf_gate':
        gate[0, 0, 2, 9] = float('-inf')
    elif case == 'nan_gate':
        gate[0, 2, 3, 3] = float('nan')
    elif case == 'zero_gates':
        gate[0, 1, ::2, 1::3] = 0.0
        gate[0, 0, 1::2, ::3] = -0.0
    elif case == 'subnormal_gates':                         # S is subnormal: no flush to zero
        gate[0, :, 4:8, 0:4] = torch.randint(1, 9, (3, 4, 4), device='cuda').float() * 1.4e-45
    elif case == 'nan_level':
        levels[1][0, 1, 2, 3] = float('nan')
    elif case == 'inf_level':
        levels[0][0, 2, 1, 1] = float('inf')
        levels[2][0, 0, 7, 1] = float('-inf')
    else:                                                   # every product is computed, those with a zero weight too
        levels[0][0, 0, 1, 2] = float('inf')
        gate[0, 0] = 0.0
    out, gl, gg = kernel(levels, gate, go, True, 1)
    want = fr.fwd_torch(levels, gate, True, 1)
    wl, wg = fr.bwd_torch(levels, gate, want, go, True, 1)
    for got, w in zip((out, gg, *gl), (want, wg, *wl)):
        assert mc.same_bits(got, w)
    # only the gates hold special values: fp64 has the same masks.  Subnormal sums are the exception: t / S overflows fp32
    # where fp64 stays finite
    if case in GATE_CASES and case != 'subnormal_gates':
        o64, gl64, gg64 = autograd64(levels, gate, go, True, 1)
        for got, w in zip((out, gg, *gl), (o64, gg64, *gl64)):
            assert masks_equal(got, w)
    if case in ('zero_pixel', 'neg_zero_pixel', 'inf_gate', 'nan_gate'):
        assert torch.isnan(out).any() and torch.isnan(gg).any()
        # w is NaN at the pixel in every level, except under an infinite gate, where the other levels get w = |g| / inf = 0
        nan_levels = (1,) if case == 'inf_gate' else (0, 1, 2)
        assert [bool(torch.isnan(g).any()) for g in gl] == [l in nan_levels for l in range(3)]
    if case == 'zero_pixel':
        assert torch.isnan(out[0, :, 4, 8]).all() and torch.isnan(gg[0, :, 4, 8]).all()


# ---- the memory contract -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,hws', [(2, 5, 13, 19, ((2, 3), (13, 19))), (1, 33, 40, 36, ((1, 2), (50, 45))),
                                          (2, 3, 16, 20, ((4, 5),))])
def test_launch_counts_and_memory_contract(B, C, H, W, hws):
    L_ = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    levels, gate, go = inputs(7, B, C, H, W, hws)
    L = len(hws)
    before = mc.snapshot([*levels, gate, go])
    ptrs, hw = _level_args(levels)
    out = mc.guarded((B, C, H, W), 4)
    assert L_.cspn_affinity_fuse2d_fwd_f32(ptrs, hw, gate.data_ptr(), out.ptr(), B, C, H, W, L, 1, 1, st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert torch.equal(mc.words(out.t), mc.words(_fuse_fwd(levels, gate, True, 1)))
    gl = [mc.guarded(tuple(x.shape), 4) for x in levels]
    gg = mc.guarded((B, L, H, W), 4)
    gptrs = (ctypes.c_void_p * L)(*[g.ptr() for g in gl])
    n = L_.cspn_affinity_fuse2d_bwd_workspace_bytes(B, C, H, W, L, hw)
    results = []
    for fill in ('sentinel', 'zero'):
        ws = mc.workspace(n, 4, fill)
        assert L_.cspn_affinity_fuse2d_bwd_f32(ptrs, hw, gate.data_ptr(), out.t.data_ptr(), go.data_ptr(), gptrs, gg.ptr(), B, C,
                                               H, W, L, 1, 1, ws.ptr(), n, st) == 0
        assert L_.cspn_last_launches() == 3
        torch.cuda.synchronize()
        assert ws.guards_intact()
        for g, x in zip(gl, levels):
            mc.assert_written(g, 'grad_levels')
        mc.assert_written(gg, 'grad_gate')
        results.append([mc.words(g.t).clone() for g in gl] + [mc.words(gg.t).clone()])
    assert all(torch.equal(a, b) for a, b in zip(*results))     # no workspace word is read before it is written
    wl, wg = _fuse_bwd(levels, gate, out.t, go, True, 1)
    assert all(torch.equal(a, mc.words(b)) for a, b in zip(results[0], [*wl, wg]))
    assert mc.unchanged(before, [*levels, gate, go])


def test_c_abi_refuses_overlapping_device_buffers():
    L_ = _lib.lib()
    buf = torch.zeros(1 << 14, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    hw = (ctypes.c_int * 2)(2, 3)                           # level 1x2x2x3 = 12 floats, gate 1x1x4x5 = 20, out 1x2x4x5 = 40
    lv = (ctypes.c_void_p * 1)(p)
    assert L_.cspn_affinity_fuse2d_fwd_f32(lv, hw, p + 4 * 1000, p + 4 * 8, 1, 2, 4, 5, 1, 1, 1, st) == -1
    assert L_.cspn_affinity_fuse2d_fwd_f32(lv, hw, p + 4 * 1000, p + 4 * 1010, 1, 2, 4, 5, 1, 1, 1, st) == -1
    n = L_.cspn_affinity_fuse2d_bwd_workspace_bytes(1, 2, 4, 5, 1, hw)
    for gl0, gg, ws in ((p + 4 * 1001, p + 4 * 4000, p + 4 * 5000), (p + 4 * 3000, p + 4 * 3005, p + 4 * 5000),
                        (p + 4 * 3000, p + 4 * 4000, p + 4 * 2030)):
        assert L_.cspn_affinity_fuse2d_bwd_f32(lv, hw, p + 4 * 1000, p + 4 * 2000, p + 4 * 2500, (ctypes.c_void_p * 1)(gl0), gg,
                                               1, 2, 4, 5, 1, 1, 1, ws, n, st) == -1
    assert L_.cspn_last_launches() == 0 and not buf.any()


def test_c_abi_takes_aliased_levels():
    """Inputs may alias: one level buffer passed twice gives the bits of two separate copies, forward and backward."""
    L_ = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    levels, gate, go = inputs(30, 2, 3, 9, 14, ((3, 5), (3, 5)))
    x, copy = levels[0], levels[0].clone()
    B, C, H, W, L = 2, 3, 9, 14, 2
    hw = (ctypes.c_int * 4)(3, 5, 3, 5)
    res = []
    for second in (x, copy):
        lv = (ctypes.c_void_p * 2)(x.data_ptr(), second.data_ptr())
        out = torch.empty(B, C, H, W, device='cuda')
        assert L_.cspn_affinity_fuse2d_fwd_f32(lv, hw, gate.data_ptr(), out.data_ptr(), B, C, H, W, L, 1, 1, st) == 0
        gl, gg = [torch.empty_like(x) for _ in range(L)], torch.empty_like(gate)
        n = L_.cspn_affinity_fuse2d_bwd_workspace_bytes(B, C, H, W, L, hw)
        ws = torch.empty(n, dtype=torch.uint8, device='cuda')
        assert L_.cspn_affinity_fuse2d_bwd_f32(lv, hw, gate.data_ptr(), out.data_ptr(), go.data_ptr(),
                                               (ctypes.c_void_p * 2)(*[g.data_ptr() for g in gl]), gg.data_ptr(), B, C, H, W, L,
                                               1, 1, ws.data_ptr(), n, st) == 0
        res.append((out, *gl, gg))
    torch.cuda.synchronize()
    assert all(torch.equal(mc.words(a), mc.words(b)) for a, b in zip(*res))


# ---- determinism -----------------------------------------------------------------------------------------------------------
def run_all(levels, gate, go, ac=False, am=0):
    out, gl, gg = kernel(levels, gate, go, ac, am)
    return (out, *gl, gg)


def test_bits_do_not_depend_on_the_stream_the_run_or_the_batch():
    B, C, H, W = 4, 40, 37, 70
    levels, gate, go = inputs(12, B, C, H, W, ((1, 2), (4, 8), (9, 17), (37, 70)))
    ref = run_all(levels, gate, go)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = run_all(levels, gate, go)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(ref, again, run_all(levels, gate, go)):
        assert torch.equal(mc.words(a), mc.words(b)) and torch.equal(mc.words(a), mc.words(c))
    for half in (slice(0, 2), slice(2, 4)):
        got = run_all([x[half].contiguous() for x in levels], gate[half].contiguous(), go[half].contiguous())
        for a, b in zip(got, ref):
            assert torch.equal(mc.words(a), mc.words(b[half]))


def test_runs_under_deterministic_algorithms():
    levels, gate, go = inputs(15, 2, 8, 21, 30, ((3, 4), (11, 15)))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        xs, g = [x.clone().requires_grad_(True) for x in levels], gate.clone().requires_grad_(True)
        out = cspn_b200.affinity_fuse2d(xs, g, False, 0)
        out.backward(go)
    finally:
        torch.use_deterministic_algorithms(prev)
    want, gl, gg = kernel(levels, gate, go, False, 0)
    assert torch.equal(out, want) and torch.equal(g.grad, gg) and all(torch.equal(x.grad, w) for x, w in zip(xs, gl))


def test_cuda_graph_capture_and_replay():
    levels, gate, go = inputs(17, 2, 8, 33, 64, ((1, 2), (4, 8), (16, 32)))
    xs, g = [x.clone().requires_grad_(True) for x in levels], gate.clone().requires_grad_(True)

    def step():
        for t in (*xs, g):
            t.grad = None
        out = cspn_b200.affinity_fuse2d(xs, g, False, 0)
        out.backward(go)
        return out

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    with torch.no_grad():
        for t in (*xs, g):
            t.copy_(torch.randn_like(t))
    graph.replay()
    torch.cuda.synchronize()
    want, gl, gg = kernel([x.detach() for x in xs], g.detach(), go, False, 0)
    assert torch.equal(out, want) and torch.equal(g.grad, gg) and all(torch.equal(x.grad, w) for x, w in zip(xs, gl))


# ---- torch integration -------------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    levels, gate, go = inputs(20, 2, 6, 19, 21, ((2, 3), (19, 21), (25, 30)))
    res = []
    for route in (lambda xs, g: torch.ops.cspn_b200.affinity_fuse2d(xs, g, True, 0),
                  lambda xs, g: _AffinityFuseFn.apply(True, 0, g, *xs)):
        xs, g = [x.clone().requires_grad_(True) for x in levels], gate.clone().requires_grad_(True)
        out = route(xs, g)
        out.backward(go)
        res.append((out.detach(), g.grad, *[x.grad for x in xs]))
    assert all(torch.equal(mc.words(x), mc.words(y)) for x, y in zip(*res))


def test_opcheck():
    torch_op.load()
    levels, gate, go = inputs(22, 2, 4, 10, 13, ((2, 3), (5, 7)))
    torch.library.opcheck(torch.ops.cspn_b200.affinity_fuse2d.default,
                          ([x.requires_grad_(True) for x in levels], gate.requires_grad_(True), False, 0))
    levels = [x.detach() for x in levels]
    out = _fuse_fwd(levels, gate.detach(), False, 0)
    torch.library.opcheck(torch.ops.cspn_b200.affinity_fuse2d_backward.default, (levels, gate.detach(), out, go, False, 0))


def test_torch_compile_fullgraph_forward_and_backward():
    levels, gate, _ = inputs(25, 2, 8, 24, 30, ((3, 4), (6, 8), (12, 15)))

    def fn(xs, g):
        return cspn_b200.affinity_fuse2d(xs, g, False, 0).square().sum()

    res = []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        xs, g = [x.clone().requires_grad_(True) for x in levels], gate.clone().requires_grad_(True)
        loss = call(xs, g)
        loss.backward()
        res.append((loss.detach(), g.grad, *[x.grad for x in xs]))
    for a, b in zip(*res):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-6)


def test_python_surface_on_the_device():
    levels, gate, _ = inputs(26, 1, 4, 9, 11, ((3, 3), (4, 5)))
    out = cspn_b200.affinity_fuse2d(levels, gate)
    assert out.shape == (1, 4, 9, 11)
    x0 = levels[0].transpose(2, 3).contiguous().transpose(2, 3)    # non-contiguous views are taken
    assert torch.equal(cspn_b200.affinity_fuse2d((x0, levels[1]), gate), out)
    torch_op.load()
    with pytest.raises(ValueError, match='align_mode'):
        torch.ops.cspn_b200.affinity_fuse2d(levels, gate, True, 3)


# ---- one training tail: affinity_pool2d, 1x1 conv branches, affinity_fuse2d, L1 loss, backward -------------------------------
def test_training_tail_matches_fp64_autograd():
    import affinity_pool_reference as apr
    gen = torch.Generator().manual_seed(27)
    B, C, H, W, ks = 2, 16, 24, 40, (8, 4, 2)
    feat = torch.randn(B, C, H, W, generator=gen)
    aff = nn.Conv2d(C, len(ks), 3, padding=1)
    branches = nn.ModuleList(nn.Conv2d(C, 8, 1, bias=False) for _ in ks)
    fuse = nn.Conv2d(C, len(ks), 3, padding=1)
    with torch.no_grad():
        for m in (aff, fuse, *branches):
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.2)
        aff.bias.zero_()
        fuse.bias.fill_(0.5)
    target = torch.randn(B, 8, H, W, generator=gen)

    def net(x, a, br, fu, pool, fuse_op):
        levels = [b(o) for b, o in zip(br, pool(x, a(x)))]
        y = fuse_op(levels, fu(x))
        return (y - target.to(y)).abs().mean()

    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                  # fp32 convolutions, not TF32
    try:
        a32, b32, f32 = aff.cuda(), branches.cuda(), fuse.cuda()
        x = feat.cuda().requires_grad_(True)
        loss = net(x, a32, b32, f32, lambda f, g: cspn_b200.affinity_pool2d(f, g, ks),
                   lambda xs, g: cspn_b200.affinity_fuse2d(xs, g, False, 0))
        loss.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    a64, b64, f64 = (m.double().cpu() for m in (nn.Conv2d(C, len(ks), 3, padding=1), nn.ModuleList(nn.Conv2d(C, 8, 1, bias=False)
                                                                                                  for _ in ks),
                                               nn.Conv2d(C, len(ks), 3, padding=1)))
    for m64, m32 in ((a64, a32), (b64, b32), (f64, f32)):
        m64.load_state_dict({k: v.double().cpu() for k, v in m32.state_dict().items()})
    x64 = feat.double().requires_grad_(True)
    ref = net(x64, a64, b64, f64, lambda f, g: apr.compose(f, g, ks), lambda xs, g: fr.compose(xs, g, False, 0))
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    pairs = [(x.grad, x64.grad), (a32.weight.grad, a64.weight.grad), (f32.weight.grad, f64.weight.grad)]
    pairs += [(p.weight.grad, q.weight.grad) for p, q in zip(b32, b64)]
    for got, want in pairs:
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
