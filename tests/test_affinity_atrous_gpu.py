"""GPU tests of atrous affinity pooling (cspn_b200/csrc/affinity_atrous.cu; DESIGN.md section 4.19): the forward and both
gradients bit for bit against the fp32 order restatement and within the a-priori bounds of fp64 autograd, at odd shapes and
the three timing shapes; each level against that level alone, the IEEE masks case by case, a cross-check against
affinity_propagate, the launch counts and the memory contract, determinism, both routes, the torch integration and one
training tail."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _AffinityAtrousFn, _atrous_bwd, _atrous_fwd, _c_sizes

import affinity_atrous_reference as ar
import memory_contract as mc
from test_affinity_atrous_cpu import IEEE, ieee_case, masks_equal

pytestmark = pytest.mark.gpu

# (B, C, H, W, rates): H, W multiples of no tile, C = 1, C = 129 (past a channel chunk), r = 1, r > H, r > W,
# r = max(H, W), repeated and unordered rates, L = 1 and L = 8, W past one row block
SHAPES = [
    (2, 3, 13, 19, (2, 3, 5)),
    (1, 1, 7, 7, (7, 1)),
    (2, 129, 11, 30, (4, 4, 1, 30)),
    (1, 4, 9, 10, (1, 2, 3, 4, 5, 6, 7, 8)),
    (3, 17, 33, 47, (16, 40, 3)),
    (1, 2, 150, 301, (301, 24, 200)),
    (2, 37, 70, 131, (64, 2)),
    (1, 33, 6, 5, (5,)),
]
# (name, B, H, W): C = 128, rates (6, 12, 18, 24), PSMNet's quarter-resolution feature map
TIMING = [('training crop', 4, 64, 128), ('KITTI inference', 1, 96, 312), ('SceneFlow test', 1, 136, 240)]
RATES = (6, 12, 18, 24)


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, device='cuda', generator=torch.Generator('cuda').manual_seed(seed)) * scale


def inputs(seed, B, C, H, W, rates):
    L = len(rates)
    return rnd(seed, B, C, H, W), rnd(seed + 1, B, 9 * L, H, W), rnd(seed + 2, B, L * C, H, W)


def kernel(feat, gate, rates, grad):
    """out, grad_feat, grad_gate through the C ABI (the ctypes route, no autograd)."""
    out = _atrous_fwd(feat, gate, rates)
    return (out, *_atrous_bwd(feat, gate, out, grad, rates))


def autograd64(feat, gate, rates, grad):
    f, g = feat.detach().double().requires_grad_(True), gate.detach().double().requires_grad_(True)
    out = ar.compose(f, g, rates)
    out.backward(grad.double())
    return out.detach(), f.grad, g.grad


def check_all(feat, gate, rates, grad):
    out, gf, gg = kernel(feat, gate, rates, grad)
    want = ar.fwd_torch(feat, gate, rates)
    assert mc.same_bits(out, want)
    for got, w in zip((gf, gg), ar.bwd_torch(feat, gate, rates, want, grad)):
        assert mc.same_bits(got, w)
    o64, gf64, gg64 = autograd64(feat, gate, rates, grad)
    assert ar.max_ratio(out, o64, ar.bound_fwd(feat, gate, rates)) <= 1.0
    for got, w, bound in zip((gf, gg), (gf64, gg64), ar.bound_bwd(feat, gate, rates, grad)):
        assert ar.max_ratio(got, w, bound) <= 1.0


# ---- exactness ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,rates', SHAPES)
def test_odd_shapes_bit_for_bit_and_within_the_bounds(B, C, H, W, rates):
    feat, gate, grad = inputs(B * 7 + W, B, C, H, W, rates)
    check_all(feat, gate, rates, grad)


@pytest.mark.parametrize('name,B,H,W', TIMING)
def test_timing_shapes(name, B, H, W):
    feat, gate, grad = inputs(11, B, 128, H, W, RATES)
    check_all(feat, gate, RATES, grad)
    torch.cuda.empty_cache()


def test_anchors_on_the_device():
    """A constant gate is the depthwise dilated box filter within the bound; a one-hot gate shifts feat bit for bit."""
    feat = rnd(1, 2, 6, 29, 35)
    rates = (1, 4, 30, 9)
    gate = torch.full((2, 36, 29, 35), 0.3, device='cuda')
    box = torch.ones(6, 1, 3, 3, dtype=torch.float64, device='cuda') / 9
    want = torch.cat([F.conv2d(feat.double(), box, padding=r, dilation=r, groups=6) for r in rates], 1)
    assert ar.max_ratio(cspn_b200.affinity_atrous_pool2d(feat, gate, rates), want, ar.bound_fwd(feat, gate, rates)) <= 1.0
    for t in range(9):
        gate = torch.zeros(2, 36, 29, 35, device='cuda')
        gate[:, t::9] = -1.7
        dy, dx = ar.OFFSETS[t]
        want = torch.cat([ar.shifted(feat, r * dy, r * dx) for r in rates], 1)
        assert torch.equal(mc.words(cspn_b200.affinity_atrous_pool2d(feat, gate, rates)), mc.words(want))


def test_each_level_is_the_level_alone():
    rates = (12, 5, 5, 1, 45)
    feat, gate, grad = inputs(2, 2, 9, 45, 38, rates)
    out, gf, gg = kernel(feat, gate, rates, grad)
    C = 9
    for l, r in enumerate(rates):
        g1 = gate[:, 9 * l:9 * l + 9].contiguous()
        go1 = grad[:, l * C:(l + 1) * C].contiguous()
        alone, _, gg1 = kernel(feat, g1, (r,), go1)
        assert torch.equal(mc.words(alone), mc.words(out[:, l * C:(l + 1) * C]))
        assert torch.equal(mc.words(gg1), mc.words(gg[:, 9 * l:9 * l + 9]))


# ---- IEEE --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', IEEE)
def test_ieee_masks_of_fp64_autograd(case):
    rates = (2, 5, 14)
    feat, gate, grad = inputs(3, 1, 4, 13, 18, rates)
    ieee_case(case, feat, gate)
    out, gf, gg = kernel(feat, gate, rates, grad)
    o64, gf64, gg64 = autograd64(feat, gate, rates, grad)
    for got, want in zip((out, gf, gg), (o64, gf64, gg64)):
        assert masks_equal(got, want)
    want = ar.fwd_torch(feat, gate, rates)
    for got, w in zip((out, gf, gg), (want, *ar.bwd_torch(feat, gate, rates, want, grad))):
        assert mc.same_bits(got, w)
    if case in ('zero_gates', 'inf_gate', 'nan_gate_on_padding'):
        assert torch.isnan(out).any()


# ---- an independent cross-check: r = 1 with the centre gate zero is affinity_propagate on the 8 normalised weights -----------
def test_rate_one_without_centre_is_affinity_propagate():
    feat, gate, _ = inputs(8, 2, 5, 21, 34, (1,))
    gate[:, 4] = 0.0
    w, _ = ar.weights(gate, 0)                                # the kernel's weights, bit for bit
    # affinity_propagate's tap k, raster (i, j) without the centre, reads offset (1 - i, 1 - j): tap 8 - (3i + j) here
    want = cspn_b200.affinity_propagate(feat, w[:, [8, 7, 6, 5, 3, 2, 1, 0]].contiguous(), 3, 1)
    got = cspn_b200.affinity_atrous_pool2d(feat, gate, (1,))
    assert ar.max_ratio(got, want, ar.bound_fwd(feat, gate, (1,))) <= 1.0


# ---- the memory contract -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,rates', [(2, 5, 13, 19, (2, 3, 13)), (1, 33, 40, 137, (16, 1)), (2, 3, 15, 14, (14,))])
@pytest.mark.parametrize('offset', [0, 4])
def test_launch_counts_and_memory_contract(B, C, H, W, rates, offset):
    L_ = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    feat, gate, go = inputs(7, B, C, H, W, rates)
    L = len(rates)
    r = _c_sizes(rates)
    before = mc.snapshot([feat, gate, go])
    out = mc.guarded((B, L * C, H, W), offset)
    assert L_.cspn_affinity_atrous2d_fwd_f32(feat.data_ptr(), gate.data_ptr(), out.ptr(), B, C, H, W, L, r, st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert torch.equal(mc.words(out.t), mc.words(_atrous_fwd(feat, gate, rates)))
    gf, gg = mc.guarded((B, C, H, W), offset), mc.guarded((B, 9 * L, H, W), offset)
    n = L_.cspn_affinity_atrous2d_bwd_workspace_bytes(B, C, H, W, L, r)
    assert n == 4 * B * 9 * L * H * W
    results = []
    for fill in ('sentinel', 'zero'):
        ws = mc.workspace(n, offset, fill)
        assert L_.cspn_affinity_atrous2d_bwd_f32(feat.data_ptr(), gate.data_ptr(), out.t.data_ptr(), go.data_ptr(), gf.ptr(),
                                                 gg.ptr(), B, C, H, W, L, r, ws.ptr(), n, st) == 0
        assert L_.cspn_last_launches() == 2
        torch.cuda.synchronize()
        assert ws.guards_intact()
        mc.assert_written(gf, 'grad_feat')
        mc.assert_written(gg, 'grad_gate')
        results.append((mc.words(gf.t).clone(), mc.words(gg.t).clone()))
    assert all(torch.equal(a, b) for a, b in zip(*results))     # no workspace word is read before it is written
    want = _atrous_bwd(feat, gate, out.t, go, rates)
    assert torch.equal(results[0][0], mc.words(want[0])) and torch.equal(results[0][1], mc.words(want[1]))
    assert mc.unchanged(before, [feat, gate, go])


def test_c_abi_refuses_overlapping_device_buffers():
    L_ = _lib.lib()
    buf = torch.zeros(1 << 14, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    r = _c_sizes((2,))                                   # feat 1x2x4x5 = 40 floats, gate 180, out 40, workspace 720 bytes
    assert L_.cspn_affinity_atrous2d_fwd_f32(p, p + 4 * 1000, p + 4 * 20, 1, 2, 4, 5, 1, r, st) == -1
    assert L_.cspn_affinity_atrous2d_fwd_f32(p, p + 4 * 1000, p + 4 * 1100, 1, 2, 4, 5, 1, r, st) == -1
    for gf, gg, ws in ((p + 4 * 2010, p + 4 * 5000, p + 4 * 6000), (p + 4 * 4000, p + 4 * 4030, p + 4 * 6000),
                       (p + 4 * 4000, p + 4 * 5000, p + 4 * 5100)):
        assert L_.cspn_affinity_atrous2d_bwd_f32(p, p + 4 * 1000, p + 4 * 2000, p + 4 * 3000, gf, gg, 1, 2, 4, 5, 1, r, ws, 720,
                                                 st) == -1
    assert L_.cspn_last_launches() == 0 and not buf.any()


# ---- determinism -----------------------------------------------------------------------------------------------------------
def test_bits_do_not_depend_on_the_stream_the_run_or_the_batch():
    rates = (32, 8, 3)
    feat, gate, grad = inputs(12, 4, 40, 37, 70, rates)
    ref = kernel(feat, gate, rates, grad)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = kernel(feat, gate, rates, grad)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(ref, again, kernel(feat, gate, rates, grad)):
        assert torch.equal(mc.words(a), mc.words(b)) and torch.equal(mc.words(a), mc.words(c))
    for half in (slice(0, 1), slice(1, 4)):
        got = kernel(feat[half].contiguous(), gate[half].contiguous(), rates, grad[half].contiguous())
        for a, b in zip(got, ref):
            assert torch.equal(mc.words(a), mc.words(b[half]))


def test_runs_under_deterministic_algorithms():
    rates = (8, 4)
    feat, gate, grad = inputs(15, 2, 8, 21, 30, rates)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)
        out = cspn_b200.affinity_atrous_pool2d(f, g, rates)
        out.backward(grad)
    finally:
        torch.use_deterministic_algorithms(prev)
    want, gf, gg = kernel(feat, gate, rates, grad)
    assert torch.equal(out, want) and torch.equal(f.grad, gf) and torch.equal(g.grad, gg)


def test_cuda_graph_capture_and_replay():
    rates = (16, 4, 4)
    feat, gate, grad = inputs(17, 2, 8, 33, 64, rates)
    f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)

    def step():
        f.grad = g.grad = None
        out = cspn_b200.affinity_atrous_pool2d(f, g, rates)
        out.backward(grad)
        return out

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    f.grad = g.grad = None
    with torch.cuda.graph(graph):
        out = step()
    with torch.no_grad():
        f.copy_(torch.randn_like(f))
        g.copy_(torch.randn_like(g))
    graph.replay()
    torch.cuda.synchronize()
    want, gf, gg = kernel(f.detach(), g.detach(), rates, grad)
    assert torch.equal(out, want) and torch.equal(f.grad, gf) and torch.equal(g.grad, gg)


# ---- torch integration -------------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    rates = (6, 2, 6)
    feat, gate, grad = inputs(20, 2, 6, 19, 21, rates)
    res = []
    for route in (lambda f, g: torch.ops.cspn_b200.affinity_atrous_pool2d(f, g, list(rates)),
                  lambda f, g: _AffinityAtrousFn.apply(f, g, rates)):
        f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)
        out = route(f, g)
        out.backward(grad)
        res.append((out.detach(), f.grad, g.grad))
    assert all(torch.equal(mc.words(x), mc.words(y)) for x, y in zip(*res))


def test_opcheck():
    torch_op.load()
    rates = (4, 3)
    feat, gate, grad = inputs(22, 2, 4, 10, 13, rates)
    torch.library.opcheck(torch.ops.cspn_b200.affinity_atrous_pool2d.default,
                          (feat.requires_grad_(True), gate.requires_grad_(True), list(rates)))
    out = _atrous_fwd(feat.detach(), gate.detach(), rates)
    torch.library.opcheck(torch.ops.cspn_b200.affinity_atrous_pool2d_backward.default,
                          (feat.detach(), gate.detach(), out, grad, list(rates)))


def test_torch_compile_fullgraph_forward_and_backward():
    rates = (8, 4, 3)
    feat, gate, _ = inputs(25, 2, 8, 24, 30, rates)

    def fn(f, g):
        return cspn_b200.affinity_atrous_pool2d(f, g, rates).square().sum()

    res = []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)
        loss = call(f, g)
        loss.backward()
        res.append((loss.detach(), f.grad, g.grad))
    for a, b in zip(*res):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-6)


def test_python_surface_on_the_device():
    feat, gate, _ = inputs(26, 1, 4, 9, 11, (3, 2))
    out = cspn_b200.affinity_atrous_pool2d(feat, gate, [3, 2])
    assert tuple(out.shape) == (1, 8, 9, 11)
    ft = feat.transpose(2, 3).contiguous().transpose(2, 3)    # non-contiguous views are taken
    assert torch.equal(cspn_b200.affinity_atrous_pool2d(ft, gate, (3, 2)), out)
    torch_op.load()
    with pytest.raises(ValueError, match='dilations'):
        torch.ops.cspn_b200.affinity_atrous_pool2d(feat, gate, [3, 12])


# ---- one training tail: gate conv, affinity_atrous_pool2d, grouped 1x1 conv, loss, backward ----------------------------------
def test_training_tail_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(27)
    B, C, H, W, rates = 2, 16, 24, 40, (6, 12, 18)
    L = len(rates)
    feat = torch.randn(B, C, H, W, generator=gen)
    aff = nn.Conv2d(C, 9 * L, 3, padding=1)
    head = nn.Conv2d(L * C, L * 4, 1, groups=L, bias=False)
    with torch.no_grad():
        for m in (aff, head):
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.2)
        aff.bias.zero_()
    target = torch.randn(B, 4 * L, H, W, generator=gen)

    def net(x, a, h, pool):
        y = h(pool(x, a(x)))
        return ((y - target.to(y)) ** 2).mean()

    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                  # fp32 convolutions, not TF32
    try:
        a32, h32 = aff.cuda(), head.cuda()
        x = feat.cuda().requires_grad_(True)
        loss = net(x, a32, h32, lambda f, g: cspn_b200.affinity_atrous_pool2d(f, g, rates))
        loss.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    a64 = nn.Conv2d(C, 9 * L, 3, padding=1).double()
    h64 = nn.Conv2d(L * C, L * 4, 1, groups=L, bias=False).double()
    a64.load_state_dict({k: v.double().cpu() for k, v in a32.state_dict().items()})
    h64.load_state_dict({k: v.double().cpu() for k, v in h32.state_dict().items()})
    x64 = feat.double().requires_grad_(True)
    ref = net(x64, a64, h64, lambda f, g: ar.compose(f, g, rates))
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    for got, want in ((x.grad, x64.grad), (a32.weight.grad, a64.weight.grad), (h32.weight.grad, h64.weight.grad)):
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
