"""GPU tests of affinity pooling (cspn_b200/csrc/affinity_pool.cu; DESIGN.md section 4.17): the forward and both gradients
bit for bit against the fp32 order restatement and within the a-priori bounds of fp64 autograd, at odd shapes and the three
timing shapes; the IEEE masks case by case, the +0.0 gradients outside the windows, each level of a pyramid against that
level alone, the memory contract, determinism, both routes, the torch integration and one training tail."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _AffinityPoolFn, _c_sizes, _pool_bwd, _pool_fwd

import affinity_pool_reference as ar
import memory_contract as mc

pytestmark = pytest.mark.gpu

# (B, C, H, W, ks): H, W multiples of no p, p = 1, p = min(H, W), repeated and unordered sizes, L = 1 and L = 8, windows
# taller than a CTA (p > 128: the forward's and the backward's row chunks), C past a channel chunk, odd C
SHAPES = [
    (2, 3, 13, 19, (2, 3, 5)),
    (1, 5, 7, 7, (7, 1)),
    (2, 2, 11, 30, (4, 4, 1, 11)),
    (1, 4, 9, 10, (1, 2, 3, 4, 5, 6, 7, 8)),
    (3, 17, 33, 47, (16, 8, 3)),
    (1, 1, 6, 5, (5,)),
    (1, 2, 300, 301, (300, 150, 129)),
    (2, 37, 70, 131, (64, 33, 2)),
]
# (name, B, H, W): C = 128, p = (64, 32, 16, 8), PSMNet's quarter-resolution feature map
TIMING = [('training crop', 4, 64, 128), ('KITTI inference', 1, 96, 312), ('SceneFlow test', 1, 136, 240)]
KS = (64, 32, 16, 8)


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, device='cuda', generator=torch.Generator('cuda').manual_seed(seed)) * scale


def inputs(seed, B, C, H, W, ks):
    return (rnd(seed, B, C, H, W), rnd(seed + 1, B, len(ks), H, W),
            tuple(rnd(seed + 2 + l, B, C, H // p, W // p) for l, p in enumerate(ks)))


def kernel(feat, gate, ks, grads):
    """levels, grad_feat, grad_gate through the C ABI (the ctypes route, no autograd)."""
    B, C, H, W = feat.shape
    flat = _pool_fwd(feat, gate, ks)
    gf, gg = _pool_bwd(feat, gate, flat, ar.pack(grads), ks)
    return ar.unpack(flat, B, C, H, W, ks), gf, gg


def autograd64(feat, gate, ks, grads):
    f, g = feat.detach().double().requires_grad_(True), gate.detach().double().requires_grad_(True)
    outs = ar.compose(f, g, ks)
    torch.autograd.backward(outs, [t.double() for t in grads])
    return tuple(o.detach() for o in outs), f.grad, g.grad


def check_all(feat, gate, ks, grads):
    outs, gf, gg = kernel(feat, gate, ks, grads)
    want = ar.fwd_torch(feat, gate, ks)
    for got, w in zip(outs, want):
        assert mc.same_bits(got, w)
    for got, w in zip((gf, gg), ar.bwd_torch(feat, gate, ks, want, grads)):
        assert mc.same_bits(got, w)
    o64, gf64, gg64 = autograd64(feat, gate, ks, grads)
    for got, w, bound in zip(outs, o64, ar.bound_fwd(feat, gate, ks)):
        assert ar.max_ratio(got, w, bound) <= 1.0
    for got, w, bound in zip((gf, gg), (gf64, gg64), ar.bound_bwd(feat, gate, ks, grads)):
        assert ar.max_ratio(got, w, bound) <= 1.0


# ---- exactness ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,ks', SHAPES)
def test_odd_shapes_bit_for_bit_and_within_the_bounds(B, C, H, W, ks):
    feat, gate, grads = inputs(B * 7 + W, B, C, H, W, ks)
    check_all(feat, gate, ks, grads)


@pytest.mark.parametrize('name,B,H,W', TIMING)
def test_timing_shapes(name, B, H, W):
    feat, gate, grads = inputs(11, B, 128, H, W, KS)
    check_all(feat, gate, KS, grads)
    torch.cuda.empty_cache()


def test_anchors_on_the_device():
    """A constant gate is avg_pool2d within the bound; a one-hot gate copies its pixel bit for bit."""
    feat = rnd(1, 2, 6, 29, 35)
    ks = (8, 4, 3, 1)
    outs = cspn_b200.affinity_pool2d(feat, torch.full((2, 4, 29, 35), 0.3, device='cuda'), ks)
    for got, p, bound in zip(outs, ks, ar.bound_fwd(feat, torch.full((2, 4, 29, 35), 0.3, device='cuda'), ks)):
        assert ar.max_ratio(got, F.avg_pool2d(feat.double(), p), bound) <= 1.0
    p = 5
    gate = torch.zeros(2, 1, 29, 35, device='cuda')
    gate[:, :, 2::p, 4::p] = -1.7                             # row 2, column 4 of every window
    out, = cspn_b200.affinity_pool2d(feat, gate, (p,))
    assert torch.equal(mc.words(out), mc.words(feat[:, :, 2:25:p, 4:35:p].contiguous()))


def test_each_level_is_the_level_alone():
    feat, gate, grads = inputs(2, 2, 9, 45, 38, (12, 5, 5, 1, 38))
    ks = (12, 5, 5, 1, 38)
    outs, gf, gg = kernel(feat, gate, ks, grads)
    for l, p in enumerate(ks):
        alone, = ar.unpack(_pool_fwd(feat, gate[:, l:l + 1].contiguous(), (p,)), 2, 9, 45, 38, (p,))
        assert torch.equal(mc.words(alone), mc.words(outs[l]))


# ---- IEEE --------------------------------------------------------------------------------------------------------------------
IEEE = ['zero_window', 'neg_zero_window', 'inf_gate', 'neg_inf_gate', 'nan_gate', 'nan_feat', 'inf_feat', 'zero_times_inf',
        'neg_zero_gates', 'subnormal_sums']


def masks_equal(got, want):
    return (torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(torch.isinf(got), torch.isinf(want))
            and torch.equal(got[torch.isinf(got)], want[torch.isinf(want)].float()))


@pytest.mark.parametrize('case', IEEE)
def test_ieee_masks_of_fp64_autograd(case):
    B, C, H, W, ks = 1, 4, 13, 18, (4, 3, 2)
    feat, gate, grads = inputs(3, B, C, H, W, ks)
    if case == 'zero_window':
        gate[0, 0, 4:8, 8:12] = 0.0
    elif case == 'neg_zero_window':
        gate[0, 1, 3:6, 6:9] = -0.0
    elif case == 'inf_gate':
        gate[0, 1, 5, 7] = float('inf')
    elif case == 'neg_inf_gate':
        gate[0, 0, 2, 9] = float('-inf')
    elif case == 'nan_gate':
        gate[0, 2, 3, 3] = float('nan')
    elif case == 'nan_feat':
        feat[0, 1, 6, 9] = float('nan')
    elif case == 'inf_feat':
        feat[0, 2, 2, 5] = float('inf')
        feat[0, 0, 7, 1] = float('-inf')
    elif case == 'zero_times_inf':
        feat[0, 0, 9, 10] = float('inf')
        gate[0, :, 9, 10] = 0.0
    elif case == 'neg_zero_gates':
        gate[0, :, ::2, 1::3] = -0.0
    else:                                                     # the windows' sums are subnormal: no flush to zero
        gate[0, 0, 4:8, 0:4] = torch.randint(1, 9, (4, 4), device='cuda').float() * 1.4e-45
        gate[0, 2, 0:2, 2:4] = 3e-45
        grads = tuple(g * 1e-30 for g in grads)
    outs, gf, gg = kernel(feat, gate, ks, grads)
    o64, gf64, gg64 = autograd64(feat, gate, ks, grads)
    for got, want in zip((*outs, gf, gg), (*o64, gf64, gg64)):
        assert masks_equal(got, want)
    want = ar.fwd_torch(feat, gate, ks)
    for got, w in zip((*outs, gf, gg), (*want, *ar.bwd_torch(feat, gate, ks, want, grads))):
        assert mc.same_bits(got, w)
    if case in ('zero_window', 'neg_zero_window', 'inf_gate', 'nan_gate'):
        assert torch.isnan(torch.cat([o.reshape(-1) for o in outs])).any()


def test_uncovered_pixels_get_positive_zero_gradients():
    """Pixels outside every level's windows get grad_feat +0.0, pixels outside level l's windows grad_gate_l +0.0, whatever
    feat and gate hold there."""
    B, C, H, W, ks = 2, 3, 11, 14, (4, 3)                    # rows 9.., columns 12.. in no window of either level
    feat, gate, grads = inputs(5, B, C, H, W, ks)
    feat[:, :, 9:, :] = float('nan')
    feat[:, :, :, 12:] = float('inf')
    gate[:, :, 9:, :] = float('nan')
    gate[:, :, :, 12:] = float('-inf')
    _, gf, gg = kernel(feat, gate, ks, grads)
    assert (mc.words(gf[:, :, 9:]) == 0).all() and (mc.words(gf[:, :, :, 12:]) == 0).all()
    for l, p in enumerate(ks):
        out_of = torch.ones(H, W, dtype=torch.bool, device='cuda')
        out_of[:(H // p) * p, :(W // p) * p] = False
        assert (mc.words(gg[:, l])[:, out_of] == 0).all()
        assert torch.isfinite(gg[:, l][:, ~out_of]).all()


# ---- the memory contract -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,ks', [(2, 5, 13, 19, (2, 3, 13)), (1, 33, 40, 37, (16, 1)), (2, 3, 150, 140, (140,))])
def test_launch_counts_and_memory_contract(B, C, H, W, ks):
    L_ = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    feat, gate, grads = inputs(7, B, C, H, W, ks)
    n = B * C * sum((H // p) * (W // p) for p in ks)
    go = ar.pack(grads)
    before = mc.snapshot([feat, gate, go])
    out = mc.guarded((n,), 4)
    assert L_.cspn_affinity_pool2d_fwd_f32(feat.data_ptr(), gate.data_ptr(), out.ptr(), B, C, H, W, len(ks), _c_sizes(ks),
                                           st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert torch.equal(mc.words(out.t), mc.words(_pool_fwd(feat, gate, ks)))
    gf, gg = mc.guarded((B, C, H, W), 4), mc.guarded((B, len(ks), H, W), 4)
    assert L_.cspn_affinity_pool2d_bwd_f32(feat.data_ptr(), gate.data_ptr(), out.t.data_ptr(), go.data_ptr(), gf.ptr(), gg.ptr(),
                                           B, C, H, W, len(ks), _c_sizes(ks), st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(gf, 'grad_feat')
    mc.assert_written(gg, 'grad_gate')
    want = _pool_bwd(feat, gate, out.t, go, ks)
    assert torch.equal(mc.words(gf.t), mc.words(want[0])) and torch.equal(mc.words(gg.t), mc.words(want[1]))
    assert mc.unchanged(before, [feat, gate, go])


def test_c_abi_refuses_overlapping_device_buffers():
    L_ = _lib.lib()
    buf = torch.zeros(1 << 14, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    ks = _c_sizes((2, 3))                                     # feat 1x2x4x5 = 40 floats, gate 40, out 10
    assert L_.cspn_affinity_pool2d_fwd_f32(p, p + 4 * 1000, p + 4 * 20, 1, 2, 4, 5, 2, ks, st) == -1
    assert L_.cspn_affinity_pool2d_bwd_f32(p, p + 4 * 1000, p + 4 * 2000, p + 4 * 3000, p + 4 * 4000, p + 4 * 4030, 1, 2, 4, 5,
                                           2, ks, st) == -1
    assert L_.cspn_last_launches() == 0 and not buf.any()


# ---- determinism -----------------------------------------------------------------------------------------------------------
def run_all(feat, gate, ks, grads):
    outs, gf, gg = kernel(feat, gate, ks, grads)
    return (*outs, gf, gg)


def test_bits_do_not_depend_on_the_stream_the_run_or_the_batch():
    B, C, H, W, ks = 4, 40, 37, 70, (32, 8, 3)
    feat, gate, grads = inputs(12, B, C, H, W, ks)
    ref = run_all(feat, gate, ks, grads)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = run_all(feat, gate, ks, grads)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(ref, again, run_all(feat, gate, ks, grads)):
        assert torch.equal(mc.words(a), mc.words(b)) and torch.equal(mc.words(a), mc.words(c))
    for half in (slice(0, 2), slice(2, 4)):
        got = run_all(feat[half].contiguous(), gate[half].contiguous(), ks, tuple(g[half].contiguous() for g in grads))
        for a, b in zip(got, ref):
            assert torch.equal(mc.words(a), mc.words(b[half]))


def test_runs_under_deterministic_algorithms():
    feat, gate, grads = inputs(15, 2, 8, 21, 30, (8, 4))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)
        outs = cspn_b200.affinity_pool2d(f, g, (8, 4))
        torch.autograd.backward(outs, list(grads))
    finally:
        torch.use_deterministic_algorithms(prev)
    want, gf, gg = kernel(feat, gate, (8, 4), grads)
    assert all(torch.equal(a, b) for a, b in zip(outs, want))
    assert torch.equal(f.grad, gf) and torch.equal(g.grad, gg)


def test_cuda_graph_capture_and_replay():
    ks = (16, 4, 4)
    feat, gate, grads = inputs(17, 2, 8, 33, 64, ks)
    f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)

    def step():
        f.grad = g.grad = None
        outs = cspn_b200.affinity_pool2d(f, g, ks)
        torch.autograd.backward(outs, list(grads))
        return outs

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    f.grad = g.grad = None
    with torch.cuda.graph(graph):
        outs = step()
    with torch.no_grad():
        f.copy_(torch.randn_like(f))
        g.copy_(torch.randn_like(g))
    graph.replay()
    torch.cuda.synchronize()
    want, gf, gg = kernel(f.detach(), g.detach(), ks, grads)
    assert all(torch.equal(a, b) for a, b in zip(outs, want))
    assert torch.equal(f.grad, gf) and torch.equal(g.grad, gg)


# ---- torch integration -------------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    ks = (6, 2, 6)
    feat, gate, grads = inputs(20, 2, 6, 19, 21, ks)
    go = ar.pack(grads)
    res = []
    for route in (lambda f, g: torch.ops.cspn_b200.affinity_pool2d(f, g, list(ks)), lambda f, g: _AffinityPoolFn.apply(f, g, ks)):
        f, g = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)
        flat = route(f, g)
        flat.backward(go)
        res.append((flat.detach(), f.grad, g.grad))
    assert all(torch.equal(mc.words(x), mc.words(y)) for x, y in zip(*res))


def test_opcheck():
    torch_op.load()
    feat, gate, grads = inputs(22, 2, 4, 10, 13, (4, 3))
    torch.library.opcheck(torch.ops.cspn_b200.affinity_pool2d.default,
                          (feat.requires_grad_(True), gate.requires_grad_(True), [4, 3]))
    flat = _pool_fwd(feat.detach(), gate.detach(), (4, 3))
    torch.library.opcheck(torch.ops.cspn_b200.affinity_pool2d_backward.default,
                          (feat.detach(), gate.detach(), flat, ar.pack(grads), [4, 3]))


def test_torch_compile_fullgraph_forward_and_backward():
    feat, gate, _ = inputs(25, 2, 8, 24, 30, (8, 4, 3))

    def fn(f, g):
        return sum(o.square().sum() for o in cspn_b200.affinity_pool2d(f, g, (8, 4, 3)))

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
    outs = cspn_b200.affinity_pool2d(feat, gate, [3, 2])
    assert [tuple(o.shape) for o in outs] == [(1, 4, 3, 3), (1, 4, 4, 5)]
    ft = feat.transpose(2, 3).contiguous().transpose(2, 3)    # non-contiguous views are taken
    assert all(torch.equal(a, b) for a, b in zip(cspn_b200.affinity_pool2d(ft, gate, (3, 2)), outs))
    torch_op.load()
    with pytest.raises(ValueError, match='kernel sizes'):
        torch.ops.cspn_b200.affinity_pool2d(feat, gate, [3, 10])


# ---- one training tail: affinity conv, affinity_pool2d, 1x1 conv, bilinear upsample, loss, backward ---------------------------
def test_training_tail_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(27)
    B, C, H, W, ks = 2, 16, 24, 40, (8, 4, 2)
    feat = torch.randn(B, C, H, W, generator=gen)
    aff = nn.Conv2d(C, len(ks), 3, padding=1)
    head = nn.Conv2d(C, 4, 1, bias=False)
    with torch.no_grad():
        for m in (aff, head):
            m.weight.copy_(torch.randn(m.weight.shape, generator=gen) * 0.2)
        aff.bias.zero_()
    target = torch.randn(B, 4 * len(ks), H, W, generator=gen)

    def net(x, a, h, pool):
        outs = pool(x, a(x))
        y = torch.cat([F.interpolate(h(o), size=(H, W), mode='bilinear', align_corners=False) for o in outs], 1)
        return ((y - target.to(y)) ** 2).mean()

    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                  # fp32 convolutions, not TF32
    try:
        a32, h32 = aff.cuda(), head.cuda()
        x = feat.cuda().requires_grad_(True)
        loss = net(x, a32, h32, lambda f, g: cspn_b200.affinity_pool2d(f, g, ks))
        loss.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    a64, h64 = nn.Conv2d(C, len(ks), 3, padding=1).double(), nn.Conv2d(C, 4, 1, bias=False).double()
    a64.load_state_dict({k: v.double().cpu() for k, v in a32.state_dict().items()})
    h64.load_state_dict({k: v.double().cpu() for k, v in h32.state_dict().items()})
    x64 = feat.double().requires_grad_(True)
    ref = net(x64, a64, h64, lambda f, g: ar.compose(f, g, ks))
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    for got, want in ((x.grad, x64.grad), (a32.weight.grad, a64.weight.grad), (h32.weight.grad, h64.weight.grad)):
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
