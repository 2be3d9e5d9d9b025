"""GPU tests of the stereo cost volumes (cspn_b200/csrc/cost_volume.cu; DESIGN.md section 4.16): the concatenation forward
bit for bit against the PSMNet loop, everything else bit for bit against the fp32 order restatement and within the
a-priori bounds of fp64, at odd shapes, at both timing shapes and on the smallest-tile fallbacks; the IEEE masks and the
+0.0 zero region, aliasing, the memory contract, determinism, the torch integration and one training tail through
disparity_regression."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _concat_bwd, _concat_fwd, _ConcatVolumeFn, _gwc_bwd, _gwc_fwd, _GwcVolumeFn

import cost_volume_reference as cr
import disparity_reference as dr
import memory_contract as mc

pytestmark = pytest.mark.gpu

# (B, F, H, W, D, G): W a multiple of 4 and not, W = 1, D = 1, D > W, F = 1, G in {1, F/2, F}, several tiles
SHAPES = [
    (2, 8, 5, 16, 6, 4),
    (1, 6, 3, 13, 5, 3),
    (2, 4, 3, 1, 3, 2),
    (1, 8, 4, 20, 1, 8),
    (2, 4, 3, 7, 12, 1),
    (1, 1, 3, 9, 4, 1),
    (1, 16, 2, 300, 48, 8),
    (2, 12, 3, 260, 40, 6),
    (1, 6, 2, 130, 9, 6),
]
# (name, B, F, H, W, D, G): the concatenation volume takes F = 32, the group-wise one F = 320 and G = 40
TIMING = [('training crop', 4, 64, 128, 48), ('KITTI inference', 1, 96, 312, 48)]
# smallest-tile fallbacks: (kind, B, F, H, W, D, G), each runs on 1-column tiles at up to 227 KB of shared memory
FALLBACKS = [('concat_fwd', 1, 1, 1, 7200, 7100, 1), ('gwc_fwd', 1, 320, 2, 160, 150, 1), ('gwc_bwd', 1, 8, 1, 2100, 2000, 4)]


def feats(seed, B, F, H, W, scale=1.0):
    gen = torch.Generator('cuda').manual_seed(seed)
    return (torch.randn(B, F, H, W, device='cuda', generator=gen) * scale,
            torch.randn(B, F, H, W, device='cuda', generator=gen) * scale)


def grad_of(seed, *shape):
    return torch.randn(*shape, device='cuda', generator=torch.Generator('cuda').manual_seed(seed))


def check_all(L, R, D, G, seed=0, fp64=True):
    """Every result of both volumes against its reference: concat forward bit for bit against the loop, the rest bit for
    bit against the fp32 order restatement and within the a-priori bounds of fp64."""
    B, F_, H, W = L.shape
    vol = _concat_fwd(L, R, D)
    assert mc.same_bits(vol, cr.concat_loop(L, R, D)) and torch.equal(mc.words(vol), mc.words(cr.concat_loop(L, R, D)))
    del vol
    gc = grad_of(seed, B, 2 * F_, D, H, W)
    gl, gr = _concat_bwd(gc)
    for got, want in zip((gl, gr), cr.concat_bwd_torch(gc)):
        assert mc.same_bits(got, want)
    if fp64:
        for got, want, bound in zip((gl, gr), cr.concat_bwd_torch(gc.double()), cr.bound_concat_bwd(gc)):
            assert cr.max_ratio(got, want, bound) <= 1.0
    del gc
    vol = _gwc_fwd(L, R, D, G)
    assert mc.same_bits(vol, cr.gwc_fwd_torch(L, R, D, G))
    if fp64:
        assert cr.max_ratio(vol, cr.gwc_loop(L.double(), R.double(), D, G), cr.bound_gwc_fwd(L, R, D, G)) <= 1.0
    torch.testing.assert_close(vol, cr.gwc_loop(L, R, D, G), rtol=1e-5, atol=1e-5)        # the GPU torch loop
    g = grad_of(seed + 1, B, G, D, H, W)
    gl, gr = _gwc_bwd(L, R, g)
    for got, want in zip((gl, gr), cr.gwc_bwd_torch(L, R, g)):
        assert mc.same_bits(got, want)
    if fp64:
        for got, want, bound in zip((gl, gr), cr.gwc_bwd_torch(L.double(), R.double(), g.double()), cr.bound_gwc_bwd(L, R, g)):
            assert cr.max_ratio(got, want, bound) <= 1.0


# ---- exactness ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,F,H,W,D,G', SHAPES)
def test_odd_shapes_bit_for_bit_and_within_the_bounds(B, F, H, W, D, G):
    L, R = feats(B * 7 + W, B, F, H, W)
    check_all(L, R, D, G, seed=W)


@pytest.mark.parametrize('B,F,H,W,D,G', SHAPES[:3])
def test_gradients_are_fp64_autograd_of_the_loops(B, F, H, W, D, G):
    L, R = feats(3, B, F, H, W)
    for build, gshape, fn in ((cr.concat_loop, (B, 2 * F, D, H, W), lambda a, b: cspn_b200.build_concat_volume(a, b, D)),
                              (cr.gwc_loop, (B, G, D, H, W), lambda a, b: cspn_b200.build_gwc_volume(a, b, D, G))):
        g = grad_of(4, *gshape)
        Ld, Rd = L.double().requires_grad_(True), R.double().requires_grad_(True)
        (build(Ld, Rd, D) if build is cr.concat_loop else build(Ld, Rd, D, G)).backward(g.double())
        Lf, Rf = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
        fn(Lf, Rf).backward(g)
        for got, want in ((Lf.grad, Ld.grad), (Rf.grad, Rd.grad)):
            torch.testing.assert_close(got.double(), want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('name,B,H,W,D', TIMING)
def test_timing_shapes(name, B, H, W, D):
    L, R = feats(11, B, 320, H, W)
    check_all(L[:, :32].contiguous(), R[:, :32].contiguous(), D, 1, seed=1)
    check_all(L, R, D, 40, seed=2)
    torch.cuda.empty_cache()


@pytest.mark.parametrize('kind,B,F,H,W,D,G', FALLBACKS)
def test_smallest_tile_fallbacks(kind, B, F, H, W, D, G):
    tx, _, smem = cr.plan(kind, W, D, F // G)
    assert tx == 1 and cr.SMEM_SOFT < smem <= cr.SMEM_HARD
    L, R = feats(D, B, F, H, W)
    if kind == 'concat_fwd':
        vol = _concat_fwd(L, R, D)
        assert torch.equal(mc.words(vol), mc.words(cr.concat_loop(L, R, D)))
    elif kind == 'gwc_fwd':
        vol = _gwc_fwd(L, R, D, G)
        assert mc.same_bits(vol, cr.gwc_fwd_torch(L, R, D, G))
        assert cr.max_ratio(vol, cr.gwc_loop(L.double(), R.double(), D, G), cr.bound_gwc_fwd(L, R, D, G)) <= 1.0
    else:
        g = grad_of(5, B, G, D, H, W)
        gl, gr = _gwc_bwd(L, R, g)
        for got, want in zip((gl, gr), cr.gwc_bwd_torch(L, R, g)):
            assert mc.same_bits(got, want)
    torch.cuda.empty_cache()


# ---- IEEE --------------------------------------------------------------------------------------------------------------------
def test_concat_forward_keeps_every_bit():
    L, R = feats(1, 2, 3, 4, 12)
    nan_payload = torch.tensor([0x7FC01234, 0x7F800001, -0x00400001], dtype=torch.int32, device='cuda').view(torch.float32)
    L[0, 1, 2, 3:6] = nan_payload
    R[1, 2, 0, 7:10] = nan_payload
    L[1, 0, 1, 5] = -0.0
    R[0, 0, 3, 0] = -0.0
    R[0, 2, 1, 11] = float('-inf')
    for D in (1, 5, 12, 15):
        vol = _concat_fwd(L, R, D)
        assert torch.equal(mc.words(vol), mc.words(cr.concat_loop(L, R, D)))


@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf'), 0.0])
def test_non_finite_features_give_the_masks_of_the_fp64_loops(value):
    B, F_, H, W, D, G = 1, 8, 3, 20, 7, 2
    L, R = feats(2, B, F_, H, W)
    L[0, 1, 1, 4] = value
    R[0, 6, 2, 9] = value
    L[0, 3, 0, 12] = float('inf')                # against a 0 on the other side: 0 * inf in the computed region only
    R[0, 3, 0, 12 - 3] = 0.0
    R[0, 5, 2, 0] = float('nan')
    for build, loop, gshape, args in ((_concat_fwd, cr.concat_loop, (B, 2 * F_, D, H, W), (D,)),
                                      (_gwc_fwd, cr.gwc_loop, (B, G, D, H, W), (D, G))):
        vol = build(L, R, *args)
        Ld, Rd = L.double().requires_grad_(True), R.double().requires_grad_(True)
        want = loop(Ld, Rd, *args)
        assert torch.equal(torch.isnan(vol), torch.isnan(want)) and torch.equal(torch.isinf(vol), torch.isinf(want))
        assert torch.equal(vol[torch.isinf(vol)], want[torch.isinf(want)].float())
        g = grad_of(3, *gshape)
        want.backward(g.double())
        got = _concat_bwd(g) if build is _concat_fwd else _gwc_bwd(L, R, g)
        for a, b in zip(got, (Ld.grad, Rd.grad)):
            assert torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.isinf(a), torch.isinf(b))
            assert torch.equal(a[torch.isinf(a)], b[torch.isinf(b)].float())


def test_the_zero_region_is_positive_zero_under_nan_inputs():
    L = torch.full((2, 4, 3, 9), float('nan'), device='cuda')
    for D in (4, 9, 13):
        x = torch.arange(9, device='cuda')
        d = torch.arange(D, device='cuda')[:, None]
        zero = (x < d)[None, None, :, None, :].expand(2, -1, D, 3, 9)
        for vol in (_concat_fwd(L, L, D), _gwc_fwd(L, L, D, 2)):
            z = zero.expand(2, vol.shape[1], D, 3, 9)
            assert (mc.words(vol)[z] == 0).all() and torch.isnan(vol[~z]).all()


# ---- aliasing and the memory contract ------------------------------------------------------------------------------------------
def test_left_may_be_right():
    X = feats(5, 2, 8, 3, 17)[0]
    for build, gshape in ((lambda a, b: cspn_b200.build_concat_volume(a, b, 6), (2, 16, 6, 3, 17)),
                          (lambda a, b: cspn_b200.build_gwc_volume(a, b, 6, 4), (2, 4, 6, 3, 17))):
        g = grad_of(6, *gshape)
        x = X.clone().requires_grad_(True)
        vol = build(x, x)
        vol.backward(g)
        a, b = X.clone().requires_grad_(True), X.clone().requires_grad_(True)
        ref = build(a, b)
        ref.backward(g)
        assert torch.equal(vol, ref) and torch.equal(x.grad, a.grad + b.grad)


@pytest.mark.parametrize('B,F,H,W,D,G', [(2, 8, 3, 16, 5, 4), (1, 6, 2, 13, 20, 3), (2, 4, 3, 131, 9, 1)])
def test_launch_counts_and_memory_contract(B, F, H, W, D, G):
    L_ = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    L, R = feats(7, B, F, H, W)
    gc, g = grad_of(8, B, 2 * F, D, H, W), grad_of(9, B, G, D, H, W)
    before = mc.snapshot([L, R, gc, g])
    for offset in (0, 4):                          # 4: the concat forward's scalar stores
        out = mc.guarded((B, 2 * F, D, H, W), offset)
        assert L_.cspn_concat_volume_fwd_f32(L.data_ptr(), R.data_ptr(), out.ptr(), B, F, H, W, D, st) == 0
        assert L_.cspn_last_launches() == 1
        torch.cuda.synchronize()
        mc.assert_written(out, 'concat out')
        assert torch.equal(mc.words(out.t), mc.words(_concat_fwd(L, R, D)))
    gl, gr = mc.guarded((B, F, H, W), 4), mc.guarded((B, F, H, W), 4)
    assert L_.cspn_concat_volume_bwd_f32(gc.data_ptr(), gl.ptr(), gr.ptr(), B, F, H, W, D, st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(gl, 'concat grad_left')
    mc.assert_written(gr, 'concat grad_right')
    out = mc.guarded((B, G, D, H, W), 4)
    assert L_.cspn_gwc_volume_fwd_f32(L.data_ptr(), R.data_ptr(), out.ptr(), B, F, H, W, D, G, st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(out, 'gwc out')
    gl, gr = mc.guarded((B, F, H, W), 4), mc.guarded((B, F, H, W), 4)
    assert L_.cspn_gwc_volume_bwd_f32(L.data_ptr(), R.data_ptr(), g.data_ptr(), gl.ptr(), gr.ptr(), B, F, H, W, D, G, st) == 0
    assert L_.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(gl, 'gwc grad_left')
    mc.assert_written(gr, 'gwc grad_right')
    assert torch.equal(gl.t, _gwc_bwd(L, R, g)[0]) and torch.equal(gr.t, _gwc_bwd(L, R, g)[1])
    assert mc.unchanged(before, [L, R, gc, g])


def test_c_abi_refuses_overlapping_device_buffers():
    L_ = _lib.lib()
    buf = torch.zeros(1 << 14, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    p = buf.data_ptr()
    # features 1x4x2x5 = 40 floats, the concat volume (D = 3) 240
    assert L_.cspn_concat_volume_fwd_f32(p, p + 4 * 1000, p + 4 * 20, 1, 4, 2, 5, 3, st) == -1
    assert L_.cspn_gwc_volume_fwd_f32(p, p + 4 * 1000, p + 4 * 1020, 1, 4, 2, 5, 3, 2, st) == -1
    assert L_.cspn_gwc_volume_bwd_f32(p, p + 4 * 1000, p + 4 * 2000, p + 4 * 3000, p + 4 * 3020, 1, 4, 2, 5, 3, 2, st) == -1
    assert L_.cspn_last_launches() == 0 and not buf.any()


# ---- determinism -----------------------------------------------------------------------------------------------------------
def run_all(L, R, gc, g, D, G):
    return (_concat_fwd(L, R, D), *_concat_bwd(gc), _gwc_fwd(L, R, D, G), *_gwc_bwd(L, R, g))


def test_bits_do_not_depend_on_the_stream_the_run_or_the_batch():
    B, F_, H, W, D, G = 4, 16, 5, 140, 24, 4
    L, R = feats(12, B, F_, H, W)
    gc, g = grad_of(13, B, 2 * F_, D, H, W), grad_of(14, B, G, D, H, W)
    ref = run_all(L, R, gc, g, D, G)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        again = run_all(L, R, gc, g, D, G)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b, c in zip(ref, again, run_all(L, R, gc, g, D, G)):
        assert torch.equal(mc.words(a), mc.words(b)) and torch.equal(mc.words(a), mc.words(c))
    for half in (slice(0, 2), slice(2, 4)):
        for a, b in zip(run_all(L[half], R[half], gc[half], g[half], D, G), ref):
            assert torch.equal(mc.words(a), mc.words(b[half]))


def test_runs_under_deterministic_algorithms():
    L, R = feats(15, 2, 8, 3, 30)
    g = grad_of(16, 2, 4, 10, 3, 30)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a, b = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
        vol = cspn_b200.build_gwc_volume(a, b, 10, 4)
        vol.backward(g)
        c = cspn_b200.build_concat_volume(L, R, 10)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(vol, _gwc_fwd(L, R, 10, 4)) and torch.equal(c, _concat_fwd(L, R, 10))
    gl, gr = _gwc_bwd(L, R, g)
    assert torch.equal(a.grad, gl) and torch.equal(b.grad, gr)


def test_cuda_graph_capture_and_replay():
    L, R = feats(17, 2, 8, 4, 64)
    a, b = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
    gc, g = grad_of(18, 2, 16, 12, 4, 64), grad_of(19, 2, 2, 12, 4, 64)

    def step():
        a.grad = b.grad = None
        c = cspn_b200.build_concat_volume(a, b, 12)
        v = cspn_b200.build_gwc_volume(a, b, 12, 2)
        torch.autograd.backward([c, v], [gc, g])
        return c, v

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    a.grad = b.grad = None
    with torch.cuda.graph(graph):
        c, v = step()
    with torch.no_grad():
        a.copy_(torch.randn_like(a))
        b.copy_(torch.randn_like(b))
    graph.replay()
    torch.cuda.synchronize()
    La, Rb = a.detach(), b.detach()
    assert torch.equal(c, _concat_fwd(La, Rb, 12)) and torch.equal(v, _gwc_fwd(La, Rb, 12, 2))
    cl, cr_ = _concat_bwd(gc)
    wl, wr = _gwc_bwd(La, Rb, g)
    assert torch.equal(a.grad, cl + wl) and torch.equal(b.grad, cr_ + wr)


# ---- torch integration -------------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    L, R = feats(20, 2, 6, 3, 21)
    for op, fn, args, gshape in ((torch.ops.cspn_b200.concat_volume, _ConcatVolumeFn.apply, (7,), (2, 12, 7, 3, 21)),
                                 (torch.ops.cspn_b200.gwc_volume, _GwcVolumeFn.apply, (7, 3), (2, 3, 7, 3, 21))):
        g = grad_of(21, *gshape)
        res = []
        for route in (op, fn):
            a, b = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
            vol = route(a, b, *args)
            vol.backward(g)
            res.append((vol.detach(), a.grad, b.grad))
        assert all(torch.equal(x, y) for x, y in zip(*res))


def test_opcheck():
    torch_op.load()
    L, R = feats(22, 2, 4, 3, 10)
    a, b = L.requires_grad_(True), R.requires_grad_(True)
    torch.library.opcheck(torch.ops.cspn_b200.concat_volume.default, (a, b, 4))
    torch.library.opcheck(torch.ops.cspn_b200.gwc_volume.default, (a, b, 4, 2))
    torch.library.opcheck(torch.ops.cspn_b200.concat_volume_backward.default, (grad_of(23, 2, 8, 4, 3, 10),))
    torch.library.opcheck(torch.ops.cspn_b200.gwc_volume_backward.default, (L.detach(), R.detach(), grad_of(24, 2, 2, 4, 3, 10)))


def test_torch_compile_fullgraph_forward_and_backward():
    L, R = feats(25, 2, 8, 3, 24)

    def fn(a, b):
        return (cspn_b200.build_gwc_volume(a, b, 6, 4).square().sum() + cspn_b200.build_concat_volume(a, b, 6).sum())

    res = []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        a, b = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
        loss = call(a, b)
        loss.backward()
        res.append((loss.detach(), a.grad, b.grad))
    for a, b in zip(*res):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-6)


def test_python_surface_on_the_device():
    L, R = feats(26, 1, 4, 2, 9)
    assert cspn_b200.build_concat_volume(L, R, 3).shape == (1, 8, 3, 2, 9)
    assert cspn_b200.build_gwc_volume(L, R, 3, 4).shape == (1, 4, 3, 2, 9)
    # non-contiguous views are taken
    Lt, Rt = L.transpose(2, 3).contiguous().transpose(2, 3), R.transpose(2, 3).contiguous().transpose(2, 3)
    assert torch.equal(cspn_b200.build_gwc_volume(Lt, Rt, 3, 2), _gwc_fwd(L, R, 3, 2))
    torch_op.load()
    with pytest.raises(RuntimeError, match='2\\^31'):
        torch.ops.cspn_b200.concat_volume(L, R, 1 << 28)
    with pytest.raises(RuntimeError, match='shared memory'):
        big = torch.zeros(1, 320, 1, 300, device='cuda')
        torch.ops.cspn_b200.gwc_volume(big, big, 250, 1)


# ---- one training tail: gwc volume, a 3D convolution, disparity regression, smooth L1, backward ------------------------------
def test_training_tail_matches_fp64_autograd():
    gen = torch.Generator().manual_seed(27)
    B, F_, G, H, W, D = 2, 16, 4, 8, 24, 6
    left, right = torch.randn(B, F_, H, W, generator=gen), torch.randn(B, F_, H, W, generator=gen)
    conv = nn.Conv3d(G, 1, 3, padding=1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * 0.3)
        conv.bias.zero_()
    size = (4 * D, 4 * H, 4 * W)
    target = torch.rand(B, 1, *size[1:], generator=gen) * size[0]
    mask = target > 2

    def loss_of(y):
        m = mask.to(y.device)
        return F.smooth_l1_loss(y[m], target.to(y)[m])

    conv32 = conv.cuda()
    lc, rc = left.cuda().requires_grad_(True), right.cuda().requires_grad_(True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False         # an fp32 convolution, not TF32
    try:
        loss = loss_of(cspn_b200.disparity_regression(conv32(cspn_b200.build_gwc_volume(lc, rc, D, G)), size))
        loss.backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    conv64 = nn.Conv3d(G, 1, 3, padding=1).double()
    conv64.load_state_dict({k: v.double().cpu() for k, v in conv32.state_dict().items()})
    ld, rd = left.double().requires_grad_(True), right.double().requires_grad_(True)
    ref = loss_of(dr.forward_torch(conv64(cr.gwc_loop(ld, rd, D, G)), size))
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref))
    for got, want in ((lc.grad, ld.grad), (rc.grad, rd.grad)):
        err = float((got.cpu().double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-3, err
