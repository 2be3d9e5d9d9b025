"""GPU tests of the guidance / depth head kernels (cspn_b200/csrc/unpool_conv.cu): forward accuracy against fp64 within the
a-priori bound, the IEEE footprint of the op sequence, determinism, the backward against fp64 autograd, launch counts and
the memory contract, the torch integration, and the reference model's heads (tests/golden/model/nyu_resnet50_heads.npz)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import cspn_b200
from cspn_b200 import _lib, torch_op
from cspn_b200.cspn import _UnpoolConv3x3Fn, _unpool_conv_fwd
from oracle import cspn_numpy as onp
from oracle import cspn_torch_port as tp

import memory_contract as mc
import unpool_conv_reference as ur

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model')


def gamma(n):
    return n * U / (1 - n * U)


def inputs(seed, B, Cin, h, w, Cout, offset=0):
    """x and weight on the GPU; offset > 0 puts both `offset` floats past a 16-byte boundary."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, h, w, generator=g)
    wt = torch.randn(Cout, Cin, 3, 3, generator=g) / 8
    if not offset:
        return x.cuda(), wt.cuda()
    bx = torch.empty(x.numel() + offset, device='cuda')[offset:].view(x.shape)
    bw = torch.empty(wt.numel() + offset, device='cuda')[offset:].view(wt.shape)
    bx.copy_(x)
    bw.copy_(wt)
    assert bx.data_ptr() % 16 == 4 * offset
    return bx, bw


def exact(x, wt, H, W):
    return ur.op_sequence(x.double(), wt.double(), H, W)


def fwd_bound(x, wt, H, W):
    return gamma(4 * x.shape[1]) * ur.op_sequence(x.double().abs(), wt.double().abs(), H, W)


# ---- forward accuracy --------------------------------------------------------------------------------------------------
FWD_CASES = [
    (1, 64, 114, 152, 8, 228, 304, 0),       # NYU guidance head
    (1, 64, 114, 152, 1, 228, 304, 0),       # NYU depth head
    (1, 64, 176, 608, 8, 352, 1216, 0),      # KITTI guidance head
    (2, 64, 176, 608, 1, 352, 1216, 0),      # KITTI depth head
    (2, 64, 40, 52, 24, 80, 104, 0),         # 5x5 guidance
    (1, 64, 40, 52, 48, 79, 103, 0),         # 7x7 guidance, odd crop
    (4, 3, 17, 23, 8, 33, 45, 0),            # H = 2h-1, odd W, B = 4
    (3, 1, 9, 11, 1, 17, 22, 0),             # Cin = 1
    (2, 65, 13, 37, 5, 26, 73, 0),           # Cin = 65 (a partial channel chunk), Cout = 5
    (1, 3, 1, 1, 2, 1, 1, 0),                # 1x1 output
    (1, 2, 3, 2, 3, 5, 3, 0),                # tiny, both odd
    (2, 64, 20, 40, 8, 39, 77, 1),           # pointers 4 bytes past 16-byte alignment
    (2, 65, 20, 40, 3, 40, 80, 1),
]


@pytest.mark.parametrize('B,Cin,h,w,Cout,H,W,offset', FWD_CASES)
def test_forward_within_the_a_priori_bound(B, Cin, h, w, Cout, H, W, offset):
    x, wt = inputs(B * 100 + Cin + Cout, B, Cin, h, w, Cout, offset)
    out = cspn_b200.unpool_conv3x3(x, wt, H, W)
    torch.cuda.synchronize()
    assert out.shape == (B, Cout, H, W)
    err = (out.double() - exact(x, wt, H, W)).abs()
    assert (err <= fwd_bound(x, wt, H, W)).all(), float(err.max())


# ---- IEEE footprint ----------------------------------------------------------------------------------------------------
def nonfinite_pattern(t):
    t = t.double().cpu()
    return torch.isnan(t), torch.isposinf(t), torch.isneginf(t)


@pytest.mark.parametrize('H,W', [(40, 66), (39, 65), (1, 1), (24, 31)])
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_ieee_footprint_of_non_finite_x(H, W, value):
    x, wt = inputs(11, 2, 19, 20, 33, 8)
    for (b, c, i, j) in [(0, 0, 0, 0), (1, 18, 19, 32), (0, 5, 15, 31), (1, 3, 16, 32), (0, 7, (H - 1) // 2, (W - 1) // 2),
                         (1, 2, 8, 15)]:                         # tile seams at i = 16, j = 32 and cropped-away cells
        xx = x.clone()
        xx[b, c, i, j] = value
        out = cspn_b200.unpool_conv3x3(xx, wt, H, W)
        ref = exact(xx, wt, H, W)
        for a, r in zip(nonfinite_pattern(out), nonfinite_pattern(ref)):
            assert torch.equal(a, r), (b, c, i, j)
        fin = torch.isfinite(ref)
        assert ((out.double() - ref).abs()[fin] <= fwd_bound(x, wt, H, W)[fin] + 1e-30).all()


@pytest.mark.parametrize('H,W', [(40, 66), (39, 65), (1, 1)])
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_ieee_footprint_of_non_finite_weights(H, W, value):
    x, wt = inputs(12, 2, 19, 20, 33, 8)
    for (co, ci, t) in [(0, 0, 0), (3, 18, 4), (7, 5, 8), (2, 2, 5), (5, 0, 7)]:
        ww = wt.clone()
        ww[co, ci, t // 3, t % 3] = value
        out = cspn_b200.unpool_conv3x3(x, ww, H, W)
        ref = exact(x, ww, H, W)
        for a, r in zip(nonfinite_pattern(out), nonfinite_pattern(ref)):
            assert torch.equal(a, r), (co, ci, t)


# ---- determinism -------------------------------------------------------------------------------------------------------
def test_forward_and_grad_x_bits_do_not_depend_on_the_batch_and_grad_weight_is_reproducible():
    B, Cin, h, w, Cout, H, W = 3, 64, 30, 45, 8, 59, 90
    x, wt = inputs(21, B, Cin, h, w, Cout)
    go = torch.randn(B, Cout, H, W, device='cuda')
    op = torch.ops.cspn_b200
    torch_op.load()
    out = op.unpool_conv3x3(x, wt, H, W)
    gx, gw = op.unpool_conv3x3_backward(x, wt, go, H, W, True, True)
    for _ in range(2):
        assert torch.equal(op.unpool_conv3x3(x, wt, H, W), out)
        gx2, gw2 = op.unpool_conv3x3_backward(x, wt, go, H, W, True, True)
        assert torch.equal(gx2, gx) and torch.equal(gw2, gw)
    for b in range(B):
        assert torch.equal(op.unpool_conv3x3(x[b:b + 1], wt, H, W), out[b:b + 1])
        gxb, _ = op.unpool_conv3x3_backward(x[b:b + 1], wt, go[b:b + 1].contiguous(), H, W, True, False)
        assert torch.equal(gxb, gx[b:b + 1])


# ---- backward ----------------------------------------------------------------------------------------------------------
BWD_CASES = [
    (1, 64, 114, 152, 8, 228, 304),
    (2, 64, 40, 52, 1, 79, 103),
    (2, 65, 17, 23, 24, 33, 45),
    (4, 3, 9, 11, 8, 18, 21),
    (1, 1, 1, 1, 1, 1, 1),
    (1, 2, 5, 4, 48, 9, 7),
]


def fp64_grads(x, wt, go, H, W, absolute=False):
    xd = x.double().abs() if absolute else x.double()
    wd = wt.double().abs() if absolute else wt.double()
    xd.requires_grad_(True)
    wd.requires_grad_(True)
    ur.op_sequence(xd, wd, H, W).backward(go.double().abs() if absolute else go.double())
    return xd.grad, wd.grad


@pytest.mark.parametrize('B,Cin,h,w,Cout,H,W', BWD_CASES)
def test_backward_within_the_a_priori_bound(B, Cin, h, w, Cout, H, W):
    x, wt = inputs(B + Cin + 7 * Cout, B, Cin, h, w, Cout)
    go = torch.randn(B, Cout, H, W, device='cuda', generator=torch.Generator('cuda').manual_seed(5))
    xr, wr = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    cspn_b200.unpool_conv3x3(xr, wr, H, W).backward(go)
    gx_ref, gw_ref = fp64_grads(x, wt, go, H, W)
    gx_abs, gw_abs = fp64_grads(x, wt, go, H, W, absolute=True)
    ex = (xr.grad.double() - gx_ref).abs()
    ew = (wr.grad.double() - gw_ref).abs()
    assert (ex <= gamma(9 * Cout) * gx_abs).all(), float(ex.max())           # grad_x: at most 9*Cout terms
    assert (ew <= gamma(B * h * w) * gw_abs).all(), float(ew.max())          # grad_w: at most B*h*w terms
    # normwise: relative to the size of the gradients, far below the componentwise bound's worst case
    assert float(ex.norm() / gx_ref.norm().clamp_min(1e-300)) < 1e-5
    assert float(ew.norm() / gw_ref.norm().clamp_min(1e-300)) < 1e-5
    # a cropped-away source pixel gets no gradient
    hv, wv = (H + 1) // 2, (W + 1) // 2
    assert not xr.grad[:, :, hv:].any() and not xr.grad[:, :, :, wv:].any()


def test_partial_gradients_give_the_full_calls_bits():
    B, Cin, h, w, Cout, H, W = 2, 64, 30, 41, 8, 59, 81
    x, wt = inputs(31, B, Cin, h, w, Cout)
    go = torch.randn(B, Cout, H, W, device='cuda')
    op = torch.ops.cspn_b200
    torch_op.load()
    gx, gw = op.unpool_conv3x3_backward(x, wt, go, H, W, True, True)
    assert torch.equal(op.unpool_conv3x3_backward(x, wt, go, H, W, True, False)[0], gx)
    assert torch.equal(op.unpool_conv3x3_backward(x, wt, go, H, W, False, True)[1], gw)


# ---- launches and the memory contract ----------------------------------------------------------------------------------
@pytest.mark.parametrize('B,Cin,h,w,Cout,H,W', [(2, 64, 30, 41, 8, 59, 81), (1, 3, 5, 6, 1, 10, 11), (3, 65, 17, 9, 24, 33, 17)])
def test_launch_counts_and_memory_contract(B, Cin, h, w, Cout, H, W):
    L = _lib.lib()
    x, wt = inputs(41, B, Cin, h, w, Cout)
    go = torch.randn(B, Cout, H, W, device='cuda')
    before = mc.snapshot([x, wt, go])
    st = torch.cuda.current_stream().cuda_stream
    out = mc.guarded((B, Cout, H, W), 4)
    assert L.cspn_unpool_conv3x3_fwd_f32(x.data_ptr(), wt.data_ptr(), out.ptr(), B, Cin, h, w, Cout, H, W, st) == 0
    assert L.cspn_last_launches() == 1
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert torch.equal(out.t, cspn_b200.unpool_conv3x3(x, wt, H, W))
    nbytes = L.cspn_unpool_conv3x3_bwd_workspace_bytes(B, Cin, h, w, Cout, H, W)
    results = []
    for fill in ('sentinel', 'zero'):
        gx, gw = mc.guarded(x.shape, 4), mc.guarded(wt.shape, 8)
        ws = mc.workspace(nbytes, 4, fill)
        assert L.cspn_unpool_conv3x3_bwd_f32(x.data_ptr(), wt.data_ptr(), go.data_ptr(), gx.ptr(), gw.ptr(), B, Cin, h, w, Cout,
                                             H, W, ws.ptr(), nbytes, st) == 0
        assert L.cspn_last_launches() == 3
        torch.cuda.synchronize()
        mc.assert_written(gx, 'grad_x')
        mc.assert_written(gw, 'grad_weight')
        assert ws.guards_intact()
        results.append((gx.t.clone(), gw.t.clone()))
    assert mc.same_bits(results[0][0], results[1][0]) and mc.same_bits(results[0][1], results[1][1])
    gx = mc.guarded(x.shape)
    assert L.cspn_unpool_conv3x3_bwd_f32(x.data_ptr(), wt.data_ptr(), go.data_ptr(), gx.ptr(), None, B, Cin, h, w, Cout, H, W,
                                         None, 0, st) == 0
    assert L.cspn_last_launches() == 1
    gw = mc.guarded(wt.shape)
    ws = mc.workspace(nbytes)
    assert L.cspn_unpool_conv3x3_bwd_f32(x.data_ptr(), wt.data_ptr(), go.data_ptr(), None, gw.ptr(), B, Cin, h, w, Cout, H, W,
                                         ws.ptr(), nbytes, st) == 0
    assert L.cspn_last_launches() == 2
    torch.cuda.synchronize()
    assert torch.equal(gx.t, results[0][0]) and torch.equal(gw.t, results[0][1])
    assert mc.unchanged(before, [x, wt, go])


# ---- torch integration -------------------------------------------------------------------------------------------------
def test_both_routes_give_the_same_bits():
    torch_op.load()
    B, Cin, h, w, Cout, H, W = 2, 64, 23, 37, 8, 45, 73
    x, wt = inputs(51, B, Cin, h, w, Cout)
    go = torch.randn(B, Cout, H, W, device='cuda')
    res = []
    for route in ('op', 'fn'):
        xr, wr = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
        out = torch.ops.cspn_b200.unpool_conv3x3(xr, wr, H, W) if route == 'op' else _UnpoolConv3x3Fn.apply(xr, wr, H, W)
        out.backward(go)
        res.append((out.detach(), xr.grad, wr.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)
    assert torch.equal(_unpool_conv_fwd(x, wt, H, W), res[0][0])


def test_opcheck():
    torch_op.load()
    x, wt = inputs(61, 2, 5, 6, 7, 3)
    x.requires_grad_(True)
    wt.requires_grad_(True)
    torch.library.opcheck(torch.ops.cspn_b200.unpool_conv3x3.default, (x, wt, 11, 13))
    go = torch.randn(2, 3, 11, 13, device='cuda')
    torch.library.opcheck(torch.ops.cspn_b200.unpool_conv3x3_backward.default, (x.detach(), wt.detach(), go, 11, 13, True, True))


def test_torch_compile_fullgraph_forward_and_backward():
    torch.manual_seed(0)
    m = cspn_b200.Simple_Gudi_UpConv_Block_Last_Layer(16, 8, 35, 47).cuda()
    x = torch.randn(2, 16, 18, 24, device='cuda')

    def fn(x):
        return m(x)

    outs, grads = [], []
    for call in (fn, torch.compile(fn, fullgraph=True)):
        m.zero_grad()
        xc = x.clone().requires_grad_(True)
        out = call(xc)
        out.square().sum().backward()
        outs.append(out.detach())
        grads.append((xc.grad, m.conv1.weight.grad.clone()))
    assert torch.equal(outs[0], outs[1])
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6)


def test_cuda_graph_capture_and_replay():
    m = cspn_b200.Simple_Gudi_UpConv_Block_Last_Layer(64, 8, 228, 304).cuda()
    x = torch.randn(1, 64, 114, 152, device='cuda')
    with torch.no_grad():
        ref = m(x)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(x)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(x)
        x.copy_(torch.randn_like(x))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, m(x)) and not torch.equal(out, ref)


# ---- the reference model's heads ---------------------------------------------------------------------------------------
# The golden holds the bottom-right window x[:, :, y0:, x0:] of the heads' input (the whole map does not fit the
# repository).  Outputs (oy >= 2*y0, ox >= 2*x0) read that window only, and it shares the image's bottom and right borders,
# so the heads on the window, cropped to (oheight - 2*y0, owidth - 2*x0), give the full run's products there.
def golden_heads():
    z = np.load(os.path.join(GOLDEN, 'nyu_resnet50_heads.npz'))
    t = np.load(os.path.join(GOLDEN, 'nyu_resnet50_tail.npz'))
    y0, x0 = int(z['y0']), int(z['x0'])
    oh, ow = int(z['oheight']) - 2 * y0, int(z['owidth']) - 2 * x0
    heads = []
    for key, cout in (('w_guidance', 8), ('w_blur', 1)):
        m = cspn_b200.Simple_Gudi_UpConv_Block_Last_Layer(64, cout, oh, ow).cuda()
        m.load_state_dict({'conv1.weight': torch.from_numpy(z[key])})
        heads.append(m)
    return torch.from_numpy(z['x']).cuda(), heads, t, (y0, x0)


def test_a_window_at_the_bottom_right_gives_the_full_runs_bits():
    x, heads, t, (y0, x0) = golden_heads()
    full = torch.zeros(1, 64, 114, 152, device='cuda')
    full[:, :, y0:, x0:] = x
    with torch.no_grad():
        for m in heads:
            whole = cspn_b200.unpool_conv3x3(full, m.conv1.weight, 228, 304)
            assert torch.equal(m(x), whole[:, :, 2 * y0:, 2 * x0:])


def test_golden_heads_reproduce_the_models_guidance_blur_and_output():
    x, (head6, head5), t, (y0, x0) = golden_heads()
    region = (slice(None), slice(None), slice(2 * y0, None), slice(2 * x0, None))
    with torch.no_grad():
        guidance, blur = head6(x), head5(x)
        for out, m, key in ((guidance, head6, 'guidance'), (blur, head5, 'blur')):
            gold = torch.from_numpy(t[key]).cuda().double()[region]
            H, W = out.shape[2:]
            assert gold.shape == out.shape
            absconv = ur.op_sequence(x.double().abs(), m.conv1.weight.double().abs(), H, W)
            # both are fp32 evaluations: ours within gamma_{4 Cin}, the reference's cuDNN/CPU convolution over the
            # zero-inserted map within gamma_{9 Cin}
            tol = (gamma(4 * 64) + gamma(9 * 64)) * absconv
            assert ((out.double() - gold).abs() <= tol).all(), key
            assert ((out.double() - exact(x, m.conv1.weight, H, W)).abs() <= gamma(4 * 64) * absconv).all(), key
        # the model's guidance / blur with the region computed here: the propagation gives the model's output
        g_all, d_all = torch.from_numpy(t['guidance']).cuda(), torch.from_numpy(t['blur']).cuda()
        g_all[region], d_all[region] = guidance, blur
        out = cspn_b200.Affinity_Propagate(24, 3, '8sum')(g_all, d_all, torch.from_numpy(t['sparse_depth']).cuda())
    ok, ratio, normwise = onp.parity_ok(out.cpu().numpy(), t['out'], 1e-4)
    assert ok, (ratio, normwise)


def test_training_step_of_the_heads_and_the_propagation_matches_fp64_autograd():
    x, (head6, head5), t, (y0, x0) = golden_heads()
    H, W = head6.oheight, head6.owidth
    sparse = torch.from_numpy(t['sparse_depth'][:, :, 2 * y0:, 2 * x0:].copy()).cuda()
    target = torch.rand(1, 1, H, W, device='cuda', generator=torch.Generator('cuda').manual_seed(3))
    mask = (target > 0.5).float()

    def loss_of(out):
        return ((out - target.to(out.dtype)).abs() * mask.to(out.dtype)).sum() / mask.sum()

    out = cspn_b200.Affinity_Propagate(24, 3, '8sum')(head6(x), head5(x), sparse)
    loss_of(out).backward()
    w6 = head6.conv1.weight.detach().double().requires_grad_(True)
    w5 = head5.conv1.weight.detach().double().requires_grad_(True)
    xd = x.double()
    ref = tp.cspn2d_torch(ur.op_sequence(xd, w6, H, W), ur.op_sequence(xd, w5, H, W), sparse.double(), 24, '8sum')
    loss_of(ref).backward()
    for got, want in ((head6.conv1.weight.grad, w6.grad), (head5.conv1.weight.grad, w5.grad)):
        err = float((got.double() - want).norm() / want.norm())
        assert torch.isfinite(got).all() and err < 1e-4, err
