"""CPU tests of disparity_regression (resize_trilinear -> softmax over d -> expectation of d; DESIGN.md section 4.15): the
restatements of tests/disparity_reference.py against PyTorch's own chain in fp64, gradcheck, sharp columns, the a-priori
bound of the softmax stage against an fp32 evaluation, the Python argument errors, the C ABI's refusals before any device
work, and the dispatcher registration."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import disparity_reference as dr
import resize_reference as rr
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn_disparity_regression_fwd_f32', 'cspn_disparity_regression_bwd_workspace_bytes',
           'cspn_disparity_regression_bwd_f32')
MODES = [(True, 1), (False, 0), (False, 1)]
SHAPES = [((5, 4, 6), (17, 9, 13)), ((7, 3, 9), (4, 8, 5)), ((4, 5, 6), (4, 5, 6)), ((1, 3, 2), (6, 5, 4))]


def rand(seed, *shape, dtype=torch.float64):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=dtype)


# ---- 1. the restatement is PyTorch's chain ------------------------------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', [(True, 1), (False, 0)])
@pytest.mark.parametrize('in_size,out_size', SHAPES)
def test_restatement_is_interpolate_softmax_sum_in_fp64(in_size, out_size, align_corners, align_mode):
    cost = rand(1, 2, 3, *in_size)
    up = F.interpolate(cost, size=out_size, mode='trilinear', align_corners=align_corners)
    want = (torch.softmax(up, dim=2) * torch.arange(out_size[0], dtype=torch.float64)[:, None, None]).sum(2)
    got = dr.forward_torch(cost, out_size, align_corners, align_mode)
    assert got.shape == (2, 3, *out_size[1:])
    # ATen forms fp64 coordinates for fp64 input, ours are fp32 (as in the resize tests); dy/dU_o = p_o (o - y), and
    # sum_o p_o |o - y| < Do
    tol_u = 8 * max(in_size) * rr.U * 2 * float(cost.abs().max())
    torch.testing.assert_close(got, want, rtol=0, atol=out_size[0] * tol_u)


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_gathered_resize_is_resize_reference(align_corners, align_mode):
    for in_size, out_size in SHAPES:
        x = rand(2, 2, 2, *in_size)
        torch.testing.assert_close(dr.resize_fp64(x, out_size, align_corners, align_mode),
                                   rr.resize_torch(x, out_size, align_corners, align_mode), rtol=1e-12, atol=1e-12)
        x32 = x.float()
        want = rr.forward_fp32(x32.numpy(), out_size, align_corners, align_mode)
        assert np.array_equal(dr.resize_fp32(x32, out_size, align_corners, align_mode).numpy().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_gradcheck_of_the_restatement(align_corners, align_mode):
    cost = rand(3, 1, 2, 3, 4, 2).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda c: dr.forward_torch(c, (7, 3, 5), align_corners, align_mode), (cost,))


def test_the_backward_formula_is_autograd():
    """gU_o = g * p_o * (o - y), then resize's adjoint: what the kernels compute, against autograd."""
    cost = rand(4, 2, 2, 5, 4, 6)
    g = rand(5, 2, 2, 9, 11)
    for ac, am in MODES:
        u = dr.resize_fp64(cost, (17, 9, 11), ac, am)
        p = torch.softmax(u, dim=2)
        o = torch.arange(17, dtype=torch.float64)[:, None, None]
        y = (p * o).sum(2, keepdim=True)
        grad = rr.adjoint_torch(g[:, :, None] * p * (o - y), (5, 4, 6), ac, am)
        torch.testing.assert_close(grad, dr.grad_torch(cost, g, (17, 9, 11), ac, am), rtol=1e-10, atol=1e-12)


def test_sharp_columns_are_exact_in_the_restatement():
    cost, k = dr.sharp_cost(2, 3, 4, 6)
    y = dr.forward_torch(cost, (17, 7, 11), True, 1)
    # every o but 4k is >= 234 below the maximum: exp(-234) ~ 1e-102 (in fp32 it is 0, and the kernels' y is 4k exactly)
    assert float((y - (4 * k).double()[:, :, None, None]).abs().max()) < 1e-90
    grad = dr.grad_torch(cost, rand(6, 2, 3, 7, 11), (17, 7, 11), True, 1)
    assert float(grad.abs().max()) < 1e-90


def test_non_finite_values_reach_only_the_columns_whose_taps_read_them():
    cost = rand(7, 1, 1, 5, 6, 7)
    cost[0, 0, 2, 3, 3] = float('inf')
    y = dr.forward_torch(cost, (9, 11, 13), True, 1)
    assert torch.isnan(y).any() and not torch.isnan(y).all()
    # the dense matrices of resize_reference multiply the inf by every zero of its row: NaN in whole rows
    dense = dr.regress_torch(rr.resize_torch(cost, (9, 11, 13), True, 1))
    assert torch.isnan(dense).sum() > torch.isnan(y).sum()


# ---- 2. the a-priori bound of the softmax stage -------------------------------------------------------------------------
@pytest.mark.parametrize('scale', [1.0, 30.0, 1e4])
def test_fp32_softmax_stage_within_its_bound(scale):
    u32 = (rand(8, 2, 2, 48, 5, 7) * scale).float()
    got = torch.from_numpy(dr.softmax_stage_fp32(u32.numpy()))
    want = dr.regress_torch(u32.double())
    bound = dr.bound_softmax(u32)
    assert dr.max_ratio(got, want, bound) <= 1.0
    assert float(bound.max()) < 1e-2 * 48


def test_whole_op_bounds_are_finite_and_small():
    cost = rand(9, 1, 2, 5, 4, 6).float()
    g = rand(10, 1, 2, 9, 11).float()
    for ac, am in MODES:
        bf = dr.bound_fwd(cost, (17, 9, 11), ac, am)
        bb = dr.bound_bwd(cost, g, (17, 9, 11), ac, am)
        assert bf.shape == (1, 2, 9, 11) and bb.shape == cost.shape
        assert torch.isfinite(bf).all() and torch.isfinite(bb).all()
        assert float(bf.max()) < 1e-3 and float(bb.max()) < 1e-3


# ---- 3. the launch plans: the spans that size shared memory bound the spans the kernels meet ------------------------------
SIZES = [(48, 192), (64, 256), (128, 512), (48, 384), (156, 1248), (6, 31), (64, 512), (5, 40), (4, 32), (3, 24), (7, 9),
         (33, 100), (100, 33), (9, 4), (1, 7), (7, 1), (2, 5), (12, 100), (10, 77), (96, 384), (312, 1248), (20, 20)]


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_plan_spans_bound_the_spans_of_every_tile(align_corners, align_mode):
    """For t outputs (forward) or t low-resolution cells (backward) at every start, along axes up 1x-8x and down, the
    tables the kernels size from span_in / span_out hold every span they meet (span_out once missed the outputs the
    half-pixel rule clamps to coordinate 0, for tiles of one or two cells)."""
    for n_in, n_out in SIZES:
        for t in (1, 2, 3, 4, 8, 16, 32):
            read, readers = dr.spans(n_in, n_out, align_corners, align_mode, t)
            assert read <= dr.span_in(n_in, n_out, align_corners, align_mode, t), (n_in, n_out, t)
            assert readers <= dr.span_out(n_in, n_out, align_corners, align_mode, t), (n_in, n_out, t)


def test_half_pixel_union_at_8x_fits_its_tile():
    """A 1/8-resolution stereo volume, 48x48x156 -> 384x384x1248, with F.interpolate's half-pixel rule: the backward falls
    back to 1-cell tiles, and the tile at h = 1 is read by 20 outputs per axis."""
    tile, (ph, pw), smem = dr.bwd_plan((48, 48, 156), (384, 384, 1248), False, 0)
    assert tile[0] == 1 and smem <= dr.SMEM_HARD
    assert dr.spans(48, 384, False, 0, tile[0])[1] == 20 <= ph and dr.spans(156, 1248, False, 0, tile[1])[1] <= pw


# ---- 4. the Python surface ----------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    f = cspn_b200.disparity_regression
    x = torch.rand(1, 2, 3, 4, 5)
    for args, kw in [((torch.rand(2, 3, 4, 5),), dict(scale=2.0)), ((x,), dict()), ((x,), dict(out_shape=(1, 2, 3), scale=1.0)),
                     ((x,), dict(scale=2.0, align_mode=2)), ((x,), dict(scale=2.0, align_mode=True)),
                     ((x,), dict(out_shape=(0, 2, 3))), ((torch.rand(1, 1, 0, 2, 2),), dict(scale=2.0))]:
        with pytest.raises(ValueError):
            f(*args, **kw)
    with pytest.raises(RuntimeError):
        f(x.double(), scale=2.0)
    for ac, am in MODES:
        with pytest.raises(cspn_b200.CspnError):
            f(x, (6, 8, 10), align_corners=ac, align_mode=am)
        with pytest.raises(cspn_b200.CspnError):
            f(x.clone().requires_grad_(True), scale=2.0, align_corners=ac, align_mode=am)


def test_sizes_the_c_abi_cannot_take_are_refused_before_anything_is_allocated():
    x = torch.empty(1, 1, 2, 2, 2, device='meta')
    for size in [(2 ** 32 + 1, 1, 1), (1 << 11, 1 << 10, 1 << 10)]:
        with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
            cspn_b200.disparity_regression(x, size)
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.disparity_regression(torch.empty(1 << 31, 1, 2, 2, 2, device='meta'), (2, 2, 2))


# ---- 5. the C ABI -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 8192)()
    base = ctypes.cast(buf, ctypes.c_void_p).value
    cost, out, go = ctypes.c_void_p(base), ctypes.c_void_p(base + 8192), ctypes.c_void_p(base + 16384)
    w = ctypes.c_void_p(base + 24576)                                 # clear of all three
    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, D=3, H=4, W=5, Do=6, Ho=7, Wo=8, ac=1, am=1)    # cost 120 floats, out / grad_out 112 floats
    names = list(ok)

    def f(c=cost, o=out, **over):
        v = dict(ok, **over)
        return L.cspn_disparity_regression_fwd_f32(c, o, *[v[k] for k in names], None)

    def g(c=cost, gout=go, gc=out, ws=w, ws_bytes=1 << 20, **over):
        v = dict(ok, **over)
        return L.cspn_disparity_regression_bwd_f32(c, gout, gc, *[v[k] for k in names], ws, ws_bytes, None)

    for call, ptrs in ((f, ('c', 'o')), (g, ('c', 'gout', 'gc'))):
        for k in names[:8]:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for k in ('ac', 'am'):
            assert call(**{k: 2}) == -1 and call(**{k: -1}) == -1
        for p in ptrs:
            assert call(**{p: None}) == -1 and b'null' in L.cspn_last_error()
            assert call(**{p: odd}) == -1 and b'aligned' in L.cspn_last_error()
        # resize's size rule: >= 2^31 elements per (B*C) slice in the cost or the upsampled volume
        assert call(D=1 << 11, H=1 << 10, W=1 << 10) == -4 and call(Do=1 << 11, Ho=1 << 10, Wo=1 << 10) == -4
        assert b'2^31' in L.cspn_last_error()
        # the tile rule: Do beyond 2^24, or columns too deep for shared memory
        assert call(Do=(1 << 24) + 1, Ho=1, Wo=1) == -4 and b'2^24' in L.cspn_last_error()
        assert call(D=20000, Do=20000, H=1, Ho=1, W=1, Wo=1) == -4 and b'shared memory' in L.cspn_last_error()
    # the destination must not overlap what is read
    assert f(o=cost) == -1 and b'out overlaps cost' in L.cspn_last_error()
    assert f(o=ctypes.c_void_p(base + 4 * 120 - 4)) == -1
    assert g(gc=cost) == -1 and b'grad_cost overlaps cost' in L.cspn_last_error()
    assert g(gc=ctypes.c_void_p(base + 16384 + 4 * 112 - 4)) == -1 and b'grad_cost overlaps grad_out' in L.cspn_last_error()
    # cost and grad_out are both read: they may overlap
    need = L.cspn_disparity_regression_bwd_workspace_bytes(3, 4, 5, 6, 7, 8)
    assert need == 8 * (3 + 4 + 5 + 6 + 7 + 8)
    # a missing, short or misaligned workspace, and one that overlaps any buffer
    assert g(ws=None) == -2 and g(ws_bytes=need - 1) == -2 and g(ws=ctypes.c_void_p(base + 24580)) == -2
    for ws, what in ((out, b'grad_cost'), (cost, b'cost'), (go, b'grad_out')):
        assert g(ws=ws) == -1 and b'workspace overlaps ' + what in L.cspn_last_error()
    assert L.cspn_last_launches() == 0
    assert L.cspn_disparity_regression_bwd_workspace_bytes(0, 4, 5, 6, 7, 8) == 0


# ---- 6. the dispatcher ops ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert ('disparity_regression(Tensor cost, int D, int H, int W, bool align_corners, int align_mode) -> Tensor'
            in str(ops.disparity_regression.default._schema))
    assert ('disparity_regression_backward(Tensor cost, Tensor grad_out, int D, int H, int W, bool align_corners, '
            'int align_mode) -> Tensor' in str(ops.disparity_regression_backward.default._schema))
    with FakeTensorMode():
        cost = torch.empty(4, 1, 48, 64, 128, device='cuda')        # PSMNet's quarter-resolution cost volume
        y = ops.disparity_regression(cost, 192, 256, 512, True, 1)
        assert y.shape == (4, 1, 256, 512) and y.dtype == torch.float32 and y.device == cost.device
        assert ops.disparity_regression_backward(cost, y, 192, 256, 512, True, 1).shape == cost.shape
        assert cspn_b200.disparity_regression(cost, scale=4.0).shape == (4, 1, 256, 512)   # the function takes the op route
        with pytest.raises(Exception):
            ops.disparity_regression(cost, 0, 4, 4, True, 1)
