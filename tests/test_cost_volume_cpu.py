"""CPU tests of the stereo cost volumes (build_concat_volume / build_gwc_volume; DESIGN.md section 4.16): the restatements of
tests/cost_volume_reference.py against the fp64 loops and their autograd, gradcheck, the a-priori bounds against fp32
evaluations, the tile plans against the columns every tile reads, the Python and C ABI refusals before any device work,
the argtypes and the dispatcher registration."""
import ctypes

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import cost_volume_reference as cr
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn_concat_volume_fwd_f32', 'cspn_concat_volume_bwd_f32', 'cspn_gwc_volume_fwd_f32', 'cspn_gwc_volume_bwd_f32')
# (B, F, H, W, D, G): D < W, D = W, D > W, W = 1, D = 1, G in {1, F/2, F}
SHAPES = [(2, 4, 3, 9, 4, 2), (1, 6, 2, 5, 5, 3), (1, 4, 2, 4, 7, 1), (2, 2, 3, 1, 3, 2), (1, 8, 2, 6, 1, 8),
          (1, 1, 2, 7, 3, 1), (2, 8, 2, 11, 6, 4)]


def rand(seed, *shape, dtype=torch.float64):
    """fp32 values (so that the fp64 references see the fp32 kernels' inputs exactly) in `dtype`."""
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def inputs(seed, B, F, H, W, D, G, dtype=torch.float64):
    return rand(seed, B, F, H, W, dtype=dtype), rand(seed + 1, B, F, H, W, dtype=dtype), rand(seed + 2, B, G, D, H, W, dtype=dtype)


# ---- 1. the restatements are the loops and their autograd ------------------------------------------------------------------
@pytest.mark.parametrize('B,F,H,W,D,G', SHAPES)
def test_order_restatements_against_the_fp64_loops(B, F, H, W, D, G):
    L, R, g = inputs(B * 11 + W, B, F, H, W, D, G)
    # the forwards: concat's copies are exact in any dtype; gwc's fp32 order is within its bound of fp64
    assert torch.equal(cr.concat_loop(L.float(), R.float(), D).double(), cr.concat_loop(L, R, D))
    want = cr.gwc_loop(L, R, D, G)
    got = cr.gwc_fwd_fp32(L.float().numpy(), R.float().numpy(), D, G)
    assert cr.max_ratio(got, want, cr.bound_gwc_fwd(L.float(), R.float(), D, G)) <= 1.0
    # the backwards, restated in fp64, are autograd of the loops
    Lr, Rr = L.clone().requires_grad_(True), R.clone().requires_grad_(True)
    gc = rand(5, B, 2 * F, D, H, W)
    cr.concat_loop(Lr, Rr, D).backward(gc)
    for a, b in zip(cr.concat_bwd_torch(gc), (Lr.grad, Rr.grad)):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    Lr.grad = Rr.grad = None
    cr.gwc_loop(Lr, Rr, D, G).backward(g)
    for a, b in zip(cr.gwc_bwd_torch(L, R, g), (Lr.grad, Rr.grad)):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    # the fp32 orders within their bounds of the fp64 gradients
    for got, want, bound in zip(cr.concat_bwd_fp32(gc.float().numpy()), cr.concat_bwd_torch(gc),
                                cr.bound_concat_bwd(gc.float())):
        assert cr.max_ratio(got, want, bound) <= 1.0
    got = cr.gwc_bwd_fp32(L.float().numpy(), R.float().numpy(), g.float().numpy())
    for a, want, bound in zip(got, (Lr.grad, Rr.grad), cr.bound_gwc_bwd(L.float(), R.float(), g.float())):
        assert cr.max_ratio(a, want, bound) <= 1.0


def test_one_term_sums_return_their_term():
    """D = 1 and n = 1: the sums start from their first term, so grad and volume are that term's bits (-0.0 included)."""
    L = torch.tensor([[[[-0.0, 1.5, -2.0]]]], dtype=torch.float32)
    R = torch.tensor([[[[3.0, 0.0, -0.25]]]], dtype=torch.float32)
    vol = cr.gwc_fwd_fp32(L.numpy(), R.numpy(), 1, 1)
    assert np.array_equal(vol.view(np.int32), (L * R).numpy()[:, :, None].view(np.int32))
    g = -torch.zeros(1, 2, 1, 1, 3)
    gl, gr = cr.concat_bwd_fp32(g.numpy())
    assert np.signbit(gl).all() and np.signbit(gr).all()


@pytest.mark.parametrize('B,F,H,W,D,G', SHAPES[:4])
def test_gradcheck_of_the_loops(B, F, H, W, D, G):
    L, R, _ = inputs(3, B, F, H, W, D, G)
    L.requires_grad_(True)
    R.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b: cr.concat_loop(a, b, D), (L, R))
    assert torch.autograd.gradcheck(lambda a, b: cr.gwc_loop(a, b, D, G), (L, R))


# ---- 2. the bounds against fp32 evaluations (torch's own fp32 loop, any summation order) -----------------------------------
@pytest.mark.parametrize('scale', [1.0, 1e3, 1e-3])
def test_bounds_hold_for_the_fp32_loops(scale):
    B, F, H, W, D, G = 2, 32, 3, 40, 12, 4
    L, R, g = (t * scale for t in inputs(9, B, F, H, W, D, G))
    want = cr.gwc_loop(L, R, D, G)
    assert cr.max_ratio(cr.gwc_loop(L.float(), R.float(), D, G), want, cr.bound_gwc_fwd(L, R, D, G)) <= 1.0
    Lr, Rr = L.float().requires_grad_(True), R.float().requires_grad_(True)
    cr.gwc_loop(Lr, Rr, D, G).backward(g.float())
    for got, want, bound in zip((Lr.grad, Rr.grad), cr.gwc_bwd_torch(L.float().double(), R.float().double(), g.float().double()),
                                cr.bound_gwc_bwd(L.float(), R.float(), g.float())):
        assert cr.max_ratio(got, want, bound) <= 1.0
    gc = rand(4, B, 2 * F, D, H, W) * scale
    Lr.grad = Rr.grad = None
    cr.concat_loop(Lr, Rr, D).backward(gc.float())
    for got, want, bound in zip((Lr.grad, Rr.grad), cr.concat_bwd_torch(gc.float().double()), cr.bound_concat_bwd(gc.float())):
        assert cr.max_ratio(got, want, bound) <= 1.0


# ---- 3. the tile plans: the staged columns hold every column a tile reads ---------------------------------------------------
@pytest.mark.parametrize('W', [1, 2, 3, 5, 8, 13, 64, 130, 312])
def test_plans_stage_every_column_each_tile_reads(W):
    for D in sorted(set(range(1, W + 3)) if W < 20 else {1, 2, 7, 48, W - 1, W, W + 1, W + 5}):
        for kind, n in (('concat_fwd', 0), ('gwc_fwd', 8), ('gwc_bwd', 8), ('gwc_fwd', 64)):
            tx, rp, smem = cr.plan(kind, W, D, n)
            assert 0 < smem <= cr.SMEM_HARD and tx >= 1 and (tx & (tx - 1)) == 0
            assert smem <= cr.SMEM_SOFT or tx == 1
            for x0 in range(0, W, tx):
                (r_lo, r_hi), (l_lo, l_hi) = cr.staged(W, D, tx, x0)
                (rd_lo, rd_hi), (ld_lo, ld_hi) = cr.read_span(W, D, tx, x0)
                assert r_lo <= rd_lo and rd_hi <= r_hi and r_hi - r_lo <= rp, (kind, W, D, x0)
                assert l_lo <= ld_lo and ld_hi <= l_hi and l_hi - l_lo <= rp, (kind, W, D, x0)


def test_the_limits_of_the_smallest_tiles():
    """The D at which a 1-column tile stops fitting (DESIGN.md section 4.16), at W >= D."""
    def first_refused(kind, n):
        lo, hi = 1, 1 << 20
        while lo < hi:
            mid = (lo + hi) // 2
            if cr.plan(kind, 1 << 20, mid, n)[2]:
                lo = mid + 1
            else:
                hi = mid
        return lo
    assert first_refused('concat_fwd', 0) == 14528
    assert first_refused('gwc_fwd', 8) == 7264 and first_refused('gwc_fwd', 320) == 181
    assert first_refused('gwc_bwd', 8) == 3229
    # the training shape's tiles: 128 columns, two CTAs per SM or better
    assert cr.plan('concat_fwd', 128, 48)[:2] == (128, 128) and cr.plan('gwc_bwd', 128, 48, 8)[0] == 128


# ---- 4. the Python surface -------------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    x = torch.rand(1, 4, 3, 5)
    for f, extra in ((cspn_b200.build_concat_volume, ()), (cspn_b200.build_gwc_volume, (2,))):
        for args in [(torch.rand(4, 3, 5), torch.rand(4, 3, 5), 2), (x, torch.rand(1, 4, 3, 6), 2), (x, x, 0), (x, x, 2.0),
                     (x, x, True), (torch.rand(1, 0, 3, 5), torch.rand(1, 0, 3, 5), 2)]:
            with pytest.raises(ValueError):
                f(*args, *extra)
        with pytest.raises(RuntimeError):
            f(x.double(), x.double(), 2, *extra)
        with pytest.raises(cspn_b200.CspnError):
            f(x, x, 2, *extra)
        with pytest.raises(cspn_b200.CspnError):
            f(x.clone().requires_grad_(True), x, 2, *extra)
    for G in (3, 0, 5, True, 2.0):
        with pytest.raises(ValueError, match='num_groups'):
            cspn_b200.build_gwc_volume(x, x, 2, G)


def test_sizes_the_c_abi_cannot_take_are_refused_before_anything_is_allocated():
    x = torch.empty(1, 2, 1 << 10, 1 << 10, device='meta')
    for f, extra in ((cspn_b200.build_concat_volume, ()), (cspn_b200.build_gwc_volume, (1,))):
        with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
            f(x, x, 1 << 11, *extra)
        big = torch.empty(1 << 31, 2, 2, 2, device='meta')
        with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
            f(big, big, 2, *extra)


# ---- 5. the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 8192)()
    base = ctypes.cast(buf, ctypes.c_void_p).value
    a, b, c, d, e = (ctypes.c_void_p(base + k * 4096) for k in range(5))   # 1024 floats apart
    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, F=4, H=2, W=5, D=3)             # features 40 floats, concat volume 240, gwc volume (G = 2) 60

    def cf(l=a, r=b, o=c, **over):
        v = dict(ok, **over)
        return L.cspn_concat_volume_fwd_f32(l, r, o, *v.values(), None)

    def cb(go=c, gl=a, gr=b, **over):
        v = dict(ok, **over)
        return L.cspn_concat_volume_bwd_f32(go, gl, gr, *v.values(), None)

    def gf(l=a, r=b, o=c, G=2, **over):
        v = dict(ok, **over)
        return L.cspn_gwc_volume_fwd_f32(l, r, o, *v.values(), G, None)

    def gb(l=a, r=b, go=c, gl=d, gr=e, G=2, **over):
        v = dict(ok, **over)
        return L.cspn_gwc_volume_bwd_f32(l, r, go, gl, gr, *v.values(), G, None)

    calls = ((cf, ('l', 'r', 'o')), (cb, ('go', 'gl', 'gr')), (gf, ('l', 'r', 'o')), (gb, ('l', 'r', 'go', 'gl', 'gr')))
    for call, ptrs in calls:
        for k in ok:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for p in ptrs:
            assert call(**{p: None}) == -1 and b'null' in L.cspn_last_error()
            assert call(**{p: odd}) == -1 and b'aligned' in L.cspn_last_error()
        assert call(D=1 << 11, H=1 << 10, W=1 << 10) == -4 and b'2^31' in L.cspn_last_error()
        assert call(F=1 << 30) == -4
    for call in (gf, gb):
        assert call(G=3) == -1 and b'divide' in L.cspn_last_error()
        assert call(G=0) == -1 and call(G=-2) == -1
        assert call(G=1, F=320, D=200, W=400) == -4 and b'shared memory' in L.cspn_last_error()
    assert gb(D=3300, W=4000, F=8, G=1) == -4 and b'shared memory' in L.cspn_last_error()
    assert cf(D=15000, W=15000, H=1) == -4 and b'shared memory' in L.cspn_last_error()
    # an output may overlap neither an input nor the other output; inputs may alias
    assert cf(o=a) == -1 and b'out overlaps left' in L.cspn_last_error()
    assert cf(o=ctypes.c_void_p(base + 4096 + 4 * 39)) == -1 and b'out overlaps right' in L.cspn_last_error()
    assert cb(gl=ctypes.c_void_p(base + 2 * 4096 + 4 * 239)) == -1 and b'grad_left overlaps grad_out' in L.cspn_last_error()
    assert cb(gr=ctypes.c_void_p(base + 4 * 39)) == -1 and b'grad_right overlaps grad_left' in L.cspn_last_error()
    assert gf(o=ctypes.c_void_p(base + 4 * 39)) == -1 and b'out overlaps left' in L.cspn_last_error()
    for over, what in ((dict(gl=a), b'grad_left overlaps left'), (dict(gr=b), b'grad_right overlaps right'),
                       (dict(gl=ctypes.c_void_p(base + 2 * 4096 + 4 * 59)), b'grad_left overlaps grad_out'),
                       (dict(gr=ctypes.c_void_p(base + 3 * 4096 + 4 * 39)), b'grad_right overlaps grad_left')):
        assert gb(**over) == -1 and what in L.cspn_last_error()
    assert L.cspn_last_launches() == 0


# ---- 6. the dispatcher ops -------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert 'concat_volume(Tensor left, Tensor right, int max_disp) -> Tensor' in str(ops.concat_volume.default._schema)
    assert 'concat_volume_backward(Tensor grad_out) -> (Tensor, Tensor)' in str(ops.concat_volume_backward.default._schema)
    assert ('gwc_volume(Tensor left, Tensor right, int max_disp, int num_groups) -> Tensor'
            in str(ops.gwc_volume.default._schema))
    assert ('gwc_volume_backward(Tensor left, Tensor right, Tensor grad_out) -> (Tensor, Tensor)'
            in str(ops.gwc_volume_backward.default._schema))
    with FakeTensorMode():
        left = torch.empty(4, 320, 64, 128, device='cuda')           # GwcNet's quarter-resolution features
        v = ops.gwc_volume(left, left, 48, 40)
        assert v.shape == (4, 40, 48, 64, 128) and v.dtype == torch.float32 and v.device == left.device
        assert all(t.shape == left.shape for t in ops.gwc_volume_backward(left, left, v))
        c = ops.concat_volume(left[:, :32], left[:, :32], 48)
        assert c.shape == (4, 64, 48, 64, 128)
        assert all(t.shape == (4, 32, 64, 128) for t in ops.concat_volume_backward(c))
        assert cspn_b200.build_gwc_volume(left, left, 48, 40).shape == v.shape       # the function takes the op route
        assert cspn_b200.build_concat_volume(left[:, :32], left[:, :32], 48).shape == c.shape
        with pytest.raises(Exception):
            ops.gwc_volume(left, left, 48, 7)
