"""CPU tests of atrous affinity pooling (affinity_atrous_pool2d; DESIGN.md section 4.19): the order restatement of
tests/affinity_atrous_reference.py against the fp64 composition and its autograd, gradcheck, the a-priori bounds against
torch's fp32 composition, the IEEE masks of the restatement, the anchors (a constant gate is the depthwise dilated box
filter, a one-hot gate shifts feat), the Python and C ABI refusals before any device work, the workspace size, the argtypes
and the dispatcher registration."""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import affinity_atrous_reference as ar
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn_affinity_atrous2d_fwd_f32', 'cspn_affinity_atrous2d_bwd_workspace_bytes', 'cspn_affinity_atrous2d_bwd_f32')
# (B, C, H, W, rates): r = 1, r > H, r > W, r = max(H, W), repeated and unordered rates, L = 1 and L = 8
SHAPES = [(2, 3, 7, 9, (1, 2)), (1, 4, 5, 6, (6, 1, 1)), (2, 2, 11, 6, (3, 11, 7, 3)), (1, 1, 6, 13, (4,)),
          (1, 3, 9, 10, (1, 2, 3, 4, 5, 6, 7, 8)), (2, 5, 8, 8, (8, 2, 2))]


def rand(seed, *shape, dtype=torch.float64):
    """fp32 values (so that the fp64 references see the fp32 kernels' inputs exactly) in `dtype`."""
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def inputs(seed, B, C, H, W, rates, dtype=torch.float64):
    L = len(rates)
    return rand(seed, B, C, H, W, dtype=dtype), rand(seed + 1, B, 9 * L, H, W, dtype=dtype), rand(seed + 2, B, L * C, H, W, dtype=dtype)


def autograd64(feat, gate, rates, grad):
    f, g = feat.detach().double().clone().requires_grad_(True), gate.detach().double().clone().requires_grad_(True)
    out = ar.compose(f, g, rates)
    out.backward(grad.double())
    return out.detach(), f.grad, g.grad


# ---- 1. the restatement is the composition and its autograd -------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,rates', SHAPES)
def test_order_restatement_against_the_fp64_composition(B, C, H, W, rates):
    feat, gate, grad = inputs(B * 13 + W, B, C, H, W, rates)
    out, gf, gg = autograd64(feat, gate, rates, grad)
    # in fp64 the restatement is the composition and its autograd
    torch.testing.assert_close(ar.fwd_torch(feat, gate, rates), out, rtol=1e-12, atol=1e-12)
    for a, b in zip(ar.bwd_torch(feat, gate, rates, out, grad), (gf, gg)):
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
    # in fp32 it is within the a-priori bounds
    f32, g32, go32 = feat.float(), gate.float(), grad.float()
    o32 = ar.fwd_torch(f32, g32, rates)
    assert ar.max_ratio(o32, out, ar.bound_fwd(f32, g32, rates)) <= 1.0
    for got, want, bound in zip(ar.bwd_torch(f32, g32, rates, o32, go32), (gf, gg), ar.bound_bwd(f32, g32, rates, go32)):
        assert ar.max_ratio(got, want, bound) <= 1.0


@pytest.mark.parametrize('B,C,H,W,rates', SHAPES[:4])
def test_gradcheck_of_the_composition(B, C, H, W, rates):
    feat, gate, _ = inputs(3, B, C, H, W, rates)
    feat.requires_grad_(True)
    gate.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda f, g: ar.compose(f, g, rates), (feat, gate))


# ---- 2. the bounds against torch's own fp32 composition and its autograd ----------------------------------------------------
@pytest.mark.parametrize('scale', [1.0, 1e3, 1e-3])
def test_bounds_hold_for_the_fp32_composition(scale):
    B, C, H, W, rates = 2, 24, 37, 45, (6, 12, 18, 40, 1)
    feat, gate, grad = inputs(9, B, C, H, W, rates)
    feat, gate, grad = feat * scale, gate * scale, grad * scale
    out, gf, gg = autograd64(feat, gate, rates, grad)
    f32, g32 = feat.float().requires_grad_(True), gate.float().requires_grad_(True)
    o32 = ar.compose(f32, g32, rates)
    o32.backward(grad.float())
    assert ar.max_ratio(o32.detach(), out, ar.bound_fwd(feat.float(), gate.float(), rates)) <= 1.0
    for got, want, bound in zip((f32.grad, g32.grad), (gf, gg), ar.bound_bwd(feat.float(), gate.float(), rates, grad.float())):
        assert ar.max_ratio(got, want, bound) <= 1.0


# ---- 3. IEEE: the restatement has the NaN / inf masks of fp64 autograd -------------------------------------------------------
IEEE = ['zero_gates', 'inf_gate', 'nan_feat', 'inf_feat', 'nan_gate_on_padding']


def masks_equal(got, want):
    return (torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(torch.isinf(got), torch.isinf(want))
            and torch.equal(got[torch.isinf(got)], want[torch.isinf(want)].to(got.dtype)))


def ieee_case(case, feat, gate):
    """Writes the special values of `case` into feat (1, 4, 13, 18) and gate (rates (2, 5, 14)), in place."""
    if case == 'zero_gates':
        gate[0, 9:18, 4, 8] = 0.0
        gate[0, 0:9, 7, 2] = -0.0
    elif case == 'inf_gate':
        gate[0, 22, 5, 7] = float('inf')
        gate[0, 3, 2, 9] = float('-inf')
    elif case == 'nan_feat':
        feat[0, 1, 6, 9] = float('nan')
    elif case == 'inf_feat':
        feat[0, 2, 2, 5] = float('inf')
        feat[0, 0, 7, 1] = float('-inf')
    else:                                                     # tap 0 of level 2 (r = 14) reads the padding at (3, 4)
        gate[0, 18, 3, 4] = float('nan')


@pytest.mark.parametrize('case', IEEE)
def test_restatement_ieee_masks_of_fp64_autograd(case):
    rates = (2, 5, 14)
    feat, gate, grad = inputs(3, 1, 4, 13, 18, rates, dtype=torch.float32)
    ieee_case(case, feat, gate)
    out = ar.fwd_torch(feat, gate, rates)
    gf, gg = ar.bwd_torch(feat, gate, rates, out, grad)
    o64, gf64, gg64 = autograd64(feat, gate, rates, grad)
    for got, want in zip((out, gf, gg), (o64, gf64, gg64)):
        assert masks_equal(got, want)
    assert not torch.isfinite(torch.cat([out.reshape(-1), gf.reshape(-1), gg.reshape(-1)])).all()


# ---- 4. the anchors --------------------------------------------------------------------------------------------------------------
def test_a_constant_gate_is_the_dilated_box_filter():
    feat = rand(4, 2, 6, 19, 23, dtype=torch.float32)
    rates = (1, 4, 20, 9)
    gate = torch.full((2, 9 * len(rates), 19, 23), -0.75)
    got = ar.fwd_torch(feat, gate, rates)
    bound = ar.bound_fwd(feat, gate, rates)
    box = torch.ones(6, 1, 3, 3, dtype=torch.float64) / 9
    want = torch.cat([F.conv2d(feat.double(), box, padding=r, dilation=r, groups=6) for r in rates], 1)
    assert ar.max_ratio(got, want, bound) <= 1.0
    torch.testing.assert_close(got, want.float(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('t', range(9))
def test_a_one_hot_gate_shifts_feat_exactly(t):
    B, C, H, W, rates = 2, 3, 13, 17, (1, 5, 14)
    feat = rand(5, B, C, H, W, dtype=torch.float32)
    gate = torch.zeros(B, 9 * len(rates), H, W)
    gate[:, t::9] = torch.rand(B, len(rates), H, W, generator=torch.Generator().manual_seed(t)) * 4 + 0.5
    gate[:, t::9] *= torch.where(torch.rand(B, len(rates), H, W) < 0.5, -1.0, 1.0)
    dy, dx = ar.OFFSETS[t]
    want = torch.cat([ar.shifted(feat, r * dy, r * dx) for r in rates], 1)
    assert torch.equal(ar.fwd_torch(feat, gate, rates).view(torch.int32), want.view(torch.int32))


# ---- 5. the Python surface -------------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    f, g = torch.rand(1, 4, 6, 5), torch.rand(1, 18, 6, 5)
    for args in [(torch.rand(4, 6, 5), g, (2, 3)), (f, torch.rand(18, 6, 5), (2, 3)), (f, g, (2,)), (f, g, (2, 3, 1)),
                 (f, g, ()), (f, g, (0, 2)), (f, g, (2, 7)), (f, g, (2, 2.0)), (f, g, (True, 2)), (f, g, 2), (f, g, '23'),
                 (torch.rand(1, 0, 6, 5), g, (2, 3)), (f, torch.rand(2, 18, 6, 5), (2, 3)), (f, torch.rand(1, 2, 6, 5), (2, 3)),
                 (f, torch.rand(1, 81, 6, 5), tuple(range(1, 10)))]:
        with pytest.raises(ValueError):
            cspn_b200.affinity_atrous_pool2d(*args)
    with pytest.raises(RuntimeError, match='fp32'):
        cspn_b200.affinity_atrous_pool2d(f.double(), g.double(), (2, 3))
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_atrous_pool2d(f, g, (2, 6))                      # r = max(H, W) is valid
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_atrous_pool2d(f.clone().requires_grad_(True), g, [2, 3])


def test_sizes_the_c_abi_cannot_take_are_refused_before_anything_is_allocated():
    f = torch.empty(1, 1, 1 << 16, 1 << 15, device='meta')
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.affinity_atrous_pool2d(f, torch.empty(1, 9, 1 << 16, 1 << 15, device='meta'), (2,))


# ---- 6. the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def rates_arg(*rates):
    return (ctypes.c_int * len(rates))(*rates)


def test_workspace_is_the_weight_planes():
    L = _lib.lib()
    # 9L weight planes of H x W per image, whatever C and the rates
    assert L.cspn_affinity_atrous2d_bwd_workspace_bytes(2, 3, 7, 9, 2, rates_arg(1, 9)) == 4 * 2 * 18 * 7 * 9
    assert L.cspn_affinity_atrous2d_bwd_workspace_bytes(4, 128, 64, 128, 4, rates_arg(6, 12, 18, 24)) == 4 * 4 * 36 * 64 * 128
    for bad in ((0, 3, 7, 9, 2, rates_arg(1, 2)), (2, 0, 7, 9, 2, rates_arg(1, 2)), (2, 3, 7, 9, 0, rates_arg(1)),
                (2, 3, 7, 9, 9, rates_arg(*[1] * 9)), (2, 3, 7, 9, 2, None), (2, 3, 7, 9, 2, rates_arg(1, 10)),
                (2, 3, 7, 9, 2, rates_arg(0, 1))):
        assert L.cspn_affinity_atrous2d_bwd_workspace_bytes(*bad) == 0


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 16384)()
    base = ctypes.cast(buf, ctypes.c_void_p).value

    def at(k, off=0):                                    # 1024 floats apart
        return ctypes.c_void_p(base + k * 4096 + off)

    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, H=4, W=5)                     # feat 40 floats, gate (L = 2) 360, out 80, workspace 1440 bytes

    def fw(ft=at(0), g=at(1), o=at(2), rates=(1, 3), nl=None, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_atrous2d_fwd_f32(ft, g, o, *v.values(), (len(rates) if rates else 2) if nl is None else nl,
                                                None if rates is None else rates_arg(*rates), None)

    def bw(ft=at(0), g=at(1), o=at(2), go=at(3), gf=at(4), gg=at(5), rates=(1, 3), nl=None, ws=at(6), wsb=4096, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_atrous2d_bwd_f32(ft, g, o, go, gf, gg, *v.values(),
                                                (len(rates) if rates else 2) if nl is None else nl,
                                                None if rates is None else rates_arg(*rates), ws, wsb, None)

    for call, ptrs in ((fw, ('ft', 'g', 'o')), (bw, ('ft', 'g', 'o', 'go', 'gf', 'gg'))):
        for k in ok:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for p in ptrs:
            assert call(**{p: None}) == -1 and b'null' in L.cspn_last_error()
            assert call(**{p: odd}) == -1 and b'aligned' in L.cspn_last_error()
        assert call(rates=None) == -1 and b'dilations' in L.cspn_last_error()
        for rates in ((2, 0), (6, 2), (-1,)):
            assert call(rates=rates) == -1 and b'max(H, W)' in L.cspn_last_error()
        assert call(rates=(1,) * 9) == -1 and b'levels' in L.cspn_last_error()
        assert call(rates=(2,), nl=0) == -1 and b'levels' in L.cspn_last_error()
        assert call(H=1 << 16, W=1 << 15, rates=(2,)) == -4 and b'2^31' in L.cspn_last_error()
        assert call(B=1 << 20, C=1 << 10, H=1 << 10, W=1 << 10, rates=(1,)) == -4 and b'grid' in L.cspn_last_error()
    # a null, short or misaligned workspace
    assert bw(ws=None) == -2 and bw(wsb=1439) == -2 and bw(ws=ctypes.c_void_p(base + 6 * 4096 + 2)) == -2
    assert b'workspace' in L.cspn_last_error()
    assert bw(wsb=1440, gf=at(0, 4 * 39)) == -1 and b'grad_feat overlaps feat' in L.cspn_last_error()   # 1440 is enough
    # an output may overlap neither an input nor another output; inputs may alias
    assert fw(o=at(0, 4 * 39)) == -1 and b'out overlaps feat' in L.cspn_last_error()
    assert fw(o=at(1, 4 * 359)) == -1 and b'out overlaps gate' in L.cspn_last_error()
    for over, what in ((dict(gf=at(0, 4 * 39)), b'grad_feat overlaps feat'), (dict(gg=at(1, 4 * 359)), b'grad_gate overlaps gate'),
                       (dict(gf=at(2, 4 * 79)), b'grad_feat overlaps out'), (dict(gg=at(3, 4 * 79)), b'grad_gate overlaps grad_out'),
                       (dict(gg=at(4, 4 * 39)), b'grad_gate overlaps grad_feat'),
                       (dict(ws=at(5, 4 * 359)), b'the workspace overlaps grad_gate'),
                       (dict(ws=at(3, 4 * 79)), b'the workspace overlaps grad_out')):
        assert bw(**over) == -1 and what in L.cspn_last_error(), (over, L.cspn_last_error())
    assert L.cspn_last_launches() == 0


# ---- 7. the dispatcher ops -------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert ('affinity_atrous_pool2d(Tensor feat, Tensor gate, int[] dilations) -> Tensor'
            in str(ops.affinity_atrous_pool2d.default._schema))
    assert ('affinity_atrous_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] dilations) -> '
            '(Tensor, Tensor)' in str(ops.affinity_atrous_pool2d_backward.default._schema))
    rates = [6, 12, 18, 24]
    with FakeTensorMode():
        feat = torch.empty(4, 128, 64, 128, device='cuda')           # PSMNet's training crop at quarter resolution
        gate = torch.empty(4, 36, 64, 128, device='cuda')
        out = ops.affinity_atrous_pool2d(feat, gate, rates)
        assert out.shape == (4, 512, 64, 128) and out.dtype == torch.float32 and out.device == feat.device
        gf, gg = ops.affinity_atrous_pool2d_backward(feat, gate, out, out, rates)
        assert gf.shape == feat.shape and gg.shape == gate.shape
        assert cspn_b200.affinity_atrous_pool2d(feat, gate, rates).shape == out.shape   # the function takes the op route
        with pytest.raises(Exception):
            ops.affinity_atrous_pool2d(feat, gate, [6, 12, 18])
        with pytest.raises(Exception):
            ops.affinity_atrous_pool2d(feat, gate, [6, 12, 18, 129])
