"""CPU tests of affinity fusion (affinity_fuse2d; DESIGN.md section 4.18): the fp32 order restatement of
tests/affinity_fuse_reference.py against the fp64 composition and its autograd, gradcheck, the a-priori bounds against
torch's own fp32 composition, the anchors against F.interpolate (a constant gate is the mean of the upsampled levels, a
full-resolution level under a one-hot gate is itself), the Python and C ABI refusals before any device work, the argtypes
and the dispatcher registration."""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import affinity_fuse_reference as fr
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn_affinity_fuse2d_fwd_f32', 'cspn_affinity_fuse2d_bwd_workspace_bytes', 'cspn_affinity_fuse2d_bwd_f32')
ALIGN = [(True, 1), (True, 0), (False, 0), (False, 1)]
# (B, C, H, W, level sizes): odd sizes, a 1 x 1 level, a full-resolution level, a downsampling level, L = 1 and L = 8
SHAPES = [(2, 3, 7, 9, ((2, 3), (4, 5))), (1, 4, 5, 6, ((5, 6), (1, 1))), (2, 2, 6, 11, ((9, 14), (3, 2), (1, 4))),
          (1, 1, 8, 8, ((3, 3),)), (1, 2, 5, 7, tuple((1 + k % 4, 1 + (k * 3) % 8) for k in range(8)))]


def rand(seed, *shape, dtype=torch.float32):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def inputs(seed, B, C, H, W, hws):
    levels = [rand(seed + l, B, C, h, w) for l, (h, w) in enumerate(hws)]
    return levels, rand(seed + 20, B, len(hws), H, W), rand(seed + 21, B, C, H, W)


def autograd64(levels, gate, grad_out, ac, am):
    xs = [x.detach().double().requires_grad_(True) for x in levels]
    g = gate.detach().double().requires_grad_(True)
    out = fr.compose(xs, g, ac, am)
    out.backward(grad_out.double())
    return out.detach(), [x.grad for x in xs], g.grad


# ---- 1. the restatement against the composition and its autograd -----------------------------------------------------------------
@pytest.mark.parametrize('ac,am', ALIGN)
@pytest.mark.parametrize('B,C,H,W,hws', SHAPES)
def test_fp32_restatement_within_the_bounds_of_fp64_autograd(B, C, H, W, hws, ac, am):
    levels, gate, go = inputs(B * 13 + W, B, C, H, W, hws)
    o64, gl64, gg64 = autograd64(levels, gate, go, ac, am)
    out = fr.fwd_torch(levels, gate, ac, am)
    assert fr.max_ratio(out, o64, fr.bound_fwd(levels, gate, ac, am)) <= 1.0
    gl, gg = fr.bwd_torch(levels, gate, out, go, ac, am)
    lb, gb = fr.bound_bwd(levels, gate, go, ac, am)
    assert fr.max_ratio(gg, gg64, gb) <= 1.0
    for got, want, bound in zip(gl, gl64, lb):
        assert fr.max_ratio(got, want, bound) <= 1.0


def test_the_level_gradient_is_the_adjoint_of_the_upsampling():
    """In fp64 the composition's level gradient is the transposed resampling of w_l * grad_out."""
    levels, gate, go = inputs(4, 2, 3, 9, 10, ((3, 4), (9, 10), (12, 5)))
    _, gl64, _ = autograd64(levels, gate, go, False, 0)
    w = gate.double().abs() / gate.double().abs().sum(1, keepdim=True)
    for l, x in enumerate(levels):
        want = fr.adjoint(w[:, l:l + 1] * go.double(), x.shape[2:], False, 0)
        torch.testing.assert_close(gl64[l], want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('ac,am', ALIGN[:3])
def test_gradcheck_of_the_composition(ac, am):
    levels, gate, _ = inputs(3, 1, 2, 5, 6, ((2, 3), (5, 6), (7, 4)))
    xs = [x.double().requires_grad_(True) for x in levels]
    g = gate.double().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda g, *xs: fr.compose(xs, g, ac, am), (g, *xs))


# ---- 2. the bounds against torch's own fp32 composition ----------------------------------------------------------------------
@pytest.mark.parametrize('scale', [1.0, 1e3, 1e-3])
def test_bounds_hold_for_the_fp32_composition(scale):
    B, C, H, W, hws = 2, 24, 33, 47, ((1, 1), (2, 3), (4, 5), (8, 11), (33, 47))
    levels, gate, go = inputs(9, B, C, H, W, hws)
    levels, gate, go = [x * scale for x in levels], gate * scale, go * scale
    o64, gl64, gg64 = autograd64(levels, gate, go, False, 0)
    xs = [x.clone().requires_grad_(True) for x in levels]
    g = gate.clone().requires_grad_(True)
    out = fr.compose(xs, g, False, 0)
    out.backward(go)
    assert fr.max_ratio(out.detach(), o64, fr.bound_fwd(levels, gate, False, 0)) <= 1.0
    lb, gb = fr.bound_bwd(levels, gate, go, False, 0)
    assert fr.max_ratio(g.grad, gg64, gb) <= 1.0
    for x, want, bound in zip(xs, gl64, lb):
        assert fr.max_ratio(x.grad, want, bound) <= 1.0


# ---- 3. the anchors against torch ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ac,am', [(True, 1), (False, 0)])
def test_a_constant_gate_is_the_mean_of_the_interpolated_levels(ac, am):
    B, C, H, W, hws = 2, 5, 17, 23, ((1, 2), (2, 3), (4, 6), (9, 12))
    levels, _, _ = inputs(5, B, C, H, W, hws)
    gate = torch.full((B, len(hws), H, W), -0.4)
    got = fr.fwd_torch(levels, gate, ac, am)
    # torch's fp32 interpolation forms its coordinates in fp32 as the kernels do (in fp64 they move by an ulp); it is one more
    # fp32 evaluation of the same blend, within the same bound of the exact mean, so the two are within twice the bound
    want = sum(F.interpolate(x, size=(H, W), mode='bilinear', align_corners=ac).double() for x in levels) / len(hws)
    assert fr.max_ratio(got, want, fr.bound_fwd(levels, gate, ac, am)) <= 2.0


def test_a_full_resolution_level_under_a_one_hot_gate_is_itself():
    B, C, H, W = 2, 3, 9, 13
    levels, _, _ = inputs(6, B, C, H, W, ((2, 3), (H, W), (4, 4)))
    gate = torch.zeros(B, 3, H, W)
    gate[:, 1] = rand(7, B, H, W).abs() + 0.1
    for ac, am in ALIGN:
        got = fr.fwd_torch(levels, gate, ac, am)
        assert torch.equal(got, levels[1])
        assert torch.equal(F.interpolate(levels[1], size=(H, W), mode='bilinear', align_corners=ac), levels[1])


# ---- 4. the Python surface -------------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    x, y, g = torch.rand(1, 4, 3, 5), torch.rand(1, 4, 6, 2), torch.rand(1, 2, 6, 5)
    for args in [(x, g), ([], g[:, :0]), ([x] * 9, torch.rand(1, 9, 6, 5)), ([x, y], g[0]), ([x, y[0]], g),
                 ([x, y], torch.rand(1, 3, 6, 5)), ([x, torch.rand(1, 3, 6, 2)], g), ([x, torch.rand(2, 4, 6, 2)], g),
                 ([x, torch.rand(1, 4, 0, 2)], g), ([x, y], torch.rand(1, 2, 0, 5)), ([x, 'y'], g), ((x, y), g, True, 2),
                 ((x, y), g, True, True)]:
        with pytest.raises(ValueError):
            cspn_b200.affinity_fuse2d(*args)
    with pytest.raises(RuntimeError, match='fp32'):
        cspn_b200.affinity_fuse2d([x, y.double()], g)
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_fuse2d([x, y], g)
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_fuse2d((x.clone().requires_grad_(True), y), g, False, 0)


def test_sizes_the_c_abi_cannot_take_are_refused_before_anything_is_allocated():
    x = torch.empty(1, 1, 2, 2, device='meta')
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.affinity_fuse2d([x], torch.empty(1, 1, 1 << 16, 1 << 15, device='meta'))
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.affinity_fuse2d([torch.empty(1, 1, 1 << 16, 1 << 15, device='meta')], torch.empty(1, 1, 4, 4, device='meta'))


# ---- 5. the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def test_workspace_bytes():
    L = _lib.lib()
    hw = (ctypes.c_int * 4)(2, 3, 16, 5)
    # the weight planes B*L*H*W, then the row pass B*C*H*w_l per level
    assert L.cspn_affinity_fuse2d_bwd_workspace_bytes(2, 3, 7, 9, 2, hw) == 4 * (2 * 2 * 7 * 9 + 2 * 3 * 7 * (3 + 5))
    for bad in ((0, 3, 7, 9, 2, hw), (2, 3, 7, 9, 0, hw), (2, 3, 7, 9, 9, hw), (2, 3, 7, 9, 2, None),
                (2, 3, 7, 9, 2, (ctypes.c_int * 4)(2, 0, 1, 1))):
        assert L.cspn_affinity_fuse2d_bwd_workspace_bytes(*bad) == 0


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 16384)()
    base = ctypes.cast(buf, ctypes.c_void_p).value

    def at(k, off=0):                                    # 1024 floats apart
        return ctypes.c_void_p(base + k * 4096 + off)

    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, H=4, W=5)                     # levels 2x2x3 = 12 and 2x4x5 = 40 floats, gate 40, out 40

    def arr(*ps):
        return (ctypes.c_void_p * len(ps))(*[p.value if p is not None else None for p in ps])

    def fw(lv=(at(0), at(1)), hw=(2, 3, 4, 5), g=at(2), o=at(3), nl=2, ac=1, am=1, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_fuse2d_fwd_f32(None if lv is None else arr(*lv), None if hw is None else (ctypes.c_int * len(hw))(*hw),
                                              g, o, *v.values(), nl, ac, am, None)

    def bw(lv=(at(0), at(1)), hw=(2, 3, 4, 5), g=at(2), o=at(3), go=at(4), gl=(at(5), at(6)), gg=at(7), nl=2, ac=1, am=1,
           ws=at(8), wsb=1 << 14, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_fuse2d_bwd_f32(None if lv is None else arr(*lv), None if hw is None else (ctypes.c_int * len(hw))(*hw),
                                              g, o, go, None if gl is None else arr(*gl), gg, *v.values(), nl, ac, am, ws, wsb, None)

    for call in (fw, bw):
        for k in ok:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        assert call(nl=0) == -1 and b'levels' in L.cspn_last_error()
        assert call(nl=9, hw=(1,) * 18, lv=(at(0),) * 9) == -1 and b'levels' in L.cspn_last_error()
        assert call(hw=None) == -1 and b'level_hw' in L.cspn_last_error()
        assert call(hw=(2, 0, 4, 5)) == -1 and b'level 0' in L.cspn_last_error()
        assert call(lv=None) == -1 and b'pointer array' in L.cspn_last_error()
        assert call(lv=(at(0), None)) == -1 and b'null' in L.cspn_last_error()
        assert call(lv=(at(0), odd)) == -1 and b'aligned' in L.cspn_last_error()
        for flag in ('ac', 'am'):
            assert call(**{flag: 2}) == -1 and call(**{flag: -1}) == -1 and b'align' in L.cspn_last_error()
        assert call(g=None) == -1 and call(o=odd) == -1
        assert call(H=1 << 16, W=1 << 15) == -4 and b'2^31' in L.cspn_last_error()
        assert call(hw=(2, 3, 1 << 16, 1 << 15)) == -4 and b'2^31' in L.cspn_last_error()
    assert bw(gl=None) == -1 and b'pointer array' in L.cspn_last_error()
    assert bw(gl=(at(5), odd)) == -1 and b'aligned' in L.cspn_last_error()
    assert bw(go=None) == -1 and bw(gg=odd) == -1
    assert bw(ws=None) == -2 and bw(wsb=10) == -2 and bw(ws=odd) == -2 and b'workspace' in L.cspn_last_error()
    # an output may overlap neither an input nor another output (aliased levels are checked on device buffers)
    assert fw(o=at(0, 40)) == -1 and b'out overlaps levels[0]' in L.cspn_last_error()
    assert fw(o=at(2, 4 * 39)) == -1 and b'out overlaps gate' in L.cspn_last_error()
    for over, what in ((dict(gg=at(2, 4 * 39)), b'grad_gate overlaps gate'), (dict(gl=(at(1), at(6))), b'grad_levels[0] overlaps levels[1]'),
                       (dict(gl=(at(5), at(5, 40))), b'grad_levels[1] overlaps grad_levels[0]'),
                       (dict(gl=(at(5), at(4, 4 * 39))), b'grad_levels[1] overlaps grad_out'),
                       (dict(ws=at(3, 4 * 39)), b'the workspace overlaps out'),
                       (dict(ws=at(7, 4 * 39)), b'the workspace overlaps grad_gate')):
        assert bw(**over) == -1 and what in L.cspn_last_error(), (over, L.cspn_last_error())
    assert L.cspn_last_launches() == 0


# ---- 6. the dispatcher ops -------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert ('affinity_fuse2d(Tensor[] levels, Tensor gate, bool align_corners, int align_mode) -> Tensor'
            in str(ops.affinity_fuse2d.default._schema))
    assert ('affinity_fuse2d_backward(Tensor[] levels, Tensor gate, Tensor out, Tensor grad_out, bool align_corners, '
            'int align_mode) -> (Tensor[], Tensor)' in str(ops.affinity_fuse2d_backward.default._schema))
    with FakeTensorMode():
        levels = [torch.empty(4, 32, 64 // p, 128 // p, device='cuda') for p in (64, 32, 16, 8)]
        gate = torch.empty(4, 4, 64, 128, device='cuda')              # PSMNet's training crop at quarter resolution
        out = ops.affinity_fuse2d(levels, gate, False, 0)
        assert out.shape == (4, 32, 64, 128) and out.dtype == torch.float32 and out.device == gate.device
        gl, gg = ops.affinity_fuse2d_backward(levels, gate, out, out, False, 0)
        assert [tuple(t.shape) for t in gl] == [tuple(x.shape) for x in levels] and gg.shape == gate.shape
        assert cspn_b200.affinity_fuse2d(levels, gate, False, 0).shape == out.shape   # the function takes the op route
        with pytest.raises(Exception):
            ops.affinity_fuse2d(levels[:3], gate, False, 0)
        with pytest.raises(Exception):
            ops.affinity_fuse2d(levels, gate, False, 2)
