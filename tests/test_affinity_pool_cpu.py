"""CPU tests of affinity pooling (affinity_pool2d; DESIGN.md section 4.17): the order restatement of
tests/affinity_pool_reference.py against the fp64 composition and its autograd, gradcheck, the a-priori bounds against
torch's fp32 composition, the anchors (a constant gate is avg_pool2d, a one-hot gate copies its pixel, one-term windows
return their term), the Python and C ABI refusals before any device work, the argtypes and the dispatcher registration."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import affinity_pool_reference as ar
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn_affinity_pool2d_fwd_f32', 'cspn_affinity_pool2d_bwd_f32')
# (B, C, H, W, ks): remainders in both axes, p = 1, p = min(H, W), repeated and unordered sizes, L = 1 and L = 8
SHAPES = [(2, 3, 7, 9, (2, 3)), (1, 4, 5, 5, (5, 1)), (2, 2, 11, 6, (4, 1, 6, 4)), (1, 1, 6, 13, (3,)),
          (1, 3, 9, 10, (1, 2, 3, 4, 5, 6, 7, 8)), (2, 5, 8, 8, (8, 4, 2, 2))]


def rand(seed, *shape, dtype=torch.float64):
    """fp32 values (so that the fp64 references see the fp32 kernels' inputs exactly) in `dtype`."""
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dtype)


def inputs(seed, B, C, H, W, ks, dtype=torch.float64):
    feat, gate = rand(seed, B, C, H, W, dtype=dtype), rand(seed + 1, B, len(ks), H, W, dtype=dtype)
    grads = tuple(rand(seed + 2 + l, B, C, H // p, W // p, dtype=dtype) for l, p in enumerate(ks))
    return feat, gate, grads


def autograd64(feat, gate, ks, grads):
    f, g = feat.detach().double().clone().requires_grad_(True), gate.detach().double().clone().requires_grad_(True)
    outs = ar.compose(f, g, ks)
    torch.autograd.backward(outs, [t.double() for t in grads])
    return tuple(o.detach() for o in outs), f.grad, g.grad


# ---- 1. the restatement is the composition and its autograd -------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,ks', SHAPES)
def test_order_restatement_against_the_fp64_composition(B, C, H, W, ks):
    feat, gate, grads = inputs(B * 13 + W, B, C, H, W, ks)
    outs, gf, gg = autograd64(feat, gate, ks, grads)
    # in fp64 the restatement is the composition and its autograd
    for a, b in zip(ar.fwd_torch(feat, gate, ks), outs):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    for a, b in zip(ar.bwd_torch(feat, gate, ks, outs, grads), (gf, gg)):
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
    # in fp32 it is within the a-priori bounds
    f32, g32, go32 = feat.float(), gate.float(), tuple(t.float() for t in grads)
    o32 = ar.fwd_torch(f32, g32, ks)
    for got, want, bound in zip(o32, outs, ar.bound_fwd(f32, g32, ks)):
        assert ar.max_ratio(got, want, bound) <= 1.0
    for got, want, bound in zip(ar.bwd_torch(f32, g32, ks, o32, go32), (gf, gg), ar.bound_bwd(f32, g32, ks, go32)):
        assert ar.max_ratio(got, want, bound) <= 1.0


@pytest.mark.parametrize('B,C,H,W,ks', SHAPES[:4])
def test_gradcheck_of_the_composition(B, C, H, W, ks):
    feat, gate, _ = inputs(3, B, C, H, W, ks)
    feat.requires_grad_(True)
    gate.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda f, g: ar.compose(f, g, ks), (feat, gate))


# ---- 2. the bounds against torch's own fp32 composition and its autograd ----------------------------------------------------
@pytest.mark.parametrize('scale', [1.0, 1e3, 1e-3])
def test_bounds_hold_for_the_fp32_composition(scale):
    B, C, H, W, ks = 2, 24, 37, 45, (16, 8, 5, 3, 1)
    feat, gate, grads = inputs(9, B, C, H, W, ks)
    feat, gate = feat * scale, gate * scale
    grads = tuple(g * scale for g in grads)
    outs, gf, gg = autograd64(feat, gate, ks, grads)
    f32, g32 = feat.float().requires_grad_(True), gate.float().requires_grad_(True)
    o32 = ar.compose(f32, g32, ks)
    torch.autograd.backward(o32, [t.float() for t in grads])
    for got, want, bound in zip(o32, outs, ar.bound_fwd(feat.float(), gate.float(), ks)):
        assert ar.max_ratio(got.detach(), want, bound) <= 1.0
    for got, want, bound in zip((f32.grad, g32.grad), (gf, gg),
                                ar.bound_bwd(feat.float(), gate.float(), ks, tuple(t.float() for t in grads))):
        assert ar.max_ratio(got, want, bound) <= 1.0


# ---- 3. the anchors --------------------------------------------------------------------------------------------------------------
def test_a_constant_gate_is_avg_pool2d():
    feat = rand(4, 2, 6, 19, 23, dtype=torch.float32)
    ks = (8, 4, 3, 1)
    gate = torch.full((2, len(ks), 19, 23), -0.75)
    for got, p, bound in zip(ar.fwd_torch(feat, gate, ks), ks, ar.bound_fwd(feat, gate, ks)):
        want = F.avg_pool2d(feat.double(), p)
        assert ar.max_ratio(got, want, bound) <= 1.0
        torch.testing.assert_close(got, F.avg_pool2d(feat, p), rtol=1e-5, atol=1e-6)


def test_a_one_hot_gate_copies_the_selected_pixel():
    B, C, H, W, p = 2, 3, 13, 17, 4
    feat = rand(5, B, C, H, W, dtype=torch.float32)
    gen = torch.Generator().manual_seed(6)
    Hl, Wl = H // p, W // p
    pick = torch.randint(0, p * p, (B, Hl, Wl), generator=gen)
    gate = torch.zeros(B, 1, H, W)
    win = ar.windows(gate, p)
    val = torch.rand(B, Hl, Wl, generator=gen) * 4 - 2 + 3 * torch.sign(torch.rand(B, Hl, Wl, generator=gen) - 0.5)
    for b in range(B):
        for i in range(Hl):
            for j in range(Wl):
                win[b, 0, i, pick[b, i, j] // p, j, pick[b, i, j] % p] = val[b, i, j]
    gate[:, :, :Hl * p, :Wl * p] = win.reshape(B, 1, Hl * p, Wl * p)
    out, = ar.fwd_torch(feat, gate, (p,))
    want = ar.windows(feat, p).reshape(B, C, Hl, p, Wl, p).permute(0, 1, 2, 4, 3, 5).reshape(B, C, Hl, Wl, p * p)
    want = torch.gather(want, 4, pick[:, None, :, :, None].expand(B, C, Hl, Wl, 1))[..., 0]
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))


def test_one_term_windows_return_their_term():
    """p = 1: w = a / a = 1, so every level is feat bit for bit (-0.0 included), and every sum starts from its first term."""
    feat = torch.tensor([[[[-0.0, 1.5, -2.0], [3.0, 1e-40, -7.25]]]])
    gate = torch.tensor([[[[0.5, -3.0, 1e-42], [2.0, 7.0, -1.0]]]])
    out, = ar.fwd_torch(feat, gate, (1,))
    assert torch.equal(out.view(torch.int32), feat.view(torch.int32))
    gf, gg = ar.bwd_torch(feat, gate, (1,), (out,), (-torch.zeros_like(feat),))
    assert torch.signbit(gf).all()                             # w * -0.0 = -0.0: the sum of one term is that term


def test_pack_layout():
    B, C, H, W, ks = 2, 3, 7, 9, (2, 3, 7)
    levels = tuple(torch.arange(B * C * (H // p) * (W // p), dtype=torch.float32).view(B, C, H // p, W // p) + 1000 * l
                   for l, p in enumerate(ks))
    flat = ar.pack(levels)
    assert flat.numel() == B * C * sum((H // p) * (W // p) for p in ks)
    assert all(torch.equal(a, b) for a, b in zip(ar.unpack(flat, B, C, H, W, ks), levels))


# ---- 4. the Python surface -------------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    f, g = torch.rand(1, 4, 6, 5), torch.rand(1, 2, 6, 5)
    for args in [(torch.rand(4, 6, 5), g, (2, 3)), (f, torch.rand(2, 6, 5), (2, 3)), (f, g, (2,)), (f, g, (2, 3, 1)),
                 (f, g, ()), (f, g, (0, 2)), (f, g, (2, 6)), (f, g, (2, 2.0)), (f, g, (True, 2)), (f, g, 2), (f, g, '23'),
                 (torch.rand(1, 0, 6, 5), g, (2, 3)), (f, torch.rand(2, 2, 6, 5), (2, 3)),
                 (f, torch.rand(1, 9, 6, 5), tuple(range(1, 10)))]:
        with pytest.raises(ValueError):
            cspn_b200.affinity_pool2d(*args)
    with pytest.raises(RuntimeError, match='fp32'):
        cspn_b200.affinity_pool2d(f.double(), g.double(), (2, 3))
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_pool2d(f, g, (2, 3))
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.affinity_pool2d(f.clone().requires_grad_(True), g, [2, 3])


def test_sizes_the_c_abi_cannot_take_are_refused_before_anything_is_allocated():
    f = torch.empty(1, 1, 1 << 16, 1 << 15, device='meta')
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.affinity_pool2d(f, torch.empty(1, 1, 1 << 16, 1 << 15, device='meta'), (2,))


# ---- 5. the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 8192)()
    base = ctypes.cast(buf, ctypes.c_void_p).value
    a, b, c, d, e, f = (ctypes.c_void_p(base + k * 4096) for k in range(6))   # 1024 floats apart
    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, H=4, W=5)                  # feat 40 floats, gate (L = 2) 40, out (p = 2, 3) 2 * (4 + 1) = 10

    def sizes(*ks):
        return (ctypes.c_int * len(ks))(*ks)

    def fw(ft=a, g=b, o=c, ks=(2, 3), nl=None, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_pool2d_fwd_f32(ft, g, o, *v.values(), (len(ks) if ks else 2) if nl is None else nl,
                                              None if ks is None else sizes(*ks), None)

    def bw(ft=a, g=b, o=c, go=d, gf=e, gg=f, ks=(2, 3), nl=None, **over):
        v = dict(ok, **over)
        return L.cspn_affinity_pool2d_bwd_f32(ft, g, o, go, gf, gg, *v.values(), (len(ks) if ks else 2) if nl is None else nl,
                                              None if ks is None else sizes(*ks), None)

    for call, ptrs in ((fw, ('ft', 'g', 'o')), (bw, ('ft', 'g', 'o', 'go', 'gf', 'gg'))):
        for k in ok:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for p in ptrs:
            assert call(**{p: None}) == -1 and b'null' in L.cspn_last_error()
            assert call(**{p: odd}) == -1 and b'aligned' in L.cspn_last_error()
        assert call(ks=None) == -1 and b'kernel_sizes' in L.cspn_last_error()
        for ks in ((2, 0), (5, 2), (-1,)):
            assert call(ks=ks) == -1 and b'min(H, W)' in L.cspn_last_error()
        assert call(ks=(1,) * 9) == -1 and b'levels' in L.cspn_last_error()
        assert call(ks=(2,), nl=0) == -1 and b'levels' in L.cspn_last_error()
        assert call(H=1 << 16, W=1 << 15, ks=(2,)) == -4 and b'2^31' in L.cspn_last_error()
        assert call(B=1 << 20, C=1 << 10, H=1 << 10, W=1 << 10, ks=(1,)) == -4 and b'grid' in L.cspn_last_error()
    # an output may overlap neither an input nor the other output; inputs may alias
    assert fw(o=a) == -1 and b'out overlaps feat' in L.cspn_last_error()
    assert fw(o=ctypes.c_void_p(base + 4096 + 4 * 39)) == -1 and b'out overlaps gate' in L.cspn_last_error()
    for over, what in ((dict(gf=a), b'grad_feat overlaps feat'), (dict(gg=ctypes.c_void_p(base + 4096 + 4 * 39)), b'grad_gate overlaps gate'),
                       (dict(gf=ctypes.c_void_p(base + 2 * 4096 + 4 * 9)), b'grad_feat overlaps out'),
                       (dict(gg=ctypes.c_void_p(base + 3 * 4096 + 4 * 9)), b'grad_gate overlaps grad_out'),
                       (dict(gg=ctypes.c_void_p(base + 4 * 4096 + 4 * 39)), b'grad_gate overlaps grad_feat')):
        assert bw(**over) == -1 and what in L.cspn_last_error()
    assert L.cspn_last_launches() == 0


# ---- 6. the dispatcher ops -------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert 'affinity_pool2d(Tensor feat, Tensor gate, int[] kernel_sizes) -> Tensor' in str(ops.affinity_pool2d.default._schema)
    assert ('affinity_pool2d_backward(Tensor feat, Tensor gate, Tensor out, Tensor grad_out, int[] kernel_sizes) -> '
            '(Tensor, Tensor)' in str(ops.affinity_pool2d_backward.default._schema))
    ks = [64, 32, 16, 8]
    with FakeTensorMode():
        feat = torch.empty(4, 128, 64, 128, device='cuda')           # PSMNet's training crop at quarter resolution
        gate = torch.empty(4, 4, 64, 128, device='cuda')
        flat = ops.affinity_pool2d(feat, gate, ks)
        assert flat.shape == (4 * 128 * (2 + 8 + 32 + 128),) and flat.dtype == torch.float32 and flat.device == feat.device
        gf, gg = ops.affinity_pool2d_backward(feat, gate, flat, flat, ks)
        assert gf.shape == feat.shape and gg.shape == gate.shape
        outs = cspn_b200.affinity_pool2d(feat, gate, ks)          # the function takes the op route
        assert [tuple(o.shape) for o in outs] == [(4, 128, 64 // p, 128 // p) for p in ks]
        with pytest.raises(Exception):
            ops.affinity_pool2d(feat, gate, [64, 32, 16])
        with pytest.raises(Exception):
            ops.affinity_pool2d(feat, gate, [64, 32, 16, 65])


def test_packed_lengths_fit_the_kernel_sizes():
    """The fake kernel's length is the C ABI's level-major buffer."""
    for H, W, ks in ((96, 312, (64, 32, 16, 8)), (136, 240, (64, 32, 16, 8)), (7, 9, (2, 3, 7))):
        n = sum((H // p) * (W // p) for p in ks)
        assert n == sum(np.prod(s[2:]) for s in [(1, 1, H // p, W // p) for p in ks])
