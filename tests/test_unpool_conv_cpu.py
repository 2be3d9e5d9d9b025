"""CPU tests of the guidance / depth head (Unpool + crop + 3x3 convolution, cspn_b200.unpool_conv3x3): the fp64 polyphase
restatement (tests/unpool_conv_reference.py) against torch's own op sequence, crops and IEEE footprint included; the C ABI's
signatures and argument errors; the Python validation; the module surface; the dispatcher registration."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import unpool_conv_reference as ur

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ('cspn_unpool_conv3x3_fwd_f32', 'cspn_unpool_conv3x3_bwd_workspace_bytes', 'cspn_unpool_conv3x3_bwd_f32')


def rand(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def same_nonfinite(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
            and np.array_equal(np.isneginf(a), np.isneginf(b)))


# ---- 1. the restatement is the op sequence -----------------------------------------------------------------------------
@pytest.mark.parametrize('B,Cin,h,w,Cout,H,W', [
    (2, 3, 5, 7, 4, 10, 14),       # no crop
    (2, 3, 5, 7, 4, 9, 14),        # H = 2h - 1
    (1, 2, 5, 7, 3, 9, 13),        # both odd
    (1, 1, 4, 6, 2, 8, 11),        # odd W
    (1, 2, 1, 1, 1, 1, 1),         # 1x1 output
    (1, 1, 1, 1, 2, 2, 2),         # 1x1 source, whole map
    (1, 2, 3, 1, 2, 5, 1),         # one column
    (1, 5, 6, 4, 3, 7, 3),         # deep crops
])
def test_restatement_equals_the_op_sequence(B, Cin, h, w, Cout, H, W):
    x, wt = rand(1, B, Cin, h, w), rand(2, Cout, Cin, 3, 3)
    ref = ur.op_sequence(x, wt, H, W).numpy()
    ours = ur.unpool_conv_numpy(x.numpy(), wt.numpy(), H, W)
    assert ours.shape == (B, Cout, H, W)
    np.testing.assert_allclose(ours, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('H,W', [(8, 10), (7, 9), (7, 10), (1, 1), (2, 1)])
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_ieee_footprint_of_a_non_finite_x(H, W, value):
    h, w = 4, 5
    for (i, j) in [(0, 0), (1, 2), (3, 4), (h - 1, 0), ((H - 1) // 2, (W - 1) // 2)]:
        x, wt = rand(3, 1, 2, h, w), rand(4, 3, 2, 3, 3)
        x[0, 1, i, j] = value
        ref = ur.op_sequence(x, wt, H, W).numpy()
        ours = ur.unpool_conv_numpy(x.numpy(), wt.numpy(), H, W)
        assert same_nonfinite(ours, ref), (i, j)
        fin = np.isfinite(ref)
        np.testing.assert_allclose(ours[fin], ref[fin], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('H,W', [(8, 10), (7, 9), (1, 1)])
@pytest.mark.parametrize('value', [float('nan'), float('inf'), float('-inf')])
def test_ieee_footprint_of_a_non_finite_weight(H, W, value):
    for co, ci, t in [(0, 0, 0), (1, 1, 4), (2, 0, 8), (1, 1, 5), (0, 1, 7)]:
        x, wt = rand(5, 2, 2, 4, 5), rand(6, 3, 2, 3, 3)
        wt[co, ci, t // 3, t % 3] = value
        ref = ur.op_sequence(x, wt, H, W).numpy()
        ours = ur.unpool_conv_numpy(x.numpy(), wt.numpy(), H, W)
        assert same_nonfinite(ours, ref), (co, ci, t)
        fin = np.isfinite(ref)
        np.testing.assert_allclose(ours[fin], ref[fin], rtol=1e-12, atol=1e-12)


def test_only_a_quarter_of_the_products_are_not_structural_zeros():
    """The claim the kernel rests on: with x = 1 and w = 1, an output sums as many ones as it has real taps (1, 2 or 4 per
    channel inside the map), 2.25 on average over a 2x2 block -- not 9."""
    x = torch.ones(1, 1, 6, 6, dtype=torch.float64)
    out = ur.op_sequence(x, torch.ones(1, 1, 3, 3, dtype=torch.float64), 12, 12)[0, 0]
    assert out[2:10:2, 2:10:2].eq(1).all() and out[3:11:2, 3:11:2].eq(4).all() and out[2:10:2, 3:11:2].eq(2).all()
    assert float(out[2:10, 2:10].mean()) == 2.25


# ---- 2. the C ABI -------------------------------------------------------------------------------------------------------
def header_signature(name):
    text = open(os.path.join(ROOT, 'include', 'cspn_b200.h')).read()
    m = re.search(r'CSPN_API\s+(int|size_t)\s+' + name + r'\s*\(([^)]*)\)', text)
    assert m, f'{name} is not declared'
    types = []
    for prm in m.group(2).split(','):
        prm = ' '.join(prm.split())
        if '*' in prm or prm.startswith('cspn_stream_t'):
            types.append(ctypes.c_void_p)
        elif prm.startswith('size_t'):
            types.append(ctypes.c_size_t)
        else:
            assert prm.startswith('int '), prm
            types.append(ctypes.c_int)
    return (ctypes.c_int if m.group(1) == 'int' else ctypes.c_size_t), types


@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 2)
    ok = dict(B=1, Cin=2, h=3, w=4, Cout=2, H=6, W=8)
    names = list(ok)

    def f(x=p, wt=p, o=p, **over):
        a = dict(ok, **over)
        return L.cspn_unpool_conv3x3_fwd_f32(x, wt, o, *[a[k] for k in names], None)

    def b(x=p, wt=p, go=p, gx=p, gw=p, ws=p, ws_bytes=1 << 30, **over):
        a = dict(ok, **over)
        return L.cspn_unpool_conv3x3_bwd_f32(x, wt, go, gx, gw, *[a[k] for k in names], ws, ws_bytes, None)

    for call in (f, b):
        for k in names:
            assert call(**{k: 0}) == -1 and call(**{k: -2}) == -1
        assert call(H=7) == -1 and call(W=9) == -1
        assert call(x=None) == -1 and call(wt=None) == -1
        assert b'null' in L.cspn_last_error()
        assert call(x=odd) == -1 and call(wt=odd) == -1
    assert f(o=None) == -1 and b(go=None) == -1
    assert b(gx=odd) == -1
    # a short or missing workspace is an error only when grad_weight is asked for
    need = L.cspn_unpool_conv3x3_bwd_workspace_bytes(*[ok[k] for k in names])
    assert need > 0
    assert b(ws=None) == -2 and b(ws_bytes=need - 1) == -2 and b(ws=odd) == -2
    assert L.cspn_last_launches() == 0
    # the launch grid: images go to gridDim.z
    assert f(B=65536) == -4 and b(B=65536) == -4


def test_workspace_is_the_partials_of_grad_weight_and_depends_on_the_shape_only():
    L = _lib.lib()
    for (B, Cin, h, w, Cout, H, W) in [(1, 64, 114, 152, 8, 228, 304), (8, 64, 176, 608, 1, 352, 1216), (2, 3, 5, 7, 24, 9, 13),
                                       (1, 1, 1, 1, 1, 1, 1)]:
        n = L.cspn_unpool_conv3x3_bwd_workspace_bytes(B, Cin, h, w, Cout, H, W)
        assert n > 0 and n % (4 * Cout * Cin * 9) == 0
        parts = n // (4 * Cout * Cin * 9)
        assert 1 <= parts <= -(-B * ((H + 1) // 2) * ((W + 1) // 2) // 32)
    assert L.cspn_unpool_conv3x3_bwd_workspace_bytes(1, 1, 2, 2, 1, 5, 4) == 0      # H > 2h
    assert L.cspn_unpool_conv3x3_bwd_workspace_bytes(0, 1, 2, 2, 1, 4, 4) == 0


# ---- 3. the Python surface ---------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    f = cspn_b200.unpool_conv3x3
    x, wt = torch.rand(1, 4, 5, 6), torch.rand(8, 4, 3, 3)
    for xx, ww, oh, ow in ((torch.rand(4, 5, 6), wt, 0, 0), (x, torch.rand(8, 3, 3, 3), 0, 0), (x, torch.rand(8, 4, 5, 5), 0, 0),
                           (x, wt, 11, 12), (x, wt, 10, 13), (x, wt, -1, 5)):
        with pytest.raises(ValueError):
            f(xx, ww, oh, ow)
    with pytest.raises(RuntimeError):
        f(x.double(), wt.double())
    for oh, ow in ((0, 0), (9, 11)):
        with pytest.raises(cspn_b200.CspnError):
            f(x, wt, oh, ow)
        with pytest.raises(cspn_b200.CspnError):
            f(x.requires_grad_(True), wt, oh, ow)
        x.requires_grad_(False)


def test_crop_rule_is_the_references():
    from cspn_b200.cspn import unpool_output_size
    assert unpool_output_size(114, 152, 228, 304) == (228, 304)
    assert unpool_output_size(176, 608, 352, 1216) == (352, 1216)
    assert unpool_output_size(5, 7, 9, 13) == (9, 13)
    assert unpool_output_size(5, 7, 0, 0) == (10, 14)
    assert unpool_output_size(5, 7, 9, 0) == (10, 14) and unpool_output_size(5, 7, 0, 13) == (10, 14)   # both or neither


def test_module_surface_matches_the_reference_head():
    M = cspn_b200.Simple_Gudi_UpConv_Block_Last_Layer
    m = M(64, 8, 228, 304)
    assert (m.oheight, m.owidth) == (228, 304)
    assert isinstance(m.conv1, nn.Conv2d) and m.conv1.bias is None
    assert (m.conv1.kernel_size, m.conv1.stride, m.conv1.padding) == ((3, 3), (1, 1), (1, 1))
    assert list(m.state_dict()) == ['conv1.weight'] and m.state_dict()['conv1.weight'].shape == (8, 64, 3, 3)
    assert [p.shape for p in m.parameters()] == [torch.Size([8, 64, 3, 3])] and list(m.buffers()) == []
    assert (M(64, 1).oheight, M(64, 1).owidth) == (0, 0)
    # a seeded construction draws the weights a plain nn.Conv2d (the reference's conv1) draws
    torch.manual_seed(7)
    a = M(64, 8, 228, 304)
    torch.manual_seed(7)
    ref = nn.Conv2d(64, 8, kernel_size=3, stride=1, padding=1, bias=False)
    assert torch.equal(a.conv1.weight, ref.weight)
    # a reference checkpoint of the head loads unchanged
    m.load_state_dict({'conv1.weight': ref.weight.detach().clone()})
    assert torch.equal(m.conv1.weight, ref.weight)
    with pytest.raises(ValueError):
        M(4, 2)(torch.rand(1, 3, 5, 5))


# ---- 4. the dispatcher ops ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert 'unpool_conv3x3(Tensor x, Tensor weight, int H, int W) -> Tensor' in str(ops.unpool_conv3x3.default._schema)
    assert ('Tensor grad_out, int H, int W, bool need_x, bool need_weight) -> (Tensor, Tensor)'
            in str(ops.unpool_conv3x3_backward.default._schema))
    with FakeTensorMode():
        x, wt = torch.empty(2, 64, 114, 152, device='cuda'), torch.empty(8, 64, 3, 3, device='cuda')
        out = ops.unpool_conv3x3(x, wt, 227, 303)
        assert out.shape == (2, 8, 227, 303) and out.dtype == torch.float32 and out.device == x.device
        gx, gw = ops.unpool_conv3x3_backward(x, wt, out, 227, 303, True, True)
        assert gx.shape == x.shape and gw.shape == wt.shape
        gx, gw = ops.unpool_conv3x3_backward(x, wt, out, 227, 303, False, True)
        assert gx.numel() == 0 and gw.shape == wt.shape
        out = cspn_b200.unpool_conv3x3(x, wt, 228, 304)          # the function takes the dispatcher route
        assert out.shape == (2, 8, 228, 304)
        with pytest.raises(Exception):
            ops.unpool_conv3x3(x, wt, 229, 304)
