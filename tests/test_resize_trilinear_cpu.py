"""CPU tests of resize_trilinear (the Paddle module's fluid.layers.resize_trilinear; DESIGN.md section 4.14): the fp32 and
fp64 restatements of tests/resize_reference.py against torch's F.interpolate in the two modes both have, the align_mode=1
example, downsampling, size-1 axes and the n_out == 1 convention, the fp64 adjoint against autograd, the Python argument
errors, the C ABI's refusals before any device work, and the dispatcher registration."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib

import resize_reference as rr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ('cspn_resize_trilinear_fwd_f32', 'cspn_resize_trilinear_bwd_workspace_bytes', 'cspn_resize_trilinear_bwd_f32')
SHARED = [(True, 1), (False, 0)]          # (align_corners, align_mode) that F.interpolate also has
MODES = [(True, 1), (False, 0), (False, 1)]


def ramp(in_size, axis, B=1, C=1):
    """x = the index along `axis` (a ramp): the output along that axis is its source coordinate."""
    shape = [1, 1, 1]
    shape[axis] = in_size[axis]
    x = np.arange(in_size[axis], dtype=np.float32).reshape(shape)
    return np.broadcast_to(x, (B, C, *in_size)).copy()


def rand(seed, *shape):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


# ---- 1. the restatements are F.interpolate in the modes both have ------------------------------------------------------
@pytest.mark.parametrize('in_size,out_size', [((4, 5, 6), (7, 9, 13)), ((7, 3, 9), (3, 8, 4)), ((48, 64, 128), (96, 128, 256)),
                                              ((5, 6, 7), (5, 6, 7)), ((2, 3, 17), (11, 2, 5))])
@pytest.mark.parametrize('align_corners,align_mode', SHARED)
def test_source_coordinates_are_atens(in_size, out_size, align_corners, align_mode):
    for axis in range(3):
        x = ramp(in_size, axis)
        ref = F.interpolate(torch.from_numpy(x), size=out_size, mode='trilinear', align_corners=align_corners).numpy()
        s = rr.ramp_output(in_size[axis], out_size[axis], align_corners, align_mode)
        shape = [1, 1, 1, 1, 1]
        shape[2 + axis] = -1
        want = np.broadcast_to(s.reshape(shape), ref.shape)
        tol = 4 * np.spacing(np.float32(in_size[axis]))
        np.testing.assert_allclose(ref, want, rtol=0, atol=tol)
        np.testing.assert_allclose(rr.forward_fp32(x, out_size, align_corners, align_mode), want, rtol=0, atol=tol)
        np.testing.assert_allclose(rr.forward_fp64(x, out_size, align_corners, align_mode), want, rtol=0, atol=tol)


@pytest.mark.parametrize('in_size,out_size', [((4, 5, 6), (7, 9, 13)), ((7, 3, 9), (3, 8, 4)), ((3, 2, 2), (9, 7, 2))])
@pytest.mark.parametrize('align_corners,align_mode', SHARED)
def test_restatements_equal_interpolate_on_random_volumes(in_size, out_size, align_corners, align_mode):
    x = rand(1, 2, 3, *in_size)
    ref = F.interpolate(torch.from_numpy(x).double(), size=out_size, mode='trilinear', align_corners=align_corners).numpy()
    # torch forms fp64 coordinates here, ours are fp32: they differ by a few fp32 ulps of the size, times |x1 - x0|
    tol = 8 * max(in_size) * rr.U * 2 * np.abs(x).max()
    for got in (rr.forward_fp32(x, out_size, align_corners, align_mode), rr.forward_fp64(x, out_size, align_corners, align_mode)):
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=0, atol=tol)


# ---- 2. the semantics ---------------------------------------------------------------------------------------------------
def test_align_mode_1_example_4_to_7():
    x = ramp((1, 1, 4), 2)
    want = np.array([0, 4, 8, 12, 16, 20, 21]) / 7.0
    want[-1] = 3.0
    for f in (rr.forward_fp32, rr.forward_fp64):
        got = f(x, (1, 1, 7), False, 1)[0, 0, 0, 0]
        np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)


def test_downsampling_7_to_3_leaves_inputs_unread():
    for align_corners, align_mode in MODES:
        i0, i1, l0, l1 = rr.taps(7, 3, align_corners, align_mode)
        read = set(i0) | set(i1[l1 != 0])
        assert len(read) < 7
        g = rand(2, 1, 1, 3, 3, 3)
        gx = rr.backward_fp64(g, (7, 7, 7), align_corners, align_mode)
        unread = [i for i in range(7) if i not in set(i0) | set(i1)]
        assert unread and not gx[:, :, unread].any() and not gx[:, :, :, unread].any()
        np.testing.assert_array_equal(rr.backward_fp32(g, (7, 7, 7), align_corners, align_mode)[:, :, unread], 0)
    # align_corners: r = 3, outputs read 0, 3 and 6
    i0, i1, l0, l1 = rr.taps(7, 3, True)
    assert list(i0) == [0, 3, 6] and not l1.any()


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_size_one_axes(align_corners, align_mode):
    x = rand(3, 2, 2, 1, 4, 5)
    # n_in == 1: every output reads the one voxel, and both of its taps do
    out = rr.forward_fp64(x, (6, 4, 5), align_corners, align_mode)
    same = rr.forward_fp64(x, (1, 4, 5), align_corners, align_mode)
    np.testing.assert_allclose(out, np.broadcast_to(same, out.shape), rtol=1e-7)
    # n_out == 1: r = 0, so the output is the first voxel in every mode (F.interpolate takes the midpoint without
    # align_corners)
    for axis in range(3):
        x = rand(4 + axis, 1, 2, 5, 6, 7)
        size = [5, 6, 7]
        size[axis] = 1
        got = rr.forward_fp32(x, tuple(size), align_corners, align_mode)
        np.testing.assert_array_equal(got, np.take(x, [0], axis=2 + axis))
        if not align_corners and axis == 0:
            torch_out = F.interpolate(torch.from_numpy(x), size=tuple(size), mode='trilinear', align_corners=False).numpy()
            assert not np.allclose(torch_out, got)


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_fp32_restatements_within_their_bounds(align_corners, align_mode):
    for in_size, out_size in [((5, 6, 7), (9, 13, 17)), ((9, 8, 6), (4, 3, 5)), ((3, 4, 5), (12, 16, 20))]:
        x = rand(5, 2, 1, *in_size)
        err = np.abs(rr.forward_fp32(x, out_size, align_corners, align_mode) - rr.forward_fp64(x, out_size, align_corners, align_mode))
        assert (err <= rr.bound_fwd(rr.forward_fp64(np.abs(x), out_size, align_corners, align_mode))).all()
        g = rand(6, 2, 1, *out_size)
        err = np.abs(rr.backward_fp32(g, in_size, align_corners, align_mode) - rr.backward_fp64(g, in_size, align_corners, align_mode))
        k = rr.bound_bwd(in_size, out_size, align_corners, align_mode)
        assert (err <= k * rr.backward_fp64(np.abs(g), in_size, align_corners, align_mode)).all()


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_the_outputs_that_read_an_input_form_one_range(align_corners, align_mode):
    for n_in, n_out in [(48, 192), (64, 256), (128, 512), (7, 3), (4, 7), (1, 5), (5, 1), (33, 100), (100, 33)]:
        i0, i1, _, _ = rr.taps(n_in, n_out, align_corners, align_mode)
        assert (np.diff(i0) >= 0).all() and i0.max() <= n_in - 1
        for i in range(n_in):
            readers = np.flatnonzero((i0 == i) | (i1 == i))
            if readers.size:
                assert (np.diff(readers) == 1).all()


# ---- 3. the adjoint -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_gradcheck_of_the_port(align_corners, align_mode):
    x = torch.randn(1, 2, 3, 4, 2, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: rr.resize_torch(t, (5, 3, 4), align_corners, align_mode), (x,))


@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('in_size,out_size', [((3, 4, 5), (7, 9, 11)), ((7, 6, 5), (3, 2, 4)), ((1, 4, 3), (3, 1, 8))])
def test_fp64_adjoint_is_autograd(align_corners, align_mode, in_size, out_size):
    x = torch.randn(2, 3, *in_size, dtype=torch.float64, requires_grad=True)
    g = torch.randn(2, 3, *out_size, dtype=torch.float64)
    rr.resize_torch(x, out_size, align_corners, align_mode).backward(g)
    np.testing.assert_allclose(rr.backward_fp64(g.numpy(), in_size, align_corners, align_mode), x.grad.numpy(), rtol=1e-12,
                               atol=1e-12)
    # and the fp32 gather order computes the same sums
    np.testing.assert_allclose(rr.backward_fp32(g.float().numpy(), in_size, align_corners, align_mode), x.grad.numpy(),
                               rtol=1e-5, atol=1e-5)


# ---- 4. the Python surface ----------------------------------------------------------------------------------------------
def test_output_size_rules():
    from cspn_b200.cspn import resize_output_size
    assert resize_output_size((48, 64, 128), out_shape=(96, 128, 256)) == (96, 128, 256)
    assert resize_output_size((48, 64, 128), scale=2) == (96, 128, 256)
    assert resize_output_size((5, 7, 9), scale=0.5) == (2, 3, 4)                  # truncation
    assert resize_output_size((5, 7, 9), scale=1.3) == (6, 9, 11)
    assert resize_output_size((5, 7, 9), out_shape=[np.int64(2), 3, 4]) == (2, 3, 4)
    for kw in (dict(), dict(out_shape=(2, 3, 4), scale=2.0), dict(out_shape=(2, 3)), dict(out_shape=(2, 3, 0)),
               dict(out_shape=(2.0, 3, 4)), dict(out_shape=(True, 3, 4)), dict(scale=0), dict(scale=-1.0),
               dict(scale=0.1), dict(scale=True), dict(scale='2')):
        with pytest.raises(ValueError):
            resize_output_size((5, 7, 9), **kw)


def test_python_validation_and_cpu_tensors_are_refused():
    f = cspn_b200.resize_trilinear
    x = torch.rand(1, 2, 3, 4, 5)
    for args, kw in [((torch.rand(2, 3, 4, 5),), dict(scale=2.0)), ((x,), dict()), ((x,), dict(out_shape=(1, 2, 3), scale=1.0)),
                     ((x,), dict(scale=2.0, align_mode=2)), ((x,), dict(scale=2.0, align_mode=-1)),
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
    """Sizes are narrowed to C int on the way down: a size >= 2^31, or a slice of >= 2^31 elements, is refused first (the
    tensors stay on the meta device, so nothing is allocated and nothing runs)."""
    from cspn_b200.cspn import _check_resize_sizes
    _check_resize_sizes((2, 3, 48, 64, 128), (192, 256, 512))
    _check_resize_sizes((2, 3, (1 << 11) - 1, 1 << 10, 1 << 10), ((1 << 11) - 1, 1 << 10, 1 << 10))
    for in_shape, out_size in [((1, 1, 2, 2, 2), (2 ** 32 + 1, 1, 1)), ((1, 1, 2, 2, 2), (1 << 11, 1 << 10, 1 << 10)),
                               ((1, 1, 1 << 11, 1 << 10, 1 << 10), (2, 2, 2)), ((1 << 31, 1, 2, 2, 2), (2, 2, 2)),
                               ((1, 2 ** 32, 2, 2, 2), (2, 2, 2))]:
        with pytest.raises(cspn_b200.CspnError):
            _check_resize_sizes(in_shape, out_size)
    x = torch.empty(1, 1, 2, 2, 2, device='meta')
    with pytest.raises(cspn_b200.CspnError, match='2\\^31'):
        cspn_b200.resize_trilinear(x, (2 ** 32 + 1, 1, 1))


# ---- 5. the C ABI -------------------------------------------------------------------------------------------------------
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
    buf = (ctypes.c_float * 4096)()
    base = ctypes.cast(buf, ctypes.c_void_p).value
    a, b = ctypes.c_void_p(base), ctypes.c_void_p(base + 8192)       # 2048 floats apart
    w = ctypes.c_void_p(base + 4096)                                  # a workspace clear of both
    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, D=3, H=4, W=5, Do=6, Ho=7, Wo=8, ac=1, am=1)    # x 120 floats, out 672 floats
    names = list(ok)

    def f(x=a, o=b, **over):
        v = dict(ok, **over)
        return L.cspn_resize_trilinear_fwd_f32(x, o, *[v[k] for k in names], None)

    def g(go=b, gx=a, ws=w, ws_bytes=1 << 20, **over):
        v = dict(ok, **over)
        return L.cspn_resize_trilinear_bwd_f32(go, gx, *[v[k] for k in names], ws, ws_bytes, None)

    for call, src, dst in ((f, 'x', 'o'), (g, 'go', 'gx')):
        for k in names[:8]:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for k in ('ac', 'am'):
            assert call(**{k: 2}) == -1 and call(**{k: -1}) == -1
        assert call(**{src: None}) == -1 and call(**{dst: None}) == -1
        assert b'null' in L.cspn_last_error()
        assert call(**{src: odd}) == -1 and call(**{dst: odd}) == -1
        # >= 2^31 elements per (B*C) slice, in the input or in the output
        assert call(D=1 << 11, H=1 << 10, W=1 << 10) == -4 and call(Do=1 << 11, Ho=1 << 10, Wo=1 << 10) == -4
        assert b'2^31' in L.cspn_last_error()
        # one element fewer passes the size check: the call then stops at the next check, the overlap of src and dst
        # (every call here is refused before anything could be launched)
        assert call(D=(1 << 11) - 1, H=1 << 10, W=1 << 10, **{src: a, dst: a}) == -1 and b'overlaps' in L.cspn_last_error()
        assert call(Do=(1 << 11) - 1, Ho=1 << 10, Wo=1 << 10, **{src: a, dst: a}) == -1 and b'overlaps' in L.cspn_last_error()
    # the destination must not overlap the source: same base, a one-float overlap at either end, and an exact neighbour
    xs, os_ = 4 * 2 * 60, 4 * 2 * 336
    assert f(x=a, o=a) == -1 and b'overlaps' in L.cspn_last_error()
    assert f(x=a, o=ctypes.c_void_p(base + xs - 4)) == -1 and f(x=ctypes.c_void_p(base + os_ - 4), o=a) == -1
    assert g(go=a, gx=ctypes.c_void_p(base + os_ - 4)) == -1 and g(go=ctypes.c_void_p(base + xs - 4), gx=a) == -1
    assert f(x=ctypes.c_void_p(base + (1 << 40)), o=ctypes.c_void_p(base + (1 << 40) + xs), B=1 << 30, C=1 << 3) == -1
    # a missing, short or misaligned workspace
    need = L.cspn_resize_trilinear_bwd_workspace_bytes(3, 4, 5, 6, 7, 8)
    assert need == 8 * (3 + 4 + 5 + 6 + 7 + 8)
    assert g(ws=None) == -2 and g(ws_bytes=need - 1) == -2 and g(ws=ctypes.c_void_p(base + 4100)) == -2
    # the workspace must not overlap grad_x or grad_out: the prep kernel would overwrite them before the gather
    assert g(ws=a) == -1 and b'workspace overlaps grad_x' in L.cspn_last_error()
    assert g(ws=ctypes.c_void_p(base + 8192 + 2688 - 8)) == -1 and b'workspace overlaps grad_out' in L.cspn_last_error()
    assert L.cspn_last_launches() == 0
    assert L.cspn_resize_trilinear_bwd_workspace_bytes(0, 4, 5, 6, 7, 8) == 0
    assert L.cspn_resize_trilinear_bwd_workspace_bytes(3, 4, 5, 6, 7, -1) == 0


# ---- 6. the dispatcher ops ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert ('resize_trilinear(Tensor input, int D, int H, int W, bool align_corners, int align_mode) -> Tensor'
            in str(ops.resize_trilinear.default._schema))
    assert ('resize_trilinear_backward(Tensor grad_out, int in_D, int in_H, int in_W, bool align_corners, int align_mode) '
            '-> Tensor' in str(ops.resize_trilinear_backward.default._schema))
    with FakeTensorMode():
        x = torch.empty(4, 1, 48, 64, 128, device='cuda')
        out = ops.resize_trilinear(x, 192, 256, 512, True, 1)
        assert out.shape == (4, 1, 192, 256, 512) and out.dtype == torch.float32 and out.device == x.device
        assert ops.resize_trilinear_backward(out, 48, 64, 128, True, 1).shape == x.shape
        assert cspn_b200.resize_trilinear(x, scale=2.0).shape == (4, 1, 96, 128, 256)   # the function takes the op route
        with pytest.raises(Exception):
            ops.resize_trilinear(x, 0, 4, 4, True, 1)
