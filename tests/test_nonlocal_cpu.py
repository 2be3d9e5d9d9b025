"""CPU tests of the non-local 2D propagation (DESIGN.md section 4.21): the explicit restatement of
tests/nonlocal_reference.py against torchvision's deform_conv2d composition in fp64, forward and every gradient, at the
window's edges and with special values; the op schemas and fake kernels; the C ABI's refusals without a device; and no
spills in the new translation unit."""
import os
import re

import pytest
import torch

import nonlocal_reference as nr
from cspn_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def both(f, o, a, s, K, N, go, tv_too=True):
    d = torch.float64
    r1 = nr.grads(nr.propagate, f, o, a, s, K, N, go, dtype=d)
    if not tv_too:
        return r1, None
    pytest.importorskip('torchvision')
    return r1, nr.grads(nr.propagate_torchvision, f, o, a, s, K, N, go, dtype=d)


def assert_same(r1, r2):
    for name, x, y in zip(('out', 'feat', 'offset', 'affinity', 'sparse'), r1, r2):
        assert (x is None) == (y is None), name
        if x is not None:
            assert torch.equal(torch.isnan(x), torch.isnan(y)), name
            fin = torch.isfinite(y)
            torch.testing.assert_close(x[fin], y[fin], rtol=1e-10, atol=1e-10, msg=name)


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('sparse', [False, True])
def test_restatement_is_the_torchvision_composition(K, C, sparse):
    f, o, a, s = nr.make_inputs(2, C, 6, 7, K, scale=3.0, seed=K * 3 + C, sparse=sparse)
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(9))
    assert_same(*both(f, o, a, s, K, 3, go))


# positions exactly at -1, inside (-1, 0), at H - 1, inside (H - 1, H), at H and beyond, integer offsets
EDGE_Y = [-1.0, -0.5, -1.5, 4.0, 4.25, 5.0, 7.5, 0.0, 2.0]


@pytest.mark.parametrize('y', EDGE_Y)
@pytest.mark.parametrize('axis', [0, 1])
def test_window_edges(y, axis):
    """Every tap's position set to y along one axis (H = W = 5), the other axis random: forward and every gradient."""
    K, H, W = 3, 5, 5
    f, o, a, s = nr.make_inputs(1, 2, H, W, K, scale=0.7, seed=13, sparse=True)
    for k, (di, dj) in enumerate(nr.taps(K)):
        base = torch.arange(H, dtype=torch.float32).view(H, 1) + di if axis == 0 else torch.arange(W, dtype=torch.float32).view(1, W) + dj
        o[:, 2 * k + axis] = y - base
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(2))
    assert_same(*both(f, o, a, s, K, 2, go))


@pytest.mark.parametrize('value', [float('inf'), float('-inf'), 1e30])
def test_non_finite_and_huge_offsets(value):
    f, o, a, s = nr.make_inputs(1, 1, 5, 6, 3, seed=4)
    o[0, 3, 1, 2] = value
    o[0, 6, 4, 5] = value
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(3))
    assert_same(*both(f, o, a, s, 3, 2, go))


def test_nan_offset_gives_nan_and_no_feat_gradient():
    """torchvision converts a NaN coordinate to an integer (undefined), so only the restatement's own definition is
    checked: S is NaN, the sample reaches no pixel's gradient, and its offset gradient is NaN along the other axis."""
    f, o, a, _ = nr.make_inputs(1, 1, 5, 6, 3, seed=4)
    o[0, 2, 2, 3] = float('nan')                      # dy of tap 1 at (2, 3)
    go = torch.zeros(f.shape, dtype=torch.float64)
    go[0, 0, 2, 3] = 1
    out, gf, goff, ga, _ = nr.grads(nr.propagate, f, o, a, None, 3, 1, go, dtype=torch.float64)
    assert torch.isnan(out[0, 0, 2, 3]) and torch.isfinite(out).sum() == out.numel() - 1
    assert torch.isfinite(gf).all()
    assert torch.isnan(goff[0, 3, 2, 3]) and torch.isnan(ga[0, 1, 2, 3])


def test_infinite_zero_weight_corner_matches_torchvision():
    f = torch.zeros(1, 1, 4, 5)
    f[0, 0, 2, 3] = float('inf')
    o = torch.zeros(1, 16, 4, 5)
    a = torch.full((1, 8, 4, 5), 0.125)
    assert_same(*both(f, o, a, None, 3, 1, torch.ones(1, 1, 4, 5)))


def test_fp32_restatement_is_close_to_fp64():
    f, o, a, s = nr.make_inputs(2, 2, 9, 10, 5, scale=4.0, seed=1, sparse=True)
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(5))
    r32 = nr.grads(nr.propagate, f, o, a, s, 5, 4, go)
    r64 = nr.grads(nr.propagate, f, o, a, s, 5, 4, go, dtype=torch.float64)
    assert all(nr.normwise(x, y) < 1e-5 for x, y in zip(r32, r64))


def test_gradcheck():
    f, o, a, s = nr.make_inputs(1, 2, 4, 5, 3, scale=0.4, seed=8, sparse=True)
    ins = [t.double().requires_grad_(True) for t in (f, o, a)] + [s.double()]
    assert torch.autograd.gradcheck(lambda f, o, a: nr.propagate(f, o, a, ins[3], K=3, N=2), tuple(ins[:3]), eps=1e-7, atol=1e-5)


# ---- the library's surface without a device -----------------------------------------------------------------------------
def test_argtypes_cover_the_entry_points():
    for name in ('cspn2d_nl_workspace_bytes', 'cspn2d_nl_fwd_f32', 'cspn2d_nl_bwd_workspace_bytes', 'cspn2d_nl_bwd_f32'):
        assert name in _lib.SIGNATURES
    L = _lib.lib()
    assert L.cspn2d_nl_fwd_f32.argtypes is not None


def test_forward_workspace_formula():
    L = _lib.lib()
    for N, bufs in ((0, 0), (1, 0), (2, 1), (3, 2), (18, 2)):
        assert L.cspn2d_nl_workspace_bytes(2, 3, 7, 9, 5, N) == bufs * 4 * 2 * 3 * 7 * 9
    assert L.cspn2d_nl_workspace_bytes(2, 3, 7, 9, 4, 2) == 0
    assert L.cspn2d_nl_workspace_bytes(0, 3, 7, 9, 3, 2) == 0
    assert L.cspn2d_nl_workspace_bytes(2, 3, 7, 9, 3, -1) == 0
    assert L.cspn2d_nl_bwd_workspace_bytes(2, 3, 7, 9, 9, 2) == 0


INVALID, WORKSPACE, UNSUPPORTED = -1, -2, -4
P = 1 << 20          # fake, 4-byte aligned "device" addresses: every refusal comes before any device work


def fwd(feat=P, off=2 * P, aff=3 * P, sp=None, out=4 * P, B=1, C=1, H=8, W=8, K=3, N=2, ws=5 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_nl_fwd_f32(feat, off, aff, sp, out, B, C, H, W, K, N, ws, wsb, None)


def bwd(gs=None, sp=None, gf=6 * P, B=1, C=1, H=8, W=8, K=3, N=2, feat=P):
    return _lib.lib().cspn2d_nl_bwd_f32(feat, 2 * P, 3 * P, sp, 4 * P, gf, 7 * P, 8 * P, gs, B, C, H, W, K, N, 9 * P, 1 << 30, None)


def test_abi_refusals_without_a_device():
    assert fwd(feat=None) == INVALID
    assert fwd(out=None) == INVALID
    assert fwd(feat=P + 2) == INVALID
    assert fwd(K=4) == INVALID
    assert fwd(N=-1) == INVALID
    assert fwd(B=0) == INVALID
    assert fwd(out=P + 64) == INVALID                              # out overlaps feat
    assert b'overlaps' in _lib.lib().cspn_last_error()
    assert fwd(ws=None) == WORKSPACE
    assert fwd(wsb=4) == WORKSPACE
    assert fwd(ws=4 * P + 16) == INVALID                           # the workspace overlaps out
    assert fwd(H=30000, W=30000) == UNSUPPORTED                    # H*W*T >= 2^31
    assert fwd(B=65535, C=5, out=1 << 44, ws=1 << 45) == UNSUPPORTED   # B*ceil(C/4) beyond the grid
    assert bwd(gs=10 * P) == INVALID                               # grad_sparse without a sparse
    assert bwd(feat=None) == INVALID
    assert bwd(K=2) == INVALID
    assert bwd(gf=P) == INVALID                                    # grad_feat overlaps feat
    assert bwd(H=30000, W=30000) == UNSUPPORTED


def test_op_schemas_and_fake_kernels():
    from cspn_b200 import torch_op
    if not torch_op.available():
        pytest.skip('the torch op library is not built')
    torch_op.load()
    op = torch.ops.cspn_b200.propagate2d_nonlocal.default
    assert str(op._schema) == ('cspn_b200::propagate2d_nonlocal(Tensor feat, Tensor offset, Tensor affinity, Tensor? sparse_depth, '
                               'int kernel_size, int prop_time) -> Tensor')
    bop = torch.ops.cspn_b200.propagate2d_nonlocal_backward.default
    assert 'bool need_sparse) -> (Tensor, Tensor, Tensor, Tensor)' in str(bop._schema)
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        f, o, a = torch.empty(2, 3, 5, 7), torch.empty(2, 48, 5, 7), torch.empty(2, 24, 5, 7)
        assert op(f, o, a, None, 5, 4).shape == f.shape
        g = bop(f, o, a, f, f, 5, 4, True, True, False, True)
        assert [tuple(x.shape) for x in g] == [(2, 3, 5, 7), (2, 48, 5, 7), (0,), (2, 3, 5, 7)]


def test_python_refusals():
    import cspn_b200
    f, o, a, s = nr.make_inputs(1, 2, 5, 6, 3, sparse=True)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_nonlocal(f, o[:, :15], a, None, 3, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_nonlocal(f, o, a, s[:, :1], 3, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_nonlocal(f, o, a, None, 4, 2)
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateNonLocal(3, 6)
    with pytest.raises(_lib.CspnError):
        cspn_b200.propagate2d_nonlocal(f, o, a, None, 3, 2)        # CPU tensors: no host entry point


def test_no_spills_in_the_new_translation_unit():
    log = os.path.join(ROOT, 'cspn_b200', '_build', 'ptxas.log')
    if not os.path.isfile(log):
        pytest.skip('the library is not built')
    text = open(log).read()
    part = text.split('== cspn2d_nonlocal.cu')[1].split('\n== ')[0]
    assert 'nl_step_kernel' in part and 'nl_finalize_kernel' in part
    spills = [int(x) for x in re.findall(r'(\d+) bytes spill stores', part)]
    assert spills and max(spills) == 0
