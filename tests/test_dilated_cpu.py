"""CPU tests of the dilated propagation (PENet's DA-CSPN++ step, DESIGN.md section 4.22): the two restatements of
tests/dilated_reference.py against each other in fp64, forward and autograd; the polyphase identity; the section 2g weight
move against a conv2d; the C ABI's refusals without a device; the op schemas and fake kernels; and no spills in the new
translation unit."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

import dilated_reference as dr
from cspn_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
D = torch.float64


def assert_same(r1, r2, tol=1e-12):
    for name, x, y in zip(('out', 'kernel', 'blur', 'sparse', 'conf'), r1, r2):
        assert (x is None) == (y is None), name
        if x is not None:
            torch.testing.assert_close(x, y, rtol=tol, atol=tol, msg=name)


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('dil', [1, 2, 4])
@pytest.mark.parametrize('samples', [None, 'soft', 'hard'])
@pytest.mark.parametrize('shape', [(2, 1, 9, 11), (1, 3, 6, 7), (1, 1, 1, 13), (2, 2, 10, 1), (1, 1, 3, 4)])
def test_restatements_agree_in_fp64(K, dil, samples, shape):
    """Includes d*R >= H or W (every neighbour outside the image), 1 x W and H x 1 images, and C = 3."""
    B, C, H, W = shape
    ins = dr.make_inputs(B, C, H, W, K, samples, seed=K * 7 + dil)
    go = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(1))
    assert_same(dr.grads(dr.composition, *ins, K, dil, 3, go, dtype=D), dr.grads(dr.explicit, *ins, K, dil, 3, go, dtype=D))


def test_all_neighbours_outside_leaves_the_centre_term():
    k, b, _, _ = dr.make_inputs(1, 1, 3, 3, 7, None, seed=2)
    out = dr.composition(k.double(), b.double(), None, None, 7, 4, 2)     # d*R = 12 > H, W
    torch.testing.assert_close(out, k[:, 24:25].double() * b.double())


def polyphase(fn, kernel, blur, sparse, conf, K, dil, N):
    """Dilation dil as dil^2 dilation-1 runs on the sub-images x[..., a::dil, b::dil], interleaved."""
    out = torch.empty_like(blur)
    for a in range(dil):
        for b in range(dil):
            if a >= blur.shape[2] or b >= blur.shape[3]:
                continue
            sub = [None if t is None else t[..., a::dil, b::dil] for t in (kernel, blur, sparse, conf)]
            out[..., a::dil, b::dil] = fn(*sub, K, 1, N)
    return out


@pytest.mark.parametrize('K,dil', [(3, 2), (5, 3), (7, 4), (3, 4)])
@pytest.mark.parametrize('shape', [(2, 2, 11, 14), (1, 1, 3, 2)])
def test_polyphase_identity(K, dil, shape):
    ins = [None if t is None else t.double() for t in dr.make_inputs(*shape, K, 'soft', seed=dil)]
    torch.testing.assert_close(dr.composition(*ins, K, dil, 4), polyphase(dr.composition, *ins, K, dil, 4), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('K', [3, 5, 7])
def test_weight_move_is_a_permutation_conv(K):
    g = torch.randn(2, K * K, 8, 9, dtype=D)
    KK, R = K * K, (K - 1) // 2
    filt = torch.zeros(KK, KK, K, K, dtype=D)
    for j in range(KK):
        filt[j, KK - 1 - j, j // K, j % K] = 1
    torch.testing.assert_close(dr.move_weights(g, K), F.conv2d(g, filt, padding=R), rtol=0, atol=0)


def test_normalise_guide_puts_the_centre_in_the_middle():
    g = torch.randn(1, 8, 4, 5, dtype=D)
    w = dr.normalise_guide(g)
    assert w.shape[1] == 9
    torch.testing.assert_close(w.sum(1), torch.ones(1, 4, 5, dtype=D))
    torch.testing.assert_close(w[:, 4], 1 - (g / g.abs().sum(1, keepdim=True)).sum(1))


def test_gradcheck():
    ins = [None if t is None else t.double().requires_grad_(True) for t in dr.make_inputs(1, 2, 5, 6, 3, 'soft', seed=3)]
    assert torch.autograd.gradcheck(lambda k, b, s, m: dr.explicit(k, b, s, m, 3, 2, 2), tuple(ins), eps=1e-6, atol=1e-5)


# ---- the library's surface without a device -----------------------------------------------------------------------------
def test_argtypes_cover_the_entry_points():
    for name in ('cspn2d_dil_workspace_bytes', 'cspn2d_dil_fwd_f32', 'cspn2d_dil_bwd_workspace_bytes', 'cspn2d_dil_bwd_f32'):
        assert name in _lib.SIGNATURES
    assert _lib.lib().cspn2d_dil_fwd_f32.argtypes is not None


def test_workspace_formulas():
    L = _lib.lib()
    P = 2 * 3 * 7 * 9 * 4
    for N in (0, 1, 2, 3, 24):
        assert L.cspn2d_dil_workspace_bytes(2, 3, 7, 9, 5, 2, N) == (P if N >= 2 else 0)
        assert L.cspn2d_dil_bwd_workspace_bytes(2, 3, 7, 9, 5, 2, N) == max(2 * N - 1, 0) * P
    assert L.cspn2d_dil_workspace_bytes(2, 3, 7, 9, 4, 1, 2) == 0
    assert L.cspn2d_dil_workspace_bytes(2, 3, 7, 9, 3, 5, 2) == 0
    assert L.cspn2d_dil_workspace_bytes(2, 3, 7, 9, 3, 0, 2) == 0
    assert L.cspn2d_dil_workspace_bytes(0, 3, 7, 9, 3, 1, 2) == 0
    assert L.cspn2d_dil_bwd_workspace_bytes(2, 3, 7, 9, 3, 1, -1) == 0


INVALID, WORKSPACE, UNSUPPORTED = -1, -2, -4
P = 1 << 20          # fake, 4-byte aligned "device" addresses: every refusal comes before any device work


def fwd(k=P, b=2 * P, s=None, m=None, out=4 * P, B=1, C=1, H=8, W=8, K=3, d=1, N=2, ws=5 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_dil_fwd_f32(k, b, s, m, out, B, C, H, W, K, d, N, ws, wsb, None)


def bwd(s=None, m=None, gk=6 * P, gb=7 * P, gs=None, gm=None, B=1, C=1, H=8, W=8, K=3, d=1, N=2, ws=10 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_dil_bwd_f32(P, 2 * P, s, m, 3 * P, gk, gb, gs, gm, B, C, H, W, K, d, N, ws, wsb, None)


def test_abi_refusals_without_a_device():
    assert fwd(k=None) == INVALID
    assert fwd(b=None) == INVALID
    assert fwd(out=None) == INVALID
    assert fwd(s=8 * P) == INVALID                                 # sparse without confidence
    assert fwd(m=8 * P) == INVALID                                 # confidence without sparse
    assert fwd(b=2 * P + 2) == INVALID                             # misaligned
    assert fwd(K=4) == INVALID
    assert fwd(d=0) == INVALID
    assert fwd(d=5) == INVALID
    assert fwd(N=-1) == INVALID
    assert fwd(B=0) == INVALID
    assert fwd(W=-3) == INVALID
    assert fwd(out=2 * P + 64) == INVALID                          # out overlaps blur
    assert b'overlaps' in _lib.lib().cspn_last_error()
    assert fwd(ws=4 * P + 16) == INVALID                           # the workspace overlaps out
    assert fwd(ws=None) == WORKSPACE
    assert fwd(wsb=4) == WORKSPACE
    assert fwd(B=65536, out=1 << 44, ws=1 << 45) == UNSUPPORTED    # B*C beyond gridDim.z
    assert fwd(B=300, C=300, out=1 << 44, ws=1 << 45) == UNSUPPORTED
    assert bwd(gs=8 * P) == INVALID                                # grad_sparse without the samples
    assert bwd(gm=8 * P) == INVALID
    assert bwd(s=8 * P) == INVALID                                 # sparse without confidence
    assert bwd(gk=P) == INVALID                                    # grad_kernel overlaps kernel
    assert bwd(gb=6 * P) == INVALID                                # two outputs overlap
    assert bwd(K=2) == INVALID
    assert bwd(wsb=16) == WORKSPACE
    assert bwd(B=65536, gk=1 << 44, gb=1 << 45, ws=1 << 46) == UNSUPPORTED


def test_op_schemas_and_fake_kernels():
    from cspn_b200 import torch_op
    if not torch_op.available():
        pytest.skip('the torch op library is not built')
    torch_op.load()
    op = torch.ops.cspn_b200.propagate2d_dilated.default
    assert str(op._schema) == ('cspn_b200::propagate2d_dilated(Tensor kernel, Tensor blur_depth, Tensor? sparse_depth, '
                               'Tensor? confidence, int kernel_size, int dilation, int prop_time) -> Tensor')
    bop = torch.ops.cspn_b200.propagate2d_dilated_backward.default
    assert 'bool need_confidence) -> (Tensor, Tensor, Tensor, Tensor)' in str(bop._schema)
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        k, b, s = torch.empty(2, 25, 5, 7), torch.empty(2, 3, 5, 7), torch.empty(2, 1, 5, 7)
        assert op(k, b, s, s, 5, 2, 4).shape == b.shape
        assert op(k, b, None, None, 5, 1, 4).shape == b.shape
        g = bop(k, b, s, s, b, 5, 2, 4, True, False, True, True)
        assert [tuple(x.shape) for x in g] == [(2, 25, 5, 7), (0,), (2, 1, 5, 7), (2, 1, 5, 7)]


def test_python_refusals():
    import cspn_b200
    k, b, s, m = dr.make_inputs(1, 2, 5, 6, 3, 'soft')
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k[:, :8], b, s, m, 3, 1, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k, b, s, None, 3, 1, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k, b, None, m, 3, 1, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k, b, s.expand(1, 2, 5, 6), m, 3, 1, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k, b, s, m, 3, 5, 2)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_dilated(k, b, s, m, 3, 1, -1)
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateDilated(3, 3, 0)
    with pytest.raises(_lib.CspnError):
        cspn_b200.propagate2d_dilated(k, b, s, m, 3, 1, 2)          # CPU tensors: no host entry point


def test_no_spills_in_the_new_translation_unit():
    log = os.path.join(ROOT, 'cspn_b200', '_build', 'ptxas.log')
    if not os.path.isfile(log):
        pytest.skip('the library is not built')
    part = open(log).read().split('== cspn2d_dilated.cu')[1].split('\n== ')[0]
    assert 'dil_step_kernel' in part and 'dil_adjoint_kernel' in part and 'dil_finalize_kernel' in part
    spills = [int(x) for x in re.findall(r'(\d+) bytes spill stores', part)]
    assert len(spills) == 27 and max(spills) == 0
