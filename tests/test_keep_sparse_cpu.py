"""The keep-sparse mode without a GPU: the explicit adjoint of tests/keep_sparse_reference.py against torch autograd through
the spec's op sequence, its tie to the reference module's arithmetic (oracle/cspn_numpy_k.py) where the two modes must
agree, and the C ABI's argument checks of the new entries."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from cspn_b200 import _lib
from oracle.cspn_numpy_k import cspn2d_k

import keep_sparse_reference as ks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(seed, B, C, H, W, K, sparse_kind='mixed'):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, K * K - 1 + 1, H, W, generator=gen, dtype=torch.float64)
    blur = torch.rand(B, C, H, W, generator=gen, dtype=torch.float64) + 0.5
    hot = torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64) < 0.2
    vals = torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64) * 4
    if sparse_kind == 'mixed':          # positive samples, zeros and negative values (not samples)
        vals = torch.where(torch.rand(B, 1, H, W, generator=gen) < 0.25, -vals, vals)
    return g, blur, torch.where(hot, vals, torch.zeros_like(vals))


@pytest.mark.parametrize('K', (3, 5, 7))
@pytest.mark.parametrize('norm', ('sum', 'sum_abs'))
@pytest.mark.parametrize('C', (1, 2))
def test_explicit_adjoint_matches_autograd(K, norm, C):
    norm = f'{K * K - 1}{norm}'
    N = 4
    g, blur, sparse = _inputs(K * 10 + C, 2, C, 9, 11, K)
    go = torch.randn(blur.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in (g, blur, sparse)]
    out = ks.op_sequence(*leaves, N, K, norm)
    out.backward(go)
    ref = ks.reference(g, blur, sparse, N, K, norm, go)
    assert torch.allclose(ref[0], out.detach(), rtol=1e-13, atol=1e-13)
    for got, leaf, name in zip(ref[1:], leaves, ('guidance', 'blur', 'sparse')):
        assert torch.allclose(got, leaf.grad, rtol=1e-11, atol=1e-11), name
    # the indicator has zero derivative: no gradient reaches an unsampled pixel
    assert (ref[3][sparse <= 0] == 0).all()


@pytest.mark.parametrize('K', (3, 5, 7))
@pytest.mark.parametrize('N', (0, 1, 6))
def test_equals_the_reference_mode_where_the_samples_are_the_blur(K, N):
    """With sparse >= 0 and sparse == blur where it is positive, replacing by the sample is replacing by blur, and the
    indicator is the sign: the restatement gives what the reference module computes (cspn_numpy_k, fp64)."""
    g, blur, sparse = _inputs(K + N, 2, 1, 10, 12, K, 'positive')
    sparse = torch.where(sparse > 0, blur, torch.zeros_like(blur))
    for norm in (f'{K * K - 1}sum', f'{K * K - 1}sum_abs'):
        ours = ks.op_sequence(g, blur, sparse, N, K, norm).numpy()
        theirs = cspn2d_k(g.numpy(), blur.numpy(), sparse.numpy(), N, K, norm, dtype=np.float64)
        np.testing.assert_allclose(ours, theirs, rtol=1e-12, atol=1e-12)


def test_samples_pass_through():
    g, blur, sparse = _inputs(3, 1, 3, 12, 14, 3)
    out = ks.op_sequence(g, blur, sparse, 5)
    hit = (sparse > 0).expand_as(out)
    assert torch.equal(out[hit], sparse.expand_as(out)[hit])


def _header_args():
    text = open(os.path.join(ROOT, 'include', 'cspn_b200.h')).read()
    out = {}
    for m in re.finditer(r'CSPN_API\s+[\w\s\*]+?\b(cspn2d_keep\w+)\s*\(([^)]*)\)', text):
        out[m.group(1)] = len([a for a in m.group(2).split(',') if a.strip()])
    return out


def test_signatures_match_the_header():
    args = _header_args()
    assert sorted(args) == ['cspn2d_keep_bwd_f32', 'cspn2d_keep_bwd_workspace_bytes', 'cspn2d_keep_fwd_f32',
                            'cspn2d_keep_fwd_gather_f32', 'cspn2d_keep_workspace_bytes']
    for name, n in args.items():
        assert len(_lib.SIGNATURES[name][1]) == n, name


def test_abi_rejects_bad_arguments_without_a_gpu():
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def fwd(g=p, d=p, s=p, o=p, B=1, C=1, H=4, W=4, gch=8, K=3, N=1, norm=0, algo=0):
        return L.cspn2d_keep_fwd_f32(g, d, s, o, B, C, H, W, gch, K, N, norm, algo, None, 0, None)

    def bwd(g=p, d=p, s=p, go=p, B=1, C=1, H=4, W=4, gch=8, K=3, N=1, norm=0):
        return L.cspn2d_keep_bwd_f32(g, d, s, go, None, None, None, B, C, H, W, gch, K, N, norm, None, 0, None)

    def gather(n_peer=0, peers=None, N=1):
        return L.cspn2d_keep_fwd_gather_f32(p, p, p, p, peers, n_peer, None, 1, 1, 4, 4, 8, 3, N, 0, None, 0, None)

    for kw, what in ((dict(g=None), 'null'), (dict(d=None), 'null'), (dict(o=None), 'null'), (dict(B=0), 'non-positive'),
                     (dict(K=4), 'kernel size'), (dict(K=9), 'kernel size'), (dict(K=5, gch=23), 'guidance channels'),
                     (dict(N=-1), 'prop_time'), (dict(norm=2), 'norm_type'), (dict(norm=5), 'norm_type'),
                     (dict(norm=-1), 'norm_type'), (dict(algo=3), 'algo'), (dict(algo=-1), 'algo')):
        assert fwd(**kw) == -1, kw
        assert what.encode() in L.cspn_last_error(), (kw, L.cspn_last_error())
    for kw in (dict(g=None), dict(go=None), dict(K=6), dict(norm=2), dict(norm=5), dict(norm=-1), dict(N=-1), dict(W=0)):
        assert bwd(**kw) == -1, kw
    assert gather(n_peer=8) == -1 and b'n_peer' in L.cspn_last_error()
    assert gather(n_peer=1, peers=None) == -1
    assert gather(N=0) == -4 and b'prop_time >= 1' in L.cspn_last_error()


def test_workspace_queries():
    L = _lib.lib()
    for args in ((0, 1, 8, 8, 3, 4, 0), (1, 1, 8, 8, 4, 4, 0), (1, 1, 8, 8, 5, 0, 0), (1, 1, 8, 8, 3, 4, 3), (1, 1, 8, 8, 3, 4, -1)):
        assert L.cspn2d_keep_workspace_bytes(*args) == 0, args
    assert L.cspn2d_keep_bwd_workspace_bytes(1, 1, 8, 8, 6, 4) == 0
    assert L.cspn2d_keep_bwd_workspace_bytes(1, 1, 8, 8, 5, -1) == 0
    B, C, H, W, n = 2, 3, 9, 13, 5
    plane = 4 * B * C * H * W
    # the launch-per-step paths hold one B*C*H*W plane (d0') more than the default mode
    assert L.cspn2d_keep_workspace_bytes(B, C, H, W, 3, n, _lib.ALGO_GENERIC) == \
        L.cspn2d_workspace_bytes(B, C, H, W, n, _lib.ALGO_GENERIC) + plane
    for K in (5, 7):
        assert L.cspn2d_keep_workspace_bytes(B, C, H, W, K, n, 0) == L.cspn2d_k_workspace_bytes(B, C, H, W, K, n) + plane
        assert L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, K, n) == L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, K, n) + plane
    assert L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, 3, n) >= L.cspn2d_bwd_workspace_bytes(B, C, H, W, n)


def test_host_tensors_are_refused():
    import cspn_b200
    g, blur, sparse = [t.float() for t in _inputs(1, 1, 1, 8, 8, 3)]
    with pytest.raises(_lib.CspnError, match='CUDA tensors only'):
        cspn_b200.propagate2d(g, blur, sparse, 3, keep_sparse=True)
    with pytest.raises(_lib.CspnError, match='CUDA tensors only'):
        cspn_b200.propagate2d_k(g[:, :8].repeat(1, 4, 1, 1), blur, sparse, 5, 3, keep_sparse=True)
    with pytest.raises(_lib.CspnError, match='CUDA tensors only'):
        cspn_b200.Affinity_Propagate(3, 3, keep_sparse=True)(g, blur, sparse)
