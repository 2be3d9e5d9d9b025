"""CPU tests of the K x K 2D propagation (K in {3, 5, 7}): the oracle's generalisation against the pinned 3x3 arithmetic
and against the torch port in fp64, the C ABI's validation and workspace formulas, the module surface, and the
dispatcher registration (fake kernels, one traced node per direction)."""
import ctypes

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx

import cspn_b200
from conftest import golden_names, load_golden
from cspn_b200 import _lib
from cspn_b200.synth import make_inputs
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_k as onk
from oracle import cspn_torch_port as tp
from oracle import cspn_torch_port_k as tpk


def test_offsets_and_pads_generalise_the_3x3_tables():
    assert onk.offsets_2d(3) == onp.OFFSETS_2D
    assert tpk.pads_2d(3) == tp.PADS
    for K in (5, 7):
        r = (K - 1) // 2
        offs, pads = onk.offsets_2d(K), tpk.pads_2d(K)
        assert len(offs) == len(set(offs)) == K * K - 1 and (0, 0) not in offs
        assert offs == tuple(reversed([(-dy, -dx) for dy, dx in offs]))      # raster order: reversed taps negate
        # a pad of (l, K-1-l, t, K-1-t) then the crop [r:-r, r:-r] reads the source at (r-t, r-l)
        assert [(r - t, r - l) for (l, _, t, _) in pads] == list(offs)


@pytest.mark.parametrize('name', golden_names())
def test_k3_gives_the_bits_of_the_pinned_3x3_oracle(name):
    c = load_golden(name)
    a = onp.cspn2d(c['guidance'], c['blur'], c['sparse_depth'], c['prop_time'], c['norm_type'])
    b = onk.cspn2d_k(c['guidance'], c['blur'], c['sparse_depth'], c['prop_time'], 3, c['norm_type'])
    assert np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize('name', ['small_8sum', 'small_8sum_abs', 'c3_shared', 'odd_w_8sum', 'gch12_extra'])
def test_k3_torch_port_gives_the_bits_of_the_3x3_port(name):
    c = load_golden(name)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a))
    with torch.no_grad():
        a = tp.cspn2d_torch(t(c['guidance']), t(c['blur']), t(c['sparse_depth']), c['prop_time'], c['norm_type'])
        b = tpk.cspn2d_torch_k(t(c['guidance']), t(c['blur']), t(c['sparse_depth']), c['prop_time'], 3, c['norm_type'])
    assert torch.equal(a, b)


@pytest.mark.parametrize('K', [5, 7])
@pytest.mark.parametrize('abs_norm', [False, True])
@pytest.mark.parametrize('shape,gch,n', [((2, 3, 13, 17), None, 4), ((1, 1, 9, 11), 60, 3), ((1, 2, 3, 11), None, 5),
                                         ((1, 1, 12, 2), None, 4), ((1, 1, 1, 1), None, 2)])
def test_numpy_fp32_agrees_with_the_torch_port_in_fp64(K, abs_norm, shape, gch, n):
    """Signed sparse, C = 3, extra guidance channels, and H or W smaller than K."""
    B, C, H, W = shape
    nt = K * K - 1
    norm = f'{nt}sum_abs' if abs_norm else f'{nt}sum'
    g, d, s = make_inputs(100 * K + H + W, B, C, H, W, gch or nt, 'signed', 8)
    out = onk.cspn2d_k(g.numpy(), d.numpy(), s.numpy(), n, K, norm)
    with torch.no_grad():
        ref = tpk.cspn2d_torch_k(g.double(), d.double(), s.double(), n, K, norm).numpy()
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (ratio, normwise)
    ref64 = onk.cspn2d_k(g.numpy(), d.numpy(), s.numpy(), n, K, norm, dtype=np.float64)
    assert np.allclose(ref64, ref, rtol=1e-12, atol=1e-12, equal_nan=True)
    if gch:                                        # channels >= K*K-1 are not read
        assert np.array_equal(out, onk.cspn2d_k(g[:, :nt].numpy(), d.numpy(), s.numpy(), n, K, norm))


@pytest.mark.parametrize('K', [5, 7])
def test_sum_abs_preserves_a_constant_field_away_from_sparse_points(K):
    B, C, H, W, n = 1, 2, 20, 23, 6
    g, _, s = make_inputs(K, B, C, H, W, K * K - 1, 'bernoulli', 4)
    const = np.full((B, C, H, W), 2.75, np.float32)
    out = onk.cspn2d_k(g.numpy(), const, s.numpy(), n, K, f'{K * K - 1}sum_abs')
    assert np.allclose(out, 2.75, rtol=1e-5)
    # and its weights sum to one at every pixel whose whole K x K window lies in the image
    _, gate_sum = onk.affinity_normalization_2d_k(g.numpy(), K, f'{K * K - 1}sum_abs')
    r = (K - 1) // 2
    assert np.allclose(gate_sum[..., r:-r, r:-r], 1.0, atol=1e-5)


def _p():
    buf = (ctypes.c_float * 64)()
    return ctypes.cast(buf, ctypes.c_void_p), buf


def test_c_abi_rejects_bad_arguments():
    L = _lib.lib()
    p, _keep = _p()
    fwd = lambda *a, **kw: L.cspn2d_k_fwd_f32(*a, None, 0, None)
    bwd = lambda *a: L.cspn2d_k_bwd_f32(*a, None, 0, None)
    ok_args = dict(B=1, C=1, H=4, W=4, gch=24, K=5, iters=2, norm=0)

    def f(g=p, d=p, s=None, o=p, **over):
        a = dict(ok_args, **over)
        return fwd(g, d, s, o, a['B'], a['C'], a['H'], a['W'], a['gch'], a['K'], a['iters'], a['norm'])

    def b(g=p, d=p, s=None, go=p, **over):
        a = dict(ok_args, **over)
        return bwd(g, d, s, go, p, p, a['B'], a['C'], a['H'], a['W'], a['gch'], a['K'], a['iters'], a['norm'])

    for call in (f, b):
        for K in (1, 2, 4, 6, 9):
            assert call(K=K, gch=100) == -1
        assert call(K=5, gch=23) == -1 and call(K=7, gch=47) == -1 and call(K=3, gch=7) == -1
        assert call(norm=2) == -1 and call(norm=-1) == -1
        assert call(iters=-1) == -1
        for dim in ('B', 'C', 'H', 'W'):
            assert call(**{dim: 0}) == -1 and call(**{dim: -3}) == -1
        assert call(g=None) == -1 and call(d=None) == -1
    assert f(o=None) == -1 and b(go=None) == -1
    assert b'null' in L.cspn_last_error()


def test_workspace_formulas(monkeypatch):
    L = _lib.lib()
    B, C, H, W = 3, 2, 10, 15
    HW = H * W
    for K in (5, 7):
        for n in (1, 2, 24):
            assert L.cspn2d_k_workspace_bytes(B, C, H, W, K, n) == 4 * (B * K * K * HW + B * C * HW)
            assert L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, K, n) == 4 * (B * K * K * HW + 2 * n * B * C * HW)
        assert L.cspn2d_k_workspace_bytes(B, C, H, W, K, 0) == 0 and L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, K, 0) == 0
    for n in (0, 1, 24):      # K = 3 is the 3x3 operator: its queries are theirs
        assert L.cspn2d_k_workspace_bytes(B, C, H, W, 3, n) == L.cspn2d_workspace_bytes(B, C, H, W, n, _lib.ALGO_AUTO)
        assert L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, 3, n) == L.cspn2d_bwd_workspace_bytes(B, C, H, W, n)
    for n in (1, 2, 24):      # the 3x3 backward's fallback is the K x K one at K = 3, whose size covers the cluster route's
        assert L.cspn2d_bwd_workspace_bytes(B, C, H, W, n) == 4 * (B * 9 * HW + 2 * n * B * C * HW)
        assert L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, 3, n) == 4 * (B * 9 * HW + (2 * n + 1) * B * C * HW)
        monkeypatch.setenv('CSPN_B200_BWD', 'steps')     # the 3x3 backward's size does not depend on its route
        assert L.cspn2d_bwd_workspace_bytes(B, C, H, W, n) == 4 * (B * 9 * HW + 2 * n * B * C * HW)
        monkeypatch.delenv('CSPN_B200_BWD')
    assert L.cspn2d_k_workspace_bytes(B, C, H, W, 4, 3) == 0 and L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, 9, 3) == 0


def test_module_surface_and_assertions():
    for K, default in ((3, '8sum'), (5, '24sum'), (7, '48sum')):
        m = cspn_b200.Affinity_PropagateK(12, K)
        assert (m.prop_time, m.prop_kernel, m.norm_type) == (12, K, default)
        assert list(m.parameters()) == [] and list(m.buffers()) == [] and m.state_dict() == {}
        assert cspn_b200.Affinity_PropagateK(12, K, default + '_abs').norm_type == default + '_abs'
    for K in (1, 2, 4, 9):
        with pytest.raises(AssertionError):
            cspn_b200.Affinity_PropagateK(12, K)
    for K, name in ((5, '8sum'), (5, '48sum_abs'), (7, '24sum'), (3, '24sum'), (5, 'paddle')):
        with pytest.raises(AssertionError):
            cspn_b200.Affinity_PropagateK(12, K, name)
    with pytest.raises(AssertionError):
        cspn_b200.Affinity_Propagate(24, 5)                  # the 3x3 drop-in keeps the reference's contract
    d = torch.rand(1, 1, 4, 4)
    assert cspn_b200.Affinity_PropagateK(0, 5)(torch.randn(1, 24, 4, 4), d) is d


def test_cpu_tensors_and_short_guidance_are_refused():
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.propagate2d_k(torch.randn(1, 24, 6, 6), torch.rand(1, 1, 6, 6), None, 5, 3)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_k(torch.randn(1, 23, 6, 6), torch.rand(1, 1, 6, 6), None, 5, 3)
    with pytest.raises(AssertionError):
        cspn_b200.propagate2d_k(torch.randn(1, 24, 6, 6), torch.rand(1, 1, 6, 6), None, 5, 3, '8sum')


@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schema_and_fake_kernels(ops):
    s = str(ops.propagate2d_k.default._schema)
    assert 'Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, int kernel_size, int prop_time, int norm_type' in s
    with FakeTensorMode():
        for K in (5, 7):
            g = torch.empty(2, K * K + 1, 16, 30, device='cuda')
            d = torch.empty(2, 3, 16, 30, device='cuda')
            sp = torch.empty(2, 1, 16, 30, device='cuda')
            out = ops.propagate2d_k(g, d, sp, K, 24, 1)
            assert out.shape == d.shape and out.device == d.device and out.dtype == torch.float32
            gg, gd = ops.propagate2d_k_backward(g, d, sp, out, K, 24, 1, True, True)
            assert gg.shape == g.shape and gd.shape == d.shape
            gg, gd = ops.propagate2d_k_backward(g, d, None, out, K, 24, 0, False, True)
            assert gg.numel() == 0 and gd.shape == d.shape
        with pytest.raises(Exception):
            ops.propagate2d_k(torch.empty(1, 23, 8, 8, device='cuda'), torch.empty(1, 1, 8, 8, device='cuda'), None, 5, 4, 0)


@pytest.mark.parametrize('K', [5, 7])
def test_forward_and_backward_trace_to_one_node_each(ops, K):
    def f(g, d, s):
        out = ops.propagate2d_k(g, d, s, K, 24, 0)
        gg, gd = torch.autograd.grad(out.sum(), (g, d))
        return out, gg, gd

    g = torch.empty(1, K * K - 1, 12, 16, device='meta', requires_grad=True)
    d = torch.empty(1, 1, 12, 16, device='meta', requires_grad=True)
    s = torch.empty(1, 1, 12, 16, device='meta')
    gm = make_fx(f)(g, d, s)
    targets = [str(n.target) for n in gm.graph.nodes if n.op == 'call_function']
    assert sum('cspn_b200.propagate2d_k.default' in t for t in targets) == 1
    assert sum('cspn_b200.propagate2d_k_backward.default' in t for t in targets) == 1


def test_module_takes_the_dispatcher_route_when_the_shim_is_built(ops):
    m = cspn_b200.Affinity_PropagateK(24, 7, '48sum_abs')
    assert m._use_op is True
    with FakeTensorMode():
        out = m(torch.empty(1, 48, 8, 8, device='cuda'), torch.empty(1, 2, 8, 8, device='cuda'), torch.empty(1, 1, 8, 8, device='cuda'))
        assert out.shape == (1, 2, 8, 8)
