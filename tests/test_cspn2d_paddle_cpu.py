"""CPU tests of the 2D propagation with the Paddle module's own-location gates (CSPN.cspn with dim_num = 2, K in {3, 5, 7}):
the numpy restatement (tests/paddle2d_reference.py) against the fp64 torch port and against the merged 3D 'paddle' rule at D = 1, its properties, the C
ABI's validation and workspace formulas, the module surface, and the dispatcher registration (fake kernels, one traced node
per direction)."""
import ctypes

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx

import cspn_b200
from cspn_b200 import _lib
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_3d_k as on3
from oracle import cspn_numpy_k as onk
from oracle import cspn_torch_port_3d_k as tp3

import paddle2d_reference as pr


def inputs(seed, B, C, H, W, K, per_channel=False, signed=True):
    gen = torch.Generator().manual_seed(seed)
    nt = K * K - 1
    shape = (B, nt * C if per_channel else nt, H, W)
    g = torch.randn(*shape, generator=gen) if signed else torch.rand(*shape, generator=gen)
    return g, torch.rand(B, C, H, W, generator=gen)


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('shape,n,per_channel', [((2, 3, 13, 17), 4, False), ((1, 2, 9, 11), 3, True),
                                                 ((1, 1, 3, 11), 5, False), ((1, 3, 12, 2), 4, True), ((1, 1, 1, 1), 2, False)])
def test_numpy_fp32_agrees_with_the_torch_port_in_fp64(K, shape, n, per_channel):
    """Shared and per-channel gates, C = 3, and H or W smaller than K."""
    B, C, H, W = shape
    g, f = inputs(10 * K + H + W, B, C, H, W, K, per_channel)
    out = pr.cspn2d_paddle(g.numpy(), f.numpy(), n, K)
    with torch.no_grad():
        ref = pr.cspn2d_torch_paddle(g.double(), f.double(), n, K).numpy()
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (ratio, normwise)
    ref64 = pr.cspn2d_paddle(g.numpy(), f.numpy(), n, K, dtype=np.float64)
    assert np.allclose(ref64, ref, rtol=1e-12, atol=1e-12, equal_nan=True)


def in_plane(K):
    """The taps of offsets_3d(K) with dz = 0: in the raster order of offsets_2d(K)."""
    idx = [k for k, (dz, _, _) in enumerate(on3.offsets_3d(K)) if dz == 0]
    assert [on3.offsets_3d(K)[k][1:] for k in idx] == list(onk.offsets_2d(K))
    return idx


@pytest.mark.parametrize('K', [3, 5])
@pytest.mark.parametrize('W', [16, 3])
def test_it_is_the_3d_paddle_rule_at_depth_one(K, W):
    """With the 2D gates in the in-plane channels of a K x K x K gate and the others zero, the merged 3D 'paddle' rule at
    D = 1 is this one: the numpy restatements agree bit for bit (adding the zero terms is exact), the fp64 ports to 1e-12."""
    B, C, H, n = 2, 2, 9, 4
    g, f = inputs(K + W, B, C, H, W, K)
    g3 = torch.zeros(B, K ** 3 - 1, 1, H, W)
    g3[:, in_plane(K), 0] = g
    a = pr.cspn2d_paddle(g.numpy(), f.numpy(), n, K)
    b = on3.cspn3d_k(g3.numpy(), f[:, :, None].numpy(), n, K, 'paddle')[:, :, 0]
    assert np.array_equal(a, b)
    with torch.no_grad():
        ta = pr.cspn2d_torch_paddle(g.double(), f.double(), n, K)
        tb = tp3.cspn3d_torch_k(g3.double(), f[:, :, None].double(), n, K, 'paddle')[:, :, 0]
    assert torch.allclose(ta, tb, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('K', [3, 5, 7])
def test_a_constant_stays_constant_away_from_the_border(K):
    """The gates sum to one at every pixel, so a constant survives wherever no tap of the N steps reaches the zero padding:
    at pixels N*r or more from the border.  At the border it decays."""
    B, C, H, W, n = 1, 2, 30, 33, 3
    r = (K - 1) // 2
    g, _ = inputs(K, B, C, H, W, K, signed=True)
    const = np.full((B, C, H, W), 2.75, np.float32)
    out = pr.cspn2d_paddle(g.numpy(), const, n, K)
    m = n * r
    assert np.allclose(out[..., m:H - m, m:W - m], 2.75, rtol=1e-5)
    assert not np.allclose(out[..., 0, :], 2.75, rtol=1e-3)


@pytest.mark.parametrize('K', [3, 5, 7])
def test_per_channel_gates_are_demo_py_slice_and_concat_loop(K):
    """demo.py:28-45 propagates channel c with guide[:, nt*c:nt*c+nt] and concatenates the results."""
    B, C, H, W, n = 2, 3, 8, 10, 3
    nt = K * K - 1
    g, f = inputs(K + 100, B, C, H, W, K, per_channel=True)
    out = pr.cspn2d_paddle(g.numpy(), f.numpy(), n, K)
    loop = np.concatenate([pr.cspn2d_paddle(g[:, nt * c:nt * (c + 1)].numpy(), f[:, c:c + 1].numpy(), n, K)
                           for c in range(C)], 1)
    assert np.array_equal(out, loop)
    with torch.no_grad():
        tout = pr.cspn2d_torch_paddle(g.double(), f.double(), n, K)
        tloop = torch.cat([pr.cspn2d_torch_paddle(g[:, nt * c:nt * (c + 1)].double(), f[:, c:c + 1].double(), n, K)
                           for c in range(C)], 1)
    assert torch.equal(tout, tloop)


def test_zero_gates_give_nan_and_the_front_moves_r_per_step():
    K, r, H, W = 5, 2, 24, 26
    g, f = inputs(3, 1, 1, H, W, K)
    g[:, :, 10:13, 11:14] = 0.0
    extents = []
    for n in (1, 2, 3):
        idx = np.nonzero(np.isnan(pr.cspn2d_paddle(g.numpy(), f.numpy(), n, K)[0, 0]))
        extents.append(tuple(int(i.max() - i.min()) for i in idx))
    assert extents == [(2, 2), (2 + 2 * r, 2 + 2 * r), (2 + 4 * r, 2 + 4 * r)]


def _p():
    buf = (ctypes.c_float * 64)()
    return ctypes.cast(buf, ctypes.c_void_p), buf


def test_c_abi_rejects_bad_arguments():
    L = _lib.lib()
    p, _keep = _p()
    ok_args = dict(B=1, C=1, H=4, W=4, K=5, iters=2)

    def f(g=p, d=p, o=p, **over):
        a = dict(ok_args, **over)
        return L.cspn2d_paddle_fwd_f32(g, d, o, a['B'], a['C'], a['H'], a['W'], a['K'], a['iters'], None, 0, None)

    def b(g=p, d=p, go=p, **over):
        a = dict(ok_args, **over)
        return L.cspn2d_paddle_bwd_f32(g, d, go, p, p, a['B'], a['C'], a['H'], a['W'], a['K'], a['iters'], None, 0, None)

    for call in (f, b):
        for K in (0, 1, 2, 4, 6, 9):
            assert call(K=K) == -1
        assert call(iters=-1) == -1
        for dim in ('B', 'C', 'H', 'W'):
            assert call(**{dim: 0}) == -1 and call(**{dim: -3}) == -1
        assert call(g=None) == -1 and call(d=None) == -1
    assert f(o=None) == -1 and b(go=None) == -1
    assert b'null' in L.cspn_last_error()
    # the K x K entry points keep refusing the own-location norm (code 2)
    assert L.cspn2d_k_fwd_f32(p, p, None, p, 1, 1, 4, 4, 24, 5, 2, 2, None, 0, None) == -1
    assert L.cspn2d_k_bwd_f32(p, p, None, p, p, p, 1, 1, 4, 4, 24, 5, 2, 2, None, 0, None) == -1


def test_workspace_formulas():
    L = _lib.lib()
    for B, C, H, W in ((3, 2, 10, 15), (1, 1, 1, 1), (8, 1, 228, 304), (2, 5, 352, 1216)):
        HW = H * W
        for K in (3, 5, 7):
            for n in (1, 2, 24):
                assert L.cspn2d_paddle_workspace_bytes(B, C, H, W, K, n) == 4 * (B * K * K * HW + B * C * HW)
                assert L.cspn2d_paddle_bwd_workspace_bytes(B, C, H, W, K, n) == 4 * (B * K * K * HW + 2 * n * B * C * HW)
            assert L.cspn2d_paddle_workspace_bytes(B, C, H, W, K, 0) == 0
            assert L.cspn2d_paddle_bwd_workspace_bytes(B, C, H, W, K, 0) == 0
    for K in (1, 4, 9):
        assert L.cspn2d_paddle_workspace_bytes(2, 1, 8, 8, K, 3) == 0 and L.cspn2d_paddle_bwd_workspace_bytes(2, 1, 8, 8, K, 3) == 0
    assert L.cspn2d_paddle_workspace_bytes(0, 1, 8, 8, 3, 3) == 0 and L.cspn2d_paddle_bwd_workspace_bytes(1, 1, 8, -1, 3, 3) == 0


def test_module_surface_and_assertions():
    for K in (3, 5, 7):
        m = cspn_b200.Affinity_Propagate2DPaddle(12, K)
        assert (m.prop_time, m.prop_kernel) == (12, K)
        assert list(m.parameters()) == [] and list(m.buffers()) == [] and m.state_dict() == {}
    assert cspn_b200.Affinity_Propagate2DPaddle(24).prop_kernel == 3
    for K in (1, 2, 4, 9):
        with pytest.raises(AssertionError):
            cspn_b200.Affinity_Propagate2DPaddle(12, K)
    with pytest.raises(AssertionError):
        cspn_b200.Affinity_PropagateK(12, 5, 'paddle')                 # the K x K module keeps its norms
    d = torch.rand(1, 2, 4, 4)
    assert cspn_b200.Affinity_Propagate2DPaddle(0, 5)(torch.randn(1, 24, 4, 4), d) is d


@pytest.mark.parametrize('K', [3, 5, 7])
def test_wrong_channel_counts_are_value_errors_and_cpu_tensors_are_refused(K):
    nt = K * K - 1
    m = cspn_b200.Affinity_Propagate2DPaddle(3, K)
    f1, f3 = torch.rand(1, 1, 6, 6), torch.rand(1, 3, 6, 6)
    for g, f in ((torch.randn(1, nt + 1, 6, 6), f1), (torch.randn(1, nt - 1, 6, 6), f1), (torch.randn(1, 2 * nt, 6, 6), f3),
                 (torch.randn(1, 2 * nt, 6, 6), f1), (torch.randn(2, nt, 6, 6), f1), (torch.randn(1, nt, 6, 5), f1)):
        with pytest.raises(ValueError):
            m(g, f)
        with pytest.raises(ValueError):
            cspn_b200.propagate2d_paddle(g, f, K, 3)
    for g, f in ((torch.randn(1, nt, 6, 6), f1), (torch.randn(1, nt, 6, 6), f3), (torch.randn(1, 3 * nt, 6, 6), f3)):
        with pytest.raises(cspn_b200.CspnError):
            m(g, f)
        with pytest.raises(cspn_b200.CspnError):
            cspn_b200.propagate2d_paddle(g, f, K, 3)
    with pytest.raises(AssertionError):
        cspn_b200.propagate2d_paddle(torch.randn(1, 15, 6, 6), f1, 4, 3)


@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schema_and_fake_kernels(ops):
    s = str(ops.propagate2d_paddle.default._schema)
    assert 'Tensor guidance, Tensor feat, int kernel_size, int prop_time' in s
    s = str(ops.propagate2d_paddle_backward.default._schema)
    assert 'Tensor grad_out, int kernel_size, int prop_time, bool need_guidance, bool need_feat' in s
    with FakeTensorMode():
        for K in (3, 5, 7):
            nt = K * K - 1
            for gch, C in ((nt, 1), (nt, 3), (3 * nt, 3)):
                g = torch.empty(2, gch, 16, 30, device='cuda')
                d = torch.empty(2, C, 16, 30, device='cuda')
                out = ops.propagate2d_paddle(g, d, K, 24)
                assert out.shape == d.shape and out.device == d.device and out.dtype == torch.float32
                gg, gd = ops.propagate2d_paddle_backward(g, d, out, K, 24, True, True)
                assert gg.shape == g.shape and gd.shape == d.shape
                gg, gd = ops.propagate2d_paddle_backward(g, d, out, K, 24, False, True)
                assert gg.numel() == 0 and gd.shape == d.shape
        with pytest.raises(Exception):
            ops.propagate2d_paddle(torch.empty(1, 25, 8, 8, device='cuda'), torch.empty(1, 1, 8, 8, device='cuda'), 5, 4)


@pytest.mark.parametrize('K', [3, 5, 7])
def test_forward_and_backward_trace_to_one_node_each(ops, K):
    def f(g, d):
        out = ops.propagate2d_paddle(g, d, K, 24)
        gg, gd = torch.autograd.grad(out.sum(), (g, d))
        return out, gg, gd

    g = torch.empty(1, K * K - 1, 12, 16, device='meta', requires_grad=True)
    d = torch.empty(1, 2, 12, 16, device='meta', requires_grad=True)
    gm = make_fx(f)(g, d)
    targets = [str(n.target) for n in gm.graph.nodes if n.op == 'call_function']
    assert sum('cspn_b200.propagate2d_paddle.default' in t for t in targets) == 1
    assert sum('cspn_b200.propagate2d_paddle_backward.default' in t for t in targets) == 1


def test_module_takes_the_dispatcher_route_when_the_shim_is_built(ops):
    m = cspn_b200.Affinity_Propagate2DPaddle(24, 7)
    assert m._use_op is True
    with FakeTensorMode():
        out = m(torch.empty(1, 48, 8, 8, device='cuda'), torch.empty(1, 2, 8, 8, device='cuda'))
        assert out.shape == (1, 2, 8, 8)
        out = m(torch.empty(1, 96, 8, 8, device='cuda'), torch.empty(1, 2, 8, 8, device='cuda'))
        assert out.shape == (1, 2, 8, 8)
