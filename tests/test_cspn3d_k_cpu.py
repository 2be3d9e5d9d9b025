"""CPU tests of the K x K x K 3D propagation (K in {3, 5}): the oracle's generalisation against the existing 3D arithmetic
and against the torch port in fp64, the C ABI's validation and workspace formulas, the module surface, and the dispatcher
registration (fake kernels, one traced node per direction)."""
import ctypes

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx

import cspn_b200
from cspn_b200 import _lib
from oracle import cspn_numpy as onp
from oracle import cspn_numpy_3d_k as onk
from oracle import cspn_torch_port as tp
from oracle import cspn_torch_port_3d_k as tpk

NORMS5 = ('124sum', '124sum_abs', 'paddle')


def inputs_3d(seed, B, C, D, H, W, K, signed=True):
    """Guidance with K**3-1 channels (randn, or rand like demo.py) and feat = rand, from a seed."""
    gen = torch.Generator().manual_seed(seed)
    nt = K ** 3 - 1
    g = torch.randn(B, nt, D, H, W, generator=gen) if signed else torch.rand(B, nt, D, H, W, generator=gen)
    return g, torch.rand(B, C, D, H, W, generator=gen)


def test_offsets_3d_follow_their_definition():
    assert onk.offsets_3d(3) == onp.OFFSETS_3D == tp.OFFSETS_3D == tpk.offsets_3d(3)
    offs = onk.offsets_3d(5)
    assert offs == tpk.offsets_3d(5)
    assert len(offs) == len(set(offs)) == 124 and (0, 0, 0) not in offs
    expected = [(2 - f, 2 - t, 2 - l) for f in range(5) for t in range(5) for l in range(5) if (f, t, l) != (2, 2, 2)]
    assert list(offs) == expected
    assert offs == tuple(reversed([(-a, -b, -c) for a, b, c in offs]))   # raster order: reversed taps negate
    with pytest.raises(AssertionError):
        onk.offsets_3d(7)


@pytest.mark.parametrize('norm', ['26sum', '26sum_abs', 'paddle'])
@pytest.mark.parametrize('shape,n', [((2, 1, 6, 10, 12), 4), ((1, 2, 5, 5, 12), 3), ((1, 1, 1, 9, 11), 3), ((1, 1, 5, 1, 1), 2)])
def test_k3_gives_the_bits_of_the_3d_oracle_and_port(norm, shape, n):
    B, C, D, H, W = shape
    g, f = inputs_3d(D + H + W, B, C, D, H, W, 3, signed=(norm != 'paddle'))
    a = onp.cspn3d(g.numpy(), f.numpy(), n, norm)
    b = onk.cspn3d_k(g.numpy(), f.numpy(), n, 3, norm)
    assert np.array_equal(a, b, equal_nan=True)
    with torch.no_grad():
        assert torch.equal(tp.cspn3d_torch(g, f, n, norm), tpk.cspn3d_torch_k(g, f, n, 3, norm))


@pytest.mark.parametrize('norm', NORMS5)
@pytest.mark.parametrize('shape,n', [((1, 2, 6, 7, 9), 3), ((2, 1, 3, 3, 3), 2), ((1, 1, 1, 6, 4), 4), ((1, 1, 9, 2, 1), 2)])
def test_k5_numpy_fp32_agrees_with_the_torch_port_in_fp64(norm, shape, n):
    """C = 2, volumes smaller than the 5 x 5 x 5 window, D / H / W of 1 or 2."""
    B, C, D, H, W = shape
    g, f = inputs_3d(7 * D + H + W, B, C, D, H, W, 5, signed=(norm == '124sum'))
    out = onk.cspn3d_k(g.numpy(), f.numpy(), n, 5, norm)
    with torch.no_grad():
        ref = tpk.cspn3d_torch_k(g.double(), f.double(), n, 5, norm).numpy()
    ok, ratio, normwise = onp.parity_ok(out, ref, 1e-4)
    assert ok, (ratio, normwise)
    assert np.allclose(onk.cspn3d_k(g.numpy(), f.numpy(), n, 5, norm, dtype=np.float64), ref, rtol=1e-12, atol=1e-12)


def test_k5_gathered_weights_sum_to_one_inside():
    g, _ = inputs_3d(3, 1, 1, 9, 10, 11, 5, signed=False)
    gate, gate_sum = onk.affinity_normalization_3d_k(g.numpy(), 5, '124sum_abs')
    assert gate.shape == (1, 124, 9, 10, 11)
    assert np.allclose(gate_sum[..., 2:-2, 2:-2, 2:-2], 1.0, atol=1e-5)
    gate, gate_sum = onk.affinity_normalization_3d_k(g.numpy(), 5, 'paddle')
    assert np.allclose(gate_sum, 1.0, atol=1e-5)


def _p():
    buf = (ctypes.c_float * 64)()
    return ctypes.cast(buf, ctypes.c_void_p), buf


def test_c_abi_rejects_bad_arguments_without_a_device():
    L = _lib.lib()
    p, _keep = _p()
    ok_args = dict(B=1, C=1, D=3, H=4, W=4, K=5, iters=2, norm=0)

    def f(g=p, d=p, o=p, **over):
        a = dict(ok_args, **over)
        return L.cspn3d_k_fwd_f32(g, d, o, a['B'], a['C'], a['D'], a['H'], a['W'], a['K'], a['iters'], a['norm'], None, 0, None)

    def b(g=p, d=p, go=p, **over):
        a = dict(ok_args, **over)
        return L.cspn3d_k_bwd_f32(g, d, go, p, p, a['B'], a['C'], a['D'], a['H'], a['W'], a['K'], a['iters'], a['norm'],
                                  None, 0, None)

    for call in (f, b):
        for K in (1, 2, 4, 6, 7, 9):
            assert call(K=K) == -1
        assert b'kernel size' in L.cspn_last_error()
        for norm in (-1, 3, 7):
            assert call(norm=norm) == -1
        assert call(iters=-1) == -1 and call(iters=-5) == -1
        for dim in ('B', 'C', 'D', 'H', 'W'):
            assert call(**{dim: 0}) == -1 and call(**{dim: -3}) == -1
        assert call(g=None) == -1 and call(d=None) == -1
    assert f(o=None) == -1 and b(go=None) == -1
    assert b'null' in L.cspn_last_error()

    def b3(g=p, d=p, go=p, **over):     # the 3x3x3 backward names the offending argument like its siblings
        a = dict(ok_args, **over)
        rc = L.cspn3d_bwd_f32(g, d, go, p, p, a['B'], a['C'], a['D'], a['H'], a['W'], a['iters'], a['norm'], None, 0, None)
        return rc, L.cspn_last_error()

    for kw, msg in ([(dict(g=None), b'null'), (dict(d=None), b'null'), (dict(go=None), b'null'), (dict(iters=-1), b'>= 0')] +
                    [({dim: v}, b'non-positive shape') for dim in ('B', 'C', 'D', 'H', 'W') for v in (0, -3)] +
                    [(dict(norm=n), b'unknown 3D norm_type') for n in (-1, 3, 7)]):
        rc, err = b3(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)


def test_workspace_formulas():
    L = _lib.lib()
    B, C, D, H, W = 3, 2, 4, 5, 6
    V = D * H * W
    # pinned numbers: forward G*(125 + C)*V floats for N > 1 (G = B here), 125*V*G for N = 1; backward (125 + (2N-1)*C)*V
    assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, 5, 2) == 182880
    assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, 5, 1) == 180000
    assert L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, 5, 2) == 62880
    assert L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, 5, 1) == 60960
    for n in (2, 12, 24):
        assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, 5, n) == 4 * B * (125 * V + C * V)
        assert L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, 5, n) == 4 * (125 * V + (2 * n - 1) * C * V)
    assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, 5, 0) == 0 and L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, 5, 0) == 0
    for n in (0, 1, 12):      # K = 3 is the 3D operator: its queries are theirs
        assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, 3, n) == L.cspn3d_workspace_bytes(B, C, D, H, W, n)
        assert L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, 3, n) == L.cspn3d_bwd_workspace_bytes(B, C, D, H, W, n)
    for n in (1, 2, 12, 24):  # the 3x3x3 backward: (27 + (2N-1)*C)*V floats
        assert L.cspn3d_bwd_workspace_bytes(B, C, D, H, W, n) == 4 * (27 * V + (2 * n - 1) * C * V)
    assert L.cspn3d_bwd_workspace_bytes(B, C, D, H, W, 0) == 0
    for K in (4, 7):
        assert L.cspn3d_k_workspace_bytes(B, C, D, H, W, K, 3) == 0 and L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, K, 3) == 0
    # the demo.py volume (3 x 1 x 48 x 64 x 128, N = 24) runs as one group: 3 * 126 planes
    V = 48 * 64 * 128
    assert L.cspn3d_k_workspace_bytes(3, 1, 48, 64, 128, 5, 24) == 4 * 3 * 126 * V


def test_volume_groups_follow_the_workspace_cap(monkeypatch):
    """The group size of the 5x5x5 path is the 3x3x3 path's group3d with 125 planes per volume."""
    L = _lib.lib()
    V = 6 * 10 * 16
    per_vol = 4 * (125 * V + V)                                    # 483840 B
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str(1000))         # two volumes per group
    assert L.cspn3d_k_workspace_bytes(5, 1, 6, 10, 16, 5, 3) == 2 * per_vol
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str(100))          # below one volume: groups of one
    assert L.cspn3d_k_workspace_bytes(5, 1, 6, 10, 16, 5, 3) == per_vol
    # the 3x3x3 path sizes its groups as before: 29 planes per volume at C = 2, N > 1
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str(300))
    assert L.cspn3d_workspace_bytes(3, 2, 6, 10, 16, 4) == 2 * 4 * 29 * V


def test_module_surface_and_assertions():
    for K, default in ((3, '26sum_abs'), (5, '124sum_abs')):
        m = cspn_b200.Affinity_Propagate3DK(12, K)
        assert (m.prop_time, m.prop_kernel, m.norm_type) == (12, K, default)
        assert list(m.parameters()) == [] and list(m.buffers()) == [] and m.state_dict() == {}
        for name in (default[:-4], 'paddle'):
            assert cspn_b200.Affinity_Propagate3DK(12, K, name).norm_type == name
    for K in (1, 2, 4, 6, 7):
        with pytest.raises(AssertionError):
            cspn_b200.Affinity_Propagate3DK(12, K)
    for K, name in ((5, '26sum'), (5, '26sum_abs'), (3, '124sum'), (5, '8sum'), (5, '24sum_abs'), (5, 'Paddle')):
        with pytest.raises(AssertionError):
            cspn_b200.Affinity_Propagate3DK(12, K, name)
    with pytest.raises(AssertionError):
        cspn_b200.Affinity_Propagate3D(12, 5)                  # the 3x3x3 module keeps its contract
    f = torch.rand(1, 1, 3, 4, 4)
    assert cspn_b200.Affinity_Propagate3DK(0, 5)(torch.randn(1, 124, 3, 4, 4), f) is f
    assert 'prop_kernel=5' in repr(cspn_b200.Affinity_Propagate3DK(4, 5, 'paddle'))


@pytest.mark.parametrize('gch,C', [(123, 1), (125, 1), (26, 1), (248, 1), (248, 3), (373, 3)])
def test_wrong_guidance_channel_counts_are_value_errors(gch, C):
    m = cspn_b200.Affinity_Propagate3DK(3, 5, 'paddle')
    with pytest.raises(ValueError):
        m(torch.randn(1, gch, 3, 4, 4), torch.rand(1, C, 3, 4, 4))
    with pytest.raises(ValueError):
        cspn_b200.propagate3d_k(torch.randn(1, gch, 3, 4, 4), torch.rand(1, C, 3, 4, 4), 5, 3)


def test_cpu_tensors_are_refused():
    for K, nt in ((5, 124), (3, 26)):
        with pytest.raises(cspn_b200.CspnError):
            cspn_b200.propagate3d_k(torch.randn(1, nt, 3, 4, 4), torch.rand(1, 1, 3, 4, 4), K, 3)
        with pytest.raises(cspn_b200.CspnError):    # the module: shared gates and per-channel gates
            cspn_b200.Affinity_Propagate3DK(3, K)(torch.randn(1, nt, 3, 4, 4), torch.rand(1, 1, 3, 4, 4))
        with pytest.raises(cspn_b200.CspnError):
            cspn_b200.Affinity_Propagate3DK(3, K)(torch.randn(1, 2 * nt, 3, 4, 4), torch.rand(1, 2, 3, 4, 4))
    with pytest.raises(AssertionError):
        cspn_b200.propagate3d_k(torch.randn(1, 124, 3, 4, 4), torch.rand(1, 1, 3, 4, 4), 5, 3, '26sum')


@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schema_and_fake_kernels(ops):
    s = str(ops.propagate3d_k.default._schema)
    assert 'Tensor guidance, Tensor feat, int kernel_size, int prop_time, int norm_type' in s
    with FakeTensorMode():
        for K in (3, 5):
            g = torch.empty(2, K ** 3 - 1, 6, 10, 12, device='cuda')
            f = torch.empty(2, 3, 6, 10, 12, device='cuda')
            out = ops.propagate3d_k(g, f, K, 12, 2)
            assert out.shape == f.shape and out.device == f.device and out.dtype == torch.float32
            gg, gf = ops.propagate3d_k_backward(g, f, out, K, 12, 1, True, True)
            assert gg.shape == g.shape and gf.shape == f.shape
            gg, gf = ops.propagate3d_k_backward(g, f, out, K, 12, 0, False, True)
            assert gg.numel() == 0 and gf.shape == f.shape
        with pytest.raises(Exception):
            ops.propagate3d_k(torch.empty(1, 123, 4, 4, 4, device='cuda'), torch.empty(1, 1, 4, 4, 4, device='cuda'), 5, 4, 0)


def test_forward_and_backward_trace_to_one_node_each(ops):
    def f(g, d):
        out = ops.propagate3d_k(g, d, 5, 12, 2)
        gg, gd = torch.autograd.grad(out.sum(), (g, d))
        return out, gg, gd

    g = torch.empty(1, 124, 4, 6, 8, device='meta', requires_grad=True)
    d = torch.empty(1, 1, 4, 6, 8, device='meta', requires_grad=True)
    gm = make_fx(f)(g, d)
    targets = [str(n.target) for n in gm.graph.nodes if n.op == 'call_function']
    assert sum('cspn_b200.propagate3d_k.default' in t for t in targets) == 1
    assert sum('cspn_b200.propagate3d_k_backward.default' in t for t in targets) == 1


def test_module_takes_the_dispatcher_route_when_the_shim_is_built(ops):
    m = cspn_b200.Affinity_Propagate3DK(24, 5, 'paddle')
    assert m._use_op is True
    with FakeTensorMode():
        out = m(torch.empty(1, 124, 4, 8, 8, device='cuda'), torch.empty(1, 2, 4, 8, 8, device='cuda'))
        assert out.shape == (1, 2, 4, 8, 8)
        out = m(torch.empty(2, 124 * 3, 4, 8, 8, device='cuda'), torch.empty(2, 3, 4, 8, 8, device='cuda'))   # per-channel gates
        assert out.shape == (2, 3, 4, 8, 8)
