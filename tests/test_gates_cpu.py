"""CPU tests of the propagation with caller-supplied gates (fluid.layers.affinity_propagate, 2D K in {3, 5, 7}, 3D K in
{3, 5}): the fp64 restatement (tests/gates_reference.py) against the 'paddle' references once the gates are normalised as
demo.py does, the C ABI's validation and workspace formulas, the Python validation, and the dispatcher registration (schemas,
fake kernels, one traced node per direction)."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx

import cspn_b200
from cspn_b200 import _lib
from oracle import cspn_torch_port_3d_k as tp3

import backward_exact as be
import gates_reference as gr
import paddle2d_reference as pr


def guidance(seed, shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


# ---- 1. the restatement is 'paddle' without its first line ------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5])
@pytest.mark.parametrize('per_channel', [False, True])
def test_normalised_gates_give_the_2d_paddle_reference(K, per_channel):
    B, C, H, W, N = 2, 3, 11, 13, 4
    nt = K * K - 1
    g = guidance(K, (B, nt * C if per_channel else nt, H, W))
    f = guidance(K + 1, (B, C, H, W))
    ours = gr.affinity_propagate_ref(f, gr.paddle_gates(g, nt), K, N)
    ref = pr.cspn2d_torch_paddle(g, f, N, K)
    assert torch.allclose(ours, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('K', [3, 5])
@pytest.mark.parametrize('per_channel', [False, True])
def test_normalised_gates_give_the_3d_paddle_reference(K, per_channel):
    B, C, D, H, W, N = 2, 2, 4, 6, 7, 3
    nt = K ** 3 - 1
    g = guidance(10 + K, (B, nt * C if per_channel else nt, D, H, W))
    f = guidance(11 + K, (B, C, D, H, W))
    ours = gr.affinity_propagate_ref(f, gr.paddle_gates(g, nt), K, N)
    ref = be.cspn3d_ref(g, f, N, K, 'paddle')
    assert torch.allclose(ours, ref, rtol=1e-12, atol=1e-12)
    if not per_channel:
        assert torch.allclose(ref, tp3.cspn3d_torch_k(g, f, N, K, 'paddle'), rtol=0, atol=0)


def test_gates_are_used_as_given():
    """Signed gates that do not sum to one: one step is the plain weighted sum of the shifted neighbours."""
    K, H, W = 3, 5, 6
    g = guidance(1, (1, 8, H, W))
    f = guidance(2, (1, 1, H, W))
    out = gr.affinity_propagate_ref(f, g, K, 1)
    y, x = 2, 3
    want = sum(g[0, k, y, x] * f[0, 0, y + dy, x + dx] for k, (dy, dx) in enumerate(be.offsets(K, 2)))
    assert torch.allclose(out[0, 0, y, x], want, rtol=1e-14, atol=0)
    assert torch.equal(gr.affinity_propagate_ref(f, g, K, 0), f)


def test_an_infinite_gate_on_a_padding_tap_gives_nan():
    g = torch.zeros(1, 8, 4, 4, dtype=torch.float64)
    g[0, 0, 0, 0] = float('inf')                  # tap 0 reads (dy, dx) = (+1, +1): inside at (0, 0)
    g[0, 7, 0, 0] = float('inf')                  # tap 7 reads (-1, -1): the padding
    f = torch.ones(1, 1, 4, 4, dtype=torch.float64)
    out = gr.affinity_propagate_ref(f, g, 3, 1)
    assert torch.isnan(out[0, 0, 0, 0]) and torch.isfinite(out[0, 0, 1:, 1:]).all()


# ---- 2. the C ABI -----------------------------------------------------------------------------------------------------
def _p():
    buf = (ctypes.c_float * 64)()
    return ctypes.cast(buf, ctypes.c_void_p), buf


@pytest.mark.parametrize('nd', [2, 3])
def test_c_abi_rejects_bad_arguments(nd):
    L = _lib.lib()
    p, _keep = _p()
    dims = ('B', 'C', 'H', 'W') if nd == 2 else ('B', 'C', 'D', 'H', 'W')
    ok_args = dict(B=1, C=1, D=2, H=4, W=4, K=5, iters=2)
    fwd, bwd = getattr(L, f'cspn{nd}d_gates_fwd_f32'), getattr(L, f'cspn{nd}d_gates_bwd_f32')

    def shape(a):
        return [a[d] for d in dims] + [a['K'], a['iters']]

    def f(g=p, d=p, o=p, **over):
        return fwd(g, d, o, *shape(dict(ok_args, **over)), None, 0, None)

    def b(g=p, d=p, go=p, gg=p, gd=p, **over):
        return bwd(g, d, go, gg, gd, *shape(dict(ok_args, **over)), None, 0, None)

    bad_k = (0, 1, 2, 4, 6, 9) if nd == 2 else (0, 1, 2, 4, 7)
    for call in (f, b):
        for K in bad_k:
            assert call(K=K) == -1
        assert call(iters=-1) == -1
        for dim in dims:
            assert call(**{dim: 0}) == -1 and call(**{dim: -3}) == -1
        assert call(g=None) == -1 and call(d=None) == -1
    assert f(o=None) == -1 and b(go=None) == -1
    assert b'null' in L.cspn_last_error()


def test_workspace_formulas():
    L = _lib.lib()
    for B, C, H, W in ((3, 2, 10, 15), (1, 1, 1, 1), (8, 1, 228, 304), (2, 5, 352, 1216)):
        n = B * C * H * W
        for K in (3, 5, 7):
            for N in (1, 2, 3, 24):
                assert L.cspn2d_gates_workspace_bytes(B, C, H, W, K, N) == (4 * n if N >= 2 else 0)
                assert L.cspn2d_gates_bwd_workspace_bytes(B, C, H, W, K, N) == 4 * (2 * N - 2) * n
            assert L.cspn2d_gates_workspace_bytes(B, C, H, W, K, 0) == 0
            assert L.cspn2d_gates_bwd_workspace_bytes(B, C, H, W, K, 0) == 0
    for B, C, D, H, W in ((2, 1, 3, 4, 5), (3, 2, 7, 19, 72), (3, 1, 48, 64, 128)):
        V = D * H * W
        for K in (3, 5):
            for N in (1, 2, 3, 24):
                # every volume of these fits one launch group
                assert L.cspn3d_gates_workspace_bytes(B, C, D, H, W, K, N) == (4 * B * C * V if N >= 2 else 0)
                assert L.cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, K, N) == 4 * (2 * N - 2) * C * V
            assert L.cspn3d_gates_workspace_bytes(B, C, D, H, W, K, 0) == 0
            assert L.cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, K, 0) == 0
    for K in (1, 4, 9):
        assert L.cspn2d_gates_workspace_bytes(2, 1, 8, 8, K, 3) == 0 and L.cspn2d_gates_bwd_workspace_bytes(2, 1, 8, 8, K, 3) == 0
    assert L.cspn3d_gates_workspace_bytes(2, 1, 4, 8, 8, 7, 3) == 0 and L.cspn3d_gates_bwd_workspace_bytes(2, 1, 4, 8, 8, 7, 3) == 0
    assert L.cspn2d_gates_workspace_bytes(0, 1, 8, 8, 3, 3) == 0 and L.cspn3d_gates_bwd_workspace_bytes(1, 1, 4, 8, -1, 3, 3) == 0


def test_3d_forward_workspace_follows_the_launch_groups(monkeypatch):
    """A cap on the workspace splits the batch into groups of G volumes; the forward workspace is then G*C*V floats."""
    L = _lib.lib()
    B, C, D, H, W = 5, 2, 4, 8, 16
    V = D * H * W
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str(2 * C * V * 4 / 1024))
    assert L.cspn3d_gates_workspace_bytes(B, C, D, H, W, 5, 3) == 4 * 2 * C * V
    assert L.cspn3d_gates_bwd_workspace_bytes(B, C, D, H, W, 5, 3) == 4 * 4 * C * V


# ---- 3. the Python surface --------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    ap = cspn_b200.affinity_propagate
    x2, x3 = torch.rand(1, 2, 6, 6), torch.rand(1, 2, 3, 6, 6)
    for K in (1, 2, 4, 9):
        with pytest.raises(AssertionError):
            ap(x2, torch.rand(1, K * K - 1, 6, 6), K)
    for K in (7, 1, 4):
        with pytest.raises(AssertionError):
            ap(x3, torch.rand(1, K ** 3 - 1, 3, 6, 6), K)
    for x, g in ((x2, torch.rand(1, 9, 6, 6)), (x2, torch.rand(1, 7, 6, 6)), (x2, torch.rand(1, 24, 6, 6)),
                 (x2, torch.rand(2, 8, 6, 6)), (x2, torch.rand(1, 8, 6, 5)), (x2, torch.rand(1, 8, 1, 6, 6)),
                 (torch.rand(1, 1, 6, 6), torch.rand(1, 16, 6, 6)), (x3, torch.rand(1, 27, 3, 6, 6)),
                 (x3, torch.rand(1, 26, 2, 6, 6)), (torch.rand(2, 6, 6), torch.rand(8, 6, 6))):
        with pytest.raises(ValueError):
            ap(x, g, 3, 2)
    with pytest.raises(ValueError):
        ap(x2, torch.rand(1, 8, 6, 6), 3, -1)
    with pytest.raises(RuntimeError):
        ap(x2.double(), torch.rand(1, 8, 6, 6).double(), 3, 2)
    for x, g, K in ((x2, torch.rand(1, 8, 6, 6), 3), (x2, torch.rand(1, 16, 6, 6), 3), (x2, torch.rand(1, 48, 6, 6), 7),
                    (x3, torch.rand(1, 26, 3, 6, 6), 3), (x3, torch.rand(1, 248, 3, 6, 6), 5)):
        for N in (0, 2):
            with pytest.raises(cspn_b200.CspnError):
                ap(x, g, K, N)
            with pytest.raises(cspn_b200.CspnError):
                ap(x.requires_grad_(True), g, K, N)
            x.requires_grad_(False)


# ---- 4. the dispatcher ops --------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import build, torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    for nd in (2, 3):
        s = str(getattr(ops, f'affinity_propagate{nd}d').default._schema)
        assert 'Tensor input, Tensor gate_weight, int kernel_size, int prop_step) -> Tensor' in s
        s = str(getattr(ops, f'affinity_propagate{nd}d_backward').default._schema)
        assert 'Tensor grad_out, int kernel_size, int prop_step, bool need_input, bool need_gate) -> (Tensor, Tensor)' in s
    with FakeTensorMode():
        for nd, sizes, sp in ((2, (3, 5, 7), (16, 30)), (3, (3, 5), (4, 8, 12))):
            op, bop = getattr(ops, f'affinity_propagate{nd}d'), getattr(ops, f'affinity_propagate{nd}d_backward')
            for K in sizes:
                nt = K ** nd - 1
                for gch, C in ((nt, 1), (nt, 3), (3 * nt, 3)):
                    g = torch.empty(2, gch, *sp, device='cuda')
                    x = torch.empty(2, C, *sp, device='cuda')
                    out = op(x, g, K, 24)
                    assert out.shape == x.shape and out.device == x.device and out.dtype == torch.float32
                    gx, gg = bop(x, g, out, K, 24, True, True)
                    assert gx.shape == x.shape and gg.shape == g.shape
                    gx, gg = bop(x, g, out, K, 24, True, False)
                    assert gx.shape == x.shape and gg.numel() == 0
        with pytest.raises(Exception):
            ops.affinity_propagate2d(torch.empty(1, 1, 8, 8, device='cuda'), torch.empty(1, 25, 8, 8, device='cuda'), 5, 4)
        with pytest.raises(Exception):
            ops.affinity_propagate3d(torch.empty(1, 1, 2, 8, 8, device='cuda'), torch.empty(1, 26, 2, 8, 8, device='cuda'), 7, 4)


@pytest.mark.parametrize('nd,K', [(2, 3), (2, 7), (3, 3), (3, 5)])
def test_forward_and_backward_trace_to_one_node_each(ops, nd, K):
    name = f'affinity_propagate{nd}d'

    def f(x, g):
        out = getattr(ops, name)(x, g, K, 6)
        gx, gg = torch.autograd.grad(out.sum(), (x, g))
        return out, gx, gg

    sp = (12, 16) if nd == 2 else (3, 6, 8)
    x = torch.empty(1, 2, *sp, device='meta', requires_grad=True)
    g = torch.empty(1, K ** nd - 1, *sp, device='meta', requires_grad=True)
    gm = make_fx(f)(x, g)
    targets = [str(n.target) for n in gm.graph.nodes if n.op == 'call_function']
    assert sum(f'cspn_b200.{name}.default' in t for t in targets) == 1
    assert sum(f'cspn_b200.{name}_backward.default' in t for t in targets) == 1


def test_the_function_takes_the_dispatcher_route_when_the_shim_is_built(ops):
    with FakeTensorMode():
        out = cspn_b200.affinity_propagate(torch.empty(1, 2, 8, 8, device='cuda'), torch.empty(1, 48, 8, 8, device='cuda'), 7, 3)
        assert out.shape == (1, 2, 8, 8)
        out = cspn_b200.affinity_propagate(torch.empty(1, 2, 3, 8, 8, device='cuda'),
                                           torch.empty(1, 248, 3, 8, 8, device='cuda'), 5, 3)
        assert out.shape == (1, 2, 3, 8, 8)
