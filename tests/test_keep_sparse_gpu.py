"""The keep-sparse mode on the GPU (DESIGN.md section 4.13): m = 1[sparse > 0], and every step replaces a sampled pixel by
its sample, so the output passes through the measurements.

1. Tied to the validated mode: with sparse = blur * 1[sampled] and blur > 0 the two modes compute the same numbers with the
   same operations, so keep-mode `out` has the default mode's bits under every forced cluster plan, on the generic path and
   for K = 5 / 7; for C = 1 grad_guidance is equal and grad_blur + grad_sparse is the default grad_blur.
2. Exact dyadic inputs (tests/cluster_exact.py) against the fp64 restatement (tests/keep_sparse_reference.py), bit for bit,
   forward and backward, under the forced plans and long runs.
3. Random inputs against fp64; the samples come out bit for bit.
4. IEEE cases against the op sequence in fp32 torch.
5. Plumbing: memory contract, fused gather with local slices as peers, the registered op, both Python routes, run to run.
"""
import ctypes

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op
from oracle import cspn_numpy as onp

import backward_exact as be
import cluster_exact as ce
import forced_plans as fpl
import keep_sparse_reference as ks
import memory_contract as mc

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def norm_code(norm):
    return 1 if norm.endswith('_abs') else 0


def keep_fwd(g, d, s, n, norm, K=3, algo=_lib.ALGO_AUTO, ws_off=0, fill='sentinel', keep=True):
    """cspn2d_keep_fwd_f32 (keep=False: the default mode's cspn2d_fwd_f32 / cspn2d_k_fwd_f32) on this thread, `out` and a
    workspace of exactly the queried size in guarded buffers, checked to be fully written and stored within.
    Returns (out on the CPU, algo run)."""
    L = _lib.lib()
    gc, dc = g.cuda().contiguous(), d.cuda().contiguous()
    sc = None if s is None else s.cuda().contiguous()
    B, C, H, W = dc.shape
    code = norm_code(norm)
    if keep:
        ws_bytes = L.cspn2d_keep_workspace_bytes(B, C, H, W, K, n, algo)
    else:
        ws_bytes = L.cspn2d_workspace_bytes(B, C, H, W, n, algo) if K == 3 else L.cspn2d_k_workspace_bytes(B, C, H, W, K, n)
    ws = mc.workspace(ws_bytes, ws_off, fill)
    out = mc.guarded(dc.shape)
    wp = ws.ptr() if ws_bytes else None
    if keep:
        rc = L.cspn2d_keep_fwd_f32(_ptr(gc), _ptr(dc), _ptr(sc), out.ptr(), B, C, H, W, gc.shape[1], K, n, code, algo, wp,
                                   ws_bytes, _stream())
    elif K == 3:
        rc = L.cspn2d_fwd_f32(_ptr(gc), _ptr(dc), _ptr(sc), out.ptr(), B, C, H, W, gc.shape[1], n, code, algo, wp, ws_bytes,
                              _stream())
    else:
        rc = L.cspn2d_k_fwd_f32(_ptr(gc), _ptr(dc), _ptr(sc), out.ptr(), B, C, H, W, gc.shape[1], K, n, code, wp, ws_bytes,
                                _stream())
    _lib.check(rc, 'forward')
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert ws.guards_intact(), 'a store landed past the workspace'
    return out.t.cpu(), L.cspn_last_algo()


def keep_bwd(g, d, s, go, n, norm, K=3, ws_off=0, fill='sentinel', keep=True):
    """cspn2d_keep_bwd_f32 (keep=False: cspn2d_k_bwd_f32) with every gradient in a guarded buffer.  Returns
    (grad_guidance, grad_blur, grad_sparse or None) on the CPU."""
    L = _lib.lib()
    gc, dc, goc = g.cuda().contiguous(), d.cuda().contiguous(), go.cuda().contiguous()
    sc = None if s is None else s.cuda().contiguous()
    B, C, H, W = dc.shape
    gg, gd = mc.guarded(gc.shape), mc.guarded(dc.shape)
    gs = mc.guarded(sc.shape) if keep and sc is not None else None
    if keep:
        ws_bytes = L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, K, n)
    else:
        ws_bytes = L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, K, n)
    ws = mc.workspace(ws_bytes, ws_off, fill)
    wp = ws.ptr() if ws_bytes else None
    if keep:
        rc = L.cspn2d_keep_bwd_f32(_ptr(gc), _ptr(dc), _ptr(sc), _ptr(goc), gg.ptr(), gd.ptr(), None if gs is None else gs.ptr(),
                                   B, C, H, W, gc.shape[1], K, n, norm_code(norm), wp, ws_bytes, _stream())
    else:
        rc = L.cspn2d_k_bwd_f32(_ptr(gc), _ptr(dc), _ptr(sc), _ptr(goc), gg.ptr(), gd.ptr(), B, C, H, W, gc.shape[1], K, n,
                                norm_code(norm), wp, ws_bytes, _stream())
    _lib.check(rc, 'backward')
    torch.cuda.synchronize()
    for buf, name in ((gg, 'grad_guidance'), (gd, 'grad_blur')) + (((gs, 'grad_sparse'),) if gs is not None else ()):
        mc.assert_written(buf, name)
    assert ws.guards_intact(), 'a store landed past the workspace'
    return gg.t.cpu(), gd.t.cpu(), None if gs is None else gs.t.cpu()


def tied_inputs(seed, B, C, H, W, gch=8):
    """Random guidance, blur > 0 and sparse = blur * 1[sampled] (one pixel in 5).  sparse is shared by the C channels, so
    at a sampled pixel every channel of blur holds the sample."""
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, gch, H, W, generator=gen)
    blur = torch.rand(B, C, H, W, generator=gen) + 0.1
    hot = torch.rand(B, 1, H, W, generator=gen) < 0.2
    blur = torch.where(hot, blur[:, :1], blur)
    go = torch.randn(B, C, H, W, generator=gen)
    return g, blur, blur[:, :1] * hot, go


def assert_tied(g, d, s, go, n, norm, K=3, algo=_lib.ALGO_AUTO, grads=True, what=''):
    ours, a1 = keep_fwd(g, d, s, n, norm, K, algo)
    theirs, a2 = keep_fwd(g, d, s, n, norm, K, algo, keep=False)
    assert a1 == a2, what
    assert torch.equal(ours, theirs), f'{what}: keep mode differs from the default mode'
    if grads and d.shape[1] == 1:
        gg, gd, gs = keep_bwd(g, d, s, go, n, norm, K)
        gg0, gd0, _ = keep_bwd(g, d, s, go, n, norm, K, keep=False)
        assert torch.equal(gg, gg0), f'{what}: grad_guidance'
        assert torch.equal(gd + gs, gd0), f'{what}: grad_blur + grad_sparse'


# ---- 1. tied to the validated mode ------------------------------------------------------------------------------------
FWD_PLANS = [(name, plan) for name in sorted(fpl.PROBLEMS) for plan in fpl.PROBLEMS[name].fwd]


@pytest.mark.parametrize('name,plan', FWD_PLANS, ids=[f'{n}-{p.cfg}-{p.cs}-{p.passes}-{int(p.chain)}' for n, p in FWD_PLANS])
def test_tied_to_default_mode_under_forced_plans(name, plan, monkeypatch):
    pb = fpl.PROBLEMS[name]
    fpl.force(monkeypatch, plan)
    if not fpl.plan_info(plan, pb.H, pb.W, pb.n)['supported']:
        pytest.skip(f'the device refuses {plan}')
    for C in sorted({pb.C, 3}):
        g, d, s, go = tied_inputs(pb.H + C, pb.B, C, pb.H, pb.W, pb.gch)
        # the backward of a forced plan: the problem's own backward plans
        grads = C == 1 and plan in pb.bwd
        for norm in fpl.NORMS:
            assert_tied(g, d, s, go, pb.n, norm, 3, _lib.ALGO_CLUSTER, grads, f'{name} {plan} C={C} {norm}')


@pytest.mark.parametrize('K', (3, 5, 7))
@pytest.mark.parametrize('W', (52, 37))
def test_tied_to_default_mode_generic_and_kxk(K, W, monkeypatch):
    for C in (1, 3):
        g, d, s, go = tied_inputs(K * W + C, 2, C, 29, W, K * K - 1)
        for norm in (f'{K * K - 1}sum', f'{K * K - 1}sum_abs'):
            for n in (1, 2, 9):
                assert_tied(g, d, s, go, n, norm, K, _lib.ALGO_GENERIC, True, f'K={K} W={W} C={C} {norm} n={n}')
                if K == 3 and W % 4 == 0:
                    assert_tied(g, d, s, go, n, norm, 3, _lib.ALGO_AUTO, True, f'auto W={W} C={C} {norm} n={n}')
    # the launch-per-step backward of the 3x3 operator
    monkeypatch.setenv('CSPN_B200_BWD', 'steps')
    if K == 3:
        g, d, s, go = tied_inputs(W, 2, 1, 29, W)
        assert_tied(g, d, s, go, 7, '8sum', 3, _lib.ALGO_GENERIC, True, f'steps W={W}')


# ---- 2. exact dyadic inputs against fp64 -------------------------------------------------------------------------------
def exact_reference(case, g, d, s, go):
    ref = ks.reference(g.double(), d.double(), s.double(), case.n, 3, case.norm, go.double())
    for t, what in zip(ref, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse')):
        be.check_exact(t, case.n, f'{case.name} {what}', ce.unit(case.family, case.n))
    return ref


def _plans_of(case):
    pb = fpl.PROBLEMS[case.problem]
    return pb.fwd, pb.bwd


@pytest.mark.parametrize('case', ce.FORCED, ids=[c.name for c in ce.FORCED])
def test_exact_under_forced_plans(case, monkeypatch):
    g, d, s, go = ce.inputs(case)
    if s is None:
        s = ce.sparse_points(torch.Generator().manual_seed(case.H), case.B, case.H, case.W, 'bernoulli')
    ref = exact_reference(case, g, d, s, go)
    fwd, bwd = _plans_of(case)
    for plan in fwd:
        fpl.force(monkeypatch, plan)
        info = fpl.plan_info(plan, case.H, case.W, case.n)
        if not info['supported']:
            continue
        out, algo = keep_fwd(g, d, s, case.n, case.norm, 3, _lib.ALGO_CLUSTER)
        assert _lib.ALGO_NAMES[algo] == 'cluster'
        ce.assert_exact(out, ref[0], info, f'{case.name} {plan} out')
    for plan in bwd if case.bwd else ():
        fpl.force(monkeypatch, plan)
        info = fpl.plan_info(plan, case.H, case.W, case.n)
        if not info['supported']:
            continue
        got = keep_bwd(g, d, s, go, case.n, case.norm)
        for t, r, what in zip(got, ref[1:], ('grad_guidance', 'grad_blur', 'grad_sparse')):
            ce.assert_exact(t, r, info, f'{case.name} {plan} {what}')


LONG_KEEP = [c for c in ce.LONG if c.name.startswith(('w516', 'tall700'))]


@pytest.mark.parametrize('case', LONG_KEEP, ids=[c.name for c in LONG_KEEP])
def test_exact_long_runs(case, monkeypatch):
    g, d, s, go = ce.inputs(case)
    if s is None:
        s = ce.sparse_points(torch.Generator().manual_seed(case.W), case.B, case.H, case.W, 'bernoulli')
    ref = exact_reference(case, g, d, s, go)
    for e in case.envs:
        ce.apply(monkeypatch, e)
        info = ce.plan_of(e, case.B, case.C, case.H, case.W, case.n)
        out, _ = keep_fwd(g, d, s, case.n, case.norm, 3, _lib.ALGO_CLUSTER)
        ce.assert_exact(out, ref[0], info, f'{case.name} {ce.describe(e)} out')
        got = keep_bwd(g, d, s, go, case.n, case.norm)
        for t, r, what in zip(got, ref[1:], ('grad_guidance', 'grad_blur', 'grad_sparse')):
            ce.assert_exact(t, r, info, f'{case.name} {ce.describe(e)} {what}')


@pytest.mark.parametrize('K', (5, 7))
@pytest.mark.parametrize('n', (1, 3, 5))
def test_exact_kxk(K, n):
    g, d, s, go = be.dyadic_2d(K * 10 + n, 2, 2, 19, 23, K, 'signed')
    norm = f'{K * K - 1}sum'
    ref = ks.reference(g.double(), d.double(), s.double(), n, K, norm, go.double())
    for t, what in zip(ref, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse')):
        be.check_exact(t, n, what)
    out, _ = keep_fwd(g, d, s, n, norm, K)
    assert torch.equal(out.double(), ref[0])
    for t, r, what in zip(keep_bwd(g, d, s, go, n, norm, K), ref[1:], ('grad_guidance', 'grad_blur', 'grad_sparse')):
        assert torch.equal(t.double(), r), what


# ---- 3. random inputs against fp64 ------------------------------------------------------------------------------------
def random_inputs(seed, B, C, H, W, K):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, K * K - 1, H, W, generator=gen)
    d = torch.rand(B, C, H, W, generator=gen) * 10
    hot = torch.rand(B, 1, H, W, generator=gen) < 0.05
    s = torch.where(hot, torch.rand(B, 1, H, W, generator=gen) * 10 + 0.01, torch.zeros(B, 1, H, W))
    s = torch.where(torch.rand(B, 1, H, W, generator=gen) < 0.02, -s - 1, s)      # negative values are not samples
    return g, d, s


def check_random(out, g, d, s, n, K, norm, what):
    ref = ks.reference(g.double(), d.double(), s.double(), n, K, norm).numpy()
    ok, ratio, normwise = onp.parity_ok(out.cpu().numpy(), ref, 1e-4)
    assert ok, f'{what}: ratio {ratio:.3g} normwise {normwise:.3g}'
    if n >= 1:
        hit = (s > 0).expand_as(d)
        assert torch.equal(out.cpu()[hit], s.expand_as(d)[hit]), f'{what}: a sample did not come out bit for bit'


SHAPES = [('nyu', 1, 1, 228, 304, (0, 1, 2, 5, 24, 48)), ('kitti', 1, 1, 352, 1216, (24, 48)),
          ('odd_w', 2, 3, 37, 133, (1, 2, 5, 24))]


@pytest.mark.parametrize('name,B,C,H,W,ns', SHAPES, ids=[s[0] for s in SHAPES])
def test_random_against_fp64(name, B, C, H, W, ns):
    for K in ((3, 5, 7) if name != 'kitti' else (3, 5)):
        g, d, s = random_inputs(H + K, B, C, H, W, K)
        for n in ns if K == 3 else ns[:3]:
            norm = f'{K * K - 1}sum_abs' if n % 2 else f'{K * K - 1}sum'
            out, _ = keep_fwd(g, d, s, n, norm, K)
            check_random(out, g, d, s, n, K, norm, f'{name} K={K} n={n}')


def test_views_at_odd_storage_offsets():
    """Views one float into their storage: AUTO takes the generic path (the cluster kernel needs 16-byte bases)."""
    B, C, H, W = 2, 2, 40, 64
    g0, d0, s0 = random_inputs(3, B, C, H, W, 3)
    g, d, s = [torch.empty(t.numel() + 1, device='cuda')[1:].view(t.shape).copy_(t) for t in (g0, d0, s0)]
    for n in (1, 5, 24):
        out = cspn_b200.propagate2d(g, d, s, n, '8sum', keep_sparse=True)
        assert _lib.ALGO_NAMES[_lib.lib().cspn_last_algo()] == 'generic'
        check_random(out, g0, d0, s0, n, 3, '8sum', f'view n={n}')
        out5 = cspn_b200.propagate2d_k(torch.cat([g] * 3, 1), d, s, 5, n, keep_sparse=True)
        check_random(out5, torch.cat([g0] * 3, 1), d0, s0, n, 5, '24sum', f'view K=5 n={n}')


# ---- 4. IEEE cases against the op sequence in fp32 ---------------------------------------------------------------------
def ieee_inputs(K):
    gen = torch.Generator().manual_seed(K)
    B, C, H, W = 1, 2, 16, 24
    g = torch.randn(B, K * K - 1, H, W, generator=gen)
    g[:, :, 2:8, 3:9] = 0            # zero affinity sums (0/0 = NaN): a patch holding sampled and unsampled pixels
    d = torch.rand(B, C, H, W, generator=gen) + 0.5
    s = torch.zeros(B, 1, H, W)
    s[0, 0, 4, 5] = 2.0              # sampled, zero affinity sum
    s[0, 0, 12, 4] = float('nan')
    s[0, 0, 13, 20] = float('inf')
    s[0, 0, 3, 18] = -float('inf')
    s[0, 0, 9, 12] = -2.0
    s[0, 0, 14, 10] = 3.0
    d[0, 0, 14, 10] = float('inf')   # inf blur at a sampled pixel
    s[0, 0, 10, 16] = 1.5
    return g, d, s


@pytest.mark.parametrize('K', (3, 5, 7))
def test_ieee_cases(K):
    g, d, s = ieee_inputs(K)
    norm = f'{K * K - 1}sum'
    for n in (1, 2, 3):
        ref = ks.op_sequence(g, d, s, n, K, norm)
        for algo in ((_lib.ALGO_CLUSTER, _lib.ALGO_GENERIC) if K == 3 else (_lib.ALGO_AUTO,)):
            out, _ = keep_fwd(g, d, s, n, norm, K, algo)
            what = f'K={K} n={n} algo={algo}'
            assert torch.equal(torch.isnan(out), torch.isnan(ref)), what
            fin = torch.isfinite(ref)
            assert torch.equal(torch.isfinite(out), fin), what
            assert torch.equal(out[torch.isinf(ref)], ref[torch.isinf(ref)]), what
            assert torch.allclose(out[fin], ref[fin], rtol=1e-5, atol=1e-5), what


# ---- 5. plumbing ------------------------------------------------------------------------------------------------------
MEMORY_CASES = [(3, _lib.ALGO_CLUSTER, None), (3, _lib.ALGO_CLUSTER, 2), (3, _lib.ALGO_GENERIC, None), (5, 0, None),
                (7, 0, None)]


@pytest.mark.parametrize('K,algo,passes', MEMORY_CASES)
def test_memory_contract(K, algo, passes, monkeypatch):
    """Exact outputs (guarded, fully written), inputs untouched, and no workspace word read before it is written: a
    sentinel-filled and a zero-filled workspace at two offsets give the same bits."""
    if passes:
        monkeypatch.setenv('CSPN_B200_FORCE_PASSES', str(passes))
    g, d, s = random_inputs(K, 2, 2, 40, 64, K)
    go = torch.randn(d.shape, generator=torch.Generator().manual_seed(1))
    norm = f'{K * K - 1}sum'
    ins = [t.cuda() for t in (g, d, s, go)]
    before = mc.snapshot(ins)
    runs = [keep_fwd(*ins[:3], 9, norm, K, algo, off, fill)[0] for off, fill in ((0, 'sentinel'), (16, 'zero'))]
    assert mc.same_bits(*runs)
    grads = [keep_bwd(*ins, 9, norm, K, off, fill) for off, fill in ((0, 'sentinel'), (16, 'zero'))]
    for a, b in zip(*grads):
        assert mc.same_bits(a, b)
    assert mc.unchanged(before, ins)


@pytest.mark.parametrize('K', (3, 5, 7))
def test_fused_gather_with_local_peers(K):
    """n_peer + 1 ranks emulated on one GPU: guarded local buffers stand in for the peers' gather buffers."""
    L = _lib.lib()
    g, d, s = [t.cuda() for t in random_inputs(K + 20, 2, 2, 40, 64, K)]
    B, C, H, W = d.shape
    norm = f'{K * K - 1}sum'
    for n in (1, 2, 5):
        ref, _ = keep_fwd(g, d, s, n, norm, K)
        ws_bytes = L.cspn2d_keep_workspace_bytes(B, C, H, W, K, n, _lib.ALGO_CLUSTER)
        for n_peer in (0, 1, 7):
            out = mc.guarded(d.shape)
            peers = [mc.guarded(d.shape) for _ in range(n_peer)]
            ws = mc.workspace(ws_bytes)
            arr = (ctypes.c_void_p * max(n_peer, 1))(*[p.ptr() for p in peers])
            rc = L.cspn2d_keep_fwd_gather_f32(g.data_ptr(), d.data_ptr(), s.data_ptr(), out.ptr(), arr if n_peer else None,
                                              n_peer, None, B, C, H, W, g.shape[1], K, n, 0, ws.ptr() if ws_bytes else None,
                                              ws_bytes, _stream())
            _lib.check(rc, 'cspn2d_keep_fwd_gather_f32')
            torch.cuda.synchronize()
            for buf in [out] + peers:
                mc.assert_written(buf, 'gather destination')
                assert torch.equal(buf.t.cpu(), ref), f'K={K} n={n} n_peer={n_peer}'


def test_opcheck():
    torch_op.load()
    g, d, s = [t.cuda() for t in random_inputs(7, 1, 1, 12, 16, 3)]
    for t in (g, d, s):
        t.requires_grad_(True)
    for K, gg in ((3, g), (5, torch.cat([g] * 3, 1).detach().requires_grad_(True))):
        torch.library.opcheck(torch.ops.cspn_b200.propagate2d_keep.default, (gg, d, s, K, 4, 0, 0),
                              test_utils=('test_schema', 'test_faketensor', 'test_autograd_registration',
                                          'test_aot_dispatch_dynamic'))


class KeepCaller(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.head = torch.nn.Conv2d(2, 9, 3, padding=1)
        self.cspn = cspn_b200.Affinity_Propagate(6, 3, '8sum', keep_sparse=True)

    def forward(self, x, sparse):
        h = self.head(x)
        return self.cspn(h[:, :8], h[:, 8:].abs() + 0.1, sparse)


def test_torch_compile_fullgraph():
    torch.manual_seed(0)
    net = KeepCaller().cuda()
    x = torch.rand(2, 2, 32, 48, device='cuda')
    sparse = (torch.rand(2, 1, 32, 48, device='cuda') < 0.1).float() * 3
    ref = net(x, sparse)
    cnet = torch.compile(net, fullgraph=True, backend='aot_eager')
    out = cnet(x, sparse)
    out.sum().backward()
    assert torch.allclose(out, ref, rtol=1e-6, atol=1e-6)
    hit = (sparse > 0).expand_as(out)
    assert torch.equal(out[hit], sparse.expand_as(out)[hit])


@pytest.mark.parametrize('K', (3, 5, 7))
def test_both_python_routes_and_two_runs_give_equal_bits(K, monkeypatch):
    g0, d0, s0 = [t.cuda() for t in random_inputs(K + 40, 2, 2, 40, 64, K)]
    go = torch.randn(d0.shape, device='cuda')
    norm = f'{K * K - 1}sum'

    def run(mod):
        g, d, s = [t.clone().requires_grad_(True) for t in (g0, d0, s0)]
        out = mod(g, d, s)
        out.backward(go)
        return [out.detach(), g.grad, d.grad, s.grad]

    make = (lambda: cspn_b200.Affinity_Propagate(7, 3, '8sum', keep_sparse=True)) if K == 3 else \
        (lambda: cspn_b200.Affinity_PropagateK(7, K, norm, keep_sparse=True))
    op = make()
    assert op._use_op
    monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', '1')
    ct = make()
    assert not ct._use_op
    a, b, c = run(op), run(ct), run(op)
    for x, y, z, what in zip(a, b, c, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse')):
        assert torch.equal(x, y), f'{what}: registered op and ctypes route differ'
        assert torch.equal(x, z), f'{what}: two runs differ'
    ref = ks.reference(g0.double().cpu(), d0.double().cpu(), s0.double().cpu(), 7, K, norm, go.double().cpu())
    for x, r, what in zip(a, ref, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse')):
        assert torch.allclose(x.double().cpu(), r, rtol=1e-3, atol=1e-3), what


def test_no_sparse_is_the_default_mode_and_n0_is_blur():
    g, d, _ = [t.cuda() for t in random_inputs(9, 1, 2, 24, 32, 3)]
    for n in (0, 3):
        assert torch.equal(cspn_b200.propagate2d(g, d, None, n, keep_sparse=True), cspn_b200.propagate2d(g, d, None, n))
    s = torch.rand(1, 1, 24, 32, device='cuda')
    gd = keep_bwd(g, d, s, torch.ones_like(d), 0, '8sum')
    assert (gd[0] == 0).all() and (gd[1] == 1).all() and (gd[2] == 0).all()
