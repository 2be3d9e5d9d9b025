"""Where every device entry point writes, and what it reads, called through the C ABI (ctypes).

Every output and gradient sits in a sentinel-filled buffer between guard bands (tests/memory_contract.py), and every
workspace has exactly the queried size.  For each case:
  - outputs: nothing is stored outside them and no element keeps the sentinel.  The values must equal the fp64
    reference, so the zeros a call owes are checked too: guidance-gradient channels >= K*K-1, guidance entries that only
    taps reading the padding would touch, metrics slot 11;
  - workspace: the call runs on a workspace at offset 0 and at 4 bytes past a 16-byte boundary (the metrics: 0 and 8),
    each filled once with the sentinel and once with zeros.  All four runs give the same bits (a read before write of
    the workspace would not), and nothing is stored past the workspace;
  - inputs, grad_out and sparse included, keep their bits;
  - backward: with either gradient pointer NULL the other one keeps its bits and nothing else is written.
A workspace 4 bytes off alignment moves the K x K, 3D and 2D-backward paths to their scalar / launch-per-step kernels.
On the dyadic inputs of tests/backward_exact.py every correct variant returns the bits of the fp64 reference.

The fused gather (cspn2d_fwd_gather_f32) is run on one GPU: slices of local buffers stand in for the other GPUs' gather
buffers, since its peer pointers are plain device addresses.  Out of scope here: stores to `multicast_out`, which need
an NVLS multicast object, and the FusedGather class, which needs a symmetric-memory rendezvous of several processes
(tools/gather_check.py runs both on a multi-GPU node).
"""
import ctypes

import numpy as np
import pytest
import torch

from cspn_b200 import _lib
from cspn_b200.synth import make_inputs

import backward_exact as be
import memory_contract as mc
from forced_plans import PROBLEMS, Plan, force, plan_info

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_WORKSPACE, ERR_UNSUPPORTED = -1, -2, -4


def stream():
    return torch.cuda.current_stream().cuda_stream


def dev(*ts):
    return [None if t is None else t.cuda().contiguous() for t in ts]


def ptr(t):
    return None if t is None else t.data_ptr()


def norm2(norm):
    return 1 if norm.endswith('_abs') else 0


def norm3(norm):
    return 2 if norm == 'paddle' else norm2(norm)


def last_error():
    return _lib.lib().cspn_last_error().decode()


def run_contract(call, inputs, out_shapes, ws_bytes, what, offsets=(0, 4)):
    """call(outs, ws_ptr) under a workspace at every offset, filled with the sentinel and with zeros.  Checks every output
    fully written with its guards intact, the workspace's guards, the inputs, and that all runs give the same bits.
    Returns the outputs of the first run (CPU)."""
    first = None
    for off in offsets:
        for fill in ('sentinel', 'zero'):
            tag = f'{what}, workspace +{off} B filled with {fill}'
            outs = [mc.guarded(s) for s in out_shapes]
            ws = mc.workspace(ws_bytes, off, fill)
            before = mc.snapshot(inputs)
            _lib.check(call([o.t for o in outs], ws.ptr()), what)
            torch.cuda.synchronize()
            for i, o in enumerate(outs):
                mc.assert_written(o, f'{tag}: output {i}')
            assert ws.guards_intact(), f'{tag}: a store landed outside the workspace'
            assert mc.unchanged(before, inputs), f'{tag}: an input changed'
            res = [o.t.cpu() for o in outs]
            if first is None:
                first = res
            for i, (a, b) in enumerate(zip(res, first)):
                assert mc.same_bits(a, b), f'{tag}: output {i} differs from the first run'
    return first


def run_null_grads(call, inputs, out_shapes, ws_bytes, full, what):
    """The backward with each gradient pointer NULL in turn: the other keeps the bits of the full call."""
    for drop in range(2):
        outs = [None if i == drop else mc.guarded(s) for i, s in enumerate(out_shapes)]
        ws = mc.workspace(ws_bytes)
        before = mc.snapshot(inputs)
        _lib.check(call([None if o is None else o.t for o in outs], ws.ptr()), what)
        torch.cuda.synchronize()
        keep = outs[1 - drop]
        mc.assert_written(keep, f'{what}, gradient {drop} NULL')
        assert mc.same_bits(keep.t.cpu(), full[1 - drop]), f'{what}: gradient {1 - drop} changed with gradient {drop} NULL'
        assert ws.guards_intact() and mc.unchanged(before, inputs), what


def assert_values(ours, refs, what):
    for i, (a, b) in enumerate(zip(ours, refs)):
        bad = a.double() != b
        assert not bad.any(), (what, i, f'{int(bad.sum())} of {bad.numel()} differ, first at {tuple(bad.nonzero()[0].tolist())}')


def bwd_ref(ref, g, x, go, N, fp32=True):
    """(grad_guidance, grad_x) of fp64 autograd of ref; at N = 0 the guidance is never read: zero and grad_out."""
    if N == 0:
        return torch.zeros(g.shape, dtype=torch.float64), go.double()
    return be.exact_reference(ref, g, x, go, N, fp32)[1:]


def fwd_ref_2d(g, d, s, N, K, norm):
    ref = be.cspn2d_shift_ref(g.double(), d.double(), None if s is None else s.double(), N, K, norm)
    be.check_exact(ref, N, 'out')
    return ref


# ---- 2D forward: cspn2d_fwd_f32 (3 x 3) and cspn2d_k_fwd_f32 (K = 5, 7) --------------------------------------------------
# (K, norm, H, W, B, C, N, sparse, gch, algo or KXK_GROUP)
FWD_2D = [
    (3, '8sum', 37, 136, 2, 3, 4, 'bernoulli', 8, _lib.ALGO_AUTO),
    (3, '8sum_abs', 37, 133, 3, 2, 2, 'signed', 10, _lib.ALGO_AUTO),
    (3, '8sum_abs', 37, 136, 1, 2, 3, None, 9, _lib.ALGO_GENERIC),
    (3, '8sum', 37, 136, 2, 1, 0, 'signed', 8, _lib.ALGO_AUTO),
    (3, '8sum', 37, 133, 1, 1, 0, None, 8, _lib.ALGO_GENERIC),
    (5, '24sum', 37, 136, 2, 2, 3, 'bernoulli', 24, None),
    (5, '24sum_abs', 37, 133, 1, 3, 2, 'signed', 26, None),
    (7, '48sum', 37, 136, 3, 1, 2, None, 50, 2),
    (7, '48sum_abs', 37, 133, 2, 2, 4, 'bernoulli', 48, None),
    (5, '24sum', 37, 136, 1, 1, 0, None, 24, None),
    (7, '48sum_abs', 37, 133, 1, 2, 0, 'signed', 48, None),
]


@pytest.mark.parametrize('K,norm,H,W,B,C,N,sparse,gch,opt', FWD_2D)
def test_2d_forward_writes_exactly_out(K, norm, H, W, B, C, N, sparse, gch, opt, monkeypatch):
    g, d, s, _ = be.dyadic_2d(H * W + N + K, B, C, H, W, K, sparse, gch)
    ref = fwd_ref_2d(g, d, s, N, K, norm)
    gc, dc, sc = dev(g, d, s)
    L = _lib.lib()
    if K == 3:
        ws_bytes = L.cspn2d_workspace_bytes(B, C, H, W, N, opt)
        call = lambda o, ws: L.cspn2d_fwd_f32(ptr(gc), ptr(dc), ptr(sc), ptr(o[0]), B, C, H, W, gch, N, norm2(norm), opt, ws,
                                              ws_bytes, stream())
    else:
        if opt:
            monkeypatch.setenv('CSPN_B200_KXK_GROUP', str(opt))
        ws_bytes = L.cspn2d_k_workspace_bytes(B, C, H, W, K, N)
        call = lambda o, ws: L.cspn2d_k_fwd_f32(ptr(gc), ptr(dc), ptr(sc), ptr(o[0]), B, C, H, W, gch, K, N, norm2(norm), ws,
                                                ws_bytes, stream())
    out = run_contract(call, [gc, dc, sc], [(B, C, H, W)], ws_bytes, f'K={K} forward')
    assert_values(out, [ref], (K, norm, H, W))


# ---- 2D backward: cspn2d_bwd_f32 (3 x 3) and cspn2d_k_bwd_f32 -------------------------------------------------------------
# (K, norm, H, W, B, C, N, sparse, gch, CSPN_B200_BWD or KXK_GROUP)
BWD_2D = [
    (3, '8sum', 37, 136, 2, 2, 3, 'bernoulli', 8, None),
    (3, '8sum_abs', 37, 133, 1, 3, 2, 'signed', 11, None),
    (3, '8sum', 37, 136, 2, 1, 4, None, 10, 'steps'),
    (3, '8sum_abs', 37, 136, 1, 1, 0, 'signed', 9, None),
    (5, '24sum', 37, 136, 2, 2, 3, 'bernoulli', 24, None),
    (5, '24sum_abs', 37, 133, 1, 2, 2, 'signed', 27, None),
    (7, '48sum', 37, 133, 3, 1, 2, None, 48, 2),
    (7, '48sum_abs', 37, 136, 1, 3, 3, 'bernoulli', 50, None),
    (5, '24sum_abs', 37, 133, 2, 1, 0, None, 25, None),
]


@pytest.mark.parametrize('K,norm,H,W,B,C,N,sparse,gch,opt', BWD_2D)
def test_2d_backward_writes_exactly_its_gradients(K, norm, H, W, B, C, N, sparse, gch, opt, monkeypatch):
    g, d, s, go = be.dyadic_2d(H * W + 7 * N + K, B, C, H, W, K, sparse, gch)
    ref_g, ref_d = bwd_ref(lambda gg, dd: be.cspn2d_shift_ref(gg, dd, s, N, K, norm), g, d, go, N)
    gc, dc, sc, goc = dev(g, d, s, go)
    L = _lib.lib()
    monkeypatch.delenv('CSPN_B200_BWD', raising=False)
    if opt == 'steps':
        monkeypatch.setenv('CSPN_B200_BWD', 'steps')
    elif opt:
        monkeypatch.setenv('CSPN_B200_KXK_GROUP', str(opt))
    if K == 3:
        ws_bytes = L.cspn2d_bwd_workspace_bytes(B, C, H, W, N)
        call = lambda o, ws: L.cspn2d_bwd_f32(ptr(gc), ptr(dc), ptr(sc), ptr(goc), ptr(o[0]), ptr(o[1]), B, C, H, W, gch, N,
                                              norm2(norm), ws, ws_bytes, stream())
    else:
        ws_bytes = L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, K, N)
        call = lambda o, ws: L.cspn2d_k_bwd_f32(ptr(gc), ptr(dc), ptr(sc), ptr(goc), ptr(o[0]), ptr(o[1]), B, C, H, W, gch, K,
                                                N, norm2(norm), ws, ws_bytes, stream())
    shapes = [(B, gch, H, W), (B, C, H, W)]
    inputs = [gc, dc, sc, goc]
    full = run_contract(call, inputs, shapes, ws_bytes, f'K={K} backward')
    assert_values(full, [ref_g, ref_d], (K, norm, H, W))
    assert torch.count_nonzero(full[0][:, K * K - 1:]) == 0
    run_null_grads(call, inputs, shapes, ws_bytes, full, f'K={K} backward')


# ---- 3D: cspn3d_{fwd,bwd}_f32 (K = 3) and cspn3d_k_{fwd,bwd}_f32 (K = 5) ---------------------------------------------------
def ragged_groups(monkeypatch, B, C, D, H, W, K, N):
    """CSPN_B200_MAX_WS3D_KB such that the forward runs its volumes in groups of 2, the last one ragged (B = 3)."""
    V = D * H * W
    per_vol = 4 * (K ** 3 * V + (C * V if N > 1 else 0))
    monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', str((2 * per_vol + per_vol // 2) / 1024))
    return 2 * per_vol


# (K, norm, D, H, W, B, C, N, env)
FWD_3D = [
    (3, '26sum', 7, 19, 72, 2, 2, 3, None),
    (3, '26sum_abs', 7, 19, 70, 1, 3, 2, None),
    (3, 'paddle', 7, 19, 72, 2, 1, 4, 'planes'),
    (3, '26sum', 7, 19, 72, 3, 1, 2, 'ragged'),
    (3, 'paddle', 7, 19, 70, 1, 1, 0, None),
    (5, '124sum', 7, 19, 72, 2, 1, 2, None),
    (5, '124sum_abs', 7, 19, 70, 1, 2, 3, None),
    (5, 'paddle', 7, 19, 72, 3, 1, 2, 'ragged'),
    (5, '124sum_abs', 7, 19, 72, 1, 1, 0, None),
]


@pytest.mark.parametrize('K,norm,D,H,W,B,C,N,env', FWD_3D)
def test_3d_forward_writes_exactly_out(K, norm, D, H, W, B, C, N, env, monkeypatch):
    g, f, _ = be.dyadic_3d(D * H * W + N + K, B, C, D, H, W, K, norm)
    ref = be.cspn3d_ref(g.double(), f.double(), N, K, norm)
    be.check_exact(ref, N, 'out')
    gc, fc = dev(g, f)
    L = _lib.lib()
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    if env in ('planes', 'ragged'):            # the grouped prep + weight-plane path, also for an aligned workspace
        monkeypatch.setenv('CSPN_B200_3D_PADDLE', 'planes')
    group_bytes = ragged_groups(monkeypatch, B, C, D, H, W, K, N) if env == 'ragged' else None
    ws_bytes = L.cspn3d_k_workspace_bytes(B, C, D, H, W, K, N)
    assert group_bytes in (None, ws_bytes)
    if K == 3:
        call = lambda o, ws: L.cspn3d_fwd_f32(ptr(gc), ptr(fc), ptr(o[0]), B, C, D, H, W, N, norm3(norm), ws, ws_bytes, stream())
    else:
        call = lambda o, ws: L.cspn3d_k_fwd_f32(ptr(gc), ptr(fc), ptr(o[0]), B, C, D, H, W, K, N, norm3(norm), ws, ws_bytes,
                                                stream())
    out = run_contract(call, [gc, fc], [(B, C, D, H, W)], ws_bytes, f'3D K={K} forward')
    assert_values(out, [ref], (K, norm, D, H, W))


BWD_3D = [
    (3, '26sum', 7, 19, 72, 2, 2, 3),
    (3, 'paddle', 7, 19, 70, 1, 3, 2),
    (3, '26sum_abs', 7, 19, 72, 1, 1, 0),
    (5, '124sum', 7, 19, 70, 1, 2, 2),
    (5, '124sum_abs', 7, 19, 72, 2, 1, 3),
    (5, 'paddle', 7, 19, 72, 1, 2, 2),
    (5, 'paddle', 7, 19, 70, 1, 1, 0),
]


@pytest.mark.parametrize('K,norm,D,H,W,B,C,N', BWD_3D)
def test_3d_backward_writes_exactly_its_gradients(K, norm, D, H, W, B, C, N):
    g, f, go = be.dyadic_3d(D * H * W + 5 * N + K, B, C, D, H, W, K, norm)
    ref_g, ref_f = bwd_ref(lambda gg, ff: be.cspn3d_ref(gg, ff, N, K, norm), g, f, go, N, fp32=K == 3)
    gc, fc, goc = dev(g, f, go)
    L = _lib.lib()
    ws_bytes = L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, K, N)
    if K == 3:
        call = lambda o, ws: L.cspn3d_bwd_f32(ptr(gc), ptr(fc), ptr(goc), ptr(o[0]), ptr(o[1]), B, C, D, H, W, N, norm3(norm),
                                              ws, ws_bytes, stream())
    else:
        call = lambda o, ws: L.cspn3d_k_bwd_f32(ptr(gc), ptr(fc), ptr(goc), ptr(o[0]), ptr(o[1]), B, C, D, H, W, K, N,
                                                norm3(norm), ws, ws_bytes, stream())
    shapes = [tuple(g.shape), (B, C, D, H, W)]
    inputs = [gc, fc, goc]
    full = run_contract(call, inputs, shapes, ws_bytes, f'3D K={K} backward')
    assert_values(full, [ref_g, ref_f], (K, norm, D, H, W))
    run_null_grads(call, inputs, shapes, ws_bytes, full, f'3D K={K} backward')


# ---- depth metrics and the masked L1 backward ------------------------------------------------------------------------------
def metric_inputs(n):
    """Integer predictions and power-of-two (or invalid 0) ground truth: every per-element term is a short dyadic, so
    the double sums are exact in any order and the 12 numbers are the reference's bits."""
    gen = torch.Generator().manual_seed(n)
    pred = torch.randint(1, 9, (n,), generator=gen).float()
    gt = torch.tensor([0.0, 1.0, 2.0, 4.0, 8.0])[torch.randint(0, 5, (n,), generator=gen)]
    return pred, gt


def metrics_ref(pred, gt):
    p, g = pred.numpy(), gt.numpy()
    v = g > np.float32(1e-4)
    out = np.zeros(12, np.float64)
    n = int(v.sum())
    out[0] = n
    p, g = p[v], g[v]
    diff = np.abs(g - p)
    out[1] = (diff.astype(np.float64) ** 2).sum() / n
    out[2] = np.sqrt(out[1])
    out[3] = diff.astype(np.float64).sum() / n
    out[4] = (diff / g).astype(np.float64).sum() / n
    ratio = np.maximum(g / p, p / g)
    thr = np.float32([1.02, 1.05, 1.10, 1.25, np.float32(1.25) * np.float32(1.25),
                      np.float32(1.25) * np.float32(1.25) * np.float32(1.25)])
    for t in range(6):
        out[5 + t] = (ratio < thr[t]).sum() / n
    return torch.from_numpy(out.astype(np.float32)).double()


def test_depth_metrics_write_twelve_floats_and_refuse_a_4_byte_aligned_workspace():
    n = 37 * 133
    pred, gt = metric_inputs(n)
    pc, gtc = dev(pred, gt)
    L = _lib.lib()
    ws_bytes = L.cspn_depth_metrics_workspace_bytes()
    call = lambda o, ws: L.cspn_depth_metrics_f32(ptr(pc), ptr(gtc), n, ptr(o[0]), ws, ws_bytes, stream())
    out = run_contract(call, [pc, gtc], [(12,)], ws_bytes, 'metrics', offsets=(0, 8))
    ref = metrics_ref(pred, gt)
    assert ref[11] == 0 and 0 < ref[0] < n
    assert_values(out, [ref], 'metrics')
    # 4 bytes off: CSPN_ERR_WORKSPACE, out12 and the workspace untouched
    o, ws = mc.guarded((12,)), mc.workspace(ws_bytes, 4)
    assert call([o.t], ws.ptr()) == ERR_WORKSPACE and '8-byte aligned' in last_error()
    torch.cuda.synchronize()
    assert o.untouched() and ws.untouched()


@pytest.mark.parametrize('grad_loss', [None, 0.5])
@pytest.mark.parametrize('offset', [0, 4])
def test_masked_l1_backward_writes_exactly_grad_pred(grad_loss, offset):
    n = 37 * 133
    pred, gt = metric_inputs(n)
    ref_stats = metrics_ref(pred, gt)
    pc, gtc, sc = dev(pred, gt, ref_stats.float())
    gl = None if grad_loss is None else torch.tensor([grad_loss], device='cuda')
    inputs = [pc, gtc, sc, gl]
    before = mc.snapshot(inputs)
    o = mc.guarded((n,), offset)
    _lib.check(_lib.lib().cspn_masked_l1_bwd_f32(ptr(pc), ptr(gtc), ptr(sc), ptr(gl), o.ptr(), n, stream()), 'masked L1')
    torch.cuda.synchronize()
    mc.assert_written(o, 'grad_pred')
    assert mc.unchanged(before, inputs)
    scale = np.float32(1) / np.float32(ref_stats[0]) * np.float32(1 if grad_loss is None else grad_loss)
    ref = torch.where(gt > 1e-4, torch.sign(pred - gt) * float(scale), torch.zeros(()))
    assert_values([o.t.cpu()], [ref.double()], 'masked L1')


# ---- a cluster plan of several passes with a misaligned workspace ----------------------------------------------------------
def fwd2d_call(gc, dc, sc, out, N, algo, ws_ptr, ws_bytes, norm=0):
    B, C, H, W = dc.shape
    return _lib.lib().cspn2d_fwd_f32(ptr(gc), ptr(dc), ptr(sc), out.ptr(), B, C, H, W, gc.shape[1], N, norm, algo, ws_ptr,
                                     ws_bytes, stream())


def multipass_inputs(case):
    if case == 'forced-2-passes':      # dyadic: the result is also the fp64 reference's
        g, d, s, _ = be.dyadic_2d(48, 2, 2, 37, 136, 3, 'bernoulli')
        return g, d, s, 4
    g, d, s = make_inputs(48, 1, 1, 228, 304, 8, 'bernoulli', 1000)     # N = 48 at NYU size: the planner's own split
    return g, d, s, 48


@pytest.mark.parametrize('case', ['forced-2-passes', 'n48'])
def test_multipass_plan_declines_a_misaligned_workspace(case, monkeypatch):
    monkeypatch.delenv('CSPN_B200_FORCE_CFG', raising=False)
    monkeypatch.delenv('CSPN_B200_FORCE_CS', raising=False)
    monkeypatch.setenv('CSPN_B200_CHAIN', '0')
    if case == 'forced-2-passes':
        monkeypatch.setenv('CSPN_B200_FORCE_PASSES', '2')
    else:
        monkeypatch.delenv('CSPN_B200_FORCE_PASSES', raising=False)
    g, d, s, N = multipass_inputs(case)
    gc, dc, sc = dev(g, d, s)
    B, C, H, W = d.shape
    L = _lib.lib()
    info = _lib.plan_info(H, W, N)
    assert info['supported'] and sum(p['count'] for p in info['passes']) > 1, info
    cl_bytes = L.cspn2d_workspace_bytes(B, C, H, W, N, _lib.ALGO_CLUSTER)
    gen_bytes = L.cspn2d_workspace_bytes(B, C, H, W, N, _lib.ALGO_GENERIC)
    assert cl_bytes == L.cspn2d_workspace_bytes(B, C, H, W, N, _lib.ALGO_AUTO) and 0 < cl_bytes < gen_bytes

    def run(algo, ws_bytes, off):
        out, ws = mc.guarded(d.shape), mc.workspace(ws_bytes, off)
        rc = fwd2d_call(gc, dc, sc, out, N, algo, ws.ptr(), ws_bytes)
        torch.cuda.synchronize()
        assert ws.guards_intact() and out.guards_intact()
        return rc, out, L.cspn_last_algo()

    inputs = [gc, dc, sc]
    before = mc.snapshot(inputs)
    # aligned: the cluster kernel in several passes; the generic path for comparison
    rc, cl, algo = run(_lib.ALGO_CLUSTER, cl_bytes, 0)
    assert rc == 0 and algo == _lib.ALGO_CLUSTER and L.cspn_last_launches() > 1
    mc.assert_written(cl, 'cluster')
    rc, gen, _ = run(_lib.ALGO_GENERIC, gen_bytes, 0)
    assert rc == 0
    mc.assert_written(gen, 'generic')
    # AUTO with a generic-sized workspace 4 bytes off: the generic path, its bits
    rc, auto, algo = run(_lib.ALGO_AUTO, gen_bytes, 4)
    assert rc == 0 and _lib.ALGO_NAMES[algo] == 'generic', (rc, last_error())
    mc.assert_written(auto, 'AUTO')
    assert mc.same_bits(auto.t.cpu(), gen.t.cpu())
    # AUTO with the cluster-sized workspace it was queried for: the workspace error that names the generic size
    rc, out, _ = run(_lib.ALGO_AUTO, cl_bytes, 4)
    assert rc == ERR_WORKSPACE and 'CSPN_ALGO_GENERIC' in last_error() and '16-byte aligned' in last_error(), last_error()
    assert out.untouched()
    # CLUSTER and the fused gather: unsupported, with the reason
    rc, out, _ = run(_lib.ALGO_CLUSTER, cl_bytes, 4)
    assert rc == ERR_UNSUPPORTED and 'workspace' in last_error() and '16-byte aligned' in last_error(), last_error()
    assert out.untouched()
    out, ws = mc.guarded(d.shape), mc.workspace(cl_bytes, 4)
    rc = gather_call(gc, dc, sc, out.ptr(), [], N, 0, ws.ptr(), cl_bytes)
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED and 'workspace' in last_error(), last_error()
    assert out.untouched() and ws.untouched()
    assert mc.unchanged(before, inputs)
    if case == 'forced-2-passes':
        assert_values([cl.t.cpu(), auto.t.cpu()], [fwd_ref_2d(g, d, s, N, 3, '8sum')] * 2, case)
        # one pass: the cluster kernel does not use the workspace, so 4 bytes off changes nothing
        monkeypatch.setenv('CSPN_B200_FORCE_PASSES', '1')
        one_bytes = L.cspn2d_workspace_bytes(B, C, H, W, N, _lib.ALGO_AUTO)
        results = []
        for off in (0, 4):
            for algo in (_lib.ALGO_AUTO, _lib.ALGO_CLUSTER):
                rc, out, used = run(algo, one_bytes, off)
                assert rc == 0 and used == _lib.ALGO_CLUSTER and L.cspn_last_launches() == 1, (off, algo, last_error())
                mc.assert_written(out, 'one pass')
                results.append(out.t.cpu())
        assert all(mc.same_bits(r, results[0]) for r in results)
        assert_values(results[:1], [fwd_ref_2d(g, d, s, N, 3, '8sum')], 'one pass')


# ---- the fused gather on one GPU ---------------------------------------------------------------------------------------------
def gather_call(gc, dc, sc, out_ptr, peers, N, norm, ws_ptr, ws_bytes, n_peer=None, mc_ptr=None):
    """cspn2d_fwd_gather_f32; peers: a list of addresses (None entries allowed) or None for a NULL array."""
    B, C, H, W = dc.shape
    arr = None if peers is None else (ctypes.c_void_p * max(len(peers), 1))(*peers)
    return _lib.lib().cspn2d_fwd_gather_f32(
        ptr(gc), ptr(dc), ptr(sc), out_ptr, None if arr is None else ctypes.cast(arr, ctypes.c_void_p),
        len(peers) if n_peer is None else n_peer, mc_ptr, B, C, H, W, gc.shape[1], N, norm, ws_ptr, ws_bytes, stream())


def block_ptr(buf, r, B):
    return buf.t[r * B:(r + 1) * B].data_ptr()


def gather_world(gc, dc, sc, N, norm, n_peer, ref):
    """Emulates n_peer + 1 ranks on one GPU and runs the gather as rank world // 2: out is block r of buffer r, peer j
    block r of buffer j.  Block r of every buffer must hold `ref`'s bits, every other block and every guard the sentinel."""
    B = dc.shape[0]
    world = n_peer + 1
    r = world // 2
    bufs = [mc.guarded((world * B, *dc.shape[1:])) for _ in range(world)]
    ws_bytes = _lib.lib().cspn2d_workspace_bytes(*dc.shape, N, _lib.ALGO_CLUSTER)
    ws = mc.workspace(ws_bytes)
    before = mc.snapshot([gc, dc, sc])
    peers = [block_ptr(bufs[j], r, B) for j in range(world) if j != r]
    _lib.check(gather_call(gc, dc, sc, block_ptr(bufs[r], r, B), peers, N, norm, ws.ptr(), ws_bytes), 'gather')
    torch.cuda.synchronize()
    assert _lib.ALGO_NAMES[_lib.lib().cspn_last_algo()] == 'cluster'
    assert ws.guards_intact() and mc.unchanged(before, [gc, dc, sc])
    for j, buf in enumerate(bufs):
        assert buf.guards_intact(), f'buffer {j}: a store landed outside it'
        for k in range(world):
            blk = buf.t[k * B:(k + 1) * B]
            if k == r:
                assert mc.same_bits(blk.cpu(), ref), f'buffer {j} (rank {r} of {world}): the gathered block differs'
            else:
                assert mc.n_unwritten(blk) == blk.numel(), f'buffer {j}: block {k} of rank {r} of {world} was written'


def cluster_forward(gc, dc, sc, N, norm):
    """cspn2d_fwd_f32(CSPN_ALGO_CLUSTER) into a guarded out: the bits the gather must deliver everywhere."""
    out = mc.guarded(dc.shape)
    ws_bytes = _lib.lib().cspn2d_workspace_bytes(*dc.shape, N, _lib.ALGO_CLUSTER)
    ws = mc.workspace(ws_bytes)
    rc = fwd2d_call(gc, dc, sc, out, N, _lib.ALGO_CLUSTER, ws.ptr(), ws_bytes, norm)
    if rc == ERR_UNSUPPORTED:
        return None
    _lib.check(rc, 'cspn2d_fwd_f32')
    torch.cuda.synchronize()
    mc.assert_written(out, 'cluster forward')
    return out.t.cpu()


@pytest.mark.parametrize('name', sorted(PROBLEMS))
def test_gather_delivers_every_forward_plan_to_seven_peers(name, monkeypatch):
    pb = PROBLEMS[name]
    g, d, s = make_inputs(300 + pb.H, pb.B, pb.C, pb.H, pb.W, pb.gch, pb.sparse, pb.H * pb.W // 20)
    gc, dc, sc = dev(g, d, s)
    ran = 0
    for plan in pb.fwd:
        force(monkeypatch, plan)
        ref = cluster_forward(gc, dc, sc, pb.n, _lib.NORM2D[pb.norm])
        if ref is None:            # the device cannot host this forced plan (tests/test_forced_plans_gpu.py reports it)
            assert not plan_info(plan, pb.H, pb.W, pb.n)['supported']
            continue
        gather_world(gc, dc, sc, pb.n, _lib.NORM2D[pb.norm], 7, ref)
        ran += 1
    assert ran > 0


@pytest.mark.parametrize('n_peer', [0, 1, 3])
def test_gather_with_fewer_peers(n_peer, monkeypatch):
    """Two passes: only the last one's result travels to the peers."""
    pb = PROBLEMS['short_cfg0']
    force(monkeypatch, Plan(0, 3, 2))
    g, d, s = make_inputs(7, pb.B, pb.C, pb.H, pb.W, pb.gch, 'signed', 500)
    gc, dc, sc = dev(g, d, s)
    ref = cluster_forward(gc, dc, sc, pb.n, 1)
    gather_world(gc, dc, sc, pb.n, 1, n_peer, ref)
    if n_peer == 0:     # with no peer the gather is the plain forward, also without forcing a plan
        for k in ('CSPN_B200_FORCE_CFG', 'CSPN_B200_FORCE_CS', 'CSPN_B200_FORCE_PASSES'):
            monkeypatch.delenv(k)
        gather_world(gc, dc, sc, pb.n, 1, 0, cluster_forward(gc, dc, sc, pb.n, 1))


def test_gather_refusals_write_nothing(monkeypatch):
    for k in ('CSPN_B200_FORCE_CFG', 'CSPN_B200_FORCE_CS', 'CSPN_B200_FORCE_PASSES', 'CSPN_B200_CHAIN'):
        monkeypatch.delenv(k, raising=False)

    def attempt(shape, N, peers, n_peer=None, mc_off=None, blur_off=0):
        B, C, H, W = shape
        g, d, s = make_inputs(11, B, C, H, W, 8, 'bernoulli', 50)
        gc, sc = dev(g, s)
        blur = mc.guarded(shape, blur_off)
        blur.t.copy_(d)
        out = mc.guarded(shape)
        bufs = [mc.guarded(shape) for _ in range(3)]
        addr = {'ok': bufs[0].ptr(), 'null': None, 'off4': bufs[1].ptr() + 4}
        plist = None if peers is None else [addr[p] for p in peers]
        ws_bytes = _lib.lib().cspn2d_workspace_bytes(B, C, H, W, max(N, 1), _lib.ALGO_CLUSTER)
        ws = mc.workspace(ws_bytes)
        rc = gather_call(gc, blur.t, sc, out.ptr(), plist, N, 0, ws.ptr(), ws_bytes, n_peer,
                         None if mc_off is None else bufs[2].ptr() + mc_off)
        torch.cuda.synchronize()
        assert out.untouched() and all(b.untouched() for b in bufs) and ws.untouched()
        return rc, last_error()

    shape = (1, 2, 40, 132)
    cases = [
        (dict(peers=['ok'], n_peer=8), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok'], n_peer=-1), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=None, n_peer=2), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok', 'null']), ERR_INVALID, 'peer_out[1] is null or not 16-byte aligned'),
        (dict(peers=['off4', 'ok']), ERR_INVALID, 'peer_out[0] is null or not 16-byte aligned'),
        (dict(peers=['ok'], mc_off=4), ERR_INVALID, 'multicast_out is not 16-byte aligned'),
        (dict(peers=['ok'], N=0), ERR_UNSUPPORTED, 'prop_time >= 1'),
        (dict(peers=['ok'], shape=(1, 2, 40, 130)), ERR_UNSUPPORTED, 'cluster kernel\'s epilogue'),
        (dict(peers=['ok'], blur_off=4), ERR_UNSUPPORTED, '16-byte aligned'),
    ]
    for kw, want, msg in cases:
        args = dict(shape=shape, N=6)
        args.update(kw)
        rc, err = attempt(**args)
        assert rc == want and msg in err, (kw, rc, err)
