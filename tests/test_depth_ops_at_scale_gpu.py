"""GPU tests of the dilated (DESIGN.md section 4.22), aggregating (section 4.20), non-local (section 4.21) and dynamic
(section 4.23) 2D propagations across CTA tiles and at 8x1x352x1216, the shape the README times them at.  The small
images of test_dilated_gpu.py, test_aggregate_gpu.py, test_nonlocal_gpu.py and test_dynamic_gpu.py fit in one or two
tiles; here the 4-pixel and 1-pixel paths read their halos from neighbouring tiles (shapes in
tests/test_depth_ops_at_scale_cpu.py, which also checks that they cross what they are meant to cross and that the exact
cases are exact), the step-weight gradient runs in two launch groups, the non-local backward index runs past 2^27
samples (a second grid-stride pass of its entries kernel, a 22-bit sort key) and with every sample in one bucket, and
the dynamic finalize's 64 attention slices take a second and a third pass over the steps (N up to 129).

Oracles: bit equality with an order-free reference where one exists (dyadic and integer-offset cases against fp64,
separate propagations for the aggregate's forward, the other path or the batch split), else the op's own tolerance
against fp64: `within` for the dilated and dynamic ops, ar.within for the aggregate's gradients, and for the non-local
op a normwise distance at most 4x that of its eager fp32 restatement.  The dynamic op also has an order-exact oracle,
tests/dynamic_reference.py's kernel_order: on random inputs every output and gradient has its bits.  At the timing
shape the library runs B = 8 and the fp64 reference the first two images (kernel_order all eight).

First runs, on an NVIDIA H100 80GB HBM3 at a 700 W power limit: every bit-for-bit check held, the largest tolerance
ratios are in each test's docstring, and the file's 201 tests of the first three ops took 62-66 s; the dynamic op's 81
took 69 s, and the whole file's 282 took 107 s.
"""
import ctypes

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib
from cspn_b200.cspn import _propagate2d_keep, norm_code_2d_k
import aggregate_reference as ar
import dilated_reference as dr
import dynamic_reference as yr
import memory_contract as mc
import nonlocal_reference as nr
import test_depth_ops_at_scale_cpu as pre

pytestmark = pytest.mark.gpu
DIL_NAMES = ('out', 'kernel', 'blur', 'sparse', 'conf')
AGG_NAMES = ('out', 'grad_guidance', 'grad_blur', 'grad_sparse', 'grad_step_weight')
NL_NAMES = ('out', 'feat', 'offset', 'affinity', 'sparse')
DYN_NAMES = ('out', 'affinity', 'attention', 'blur', 'sparse', 'conf')


def bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def randn(*shape, seed=0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).cuda()


def cuda(ts):
    return [None if t is None else t.cuda() for t in ts]


def misaligned(t):
    """t's values 4 bytes into a buffer: contiguous, so taken as is, but not 16-byte aligned, so on the 1-pixel path."""
    if t is None:
        return None
    buf = torch.empty(t.numel() + 1, device='cuda')
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def place(ts, aligned):
    return list(ts) if aligned else [misaligned(t) for t in ts]


# ---- dilated ------------------------------------------------------------------------------------------------------------------
def dil_op(k, b, s, m, K, dil, N):
    return cspn_b200.propagate2d_dilated(k, b, s, m, K, dil, N)


def dil_run(ins, K, dil, N, go):
    return dr.grads(dil_op, *ins, K, dil, N, go)


def dil_ref(ins, K, dil, N, go):
    return dr.grads(dr.composition, *cuda(ins), K, dil, N, go.cuda(), dtype=torch.float64)


def dil_within(got, ref, fwd_tol=1e-5, grad_tol=2e-3, names=DIL_NAMES):
    """test_dilated_gpu.py's `within` (and test_dynamic_gpu.py's, with names=DYN_NAMES), element by element (a NaN fails
    it), returning the largest |got - ref| / bound per name for the record."""
    out = {}
    for name, g, r in zip(names, got, ref):
        assert (g is None) == (r is None), name
        if r is not None:
            tol = fwd_tol if name == 'out' else grad_tol
            g, r = g.double(), r.to(g.device)
            err, bound = (g - r).abs(), tol * (r.abs() + r.abs().mean())
            ok = err <= bound
            out[name] = float(torch.where(ok, err / bound.clamp_min(1e-300), torch.full_like(err, float('inf'))).max())
            assert bool(ok.all()), (name, out[name])
    return out


@pytest.mark.parametrize('aligned', [True, False])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('dil', [1, 2, 3, 4])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('shape', pre.DIL_SEAMS)
def test_dilated_dyadic_seams_equal_fp64_bit_for_bit(shape, samples, dil, K, aligned):
    """Three or more tiles in x and y with partial last tiles; aligned: the 4-pixel step, else the 1-pixel one."""
    ins, go = pre.dilated_dyadic(*shape, K, samples, pre.dil_seed(shape, K, dil, samples))
    N = pre.DIL_N[K]
    ref = dil_ref(ins, K, dil, N, go)
    got = dil_run(place(cuda(ins), aligned), K, dil, N, go.cuda())
    for name, g, r in zip(DIL_NAMES, got, ref):
        assert (g is None) == (r is None), name
        assert r is None or torch.equal(g, r.float()), name


def test_dilated_vector_and_scalar_paths_give_the_same_bits_across_tiles():
    """2x1x45x1216: ten 4-pixel tiles (the last half full) against 38 one-pixel tiles, random inputs."""
    ins = dr.make_inputs(2, 1, 45, 1216, 5, 'soft', seed=12, device='cuda')
    go = randn(2, 1, 45, 1216)
    ref = dil_run(ins, 5, 2, 6, go)
    got = dil_run(place(ins, False), 5, 2, 6, go)
    for name, x, y in zip(DIL_NAMES, got, ref):
        assert bits(x, y), name


DEGENERATE = [(H, W) for H in (1, 2) for W in (1, 3, 4, 8)] + [(1, 260), (45, 3), (9, 11)]


@pytest.mark.parametrize('K,dil', [(7, 4), (3, 1)])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('H,W', DEGENERATE)
def test_dilated_degenerate_shapes_within_tolerance_of_fp64(H, W, samples, K, dil):
    """1 x W, H x 1, one 4-pixel thread (W = 4) and images smaller than the d*R = 12 halo of K = 7, d = 4.  First H100
    run: largest ratio to the bound 0.019."""
    ins = dr.make_inputs(2, 2, H, W, K, samples, seed=H * 31 + W, device='cuda')
    go = randn(2, 2, H, W)
    ratios = dil_within(dil_run(ins, K, dil, 5, go), dil_ref(ins, K, dil, 5, go))
    print(f'dilated {H}x{W} K={K} d={dil} {samples}:', ratios)


@pytest.mark.parametrize('K', [3, 5, 7])
def test_dilated_timing_shape_within_tolerance_of_fp64(K):
    """8x1x352x1216, d = 2, N = 6, soft samples: the library at B = 8, the fp64 composition for images 0 and 1.  First
    H100 run: largest ratio to the bound 0.033 (out, K = 7), 0.0012 for a gradient (kernel, K = 5)."""
    ins = dr.make_inputs(8, 1, 352, 1216, K, 'soft', seed=K, device='cuda')
    go = randn(8, 1, 352, 1216)
    got = [None if t is None else t[:2] for t in dil_run(ins, K, 2, 6, go)]
    ratios = dil_within(got, dil_ref([t[:2] for t in ins], K, 2, 6, go[:2]))
    print(f'dilated timing shape K={K}:', ratios)


# ---- aggregate ----------------------------------------------------------------------------------------------------------------
def agg_inputs(seed, B, C, H, W, K, T):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, K * K - 1, H, W, generator=gen)
    d = torch.rand(B, C, H, W, generator=gen)
    s = (torch.rand(B, 1, H, W, generator=gen) < 0.3).float() * torch.rand(B, 1, H, W, generator=gen)
    s[:, :, :2] *= -1                                   # some negative samples: sign() and 1[> 0] differ there
    sw = torch.randn(B, T, H, W, generator=gen)
    go = torch.randn(B, C, H, W, generator=gen)
    return [t.cuda() for t in (g, d, s, sw, go)]


def agg_iterate(g, d, s, K, n, keep):
    """d_n from the library's own K x K propagation (K = 3 on its generic route)."""
    if keep:
        return _propagate2d_keep(g, d, s, K, n, norm_code_2d_k(K), _lib.ALGO_GENERIC)
    if K == 3:
        return cspn_b200.propagate2d(g, d, s, n, '8sum', _lib.ALGO_GENERIC)
    return cspn_b200.propagate2d_k(g, d, s, K, n)


def agg_run(g, d, s, sw, go, steps, K, keep):
    """(out, grad_guidance, grad_blur, grad_sparse, grad_step_weight); the leaves keep the inputs' addresses."""
    leaves = [t.detach().requires_grad_(True) for t in (g, d, s, sw)]
    out = cspn_b200.propagate2d_aggregate(leaves[0], leaves[1], leaves[3], leaves[2], K, None, keep, steps)
    live = [t for i, t in enumerate(leaves) if i != 2 or keep]
    gs = iter(torch.autograd.grad(out, live, go))
    return [out.detach()] + [next(gs) if i != 2 or keep else None for i in range(4)]


def agg_autograd64(g, d, s, sw, go, steps, K, keep):
    leaves = [t.detach().double().requires_grad_(True) for t in (g, d, s, sw)]
    out = ar.composition(*leaves, steps, K, None, keep)
    out.backward(go.double())
    return [out.detach()] + [t.grad for t in leaves]


def agg_check(got, ref, keep, what):
    ratios = {}
    for a, b, name in zip(got[1:], ref[1:], AGG_NAMES[1:]):
        if name == 'grad_sparse' and not keep:
            assert a is None
            continue
        ok, err, scale = ar.within(a, b)
        x, r = a.double(), b.to(a.device)
        ratios[name] = float(((x - r).abs() / (2e-3 * (r.abs() + r.abs().mean()))).max())    # ar.within's bound
        assert ok, (what, name, err, scale)
    return ratios


@pytest.mark.parametrize('aligned', [True, False])
@pytest.mark.parametrize('steps', pre.AGG_STEPS, ids=['T3', 'T70'])
@pytest.mark.parametrize('keep', [False, True])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('shape', pre.AGG_SEAMS)
def test_aggregate_seams_and_launch_groups(shape, K, keep, steps, aligned):
    """The forward has the bits of sum_j w_j propagate2d_k(..., steps[j]) (stepk_agg_vec_kernel when aligned, else
    stepk_agg_scalar_kernel, across every tile); the gradients are within the K x K tolerance of fp64 autograd, with
    the step-weight gradient in two launch groups at T = 70.  First H100 run: largest gradient ratio to the bound 0.20."""
    B, C, H, W = shape
    g, d, s, sw, go = agg_inputs(K * 100 + len(steps) + W, B, C, H, W, K, len(steps))
    g, d, s, sw = place((g, d, s, sw), aligned)
    got = agg_run(g, d, s, sw, go, steps, K, keep)
    assert bits(got[0], ar.aggregate([agg_iterate(g, d, s, K, n, keep) for n in steps], sw))
    ratios = agg_check(got, agg_autograd64(g, d, s, sw, go, steps, K, keep), keep, 'seams')
    print(f'aggregate {shape} K={K} keep={keep} T={len(steps)} aligned={aligned}: {max(ratios.values()):.3g}')


def test_aggregate_timing_shape():
    """8x1x352x1216, keep mode, K = 5, N = T = 24: the forward bit for bit against separate propagations at B = 8, the
    gradients against fp64 autograd for images 0 and 1 of the same call.  First H100 run: largest ratio to the bound
    0.0072 (grad_guidance)."""
    K, steps = 5, tuple(range(1, 25))
    g, d, s, sw, go = agg_inputs(24, 8, 1, 352, 1216, K, 24)
    got = agg_run(g, d, s, sw, go, steps, K, True)
    assert bits(got[0], ar.aggregate([agg_iterate(g, d, s, K, n, True) for n in steps], sw))
    ratios = agg_check([t[:2] for t in got], agg_autograd64(*[t[:2] for t in (g, d, s, sw, go)], steps, K, True), True, 'timing')
    print('aggregate timing shape:', ratios)


# ---- non-local ----------------------------------------------------------------------------------------------------------------
def nl_run(f, o, a, s, K, N, go):
    return nr.grads(lambda f, o, a, s, K, N: cspn_b200.propagate2d_nonlocal(f, o, a, s, K, N), f, o, a, s, K, N, go)


def nl_normwise(got, f, o, a, s, K, N, go, floor=0.0):
    """ours / eager fp32, each the normwise distance to the fp64 restatement, per name; ours may be at most 4x eager
    fp32's distance or, for the gradients, `floor`, whichever is larger."""
    e32 = nr.grads(nr.propagate, f, o, a, s, K, N, go)
    ref = nr.grads(nr.propagate, f, o, a, s, K, N, go, dtype=torch.float64)
    out = {}
    for name, g, e, r in zip(NL_NAMES, got, e32, ref):
        if r is None:
            assert g is None
            continue
        dk, de = nr.normwise(g, r), nr.normwise(e, r)
        bound = 4 * de if name == 'out' else max(4 * de, floor)
        assert dk <= bound + 1e-7, (name, dk, de, bound)
        out[name] = dk / max(de, 1e-30)
    return out


def test_nonlocal_past_2_27_samples_equals_fp64_per_image():
    """8x1x352x1216, K = 7, N = 2, integer offsets, with samples: n = 164,364,288 samples, so the entries kernel makes a
    second grid-stride pass.  One library call at B = 8; each image against the fp64 restatement of that image alone."""
    K, N = pre.NL_LARGE_K, pre.NL_LARGE_N
    _, C, H, W = pre.TIMING
    imgs = [pre.nonlocal_exact(1, C, H, W, K, pre.nl_seed(b)) for b in range(pre.TIMING[0])]
    f, o, a, s, go = [torch.cat(ts).cuda() for ts in zip(*imgs)]
    got = nl_run(f, o, a, s, K, N, go)
    del f, o, a, s, go
    for b, img in enumerate(imgs):
        fb, ob, ab, sb, gb = cuda(img)
        ref = nr.grads(nr.propagate, fb, ob, ab, sb, K, N, gb, dtype=torch.float64)
        r32 = nr.grads(nr.propagate, fb, ob, ab, sb, K, N, gb)
        for name, g, x, r in zip(NL_NAMES, got, r32, ref):
            assert torch.equal(x, r.float()), (b, name, 'premise')    # exact, so the reference's order does not matter
            assert torch.equal(g[b:b + 1], r.float()), (b, name)


def test_nonlocal_batch_split_at_the_timing_shape():
    """Random inputs, offsets at scale 2.5, K = 7, N = 2: the B = 8 call (past 2^27 samples) has the bits of eight B = 1
    calls (below it)."""
    f, o, a, s = nr.make_inputs(8, 1, 352, 1216, 7, scale=2.5, seed=8, sparse=True, device='cuda')
    go = randn(*f.shape)
    ref = nl_run(f, o, a, s, 7, 2, go)
    for b in range(8):
        one = nl_run(f[b:b + 1], o[b:b + 1], a[b:b + 1], s[b:b + 1], 7, 2, go[b:b + 1])
        for name, x, y in zip(NL_NAMES, one, ref):
            assert bits(x, y[b:b + 1]), (b, name)


def test_nonlocal_timing_shape_k3_n18():
    """8x1x352x1216, K = 3, N = 18, offsets at scale 2.5, with samples: the library at B = 8, the fp64 and eager fp32
    restatements for images 0 and 1.  First H100 run: ours / eager fp32 at most 1.0006 (grad_feat), the bound being 4."""
    f, o, a, s = nr.make_inputs(8, 1, 352, 1216, 3, scale=2.5, seed=18, sparse=True, device='cuda')
    go = randn(*f.shape)
    got = [t[:2] for t in nl_run(f, o, a, s, 3, 18, go)]
    ratios = nl_normwise(got, *[t[:2] for t in (f, o, a, s)], 3, 18, go[:2])
    print('non-local timing shape K=3 N=18:', ratios)


@pytest.mark.parametrize('outside_half', [False, True])
def test_nonlocal_hot_bucket(outside_half):
    """1x2x64x96, K = 3, N = 4: every sample at (10.25, 20.5), so one bucket holds all 49,152 entries and four pixels
    gather them all; or half of them there and half outside the window, under the sentinel key.  Two calls give the
    same bits.

    The output, which does not use the bucket index, keeps the bound of 4x eager fp32's normwise distance.  For the
    gradients it is that or u * sqrt(n), u = 2^-24 and n the entries in the bucket, whichever is larger.  The four corner
    pixels dominate every gradient's norm here, and each is one long sum: the adjoint adds a pixel's
    entries one after another in the fixed order that makes it deterministic (DESIGN.md section 4.21), while the eager
    restatement adds them in eight per-tap scatters of 6,144 and then sums the eight.  A sequential sum of n terms of
    random sign is off by about u * sqrt(n) relative, so at n = 49,152 the kernel's error is expected to be several
    times eager's.  On the first H100 runs grad_feat was 10-12.6x eager fp32's distance (3.7e-6 against 2.96e-7 in
    one; eager's own distance varies from run to run, its scatters being atomic), grad_offset up to 6.6x and grad_sparse
    up to 6.5x; the largest ratio to u * sqrt(n) was 0.28, and the output stayed at eager's distance (ratio 1.0).  A
    lost or repeated entry moves a corner by one term, about 1e-2 of its value, far past this bound."""
    B, C, H, W = pre.NL_HOT
    f, _, a, s = nr.make_inputs(B, C, H, W, 3, seed=64 + outside_half, sparse=True, device='cuda')
    o = pre.hot_offsets(B, H, W, 3, outside_half).cuda()
    go = torch.randn(f.shape, generator=torch.Generator().manual_seed(2)).cuda()
    got = nl_run(f, o, a, s, 3, 4, go)
    n = B * H * W * 8 // (2 if outside_half else 1)
    ratios = nl_normwise(got, f, o, a, s, 3, 4, go, floor=2.0 ** -24 * n ** 0.5)
    print(f'non-local hot bucket outside_half={outside_half}:', ratios)
    again = nl_run(f, o, a, s, 3, 4, go)
    for name, x, y in zip(NL_NAMES, again, got):
        assert bits(x, y), name


# ---- memory contract at the seam shapes -------------------------------------------------------------------------------------
def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def contract(forward, backward, n_out):
    """Runs forward(out, ws) and backward(outs, ws) on sentinel- and zero-filled workspaces: every output element
    written, nothing stored outside, the same bits from both fills.  Returns (out, grads) of the sentinel run."""
    fw, bw = [], []
    for fill in ('sentinel', 'zero'):
        out, ws = forward(fill)
        torch.cuda.synchronize()
        mc.assert_written(out, 'out')
        assert ws.guards_intact()
        fw.append(out.t.clone())
        outs, ws = backward(fill)
        torch.cuda.synchronize()
        assert len(outs) == n_out
        for i, x in enumerate(outs):
            mc.assert_written(x, f'grad {i}')
        assert ws.guards_intact()
        bw.append([x.t.clone() for x in outs])
    assert mc.same_bits(*fw)
    assert all(mc.same_bits(x, y) for x, y in zip(*bw))
    return fw[0], bw[0]


def test_memory_contract_dilated_at_a_seam_shape():
    B, C, H, W, K, dil, N = 2, 2, 45, 260, 5, 3, 4
    L = _lib.lib()
    k, b, s, m = dr.make_inputs(B, C, H, W, K, 'soft', seed=45, device='cuda')
    go = randn(B, C, H, W)
    before = mc.snapshot([k, b, s, m, go])

    def fwd(fill):
        out = mc.guarded(b.shape)
        ws = mc.workspace(L.cspn2d_dil_workspace_bytes(B, C, H, W, K, dil, N), 0, fill)
        rc = L.cspn2d_dil_fwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), out.t.data_ptr(), B, C, H, W, K, dil, N,
                                  ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return out, ws

    def bwd(fill):
        outs = [mc.guarded(t.shape) for t in (k, b, s, m)]
        ws = mc.workspace(L.cspn2d_dil_bwd_workspace_bytes(B, C, H, W, K, dil, N), 0, fill)
        rc = L.cspn2d_dil_bwd_f32(k.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), go.data_ptr(),
                                  *[x.t.data_ptr() for x in outs], B, C, H, W, K, dil, N, ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return outs, ws

    out, grads = contract(fwd, bwd, 4)
    assert mc.unchanged(before, [k, b, s, m, go])
    want = dil_run((k, b, s, m), K, dil, N, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


def test_memory_contract_aggregate_at_a_seam_shape():
    B, C, H, W, K, keep, steps = 2, 2, 45, 260, 5, True, (2, 3, 5)
    L = _lib.lib()
    g, d, s, sw, go = agg_inputs(260, B, C, H, W, K, len(steps))
    before = mc.snapshot([g, d, s, sw, go])
    st = (ctypes.c_int * len(steps))(*steps)

    def fwd(fill):
        out = mc.guarded(d.shape)
        ws = mc.workspace(L.cspn2d_agg_workspace_bytes(B, C, H, W, K, st, len(steps), int(keep)), 0, fill)
        rc = L.cspn2d_agg_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(sw), out.ptr(), B, C, H, W, g.shape[1], K, st, len(steps), 0,
                                  int(keep), ws.ptr(), ws.nbytes, _stream())
        _lib.check(rc, 'cspn2d_agg_fwd_f32')
        return out, ws

    def bwd(fill):
        outs = [mc.guarded(t.shape) for t in (g, d, s, sw)]
        ws = mc.workspace(L.cspn2d_agg_bwd_workspace_bytes(B, C, H, W, K, st, len(steps), int(keep)), 0, fill)
        rc = L.cspn2d_agg_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(sw), _ptr(go), *[o.ptr() for o in outs], B, C, H, W, g.shape[1],
                                  K, st, len(steps), 0, int(keep), ws.ptr(), ws.nbytes, _stream())
        _lib.check(rc, 'cspn2d_agg_bwd_f32')
        return outs, ws

    out, grads = contract(fwd, bwd, 4)
    assert mc.unchanged(before, [g, d, s, sw, go])
    want = agg_run(g, d, s, sw, go, steps, K, keep)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


def test_memory_contract_nonlocal_at_a_seam_shape():
    B, C, H, W, K, N = 2, 1, 64, 96, 3, 4
    L = _lib.lib()
    f, o, a, s = nr.make_inputs(B, C, H, W, K, scale=6.0, seed=96, sparse=True, device='cuda')
    go = randn(*f.shape)
    before = mc.snapshot([f, o, a, s, go])

    def fwd(fill):
        out = mc.guarded(f.shape)
        ws = mc.workspace(L.cspn2d_nl_workspace_bytes(B, C, H, W, K, N), 0, fill)
        rc = L.cspn2d_nl_fwd_f32(f.data_ptr(), o.data_ptr(), a.data_ptr(), s.data_ptr(), out.t.data_ptr(), B, C, H, W, K, N,
                                 ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return out, ws

    def bwd(fill):
        outs = [mc.guarded(t.shape) for t in (f, o, a, s)]
        ws = mc.workspace(L.cspn2d_nl_bwd_workspace_bytes(B, C, H, W, K, N), 0, fill)
        rc = L.cspn2d_nl_bwd_f32(f.data_ptr(), o.data_ptr(), a.data_ptr(), s.data_ptr(), go.data_ptr(), *[x.t.data_ptr() for x in outs],
                                 B, C, H, W, K, N, ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return outs, ws

    out, grads = contract(fwd, bwd, 4)
    assert mc.unchanged(before, [f, o, a, s, go])
    want = nl_run(f, o, a, s, K, N, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


# ---- dynamic ------------------------------------------------------------------------------------------------------------------
def dyn_op(a, t, b, s, m, K):
    return cspn_b200.propagate2d_dynamic(a, t, b, s, m, K)


def dyn_run(ins, K, go):
    return yr.grads(dyn_op, *ins, K, go)


def dyn_ref(ins, K, go):
    return yr.grads(yr.composition, *cuda(ins), K, go.cuda(), dtype=torch.float64)


def dyn_bits(got, want, what):
    for name, g, r in zip(DYN_NAMES, got, want):
        assert bits(g, r), (what, name)


def dyn_within(got, ref):
    return dil_within(got, ref, names=DYN_NAMES)


DYN_SEAM_N = 5


@pytest.mark.parametrize('aligned', [True, False])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('shape', pre.DIL_SEAMS)
def test_dynamic_seams_bit_for_bit(shape, samples, K, aligned):
    """Three or more tiles in x and y with partial last tiles, and a partial last finalize block; aligned: the 4-pixel
    step, else the 1-pixel one.  Dyadic inputs give the fp64 composition's bits; random ones, N = 5, the bits of the
    kernels' stated order of operations (yr.kernel_order), which no order-free reference can check."""
    ins, go = yr.dyadic_inputs(*shape, K, pre.DIL_N[K], samples, pre.dyn_seed(shape, K, samples))
    ref = dyn_ref(ins, K, go)
    got = dyn_run(place(cuda(ins), aligned), K, go.cuda())
    for name, g, r in zip(DYN_NAMES, got, ref):
        assert (g is None) == (r is None), name
        assert r is None or torch.equal(g, r.float()), ('dyadic', name)
    ins = yr.make_inputs(*shape, K, DYN_SEAM_N, samples, seed=pre.dyn_seed(shape, K, samples), device='cuda')
    go = randn(*shape, seed=K)
    dyn_bits(dyn_run(place(ins, aligned), K, go), yr.kernel_order(*ins, K, go), 'random')


@pytest.mark.parametrize('K', [7, 3])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('H,W', DEGENERATE)
def test_dynamic_degenerate_shapes(H, W, samples, K):
    """1 x W, H x 1, one 4-pixel thread (W = 4) and images smaller than the R = 3 halo of K = 7, N = 5: the bits of
    yr.kernel_order, and within `within` of fp64.  First H100 run: largest ratio to the bound 0.031 (out, 9x11, K = 7),
    0.0015 for a gradient (attention, 9x11, K = 3)."""
    ins = yr.make_inputs(2, 2, H, W, K, 5, samples, seed=H * 31 + W, device='cuda')
    go = randn(2, 2, H, W)
    got = dyn_run(ins, K, go)
    dyn_bits(got, yr.kernel_order(*ins, K, go), 'kernel order')
    ratios = dyn_within(got, dyn_ref(ins, K, go))
    print(f'dynamic {H}x{W} K={K} {samples}:', ratios)


def wrap_inputs(N, seed=0):
    ins = yr.make_inputs(*pre.DYN_WRAP_SHAPE, pre.DYN_WRAP_K, N, 'soft', seed=N + seed, device='cuda')
    return ins, randn(*pre.DYN_WRAP_SHAPE, seed=N + seed)


@pytest.mark.parametrize('N', pre.DYN_WRAP_N)
def test_dynamic_attention_slices_wrap(N):
    """1x2x17x132, K = 5: the finalize's 64 attention slices take a second step from N = 65 on, a third at N = 129.
    Every gradient has the bits of yr.kernel_order and is within `within` of fp64.  First H100 run: largest ratio to
    the bound 0.052 (out, N = 70), 0.028 for a gradient (attention, N = 63); at N = 129 0.036 and 0.014, so the bound
    holds past two wraps."""
    ins, go = wrap_inputs(N)
    got = dyn_run(ins, pre.DYN_WRAP_K, go)
    dyn_bits(got, yr.kernel_order(*ins, pre.DYN_WRAP_K, go), N)
    ratios = dyn_within(got, dyn_ref(ins, pre.DYN_WRAP_K, go))
    print(f'dynamic slice wrap N={N}:', ratios)


def test_dynamic_requested_gradients_past_the_attention_slices():
    """N = 70: each requested subset gives the full call's bits.  Without the affinity gradient there are no affinity
    slices, so the attention slices start at grid z = 0 (attention alone, and with the confidence)."""
    K = pre.DYN_WRAP_K
    ins, go = wrap_inputs(70, seed=1)
    full = dyn_run(ins, K, go)
    for need in [(0,), (1,), (2,), (3,), (4,), (0, 1), (1, 4), (2, 3)]:
        leaves = [t.clone().requires_grad_(j in need) for j, t in enumerate(ins)]
        gs = torch.autograd.grad(dyn_op(*leaves, K), [leaves[j] for j in need], go)
        for j, g in zip(need, gs):
            assert bits(g, full[1 + j]), (need, DYN_NAMES[1 + j])


@pytest.mark.parametrize('offset', [0, 4])
def test_memory_contract_dynamic_past_the_attention_slices(offset):
    """N = 70 at 1x2x17x132, outputs and workspaces `offset` bytes into their allocations (4: the 1-pixel path): every
    output word written, among them the attention gradient of steps 64-69 that the slices' second pass forms."""
    B, C, H, W = pre.DYN_WRAP_SHAPE
    K, N, NR = pre.DYN_WRAP_K, 70, (pre.DYN_WRAP_K + 1) // 2
    L = _lib.lib()
    (a, t, b, s, m), go = wrap_inputs(N, seed=offset)
    before = mc.snapshot([a, t, b, s, m, go])

    def fwd(fill):
        out = mc.guarded(b.shape, offset)
        ws = mc.workspace(L.cspn2d_dyn_workspace_bytes(B, C, H, W, K, N), offset, fill)
        rc = L.cspn2d_dyn_fwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), out.ptr(), B, C, H, W, K, N,
                                  ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return out, ws

    def bwd(fill):
        outs = [mc.guarded(x.shape, offset) for x in (a, t, b, s, m)]
        ws = mc.workspace(L.cspn2d_dyn_bwd_workspace_bytes(B, C, H, W, K, N), offset, fill)
        rc = L.cspn2d_dyn_bwd_f32(a.data_ptr(), t.data_ptr(), b.data_ptr(), s.data_ptr(), m.data_ptr(), go.data_ptr(),
                                  *[x.ptr() for x in outs], B, C, H, W, K, N, ws.ptr(), ws.nbytes, _stream())
        assert rc == 0, L.cspn_last_error()
        return outs, ws

    out, grads = contract(fwd, bwd, 5)
    assert mc.n_unwritten(grads[1][:, 64 * NR:]) == 0
    assert mc.unchanged(before, [a, t, b, s, m, go])
    want = dyn_run((a, t, b, s, m), K, go)
    assert bits(out, want[0]) and all(bits(x, y) for x, y in zip(grads, want[1:]))


@pytest.mark.parametrize('K,N', pre.DYN_TIMING)
def test_dynamic_timing_shape(K, N):
    """8x1x352x1216, soft samples: every image bit for bit to yr.kernel_order, and images 0 and 1 within `within` of
    the fp64 composition.  First H100 run: largest ratio to the bound 0.074 (out, K = 7, N = 6), 0.020 for a gradient
    (attention, K = 5, N = 24)."""
    ins = yr.make_inputs(*pre.TIMING, K, N, 'soft', seed=K * 100 + N, device='cuda')
    go = randn(*pre.TIMING, seed=N)
    got = dyn_run(ins, K, go)
    dyn_bits(got, yr.kernel_order(*ins, K, go), 'kernel order')
    ratios = dyn_within([t[:2] for t in got], dyn_ref([t[:2] for t in ins], K, go[:2]))
    print(f'dynamic timing shape K={K} N={N}:', ratios)


def test_dynamic_batch_split_at_the_timing_shape():
    """K = 7, N = 6, soft samples: the B = 8 call has the bits of eight B = 1 calls."""
    ins = yr.make_inputs(*pre.TIMING, 7, 6, 'soft', seed=8, device='cuda')
    go = randn(*pre.TIMING, seed=8)
    ref = dyn_run(ins, 7, go)
    for b in range(8):
        one = dyn_run([t[b:b + 1] for t in ins], 7, go[b:b + 1])
        for name, x, y in zip(DYN_NAMES, one, ref):
            assert bits(x, y[b:b + 1]), (b, name)
