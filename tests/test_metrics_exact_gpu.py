"""The depth-metrics and masked-L1 kernels (cspn_b200/csrc/metrics.cu behind cspn_b200/metrics.py) against the restatement
of tests/metrics_reference.py: the six delta counts and n_valid exactly, the four means within one fp32 ulp of their fp64
values (the double atomics make the last bits of the double sums depend on the order), the gradient bit for bit.

  a. sizes around a warp, a block and the grid cap of 132 * 8 * 256 threads, several trips of the grid-stride loops, the
     benchmark's 32 x 1 x 352 x 1216 and one count above 2^24;
  b. ratios on, one ulp under and one ulp over every threshold, from exact and from rounded quotients;
  c. special values, one at a time and together, also against what the reference's own functions returned
     (tests/golden/metrics/edges/, tests/test_metrics_cpu.py);
  d. nothing valid;   e. the backward's calling forms;   f. side stream, CUDA graph, repeated calls, the C ABI's workspace;
  g. the Python interface;   h. heads -> propagation -> loss -> backward against fp64 autograd.
"""
import glob
import os

import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, metrics

import backward_exact as be
import metrics_reference as mr
import unpool_conv_reference as ur

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
EDGE_DIR = os.path.join(HERE, 'golden', 'metrics', 'edges')
EDGES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(EDGE_DIR, '*.npz')))
CAP = 132 * 8 * 256          # threads of the largest grid both kernels launch: beyond it a thread takes a second element


# ---- inputs (built on the CPU: the restatement and the GPU see the same bits) ------------------------------------------
def spread_inputs(n, seed, p_valid=0.3, n_valid=None):
    """1-D gt / pred with distinct values: gt in [1, 10), pred / gt log-uniform over [0.45, 2.2] so that every threshold
    splits the elements, a fraction p_valid of them valid (or exactly n_valid).  The elements next to a multiple of CAP and
    the last two are valid, so an index visited twice or not at all there changes n_valid."""
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand(n, generator=gen) * 9 + 1
    pred = gt * torch.exp((torch.rand(n, generator=gen) - 0.5) * 1.6)
    if n_valid is None:
        keep = torch.rand(n, generator=gen) < p_valid
        at = torch.arange(n) % CAP
        keep |= (at < 2) | (at >= CAP - 2)
        keep[-2:] = True
    else:
        keep = torch.ones(n, dtype=torch.bool)
        keep[torch.arange(n - n_valid) * (n // (n - n_valid)) + 5] = False
        assert int(keep.sum()) == n_valid
    return gt * keep, pred


def dyadic_inputs(n, seed):
    """Integer predictions and power-of-two or missing ground truth: every term is a short dyadic, the double sums are exact
    in any order, and two correct runs give the same twelve floats."""
    gen = torch.Generator().manual_seed(seed)
    pred = torch.randint(1, 9, (n,), generator=gen).float()
    gt = torch.tensor([0.0, 1.0, 2.0, 4.0, 8.0])[torch.randint(0, 5, (n,), generator=gen)]
    return gt, pred


def exact_tie_inputs():
    """gt a power of two and pred = gt * r with r one ulp under, on and one ulp over each threshold: pred / gt == r exactly.
    -> gt, pred, r (float32 arrays)."""
    gts, rs = [], []
    for t in mr.THRESHOLDS:
        for g in (0.25, 1.0, 2.0, 8.0, 64.0):
            for r in (np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(4))):
                gts.append(g)
                rs.append(r)
    gt, r = np.float32(gts), np.float32(rs)
    return gt, gt * r, r


def rounded_tie_inputs():
    """Quotients that are rounded: for gt a power of two or not, every pred within 8 ulps of gt / t and of gt * t."""
    gts, preds = [], []
    for t in mr.THRESHOLDS:
        for g in np.float32([1.0, 2.0, 3.0, 5.7, 0.37, 9.99]):
            for centre in (g / t, g * t):
                p = np.float32(centre)
                for _ in range(8):
                    p = np.nextafter(p, np.float32(0))
                for _ in range(17):
                    gts.append(g)
                    preds.append(p)
                    p = np.nextafter(p, np.float32(np.inf))
    return np.float32(gts), np.float32(preds)


def tiled(gt, pred, times=7, seed=0):
    """`times` copies of the pairs and as many missing ones, in one fixed random order: several blocks, every pair in
    several lanes."""
    gen = torch.Generator().manual_seed(seed)
    g = torch.cat([torch.from_numpy(gt).repeat(times), torch.zeros(gt.size * times)])
    p = torch.cat([torch.from_numpy(pred).repeat(times), torch.ones(gt.size * times)])
    order = torch.randperm(g.numel(), generator=gen)
    return g[order].contiguous(), p[order].contiguous()


# ---- running the kernels ---------------------------------------------------------------------------------------------------
def stats(gt, pred):
    return metrics._stats(pred.cuda(), gt.cuda()).cpu().numpy()


def loss_and_grad(gt, pred, upstream=None):
    """(loss as a float32, pred.grad on the CPU) of upstream * loss; upstream None is a plain loss.backward()."""
    p = pred.cuda().requires_grad_(True)
    loss = metrics.Wighted_L1_Loss()(p, gt.cuda())
    assert loss.is_cuda and loss.dim() == 0 and loss.dtype == torch.float32
    (loss if upstream is None else upstream * loss).backward()
    return np.float32(loss.item()), p.grad.cpu()


def assert_grad_bits(grad, gt, pred, grad_loss=1.0, case='', count_dtype=np.float64):
    ref = torch.from_numpy(mr.masked_l1_grad(gt, pred, grad_loss, count_dtype))
    assert grad.dtype == torch.float32 and grad.shape == ref.shape, case
    assert not torch.isnan(grad).any(), case                      # then equal values are equal bits, but for the sign of a zero
    bad = grad != ref
    assert not bad.any(), (case, int(bad.sum()), int(bad.flatten().nonzero()[0]))


def assert_all(gt, pred, case):
    mr.assert_stats(stats(gt, pred), gt, pred, case)
    loss, grad = loss_and_grad(gt, pred)
    mae = mr.stats12(gt, pred)[3]
    assert abs(float(loss) - mae) <= mr.ulp32(mae), (case, float(loss), mae)
    assert_grad_bits(grad, gt, pred, 1.0, case)


# ---- a. sizes --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 31, 32, 33, 255, 256, 257, CAP - 1, CAP, CAP + 1, 2 * CAP + 5])
def test_sizes_around_a_warp_a_block_and_the_grid_cap(n):
    gt, pred = spread_inputs(n, n)
    n_valid = mr.counts(gt, pred)[0]
    assert n < 300 or 0.25 * n < n_valid < 0.35 * n
    assert_all(gt, pred, n)


@pytest.mark.parametrize('shape', [(32, 1, 352, 1216), (100003,), (3, 37, 53), (2, 3, 4, 5, 7)])
def test_shapes_of_any_rank_and_the_benchmark_size(shape):
    """32 x 1 x 352 x 1216 is about 50 trips of each thread through the grid-stride loops."""
    n = int(np.prod(shape))
    gt, pred = [t.view(shape) for t in spread_inputs(n, len(shape))]
    mr.assert_stats(stats(gt, pred), gt, pred, shape)
    loss, grad = loss_and_grad(gt, pred, 0.5)
    assert grad.shape == shape
    assert_grad_bits(grad, gt, pred, 0.5, shape)


@pytest.mark.parametrize('n', [CAP + 1, 2 * CAP + 5])
def test_backward_stores_every_element_on_every_trip_of_its_loop(n):
    """Through the C ABI into a NaN-filled buffer: an element that a trip skipped keeps its NaN.  (Autograd hands the kernel
    an uninitialised buffer, in which a missing store can go unseen.)"""
    gt, pred = spread_inputs(n, n + 1)
    g, p = gt.cuda(), pred.cuda()
    twelve = metrics._stats(p, g)
    grad = torch.full((n,), float('nan'), device='cuda')
    gl = torch.tensor([-2.5], device='cuda')
    rc = _lib.lib().cspn_masked_l1_bwd_f32(p.data_ptr(), g.data_ptr(), twelve.data_ptr(), gl.data_ptr(), grad.data_ptr(), n,
                                           torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'cspn_masked_l1_bwd_f32')
    assert_grad_bits(grad.cpu(), gt, pred, -2.5, n)


def test_a_count_above_2_to_24_is_rounded_to_float_before_the_backward_inverts_it():
    """n_valid travels to the backward as a float: above 2^24 it is rounded to even first.  The gradient's scale is then
    fl(1 / fl(n_valid)), at most one ulp from fl(1 / n_valid); here the two differ, and the kernel gives the former."""
    shape = (40, 1, 352, 1216)
    n = int(np.prod(shape))
    if torch.cuda.mem_get_info()[0] < (1 << 30):
        pytest.skip('less than 1 GB of device memory free')
    differs = lambda m: mr.grad_scale(m) != mr.grad_scale(m, count_dtype=np.float32)
    n_valid = next(m for m in range(2 ** 24 + 1001, n, 2) if differs(m))
    gt, pred = [t.view(shape) for t in spread_inputs(n, 40, n_valid=n_valid)]
    ours = stats(gt, pred)
    assert float(ours[0]) == float(np.float32(n_valid)) != n_valid
    mr.assert_stats(ours, gt, pred, 'above 2^24')
    _, grad = loss_and_grad(gt, pred)
    assert_grad_bits(grad, gt, pred, 1.0, 'above 2^24', count_dtype=np.float32)
    exact, rounded = mr.grad_scale(n_valid), mr.grad_scale(n_valid, count_dtype=np.float32)
    assert abs(float(rounded) - float(exact)) == mr.ulp32(exact) and float(grad.abs().max()) == float(rounded)


# ---- b. threshold ties -----------------------------------------------------------------------------------------------------
def test_a_ratio_equal_to_a_threshold_is_not_counted_and_one_ulp_under_it_is():
    gt, pred, r = exact_tie_inputs()
    assert (pred / gt == r).all() and (gt / pred < 1).all()                       # premise: the quotient is r itself
    times = 7
    # expected without any fp32 division: r and the thresholds are exact in double
    expected = [times * int((r.astype(np.float64) < float(t)).sum()) for t in mr.THRESHOLDS]
    on = [int((r == t).sum()) for t in mr.THRESHOLDS]
    assert on == [5] * 6 and expected == [times * 5 * (1 + 3 * j) for j in range(6)]
    g, p = tiled(gt, pred, times)
    assert g.numel() > 4 * 256
    ours = stats(g, p)
    n = times * gt.size
    assert ours[0] == n and [float(x) for x in ours[5:11]] == [float(np.float32(e / n)) for e in expected]
    mr.assert_stats(ours, g, p, 'exact ties')


def test_rounded_quotients_one_ulp_either_side_of_a_threshold_are_counted_as_ieee_division_rounds_them():
    gt, pred = rounded_tie_inputs()
    ratio = mr.max_ratio(gt, pred)
    for t in mr.THRESHOLDS:      # premise: both directions reach t itself and both of its neighbours
        for down in (True, False):
            side = ratio[(pred < gt) == down]
            assert all((side == v).any() for v in (np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(4)))), (t, down)
    g, p = tiled(gt, pred, 3, seed=1)
    mr.assert_stats(stats(g, p), g, p, 'rounded ties')


# ---- c. special values -----------------------------------------------------------------------------------------------------
def test_edge_fixtures_are_present():
    assert len(EDGES) == 21


@pytest.mark.parametrize('name', EDGES)
def test_special_values_as_the_reference_treats_them(name):
    z = np.load(os.path.join(EDGE_DIR, name + '.npz'))
    gt, pred = torch.from_numpy(z['gt']), torch.from_numpy(z['pred'])
    ours = stats(gt, pred)
    mr.assert_stats(ours, gt, pred, name)
    # against the reference's own numbers
    n = int(z['n_valid'])
    assert ours[0] == n
    ref = dict(zip([str(k) for k in z['keys']], z['metrics']))
    got = dict(zip(mr.KEYS, ours[1:11]))
    for k in mr.KEYS[4:]:
        assert got[k] == np.float32(ref[k]), (name, k)
    def same(a, b):          # NaN where the reference has NaN, the same inf, else its fp32-summed value to rounding
        return np.isnan(a) if np.isnan(b) else (a == b if np.isinf(b) else abs(float(a) - b) <= 2e-6 * abs(b))

    for k in ('MSE', 'MAE', 'ABS_REL'):
        assert same(got[k], ref[k]), (name, k, got[k], ref[k])
    # RMSE is the root of the fp64 mean: finite (4.4e37) where pred = FLT_MAX pushes MSE itself, and the reference's root of
    # it, to inf
    if name == 'pred_fltmax':
        assert np.isinf(got['MSE']) and np.isinf(ref['RMSE']) and 4e37 < got['RMSE'] < 5e37
    else:
        assert same(got['RMSE'], ref['RMSE']), (name, got['RMSE'], ref['RMSE'])
    loss, grad = loss_and_grad(gt, pred)
    assert same(loss, float(z['loss'])), (name, loss, float(z['loss']))
    assert_grad_bits(grad, gt, pred, 1.0, name)
    assert torch.equal(grad, torch.from_numpy(z['grad_pred']))


def test_special_values_spread_over_many_blocks():
    z = np.load(os.path.join(EDGE_DIR, 'all_together.npz'))
    gt, pred = tiled(z['gt'], z['pred'], 40, seed=2)
    assert gt.numel() > 20 * 256
    mr.assert_stats(stats(gt, pred), gt, pred, 'all_together x 40')
    _, grad = loss_and_grad(gt, pred, -2.5)
    assert_grad_bits(grad, gt, pred, -2.5, 'all_together x 40')


# ---- d. nothing valid ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fill', [0.0, -1.0, float(mr.VALID_CUT), float('nan')])
@pytest.mark.parametrize('upstream', [None, 3.0, float('inf')])
def test_nothing_valid_gives_zero_metrics_and_a_zero_loss_with_a_zero_gradient(fill, upstream):
    """The reference's metrics are all 0 here (utils.py:31) and so are ours.  Its loss is 0 / 0 = NaN; ours is 0 with a zero
    gradient, so that a frame without ground truth does not poison a training run (DESIGN.md section 4.7)."""
    gt = torch.full((1, 1, 8, 9), fill)
    pred = torch.rand(1, 1, 8, 9, generator=torch.Generator().manual_seed(1))
    err = metrics.evaluate_error(gt.cuda(), pred.cuda())
    assert all(float(err[k]) == 0 for k in metrics.KEYS)
    assert not stats(gt, pred).any()
    loss, grad = loss_and_grad(gt, pred, upstream)
    assert loss == 0 and grad.shape == pred.shape and not grad.any()


# ---- e. backward -----------------------------------------------------------------------------------------------------------
def kink_inputs(n=3001, seed=9):
    """Spread inputs with pred == gt at every third element and a NaN pred at every eleventh."""
    gt, pred = spread_inputs(n, seed, 0.6)
    pred[::3] = gt[::3]
    pred[::11] = float('nan')
    return gt, pred


@pytest.mark.parametrize('upstream', [1.0, -2.5, 0.0])
def test_gradient_bits_at_the_kink_for_nan_and_under_an_upstream_gradient(upstream):
    gt, pred = kink_inputs()
    valid = mr.valid_mask(gt)
    assert (valid & (pred == gt).numpy()).sum() > 300 and (valid & torch.isnan(pred).numpy()).sum() > 100
    _, grad = loss_and_grad(gt, pred, upstream)
    assert_grad_bits(grad, gt, pred, upstream, upstream)
    assert not grad[::3].any() and not grad[::11].any()


def test_upstream_gradient_from_autograd_and_the_loss_used_twice():
    gt, pred = kink_inputs()
    g = gt.cuda()
    p = pred.cuda().requires_grad_(True)
    w = torch.tensor(0.75, device='cuda', requires_grad=True)
    loss = metrics.Wighted_L1_Loss()(p, g)
    ((loss * w).sum() + 2.0 * loss).backward()              # grad_loss = 0.75 + 2 arrives as a tensor autograd made
    assert_grad_bits(p.grad.cpu(), gt, pred, 2.75, 'non-leaf upstream')
    assert np.isnan(loss.item()) and np.isnan(w.grad.item())        # d/dw = the loss, NaN from the NaN predictions
    p2 = pred.cuda().requires_grad_(True)                   # two applications in one graph: the gradients add
    crit = metrics.Wighted_L1_Loss()
    (crit(p2, g) + crit(p2, g)).backward()
    assert_grad_bits(p2.grad.cpu(), gt, pred, 2.0, 'used twice')


def test_label_gets_no_gradient_and_a_pred_without_one_is_fine():
    gt, pred = spread_inputs(500, 3)
    g = gt.cuda().requires_grad_(True)
    p = pred.cuda().requires_grad_(True)
    metrics.Wighted_L1_Loss()(p, g).backward()
    assert g.grad is None
    assert_grad_bits(p.grad.cpu(), gt, pred, 1.0, 'label requires grad')
    loss = metrics.Wighted_L1_Loss()(pred.cuda(), gt.cuda())
    assert not loss.requires_grad and abs(float(loss) - mr.stats12(gt, pred)[3]) <= mr.ulp32(float(loss))
    loss = metrics.Wighted_L1_Loss()(pred.cuda(), g)        # only the label requires a gradient: backward must not raise
    loss.backward()
    assert g.grad is None


def test_views_of_pred_channels_last_transposed_and_4_bytes_off_alignment():
    shape = (2, 3, 17, 23)
    n = int(np.prod(shape))
    gt, pred = [t.view(shape) for t in spread_inputs(n, 4, 0.5)]
    ref = torch.from_numpy(mr.masked_l1_grad(gt, pred, 1.0))
    g = gt.cuda()

    def check(p, case):
        assert torch.equal(p.detach().cpu(), pred if p.dim() == 4 else pred.view(p.shape))
        q = p.detach().requires_grad_(True)
        metrics.Wighted_L1_Loss()(q, g if q.dim() == 4 else g.view(q.shape)).backward()
        assert q.grad.shape == q.shape and torch.equal(q.grad.cpu().reshape(shape), ref), case
        mr.assert_stats(metrics._stats(q.detach(), g.view(q.shape)).cpu().numpy(), gt, pred, case)

    cl = pred.cuda().contiguous(memory_format=torch.channels_last)
    assert not cl.is_contiguous()
    check(cl, 'channels_last')
    tr = pred.view(6, -1).t().contiguous().cuda().t()       # logical (6, 17 * 23), stored transposed
    assert not tr.is_contiguous()
    check(tr, 'transposed')
    off = torch.empty(n + 1, device='cuda')[1:]
    off.copy_(pred.view(-1))
    assert off.data_ptr() % 16 == 4 and off.is_contiguous()
    check(off, 'offset')
    goff = torch.empty(n + 1, device='cuda')[1:]
    goff.copy_(gt.view(-1))
    mr.assert_stats(metrics._stats(off, goff).cpu().numpy(), gt, pred, 'both offset')


def test_a_double_backward_raises():
    gt, pred = spread_inputs(100, 5)
    p = pred.cuda().requires_grad_(True)
    loss = metrics.Wighted_L1_Loss()(p, gt.cuda())
    (grad,) = torch.autograd.grad(loss, p, create_graph=True, retain_graph=True)
    assert not grad.requires_grad                       # a constant upstream gradient: nothing to differentiate, and torch says so
    with pytest.raises(RuntimeError, match='does not require grad'):
        grad.sum().backward()
    w = torch.tensor(2.0, device='cuda', requires_grad=True)
    (grad,) = torch.autograd.grad(loss * w, p, create_graph=True)
    assert grad.requires_grad                           # through the upstream gradient it would be differentiable: refused
    with pytest.raises(RuntimeError, match='once_differentiable'):
        grad.sum().backward()


# ---- f. calling context ----------------------------------------------------------------------------------------------------
def test_on_a_side_stream_the_kernels_wait_for_the_work_that_produces_pred():
    n = 1 << 22
    gt, pred = dyadic_inputs(n, 6)
    g, p = gt.cuda(), pred.cuda()
    buf = p + 1024.0                          # stale values; the side stream takes them down to pred in 64 exact steps
    metrics._stats(p, g)                      # the library is loaded before anything is queued
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(64):
            buf.sub_(16.0)
        out = metrics._stats(buf, g)
        q = buf.requires_grad_(True)
        metrics.Wighted_L1_Loss()(q, g).backward()
    side.synchronize()
    assert torch.equal(buf.detach(), p)
    mr.assert_stats(out.cpu().numpy(), gt, pred, 'side stream')
    assert_grad_bits(q.grad.cpu(), gt, pred, 1.0, 'side stream')


def test_captured_in_a_cuda_graph_and_replayed_on_new_values():
    n = CAP + 1000
    gt0, pred0 = dyadic_inputs(n, 7)
    gt1, pred1 = dyadic_inputs(n, 8)
    sg, sp = gt0.cuda(), pred0.cuda().requires_grad_(True)
    crit = metrics.Wighted_L1_Loss()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):             # warm-up off the default stream, as graph capture wants it
        crit(sp, sg).backward()
        metrics.evaluate_error(sg, sp.detach())
    torch.cuda.current_stream().wait_stream(side)
    sp.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        err = metrics.evaluate_error(sg, sp.detach())
        twelve = metrics._stats(sp.detach(), sg)
        loss = crit(sp, sg)
        loss.backward()
    for gt, pred in ((gt1, pred1), (gt0, pred0)):
        with torch.no_grad():
            sg.copy_(gt)
            sp.copy_(pred)
        graph.replay()
        torch.cuda.synchronize()
        eager = metrics._stats(pred.cuda(), gt.cuda())
        assert torch.equal(twelve, eager)                                   # dyadic inputs: the sums are exact in any order
        mr.assert_stats(twelve.cpu().numpy(), gt, pred, 'graph replay')
        assert all(float(err[k]) == float(eager[metrics._SLOT[k]]) for k in metrics.KEYS)
        assert loss.item() == eager[3].item()
        assert_grad_bits(sp.grad.cpu(), gt, pred, 1.0, 'graph replay')
    assert mr.counts(gt0, pred0) != mr.counts(gt1, pred1)


def test_two_calls_in_a_row_give_the_same_twelve_floats():
    gt, pred = dyadic_inputs(3 * CAP + 17, 9)
    g, p = gt.cuda(), pred.cuda()
    a, b = metrics._stats(p, g), metrics._stats(p, g)
    assert torch.equal(a, b)
    mr.assert_stats(a.cpu().numpy(), gt, pred, 'twice')


def test_c_abi_ignores_what_the_workspace_holds_also_for_no_elements_and_when_reused():
    L = _lib.lib()
    ws_bytes = L.cspn_depth_metrics_workspace_bytes()
    assert ws_bytes == 80
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device='cuda')          # every double a NaN
    out = torch.full((12,), 7.0, device='cuda')
    gt, pred = dyadic_inputs(1000, 10)
    g, p = gt.cuda(), pred.cuda()
    stream = torch.cuda.current_stream().cuda_stream
    call = lambda n: L.cspn_depth_metrics_f32(p.data_ptr(), g.data_ptr(), n, out.data_ptr(), ws.data_ptr(), ws_bytes, stream)
    assert call(0) == 0                                                           # CSPN_OK
    assert not out.cpu().any()
    assert call(1000) == 0
    first = out.clone()
    mr.assert_stats(first.cpu().numpy(), gt, pred, 'stale workspace')
    assert call(1000) == 0                                                        # the workspace now holds the first call's sums
    assert torch.equal(out, first)
    assert call(0) == 0 and not out.cpu().any()


# ---- g. interface ----------------------------------------------------------------------------------------------------------
def test_evaluate_error_takes_gt_first_and_returns_the_reference_keys_as_0_d_cuda_tensors():
    gen = torch.Generator().manual_seed(11)
    gt = torch.rand(2000, generator=gen) * 9 + 1
    pred = gt * (torch.rand(2000, generator=gen) * 0.8 + 1.2)                     # always above gt: swapping the two shows
    err = metrics.evaluate_error(gt.cuda(), pred.cuda())
    assert set(err) == set(metrics.KEYS) | {'LG10'} and err['LG10'] == 0 and len(err) == 11
    assert all(err[k].is_cuda and err[k].dim() == 0 and err[k].dtype == torch.float32 for k in metrics.KEYS)
    ref, swapped = mr.stats12(gt, pred), mr.stats12(pred, gt)
    assert abs(ref[4] - swapped[4]) > 1e-3 * ref[4]                               # ABS_REL divides by gt: not symmetric
    assert abs(float(err['ABS_REL']) - ref[4]) <= mr.ulp32(ref[4])
    assert abs(float(metrics.evaluate_error(pred.cuda(), gt.cuda())['ABS_REL']) - swapped[4]) <= mr.ulp32(swapped[4])
    assert abs(float(metrics.evaluate_error(gt_depth=gt.cuda(), pred_depth=pred.cuda())['ABS_REL']) - ref[4]) <= mr.ulp32(ref[4])


def test_wrong_inputs_raise():
    g, p = torch.rand(2, 3, device='cuda') + 1, torch.rand(2, 3, device='cuda')
    bad = [
        (g.cpu(), p.cpu(), _lib.CspnError), (g, p.cpu(), _lib.CspnError), (g.cpu(), p, _lib.CspnError),
        (g.half(), p.half(), ValueError), (g.bfloat16(), p, ValueError), (g, p.double(), ValueError),
        (g, p.t(), ValueError), (g, p.view(-1), ValueError), (g[:1], p, ValueError),
    ]
    for gt, pred, exc in bad:
        with pytest.raises(exc):
            metrics.evaluate_error(gt, pred)
        with pytest.raises(exc):
            metrics.Wighted_L1_Loss()(pred, gt)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            metrics.evaluate_error(g, p.to('cuda:1'))


# ---- h. one whole training tail against fp64 -------------------------------------------------------------------------------
def test_training_tail_heads_propagation_loss_and_backward_match_fp64_autograd():
    """unpool_conv3x3 guidance and depth heads -> Affinity_Propagate -> Wighted_L1_Loss -> backward(): the loss and the
    gradients of the feature map and of both head weights against fp64 autograd through the restatements of each stage."""
    B, Cin, h, w, H, W, N = 2, 16, 23, 29, 45, 57, 6
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(B, Cin, h, w, generator=gen)
    wg = torch.randn(8, Cin, 3, 3, generator=gen) / 8
    wd = torch.randn(1, Cin, 3, 3, generator=gen) / 8
    sparse = 3.0 * (torch.rand(B, 1, H, W, generator=gen) < 0.1)

    def forward64(x, wg, wd):
        return be.cspn2d_shift_ref(ur.op_sequence(x, wg, H, W), ur.op_sequence(x, wd, H, W), sparse.double(), N, 3, '8sum')

    leaves64 = [t.double().requires_grad_(True) for t in (x, wg, wd)]
    out64 = forward64(*leaves64)
    # ground truth at least 1 away from the prediction, so that no sign(pred - gt) differs between fp32 and fp64
    away = (torch.rand(out64.shape, generator=gen) + 1) * (torch.randint(0, 2, out64.shape, generator=gen) * 2 - 1)
    target = ((out64.detach() + away) * (torch.rand(out64.shape, generator=gen) < 0.7)).float()
    n_valid = int(mr.valid_mask(target).sum())
    assert 0.2 * target.numel() < n_valid < 0.6 * target.numel()
    loss64 = mr.masked_l1_torch(out64, target.double())
    loss64.backward()

    leaves = [t.cuda().requires_grad_(True) for t in (x, wg, wd)]
    guidance = cspn_b200.unpool_conv3x3(leaves[0], leaves[1], H, W)
    blur = cspn_b200.unpool_conv3x3(leaves[0], leaves[2], H, W)
    out = cspn_b200.Affinity_Propagate(N, 3, '8sum')(guidance, blur, sparse.cuda())
    loss = metrics.Wighted_L1_Loss()(out, target.cuda())
    loss.backward()
    assert (out.detach().cpu().double() - target.double()).abs()[torch.from_numpy(mr.valid_mask(target))].min() > 0.5
    assert abs(loss.item() - loss64.item()) <= 1e-5 * loss64.item(), (loss.item(), loss64.item())
    for ours, ref, name in zip(leaves, leaves64, ('grad_x', 'grad_guidance_weight', 'grad_depth_weight')):
        a, b = ours.grad.double().cpu(), ref.grad
        assert b.abs().mean() > 0
        err = (a - b).abs()
        assert (err <= 2e-3 * (b.abs() + b.abs().mean())).all(), (name, float(err.max()), float(b.abs().mean()))
