"""CPU tests of the independent stereo-head model (tests/stereo_head_reference.py): its pieces equal the stock torch ops
that define them (F.avg_pool2d, F.unfold, F.conv2d, F.interpolate) and the networks' conventions, they agree in fp64 with
the per-op restatements the op suites use, and the comparator of tests/test_stereo_head_gpu.py rejects the head with any
one of six planted convention errors against the unmutated one."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

import stereo_head_reference as sh

import affinity_atrous_reference as aar
import affinity_fuse_reference as afr
import affinity_pool_reference as apr
import cost_volume_reference as cvr
import disparity_reference as dr
import gates_reference as gr
from oracle import cspn_torch_port as tp

ALIGN = [(True, 1), (True, 0), (False, 0), (False, 1)]


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


# ---- the pieces against the stock ops that define them ----------------------------------------------------------------------
def test_pool_under_a_constant_gate_is_avg_pool2d():
    feat = rnd(0, 2, 3, 37, 50)
    ks = (16, 5, 1, 37)
    for l, out in enumerate(sh.affinity_pool(feat, torch.full((2, 4, 37, 50), -2.5, dtype=torch.float64), ks)):
        torch.testing.assert_close(out, F.avg_pool2d(feat, ks[l]), rtol=1e-13, atol=1e-14)


def test_pool_weights_each_window_by_its_own_gates():
    feat, gate = rnd(1, 1, 2, 8, 12), rnd(2, 1, 1, 8, 12)
    out, = sh.affinity_pool(feat, gate, (4,))
    a = gate.abs()
    want = F.avg_pool2d(a * feat, 4) / F.avg_pool2d(a, 4)
    torch.testing.assert_close(out, want, rtol=1e-13, atol=1e-14)


@pytest.mark.parametrize('r', [1, 2, 5])
def test_atrous_taps_follow_the_unfold_order_and_the_dilation(r):
    B, C, H, W = 2, 3, 9, 11
    feat = rnd(3, B, C, H, W)
    for t in range(9):
        gate = torch.zeros(B, 9, H, W, dtype=torch.float64)
        gate[:, t] = -0.5
        dy, dx = (t // 3 - 1) * r, (t % 3 - 1) * r
        want = torch.zeros_like(feat)
        ys, xs = slice(max(0, -dy), H - max(0, dy)), slice(max(0, -dx), W - max(0, dx))
        yd, xd = slice(max(0, dy), H + min(0, dy)), slice(max(0, dx), W + min(0, dx))
        want[..., ys, xs] = feat[..., yd, xd]
        assert torch.equal(sh.affinity_atrous(feat, gate, (r,)), want), t
    box = F.conv2d(feat, torch.full((C, 1, 3, 3), 1 / 9, dtype=torch.float64), padding=r, dilation=r, groups=C)
    torch.testing.assert_close(sh.affinity_atrous(feat, torch.ones(B, 9, H, W, dtype=torch.float64), (r,)), box,
                               rtol=1e-13, atol=1e-14)


def test_atrous_levels_are_concatenated_level_major():
    feat, gate = rnd(4, 1, 2, 6, 7), rnd(5, 1, 27, 6, 7)
    out = sh.affinity_atrous(feat, gate, (1, 3, 2))
    for l, r in enumerate((1, 3, 2)):
        assert torch.equal(out[:, 2 * l:2 * l + 2], sh.affinity_atrous(feat, gate[:, 9 * l:9 * l + 9], (r,)))


@pytest.mark.parametrize('align_corners', [True, False])
def test_fuse_under_a_one_hot_gate_is_interpolate(align_corners):
    levels = [rnd(6, 2, 3, 1, 2), rnd(7, 2, 3, 5, 9), rnd(8, 2, 3, 17, 23)]
    for l, x in enumerate(levels):
        gate = torch.zeros(2, 3, 17, 23, dtype=torch.float64)
        gate[:, l] = 3.0
        want = F.interpolate(x, (17, 23), mode='bilinear', align_corners=align_corners)
        assert torch.equal(sh.affinity_fuse(levels, gate, align_corners, 0), want)
    mean = sum(F.interpolate(x, (17, 23), mode='bilinear', align_corners=align_corners) for x in levels) / 3
    torch.testing.assert_close(sh.affinity_fuse(levels, torch.ones(2, 3, 17, 23, dtype=torch.float64), align_corners, 0),
                               mean, rtol=1e-13, atol=1e-14)


def test_paddle_rule_worked_example():
    """DESIGN.md section 4.14: align_mode=1, 4 -> 7 gives s = 4o/7 and, for x = [0, 1, 2, 3], [0, 4/7, ..., 20/7, 3]."""
    x = torch.arange(4, dtype=torch.float64).view(1, 1, 1, 4)
    want = torch.tensor([0, 4 / 7, 8 / 7, 12 / 7, 16 / 7, 20 / 7, 3], dtype=torch.float64)
    torch.testing.assert_close(sh.resample(x, (1, 7), False, 1).flatten(), want, rtol=1e-15, atol=1e-15)


@pytest.mark.parametrize('size_in,size_out', [((5, 9), (17, 23)), ((6, 4), (3, 11)), ((1, 7), (4, 7)), ((12, 24), (48, 96)),
                                              ((3, 5, 7), (13, 9, 28)), ((12, 16, 32), (48, 64, 128))])
def test_paddle_rule_is_interpolate_of_the_edge_padded_input(size_in, size_out):
    """s(o) = o * n_in / n_out is F.interpolate(align_corners=True) from n_in + 1 samples (the last one repeated) to
    n_out + 1, the last output dropped: the ratio (n_in + 1 - 1) / (n_out + 1 - 1) is n_in / n_out, and past n_in - 1
    both rules read the last sample only."""
    x = rnd(9, 2, 3, *size_in)
    nd = len(size_in)
    mode = 'bilinear' if nd == 2 else 'trilinear'
    padded = F.pad(x, (0, 1) * nd, mode='replicate')
    want = F.interpolate(padded, tuple(n + 1 for n in size_out), mode=mode, align_corners=True)
    want = want[(Ellipsis,) + tuple(slice(0, n) for n in size_out)]
    torch.testing.assert_close(sh.resample(x, size_out, False, 1), want, rtol=1e-13, atol=1e-14)


def test_paddle_rule_is_the_identity_and_nearest_where_torch_agrees():
    x = rnd(10, 2, 3, 8, 12)
    assert torch.equal(sh.resample(x, (8, 12), False, 1), x)
    torch.testing.assert_close(sh.resample(x, (8, 12), False, 1), F.interpolate(x, (8, 12), mode='bilinear',
                                                                                align_corners=False))
    for k in (2, 4):
        assert torch.equal(sh.resample(x, (8 // k, 12 // k), False, 1), F.interpolate(x, (8 // k, 12 // k), mode='nearest'))


@pytest.mark.parametrize('align_corners,align_mode', [(True, 1), (False, 0)])
def test_regression_is_interpolate_softmax_expectation(align_corners, align_mode):
    cost = rnd(11, 2, 1, 5, 6, 7) * 3
    size = (20, 24, 28)
    u = F.interpolate(cost, size, mode='trilinear', align_corners=align_corners)
    want = (torch.softmax(u, 2) * torch.arange(20, dtype=torch.float64).view(1, 1, -1, 1, 1)).sum(2)
    assert torch.equal(sh.disparity_regression(cost, size, align_corners, align_mode), want)


def test_regression_counts_disparity_from_the_first_plane_in_output_pixels():
    """A cost peaked on low-resolution plane k regresses to the upsampled index of that plane, where the upsampled column
    is symmetric about it: k * (Do - 1) / (D - 1) = 4k with align_corners (D = 12 -> Do = 45), 4k + 1.5 under torch's
    half-pixel rule at x4 (the centre of the four upsampled planes k covers), 4k under Paddle's rule; so plane 0 is
    disparity 0 and the unit is a full-resolution pixel."""
    D, k = 12, 7
    cost = torch.full((1, 1, D, 3, 4), -60.0, dtype=torch.float64)
    cost[:, :, k] = 60.0
    for (ac, am), Do, want in (((True, 1), 45, 4 * k), ((False, 0), 48, 4 * k + 1.5), ((False, 1), 48, 4 * k)):
        y = sh.disparity_regression(cost, (Do, 12, 16), ac, am)
        torch.testing.assert_close(y, torch.full_like(y, want), rtol=0, atol=1e-9)


def test_cost_volumes_match_left_x_with_right_x_minus_d():
    """A right image that is the left one moved k pixels to the left (a true disparity of k) correlates best at d = k."""
    B, C, H, W, D, k = 1, 64, 4, 40, 12, 5
    left = rnd(12, B, C, H, W)
    right = torch.zeros_like(left)
    right[..., :W - k] = left[..., k:]                       # right[x - k] = left[x]
    gwc = sh.gwc_volume(left, right, D, 1)
    assert (gwc[0, 0, :, :, D:].argmax(dim=0) == k).all()
    cat = sh.concat_volume(left, right, D)
    assert torch.equal(cat[:, C:, k, :, k:], cat[:, :C, k, :, k:])
    assert (cat[:, :, 3, :, :3] == 0).all() and torch.equal(cat[:, C:, 3, :, 3:], right[..., :W - 3])


def test_propagation_taps_read_the_documented_offsets():
    """Tap k enumerates (f, t, l) in raster order without the centre and reads p + (1 - f, 1 - t, 1 - l)."""
    feat = rnd(13, 1, 1, 4, 5, 6)
    for k in (0, 4, 12, 13, 25):
        gates = torch.zeros(1, 26, 4, 5, 6, dtype=torch.float64)
        gates[:, k] = 1.0
        dz, dy, dx = sh.OFFSETS_3D[k]
        want = F.pad(feat, (1,) * 6)[..., 1 + dz:5 + dz, 1 + dy:6 + dy, 1 + dx:7 + dx]
        assert torch.equal(sh.affinity_propagate3d(feat, gates, 1), want), k
    assert sh.OFFSETS_3D[0] == (1, 1, 1) and sh.OFFSETS_3D[25] == (-1, -1, -1) and sh.OFFSETS_3D[12] == (0, 0, 1)
    torch.testing.assert_close(sh.paddle_gates(rnd(14, 2, 26, 3, 4, 5)).sum(1), torch.ones(2, 3, 4, 5, dtype=torch.float64))


# ---- agreement with the per-op restatements, fp64 ----------------------------------------------------------------------------
@pytest.mark.parametrize('D', [1, 12, 45])
def test_volumes_agree_with_the_restated_loops(D):
    left, right = rnd(20, 2, 8, 5, 40), rnd(21, 2, 8, 5, 40)
    assert torch.equal(sh.concat_volume(left, right, D), cvr.concat_loop(left, right, D))
    for G in (1, 4, 8):
        torch.testing.assert_close(sh.gwc_volume(left, right, D, G), cvr.gwc_loop(left, right, D, G), rtol=1e-14, atol=1e-15)


def test_pool_agrees_with_the_restated_composition():
    feat, gate = rnd(22, 2, 5, 33, 47), rnd(23, 2, 4, 33, 47)
    for a, b in zip(sh.affinity_pool(feat, gate, (32, 8, 3, 1)), apr.compose(feat, gate, (32, 8, 3, 1))):
        torch.testing.assert_close(a, b, rtol=1e-13, atol=1e-14)


def test_atrous_agrees_with_the_restated_composition():
    feat, gate = rnd(24, 2, 5, 17, 23), rnd(25, 2, 36, 17, 23)
    torch.testing.assert_close(sh.affinity_atrous(feat, gate, (1, 4, 9, 20)), aar.compose(feat, gate, (1, 4, 9, 20)),
                               rtol=1e-13, atol=1e-14)


# The restatements of fusion and regression form the kernels' taps in fp32 (resize_reference.taps); the model forms them in
# its own dtype, as F.interpolate does.  At sizes whose ratio r is a power of two every source coordinate r * o (or
# r * (o + 1/2) - 1/2) is exact in both, so the two must agree to fp64 rounding: 16 -> 64 without align_corners,
# 17 -> 65 with it ((17 - 1) / (65 - 1) = 1/4).
@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_fuse_agrees_with_the_restated_composition(align_corners, align_mode):
    e = int(align_corners)
    levels = [rnd(26 + k, 2, 3, h + e, w + e) for k, (h, w) in enumerate(((1, 2), (4, 8), (16, 32), (64, 128)))]
    gate = rnd(30, 2, 4, 64 + e, 128 + e)
    got = sh.affinity_fuse(levels, gate, align_corners, align_mode)
    torch.testing.assert_close(got, afr.compose(levels, gate, align_corners, align_mode), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_regression_agrees_with_the_restated_composition(align_corners, align_mode):
    e = int(align_corners)
    cost = rnd(31, 2, 1, 12 + e, 16 + e, 32 + e) * 4
    size = (48 + e, 64 + e, 128 + e)
    got = sh.disparity_regression(cost, size, align_corners, align_mode)
    torch.testing.assert_close(got, dr.forward_torch(cost, size, align_corners, align_mode), rtol=1e-12, atol=1e-10)


def test_propagation_agrees_with_the_restated_gates_op_and_the_paddle_port():
    guide, feat = rnd(32, 2, 26, 6, 7, 9), rnd(33, 2, 1, 6, 7, 9)
    got = sh.affinity_propagate3d(feat, sh.paddle_gates(guide), 5)
    torch.testing.assert_close(got, gr.affinity_propagate_ref(feat, gr.paddle_gates(guide, 26), 3, 5), rtol=1e-13, atol=1e-14)
    torch.testing.assert_close(got, tp.cspn3d_torch(guide, feat, 5, 'paddle'), rtol=1e-13, atol=1e-14)


# ---- sensitivity: the comparator rejects each planted convention error ---------------------------------------------------------
# The head at a reduced size, with the GPU tests' layer structure: B = 2, 64 x 128 images, features at 16 x 32, D = 12 -> 48.
CFG = dict(channels=8, kernel_sizes=(16, 8, 4, 2), rates=(2, 3, 5, 7), max_disp=12, groups=4, out_channels=8,
           prop_steps=6)
MODES = [(True, 1), (False, 0)]


def _load_copy():
    spec = importlib.util.spec_from_file_location('stereo_head_mutant',
                                                  os.path.join(os.path.dirname(__file__), 'stereo_head_reference.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _concat_plus(left, right, D):
    B, C, H, W = left.shape
    vol = left.new_zeros((B, 2 * C, D, H, W))
    for d in range(min(D, W)):
        vol[:, :C, d, :, :W - d] = left[:, :, :, :W - d]
        vol[:, C:, d, :, :W - d] = right[:, :, :, d:]
    return vol


def _gwc_plus(left, right, D, G):
    B, C, H, W = left.shape
    vol = left.new_zeros((B, G, D, H, W))
    for d in range(min(D, W)):
        vol[:, :, d, :, :W - d] = (left[:, :, :, :W - d] * right[:, :, :, d:]).view(B, G, C // G, H, W - d).mean(dim=2)
    return vol


def _regression_reversed(mod):
    def regress(cost, size, align_corners, align_mode):
        p = torch.softmax(mod.resample(cost, size, align_corners, align_mode), dim=2)
        o = torch.arange(size[0], dtype=cost.dtype).flip(0).view(1, 1, -1, 1, 1)
        return (p * o).sum(dim=2)
    return regress


def _resample_half_pixel(x, size, align_corners, align_mode):
    """Every sample taken half an output pixel later than the rule says: s(o + 1/2), clamped to the input."""
    for k, n_out in enumerate(size):
        dim, n_in = 2 + k, x.shape[2 + k]
        o = torch.arange(n_out, dtype=x.dtype) + 0.5
        if align_corners:
            s = o * ((n_in - 1) / max(n_out - 1, 1))
        elif align_mode == 0:
            s = (o + 0.5) * (n_in / n_out) - 0.5
        else:
            s = o * (n_in / n_out)
        s = s.clamp(0, n_in - 1)
        i0 = s.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        lam = (s - i0.to(x.dtype)).view([-1] + [1] * (x.dim() - 1 - dim))
        x = (1 - lam) * x.index_select(dim, i0) + lam * x.index_select(dim, i1)
    return x


def _atrous_gate_order(feat, gate, rates):
    B, C, H, W = feat.shape
    L, outs = len(rates), []
    for l, r in enumerate(rates):
        taps = F.unfold(feat, 3, dilation=r, padding=r).view(B, C, 9, H, W)
        a = gate[:, l::L].abs()                                  # channel t * L + l
        outs.append(((a / a.sum(1, keepdim=True)).unsqueeze(1) * taps).sum(2))
    return torch.cat(outs, 1)


def _atrous_dilation_minus_one(mod):
    real = mod.affinity_atrous
    return lambda feat, gate, rates: real(feat, gate, tuple(r - 1 for r in rates))


def _fuse_unnormalised(mod):
    def fuse(levels, gate, align_corners, align_mode):
        a = gate.abs()
        return sum(a[:, l:l + 1] * mod.resample(x, gate.shape[2:], align_corners, align_mode) for l, x in enumerate(levels))
    return fuse


MUTATIONS = {
    'disparity sign flipped (x + d)': lambda m: {'concat_volume': _concat_plus, 'gwc_volume': _gwc_plus},
    'regression index reversed': lambda m: {'disparity_regression': _regression_reversed(m)},
    'resampling half a pixel off': lambda m: {'resample': _resample_half_pixel},
    'ACSPP gate order t*L + l': lambda m: {'affinity_atrous': _atrous_gate_order},
    'ACSPP dilation r - 1': lambda m: {'affinity_atrous': _atrous_dilation_minus_one(m)},
    'fusion weights not normalised': lambda m: {'affinity_fuse': _fuse_unnormalised(m)},
}

_BASE = {}


def _base(align_corners, align_mode):
    """(head fp32, inputs, fp32 results, fp64 results) of the unmutated model, once per alignment rule."""
    key = (align_corners, align_mode)
    if key not in _BASE:
        head = sh.StereoHead(**CFG, align_corners=align_corners, align_mode=align_mode)
        args = sh.inputs(1, 2, 64, 128, CFG['max_disp'], 'cpu')
        _BASE[key] = (head, args, sh.run(head, *args), sh.run(sh.as_dtype(head, torch.float64), *args))
    return _BASE[key]


@pytest.mark.parametrize('align_corners,align_mode', MODES)
def test_the_unmutated_fp32_model_passes_the_comparator(align_corners, align_mode):
    head, args, r32, r64 = _base(align_corners, align_mode)
    ok, rows = sh.compare(r32, r32, r64)
    assert ok and len(rows) == 1 + 2 + len(list(head.parameters()))
    assert all(0 < e < 1e-4 for _, _, e, _, _ in rows), sh.report(rows)


@pytest.mark.parametrize('align_corners,align_mode', MODES)
@pytest.mark.parametrize('name', list(MUTATIONS))
def test_the_comparator_rejects_a_planted_convention_error(name, align_corners, align_mode):
    head, args, r32, r64 = _base(align_corners, align_mode)
    mod = _load_copy()
    for attr, fn in MUTATIONS[name](mod).items():
        setattr(mod, attr, fn)
    mutant = mod.StereoHead(**CFG, align_corners=align_corners, align_mode=align_mode)
    mutant.load_state_dict(head.state_dict())
    ok, rows = sh.compare(sh.run(mutant, *args), r32, r64)
    print(f'\n{name}, align_corners={align_corners}, align_mode={align_mode}: {"accepted" if ok else "rejected"}\n'
          + sh.report(rows))
    assert not ok
    assert not dict((r[0], r[-1]) for r in rows)['disparity'], sh.report(rows)
