"""The premises of tests/test_depth_ops_at_scale_gpu.py, without a GPU.  That file runs the dilated (DESIGN.md section
4.22), aggregating (section 4.20), non-local (section 4.21) and dynamic (section 4.23) 2D propagations across CTA tiles
and at the shapes the README times; here:

- the tile constants, read from the CUDA sources, and each seam shape crossing what it is meant to cross (at least three
  tiles in x and in y with a partial last tile, halos reaching into the neighbouring tile, two aggregate launch groups,
  more than 2^27 non-local samples with a sort key wider than 16 bits, a partial last block of the dynamic finalize, step
  counts on both sides of its 64 attention slices).  A retuned tile fails here, not silently there.
- the exactness the GPU file's bit-for-bit checks rest on: on the dyadic dilated and dynamic cases at the seam shapes
  and on the non-local integer-offset case at the timing shape, the fp32 restatement equals the fp64 reference, output
  and every gradient.  (The dynamic op's random-input checks need no such premise: tests/dynamic_reference.py's
  kernel_order states the kernels' order of operations, and the GPU file compares with it bit for bit.)
- the hot bucket: every sample of the case lands on one fractional point, so one bucket holds them all.

The input generators live here so that both files use the same inputs."""
import os
import re

import pytest
import torch

import dilated_reference as dr
import dynamic_reference as yr
import nonlocal_reference as nr

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), 'cspn_b200', 'csrc')

# ---- shapes (B, C, H, W) ----------------------------------------------------------------------------------------------------
TIMING = (8, 1, 352, 1216)                          # the README's timing shape of the four ops
DIL_SEAMS = [(2, 2, 45, 260), (1, 3, 37, 1216)]     # the seam shapes of the dilated and the dynamic op
DIL_N = {3: 3, 5: 2, 7: 2}                          # steps of the dyadic cases of both: every intermediate stays exact
AGG_SEAMS = [(2, 2, 37, 200), (1, 1, 45, 1216)]
AGG_STEPS = [(1, 2, 5), tuple(range(1, 71))]        # T = 70: two launch groups of the step-weight gradient
NL_LARGE_K, NL_LARGE_N = 7, 2
NL_HOT = (1, 2, 64, 96)
NL_HOT_POINT = (10.25, 20.5)
DYN_WRAP_SHAPE, DYN_WRAP_K = (1, 2, 17, 132), 5
DYN_WRAP_N = (63, 64, 65, 70, 129)                  # one short of the 64 attention slices, one step each, then wrapping
DYN_TIMING = [(3, 6), (5, 6), (7, 6), (5, 24)]      # (K, N) at TIMING


def ceil_div(a, b):
    return -(-a // b)


def _constants(name, keys):
    with open(os.path.join(CSRC, name)) as f:
        src = f.read()
    out = {}
    for k in keys:
        m = re.search(r'constexpr int [^;]*\b' + k + r'\s*=\s*(\d+)', src)
        assert m, (name, k)
        out[k] = int(m.group(1))
    return out, src


def dilated_tiles():
    c, _ = _constants('cspn2d_dilated.cu', ('kTX', 'kTY', 'kRows'))
    th = c['kTY'] * c['kRows']
    # (tile width, tile height) of the 4-pixel step, the 1-pixel step and the adjoint (always 1 pixel per thread)
    return {'vec': (4 * c['kTX'], th), 'scalar': (c['kTX'], th), 'adjoint': (c['kTX'], th)}


def dynamic_tiles():
    """(tiles as dilated_tiles gives them, finalize threads per block, attention slices) of cspn2d_dynamic.cu."""
    c, _ = _constants('cspn2d_dynamic.cu', ('kTX', 'kTY', 'kRows', 'kFinThreads', 'kAttSlices'))
    th = c['kTY'] * c['kRows']
    return {'vec': (4 * c['kTX'], th), 'scalar': (c['kTX'], th), 'adjoint': (c['kTX'], th)}, c['kFinThreads'], c['kAttSlices']


def attention_slices(N, slices):
    """The steps each grid slice of the dynamic finalize forms grad_attention for: min(N, slices) slices, slice z taking
    steps z, z + min(N, slices), ..."""
    n = min(N, slices)
    return [list(range(z, N, n)) for z in range(n)]


def wide_tiles():
    c, _ = _constants('cspn2d_wide.cu', ('kVecTW', 'kVecTH', 'kSclTW', 'kSclTH', 'kAggStepsPerLaunch'))
    return {'vec': (c['kVecTW'], c['kVecTH']), 'scalar': (c['kSclTW'], c['kSclTH'])}, c['kAggStepsPerLaunch']


def nonlocal_grid():
    """(threads per block, block cap) of nl_entries_kernel's grid-stride launch."""
    c, src = _constants('cspn2d_nonlocal.cu', ('kThreads',))
    m = re.search(r'nl_entries_kernel<K><<<\(unsigned\)min\(ceil_div\(n, kThreads\), 1ll << (\d+)\)', src)
    assert m, 'the launch of nl_entries_kernel'
    return c['kThreads'], 1 << int(m.group(1))


def key_bits(sentinel):
    """cspn2d_nonlocal.cu's key_bits: the radix sort's key width for buckets 0 .. sentinel."""
    bits = 1
    while bits < 32 and (sentinel >> bits) != 0:
        bits += 1
    return bits


def nl_samples(B, H, W, K):
    return B * H * W * (K * K - 1)


# ---- inputs -----------------------------------------------------------------------------------------------------------------
def dilated_dyadic(B, C, H, W, K, samples, seed):
    """Weights in {0, +-1/4, +-1/2, +-1}, integer blur, samples and grad_out, confidences in {0, 1/2, 1}: every
    intermediate of DIL_N[K] steps is exact in fp32.  ([kernel, blur, sparse, conf], grad_out) on the CPU."""
    g = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, 0.0, 0.0, 0.25, -0.25, 0.5, -0.5, 1.0, -1.0])
    kernel = vals[torch.randint(0, 9, (B, K * K, H, W), generator=g)]
    blur = torch.randint(-4, 5, (B, C, H, W), generator=g).float()
    sparse = conf = None
    if samples:
        sparse = torch.randint(0, 5, (B, 1, H, W), generator=g).float()
        conf = torch.tensor([0.0, 0.5, 1.0])[torch.randint(0, 3, (B, 1, H, W), generator=g)]
    go = torch.randint(-2, 3, (B, C, H, W), generator=g).float()
    return [kernel, blur, sparse, conf], go


def dil_seed(shape, K, dil, samples):
    return shape[3] + 10 * K + dil + (100 if samples else 0)


def nonlocal_exact(B, C, H, W, K, seed):
    """Integer offsets in [-12, 12], affinities in {0, +-1/4, +-1/2}, integer feat, samples and grad_out: every bilinear
    weight is 0 or 1 and every intermediate of N = 2 steps is exact in fp32.  (feat, offset, affinity, sparse, grad_out)."""
    g = torch.Generator().manual_seed(seed)
    T = K * K - 1
    feat = torch.randint(-8, 9, (B, C, H, W), generator=g).float()
    offset = torch.randint(-12, 13, (B, 2 * T, H, W), generator=g).float()
    affinity = torch.tensor([0.0, 0.25, -0.25, 0.5, -0.5])[torch.randint(0, 5, (B, T, H, W), generator=g)]
    sparse = torch.where(torch.rand(B, C, H, W, generator=g) < 0.3, torch.randint(1, 9, (B, C, H, W), generator=g).float(),
                         torch.zeros(()))
    go = torch.randint(-4, 5, (B, C, H, W), generator=g).float()
    return feat, offset, affinity, sparse, go


def dyn_seed(shape, K, samples):
    return shape[3] + 10 * K + (100 if samples else 0)


def nl_seed(b):
    """The seed of image b of the large exact case: images are drawn one at a time, so any one is cheap to rebuild."""
    return 700 + b


def hot_offsets(B, H, W, K, outside_half=False):
    """Offsets that send every sample (p, k) to NL_HOT_POINT; with outside_half, the samples of odd pixels to y = -5,
    outside the window (their keys are the sentinel)."""
    T = K * K - 1
    py = torch.arange(H, dtype=torch.float32).view(H, 1).expand(H, W)
    px = torch.arange(W, dtype=torch.float32).view(1, W).expand(H, W)
    off = torch.empty(B, 2 * T, H, W)
    odd = ((py * W + px) % 2 == 1)
    for k, (di, dj) in enumerate(nr.taps(K)):
        ty = torch.where(odd, torch.full_like(py, -5.0), torch.full_like(py, NL_HOT_POINT[0])) if outside_half else NL_HOT_POINT[0]
        off[:, 2 * k] = ty - (py + di)
        off[:, 2 * k + 1] = NL_HOT_POINT[1] - (px + dj)
    return off


# ---- the tiles and what the shapes cross --------------------------------------------------------------------------------
def test_tile_constants_are_the_ones_the_shapes_were_chosen_for():
    assert dilated_tiles() == {'vec': (128, 16), 'scalar': (32, 16), 'adjoint': (32, 16)}
    assert wide_tiles() == ({'vec': (64, 16), 'scalar': (32, 8)}, 64)
    assert nonlocal_grid() == (128, 1 << 20)
    assert dynamic_tiles() == ({'vec': (128, 16), 'scalar': (32, 16), 'adjoint': (32, 16)}, 128, 64)


def crossings(extent, tile):
    """(tiles, pixels in the last tile)"""
    return ceil_div(extent, tile), extent - (ceil_div(extent, tile) - 1) * tile


def seam_tiles():
    """The dilated and the dynamic op's tiles: both run their seam cases on DIL_SEAMS."""
    return {'dilated': dilated_tiles(), 'dynamic': dynamic_tiles()[0]}


@pytest.mark.parametrize('shape', DIL_SEAMS)
def test_dilated_seam_shapes_cross_three_partial_tiles(shape):
    _, _, H, W = shape
    for op, tiles in seam_tiles().items():
        for path, (tw, th) in tiles.items():
            nx, _ = crossings(W, tw)
            ny, last_y = crossings(H, th)
            assert nx >= 3 and ny >= 3, (op, path, nx, ny)
            assert 0 < last_y < th, (op, path)                         # the last row tile is partial
        nx, last_x = crossings(W, tiles['vec'][0])
        assert 0 < last_x < tiles['vec'][0], op                        # and so is the last 4-pixel tile in x


def test_dilated_seam_shapes_partial_in_x_on_every_path():
    for op, tiles in seam_tiles().items():
        for path, (tw, _) in tiles.items():
            assert any(0 < crossings(W, tw)[1] < tw for _, _, _, W in DIL_SEAMS), (op, path)


def test_dynamic_shapes_leave_a_partial_finalize_block():
    """The finalize runs ceil(H*W / kFinThreads) blocks per image; at the seam, slice-wrap and degenerate shapes the last
    one is partial, so a block count one short leaves pixels unwritten there."""
    _, threads, _ = dynamic_tiles()
    for _, _, H, W in DIL_SEAMS + [DYN_WRAP_SHAPE]:
        assert (H * W) % threads != 0, (H, W)
    assert ceil_div(DYN_WRAP_SHAPE[2] * DYN_WRAP_SHAPE[3], threads) == 18
    tiles = dynamic_tiles()[0]
    _, _, H, W = DYN_WRAP_SHAPE
    assert crossings(W, tiles['vec'][0])[0] == 2 and crossings(H, tiles['vec'][1])[0] == 2   # and a seam in x and y


def test_dynamic_slice_wrap_step_counts():
    """N = 63 uses 63 of the 64 attention slices, N = 64 all of them with one step each; from N = 65 on slice 0 takes
    step 64 on a second pass, at N = 70 slices 0-5 do, and at N = 129 slice 0 takes steps 0, 64 and 128."""
    _, _, slices = dynamic_tiles()
    plan = {N: attention_slices(N, slices) for N in DYN_WRAP_N}
    for N, p in plan.items():
        assert sorted(t for steps in p for t in steps) == list(range(N)), N    # every step once
    assert len(plan[63]) == 63 and all(len(x) == 1 for x in plan[63])
    assert len(plan[64]) == 64 and all(len(x) == 1 for x in plan[64])
    assert plan[65][0] == [0, 64] and all(len(x) == 1 for x in plan[65][1:])
    assert [z for z, x in enumerate(plan[70]) if len(x) == 2] == list(range(6)) and max(map(len, plan[70])) == 2
    assert plan[129][0] == [0, 64, 128] and plan[129][1] == [1, 65] and plan[129][63] == [63, 127]


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('dil', [1, 2, 3, 4])
@pytest.mark.parametrize('shape', DIL_SEAMS)
def test_dilated_halos_reach_into_the_neighbouring_tile(K, dil, shape):
    """At every seam of every path, the d*R halo on each side lies in the image and in the neighbouring tile only."""
    _, _, H, W = shape
    h = dil * (K - 1) // 2
    for path, (tw, th) in dilated_tiles().items():
        assert 0 < h <= min(tw, th), path
        for extent, t in ((W, tw), (H, th)):
            seams = range(t, extent, t)
            assert len(seams) >= 2 and all(s - h >= 0 for s in seams) and seams[0] + h <= extent, (path, extent)


@pytest.mark.parametrize('shape', AGG_SEAMS)
def test_aggregate_seam_shapes_cross_three_tiles(shape):
    _, _, H, W = shape
    tiles, _ = wide_tiles()
    for path, (tw, th) in tiles.items():
        nx, _ = crossings(W, tw)
        ny, last_y = crossings(H, th)
        assert nx >= 3 and ny >= 3, (path, nx, ny)
        assert 0 < last_y < th, path
    for path, (tw, _) in tiles.items():
        assert any(0 < crossings(W, tw)[1] < tw for _, _, _, W in AGG_SEAMS), path
    assert crossings(200, tiles['vec'][0]) == (4, 8)


def test_aggregate_step_sets_take_more_than_one_launch_group():
    _, per_launch = wide_tiles()
    assert max(len(s) for s in AGG_STEPS) > per_launch
    assert ceil_div(len(AGG_STEPS[1]), per_launch) == 2


def test_nonlocal_large_case_takes_a_second_grid_stride_pass_and_a_wide_key():
    threads, cap = nonlocal_grid()
    B, _, H, W = TIMING
    n = nl_samples(B, H, W, NL_LARGE_K)
    assert n == 164_364_288
    assert n > threads * cap == 1 << 27                             # the second pass of nl_entries_kernel runs
    assert nl_samples(1, H, W, NL_LARGE_K) <= threads * cap          # the one-image calls of the batch split do not
    assert key_bits(B * (H + 1) * (W + 1)) == 22 > 16
    assert n < 1 << 31                                              # and the call is within the op's limits


def test_hot_bucket_sends_every_sample_to_one_point():
    B, _, H, W = NL_HOT
    K = 3
    for outside_half in (False, True):
        off = hot_offsets(B, H, W, K, outside_half)
        hit = 0
        for k, (di, dj) in enumerate(nr.taps(K)):
            py = torch.arange(H, dtype=torch.float32).view(H, 1) + di
            px = torch.arange(W, dtype=torch.float32).view(1, W) + dj
            y, x = py + off[:, 2 * k], px + off[:, 2 * k + 1]          # the kernels' fp32 sums, exact
            at = (y == NL_HOT_POINT[0]) & (x == NL_HOT_POINT[1])
            assert bool((at | (y <= -1)).all())
            hit += int(at.sum())
        assert hit == (B * H * W * (K * K - 1)) // (2 if outside_half else 1)
    assert B * H * W * (K * K - 1) == 49_152


# ---- exactness premises -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('dil', [1, 2, 3, 4])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('shape', DIL_SEAMS)
def test_dilated_dyadic_cases_are_exact_at_the_seam_shapes(K, dil, samples, shape):
    """The fp32 explicit restatement gives the fp64 composition's bits: every intermediate is exact, so fp32 in any
    order gives fp64's values."""
    ins, go = dilated_dyadic(*shape, K, samples, dil_seed(shape, K, dil, samples))
    ref = dr.grads(dr.composition, *ins, K, dil, DIL_N[K], go, dtype=torch.float64)
    r32 = dr.grads(dr.explicit, *ins, K, dil, DIL_N[K], go)
    for name, x, y in zip(('out', 'kernel', 'blur', 'sparse', 'conf'), r32, ref):
        assert (x is None) == (y is None), name
        assert x is None or torch.equal(x, y.float()), name


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('samples', [None, 'soft'])
@pytest.mark.parametrize('shape', DIL_SEAMS)
def test_dynamic_dyadic_cases_are_exact_at_the_seam_shapes(K, samples, shape):
    """The kernel-order restatement gives the fp64 composition's values on the dyadic cases, output and every gradient:
    every intermediate is exact, so the GPU file may compare the library with fp64 bit for bit there."""
    ins, go = yr.dyadic_inputs(*shape, K, DIL_N[K], samples, dyn_seed(shape, K, samples))
    ref = yr.grads(yr.composition, *ins, K, go, dtype=torch.float64)
    for name, x, y in zip(('out', 'affinity', 'attention', 'blur', 'sparse', 'conf'), yr.kernel_order(*ins, K, go), ref):
        assert (x is None) == (y is None), name
        assert x is None or torch.equal(x, y.float()), name


@pytest.mark.parametrize('b', [0, TIMING[0] - 1])
def test_nonlocal_integer_offset_case_is_exact_at_the_timing_shape(b):
    """Image b of the large exact case: the fp32 restatement gives the fp64 one's bits, output and every gradient.  The
    first and the last image here (the last one's entries are the ones the second grid-stride pass handles); the GPU file
    checks the same premise on every image before it compares."""
    _, C, H, W = TIMING
    f, o, a, s, go = nonlocal_exact(1, C, H, W, NL_LARGE_K, seed=nl_seed(b))
    r32 = nr.grads(nr.propagate, f, o, a, s, NL_LARGE_K, NL_LARGE_N, go)
    ref = nr.grads(nr.propagate, f, o, a, s, NL_LARGE_K, NL_LARGE_N, go, dtype=torch.float64)
    for name, x, y in zip(('out', 'feat', 'offset', 'affinity', 'sparse'), r32, ref):
        assert torch.equal(x, y.float()), name
