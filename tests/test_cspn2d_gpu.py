"""GPU parity tests of the 2D path, through the C ABI (cspn_b200._lib -> libcspn_b200.so).

Tolerance (BASELINE.md section 4, SURVEY.md 7.3-6): |a-b| <= 1e-4 * (|b| + mean|b|) elementwise -- the
north_star's "1e-4 relative fp32", made well-posed for '8sum' outputs that cross zero -- and NaNs
must coincide.  In practice the kernels sit ~1e-6 normwise from the oracle.
"""
import numpy as np
import pytest
import torch

import cspn_b200
from conftest import golden_names, load_golden
from cspn_b200 import _lib
from cspn_b200.synth import make_inputs
from forced_plans import SPECIAL
from oracle import c_oracle, cspn_numpy as onp

pytestmark = pytest.mark.gpu

ALGOS = [_lib.ALGO_GENERIC, _lib.ALGO_CLUSTER]
RTOL = 1e-4


def cluster_accepts(W):
    """The one shape restriction of the cluster kernel (DESIGN.md 4.1): TMA row pitch / float4 accesses need W % 4 == 0."""
    return W % 4 == 0


def run(g, d, s, n, norm, algo):
    """numpy/torch CPU inputs -> GPU -> numpy.  A shape the cluster kernel cannot take must be REFUSED loudly
    (CspnError 'unsupported'), never computed some other way: that is asserted here, and None is returned for it."""
    t = lambda a: None if a is None else torch.as_tensor(a).cuda()
    W = np.shape(g)[-1]
    if algo == _lib.ALGO_CLUSTER and not cluster_accepts(W):
        with pytest.raises(cspn_b200.CspnError, match='unsupported'):
            cspn_b200.propagate2d(t(g), t(d), t(s), n, norm, algo)
        return None
    out = cspn_b200.propagate2d(t(g), t(d), t(s), n, norm, algo)
    torch.cuda.synchronize()
    if algo == _lib.ALGO_CLUSTER:
        assert _lib.ALGO_NAMES[_lib.lib().cspn_last_algo()] == 'cluster'
    return out.cpu().numpy()


def assert_parity(out, ref, what=''):
    ok, ratio, normwise = onp.parity_ok(out, ref, RTOL)
    assert ok, f'{what}: violation ratio {ratio:.3g}, normwise {normwise:.3g}'
    return ratio, normwise


@pytest.mark.parametrize('algo', ALGOS)
@pytest.mark.parametrize('name', golden_names())
def test_golden_vectors_from_reference(name, algo):
    c = load_golden(name)
    out = run(c['guidance'], c['blur'], c['sparse_depth'], c['prop_time'], c['norm_type'], algo)
    if out is not None:          # None: the cluster kernel refused an odd-W shape (asserted inside run)
        assert_parity(out, c['out'], name)


@pytest.mark.parametrize('algo', ALGOS)
@pytest.mark.parametrize('norm', ['8sum', '8sum_abs'])
@pytest.mark.parametrize('shape,n', [((2, 1, 100, 160), 24), ((1, 2, 37, 64), 9), ((3, 1, 64, 128), 16),
                                      ((1, 1, 352, 1216), 24), ((2, 1, 228, 304), 48), ((1, 1, 228, 304), 4),
                                      ((1, 1, 228, 912), 24), ((5, 1, 16, 16), 3)])
def test_against_c_oracle(shape, n, norm, algo):
    B, C, H, W = shape
    g, d, s = make_inputs(1000 + H + W + n, B, C, H, W, 8, 'signed', 500)
    ref = c_oracle.cspn2d(g.numpy(), d.numpy(), s.numpy(), n, norm)
    out = run(g, d, s, n, norm, algo)
    assert out is not None
    assert_parity(out, ref, f'{shape} n={n} {norm}')


@pytest.mark.parametrize('algo', ALGOS)
@pytest.mark.parametrize('n', [4, 8, 16, 24, 48])
def test_cfg3_iteration_sweep_against_c_oracle(n, algo):
    """BASELINE configs[2]: every point of the {4,8,16,24,48} sweep at the NYU shape, both paths, against the oracle."""
    g, d, s = make_inputs(2000 + n, 2, 1, 228, 304)
    ref = c_oracle.cspn2d(g.numpy(), d.numpy(), s.numpy(), n, '8sum')
    assert_parity(run(g, d, s, n, '8sum', algo), ref, f'228x304 n={n}')


@pytest.mark.parametrize('algo', ALGOS)
def test_edge_shapes_and_layouts(algo):
    # ragged / degenerate shapes, extra guidance channels, non-contiguous inputs, no sparse
    for (B, C, H, W, gch) in [(1, 1, 1, 1, 8), (1, 1, 1, 40, 8), (1, 1, 40, 1, 8), (2, 3, 5, 7, 11), (1, 1, 3, 4, 8),
                              (1, 1, 33, 36, 8)]:
        g, d, s = make_inputs(7 + H * W, B, C, H, W, gch, 'bernoulli', 5)
        for sp in (s, None):
            ref = onp.cspn2d(g.numpy(), d.numpy(), None if sp is None else sp.numpy(), 6, '8sum')
            out = run(g, d, sp, 6, '8sum', algo)
            if out is not None:
                assert_parity(out, ref, f'{(B, C, H, W, gch)}')
    g, d, s = make_inputs(3, 2, 1, 24, 32, 8, 'bernoulli', 20)
    gn = torch.randn(2, 24, 32, 8).permute(0, 3, 1, 2)            # channels-last view: non-contiguous
    gn.copy_(g)
    assert not gn.is_contiguous()
    ref = onp.cspn2d(g.numpy(), d.numpy(), s.numpy(), 5, '8sum_abs')
    out = cspn_b200.propagate2d(gn.cuda(), d.cuda(), s.cuda(), 5, '8sum_abs', algo)
    assert_parity(out.cpu().numpy(), ref, 'non-contiguous guidance')


@pytest.mark.parametrize('algo', ALGOS)
def test_nan_semantics_match_reference(algo):
    c = load_golden('zero_guidance_nan')                         # 0/0 affinities -> NaN (cspn.py:138); W=5: generic only
    out = run(c['guidance'], c['blur'], None, c['prop_time'], c['norm_type'], algo)
    assert out is None or np.isnan(out).all()
    c = load_golden('nan_zero_guidance_4x8')                     # the same on a shape the cluster kernel takes
    out = run(c['guidance'], c['blur'], None, c['prop_time'], c['norm_type'], algo)
    assert np.isnan(out).all()
    # a single all-zero-affinity pixel poisons exactly what the reference poisons
    g, d, s = make_inputs(5, 1, 1, 12, 16, 8, 'bernoulli', 10)
    g[0, :, 3:8, 4:9] = 0
    ref = onp.cspn2d(g.numpy(), d.numpy(), s.numpy(), 3, '8sum')
    assert np.isnan(ref).any() and not np.isnan(ref).all()
    assert_parity(run(g, d, s, 3, '8sum', algo), ref, 'partial NaN')


@pytest.mark.parametrize('algo', ALGOS)
def test_nan_sparse_pixel_masks_nothing(algo):
    """torch.sign(NaN) is 0 on CUDA as on the CPU (the reference's mask, cspn.py:64): a NaN sparse pixel is not a sparse
    pixel, and both algorithms agree with the torch port there."""
    from oracle import cspn_torch_port as tp
    assert torch.sign(torch.tensor([float('nan')], device='cuda')).item() == 0
    g, d, s = make_inputs(5, 1, 1, 12, 16, 8, 'bernoulli', 10)
    s[0, 0, 6, 7] = float('nan')
    ref = tp.cspn2d_torch(g, d, s, 3, '8sum').numpy()
    out = run(g, d, s, 3, '8sum', algo)
    assert not np.isnan(out).any()
    assert_parity(out, ref, 'NaN sparse pixel')


@pytest.mark.parametrize('algo', ALGOS)
@pytest.mark.parametrize('name', SPECIAL)
def test_non_finite_and_degenerate_affinities_match_reference(name, algo):
    """Goldens from the unmodified reference for 0/0, a NaN source whose front moves one pixel per step (also next to a
    strip cut and in the image corner), subnormal and near-overflow sums of |affinity| and +-inf guidance: the NaN
    pattern must coincide and finite values agree (cspn.py:135-138; the cluster prologue's reciprocal has an IEEE
    division fallback for exactly these inputs)."""
    c = load_golden(name)
    out = run(c['guidance'], c['blur'], c['sparse_depth'], c['prop_time'], c['norm_type'], algo)
    assert out is not None, 'every special case has W % 4 == 0: the cluster kernel must run it'
    assert np.array_equal(np.isnan(out), np.isnan(c['out'])), name
    assert np.array_equal(np.isinf(out), np.isinf(c['out'])), name
    assert_parity(out, c['out'], name)


def test_inputs_not_mutated_and_fresh_output():
    g, d, s = [t.cuda() for t in make_inputs(9, 2, 1, 20, 24, 8, 'bernoulli', 10)]
    g0, d0, s0 = g.clone(), d.clone(), s.clone()
    out = cspn_b200.Affinity_Propagate(4, 3)(g, d, s)
    assert out.data_ptr() != d.data_ptr() and out.shape == d.shape and out.dtype == d.dtype and out.device == d.device
    assert torch.equal(g, g0) and torch.equal(d, d0) and torch.equal(s, s0)


def test_sparse_pixels_return_blur_depth_exactly():
    g, d, s = [t.cuda() for t in make_inputs(11, 2, 1, 60, 80, 8, 'bernoulli', 300)]
    out = cspn_b200.propagate2d(g, d, s, 24, '8sum')
    mask = s > 0
    assert mask.any() and torch.equal(out[mask], d[mask])        # cspn.py:81 with m == 1


# ---- BASELINE.json full sizes: size-independent properties (the oracle would take minutes) --------

FULL = [pytest.param((32, 1, 352, 1216), 24, id='cfg2_kitti'), pytest.param((64, 1, 228, 304), 24, id='cfg3_nyu')]


@pytest.mark.parametrize('shape,n', FULL)
@pytest.mark.parametrize('algo', ALGOS)
def test_full_size_properties(shape, n, algo):
    B, C, H, W = shape
    g, d, s = [t.cuda() for t in make_inputs(42, B, C, H, W)]
    f = lambda dd, ss, norm: cspn_b200.propagate2d(g, dd, ss, n, norm, algo)
    out = f(d, s, '8sum')
    assert torch.isfinite(out).all()
    # (1) the map blur_depth -> out is linear (d_N = L(d_0): kappa*d0 + sum w' shift(d))
    d2 = torch.rand_like(d) * 10
    lhs = f(0.25 * d + 2.0 * d2, s, '8sum')
    rhs = 0.25 * out + 2.0 * f(d2, s, '8sum')
    scale = rhs.abs().mean()
    assert ((lhs - rhs).abs() <= 1e-4 * (rhs.abs() + scale)).all()
    # (2) '8sum_abs' weights sum to one over the in-image neighbours: constants are fixed points
    const = torch.full_like(d, 3.5)
    assert torch.allclose(f(const, None, '8sum_abs'), const, rtol=1e-5, atol=0)
    # (3) sparse pixels come back as the blur depth, bit-exact
    m = s > 0
    assert torch.equal(out[m], d[m])
    # (4) images are independent: a slice of the batch gives the same bits as the full batch
    sub = cspn_b200.propagate2d(g[3:5], d[3:5], s[3:5], n, '8sum', algo)
    assert torch.equal(sub, out[3:5])
    # (5) one image of the batch against the C oracle
    ref = c_oracle.cspn2d(g[7:8].cpu().numpy(), d[7:8].cpu().numpy(), s[7:8].cpu().numpy(), n, '8sum')
    ok, ratio, normwise = onp.parity_ok(out[7:8].cpu().numpy(), ref, RTOL)
    assert ok, (ratio, normwise)


def test_cluster_and_generic_agree_at_full_size():
    g, d, s = [t.cuda() for t in make_inputs(43, 8, 1, 352, 1216)]
    a = cspn_b200.propagate2d(g, d, s, 24, '8sum', _lib.ALGO_GENERIC)
    b = cspn_b200.propagate2d(g, d, s, 24, '8sum', _lib.ALGO_CLUSTER)
    ok, ratio, normwise = onp.parity_ok(b.cpu().numpy(), a.cpu().numpy(), RTOL)
    assert ok and normwise < 1e-5, (ratio, normwise)


def test_host_buffer_entry_point_matches_device_entry_point():
    g, d, s = make_inputs(17, 7, 1, 228, 304)
    out_host = cspn_b200.propagate2d(g.pin_memory(), d.pin_memory(), s.pin_memory(), 24, '8sum')      # CPU tensors -> *_host
    assert not out_host.is_cuda
    out_dev = cspn_b200.propagate2d(g.cuda(), d.cuda(), s.cuda(), 24, '8sum').cpu()
    assert torch.equal(out_host, out_dev)
    g12 = torch.cat([g, torch.randn(7, 4, 228, 304)], 1)                                              # gch=12, pageable
    assert torch.equal(cspn_b200.propagate2d(g12, d, s, 24, '8sum'), out_dev)


def test_runs_on_the_callers_stream():
    g, d, s = [t.cuda() for t in make_inputs(19, 4, 1, 96, 128)]
    ref = cspn_b200.propagate2d(g, d, s, 8, '8sum')
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        d2 = d * 2                                  # produced on `st`; the op must be ordered after it
        out = cspn_b200.propagate2d(g, d2, s, 8, '8sum')
    st.synchronize()
    assert torch.allclose(out, 2 * ref, rtol=1e-5, atol=1e-5)


def test_errors_are_loud():
    g, d, _ = [None if t is None else t.cuda() for t in make_inputs(1, 1, 1, 8, 8, 8, None)]
    L = _lib.lib()
    out = torch.empty_like(d)
    rc = L.cspn2d_fwd_f32(g.data_ptr(), d.data_ptr(), None, out.data_ptr(), 1, 1, 8, 8, 8, 4, 0, _lib.ALGO_GENERIC,
                          None, 0, None)
    assert rc == -2 and b'workspace' in L.cspn_last_error()
