"""Inputs on which the 3x3 2D propagation stays exact at any step count, the explicit fp64 reference they are checked
against, and the case matrix of tests/test_cluster_exact_gpu.py (tests/test_cluster_exact_cpu.py checks its premises
without a GPU).

Why bits.  A strip overlaps its neighbours by a halo of `iters` columns and the stale region creeps inwards one column
per step; row bands, chained strips (one recorded column handed over per step) and persistent clusters (staging buffers
and mbarrier phases reused from task to task) have the same kind of bookkeeping.  Under random gates an off-by-one in it
reaches a stored pixel only along a path of about N hops of weight ~3/8 each, far below any tolerance at N = 24.  On the
inputs below every value is a short dyadic rational, so any correct fp32 implementation returns the bits of the fp64
reference, and a stale value is a wrong number:
  directed   item k of every 8 has tap k hot (+-1) at every site, reflected into the image at the border
             (be.one_tap_guidance): S = 1, and each step is an integer shift, plus 0 or 2 x blur.  Values are integers
             that grow at most linearly with N; the stale front moves one column (row) per step with weight 1;
  mixed      m in {1, 2} hot taps per site, gates +-1, so w = +-1 or +-1/2 (be.dyadic_guidance): the multi-tap
             arithmetic and the S computation, at the forced-plan matrix's own step counts (n <= 15).
blur and grad_out are integers in [-4, 4]; sparse_depth is 0 but at one pixel in 20, where it is 3 ('bernoulli') or +-3
('signed').  Where sparse_depth is negative (m = -1) a value doubles at every visit, so 'signed' runs at n <= 3 only.
Under '8sum_abs' one hot tap has w = 1 whatever its value, so the directed taps' guidance gradient is identically 0: every
directed case with a backward runs '8sum', and '8sum_abs' is checked backward on the mixed taps.  be.check_exact asserts
of every reference tensor that it lies on the grid of `unit` and far inside 24 bits.
"""
import math
from collections import namedtuple

import torch

from cspn_b200 import _lib
from oracle.cspn_numpy_k import offsets_2d

import backward_exact as be
import forced_plans as fpl

OFFS = offsets_2d(3)          # the tap order of the guidance channels, as in be.cspn2d_shift_ref
FAMILIES = ('directed', 'mixed')


# ---- the explicit fp64 reference --------------------------------------------------------------------------------------
def _neg(o):
    return tuple(-c for c in o)


def gates(g, norm):
    """(a, w, S, s): the gathered gates a_k(p) = g'_k(p + off_k) (g' = |g| for '8sum_abs'), S = sum |a|, w = a / S and
    s = sum w, each (B, 8 or 1, H, W)."""
    gn = g[:, :8].abs() if norm == '8sum_abs' else g[:, :8]
    a = torch.stack([be.shift(gn[:, k], o, 1) for k, o in enumerate(OFFS)], 1)
    S = a.abs().sum(1, keepdim=True)
    w = a / S
    return a, w, S, w.sum(1, keepdim=True)


def reference(g, blur, sparse, N, norm, grad_out=None):
    """be.cspn2d_shift_ref (K = 3) with its adjoint written out: the forward keeps its N + 1 iterates, the adjoint walks
    them back, so memory is (N + 1) images instead of autograd's ~8 saved tensors per step.  Runs in the dtype and on the
    device of its inputs.  Returns `out`, or with grad_out (out, grad_guidance, grad_blur).

        d_0 = blur,  e_{t+1} = (1 - s) blur + sum_k w_k shift(d_t, off_k),  d_{t+1} = (1 - m) e_{t+1} + m blur
    with m = sign(sparse).  The transpose of b(p) = a(p + off) (zero outside) is shift(b, -off)."""
    a, w, S, s = gates(g, norm)
    m = None if sparse is None else sparse.sign()
    ds = [blur]
    for _ in range(N):
        acc = 0
        for k, o in enumerate(OFFS):
            acc = acc + w[:, k:k + 1] * be.shift(ds[-1], o, 1)
        e = (1.0 - s) * blur + acc
        ds.append(e if m is None else (1 - m) * e + m * blur)
    if grad_out is None:
        return ds[-1]
    out = ds[-1]
    lam = grad_out                      # lambda_{t+1} = dL/dd_{t+1}
    gw = torch.zeros_like(w)            # dL/dw_k, summed over steps and channels (s = sum w folded in below)
    gs = torch.zeros_like(s)
    gblur = torch.zeros_like(blur)
    for t in range(N - 1, -1, -1):
        ds.pop()
        mu = lam if m is None else (1 - m) * lam             # dL/de_{t+1}
        if m is not None:
            gblur = gblur + m * lam
        gblur = gblur + (1.0 - s) * mu
        gs = gs - (mu * blur).sum(1, keepdim=True)
        for k, o in enumerate(OFFS):
            gw[:, k] += (mu * be.shift(ds[t], o, 1)).sum(1)
        nxt = 0
        for k, o in enumerate(OFFS):
            nxt = nxt + be.shift(w[:, k:k + 1] * mu, _neg(o), 1)
        lam = nxt
    gblur = gblur + lam                 # d_0 = blur
    gw = gw + gs
    # w_j = a_j / S, S = sum |a|:  dL/da_j = (gw_j - sign(a_j) sum_k gw_k w_k) / S   (abs' subgradient at 0 is 0)
    ga = (gw - a.sign() * (gw * w).sum(1, keepdim=True)) / S
    gn = torch.stack([be.shift(ga[:, k], _neg(o), 1) for k, o in enumerate(OFFS)], 1)
    gg = torch.zeros_like(g)
    gg[:, :8] = gn * g[:, :8].sign() if norm == '8sum_abs' else gn
    return out, gg, gblur


# ---- inputs -----------------------------------------------------------------------------------------------------------
def sparse_points(gen, B, H, W, mode):
    if mode is None:
        return None
    hot = (torch.rand(B, 1, H, W, generator=gen) < 0.05).float()
    return 3 * hot * (be.signs(gen, (B, 1, H, W)) if mode == 'signed' else 1)


def _extra(gen, g, gch):
    B, _, H, W = g.shape
    return torch.cat([g, be.small_ints(gen, (B, gch - 8, H, W))], 1) if gch > 8 else g


def directed(seed, B, C, H, W, gch=8, sparse=None):
    """(guidance, blur, sparse, grad_out): image b has tap b % 8 hot at every site (reflected at the border), signs drawn
    afresh for every 8 images."""
    g = torch.cat([be.one_tap_guidance(seed * 97 + i, (H, W), 3, True) for i in range(math.ceil(B / 8))])[:B]
    gen = torch.Generator().manual_seed(seed)
    return (_extra(gen, g, gch), be.small_ints(gen, (B, C, H, W)), sparse_points(gen, B, H, W, sparse),
            be.small_ints(gen, (B, C, H, W)))


def mixed(seed, B, C, H, W, gch=8, sparse=None):
    """(guidance, blur, sparse, grad_out): m in {1, 2} hot taps at every site, gates +-1.  grad_out is nonzero at one
    pixel in 4, which keeps the guidance gradient inside 24 bits at n <= 15."""
    gen = torch.Generator().manual_seed(seed)
    g = be.dyadic_guidance(gen, B, (H, W), 3, True, ms=(1, 2))
    go = be.small_ints(gen, (B, C, H, W)) * (torch.rand(B, C, H, W, generator=gen) < 0.25)
    return _extra(gen, g, gch), be.small_ints(gen, (B, C, H, W)), sparse_points(gen, B, H, W, sparse), go


def unit(family, N):
    """The grid every value of the family lies on: integers, or with w = +-1/2 one halving per step, plus one for the
    division by S in the guidance gradient."""
    return 1.0 if family == 'directed' else 2.0 ** -(N + 1)


def make(family, seed, B, C, H, W, gch, sparse):
    return (directed if family == 'directed' else mixed)(seed, B, C, H, W, gch, sparse)


def check_exact(ref, family, N, what):
    for t, name in zip(ref, ('out', 'grad_guidance', 'grad_blur')):
        be.check_exact(t, N, f'{what} {name}', unit(family, N))


# ---- locating a mismatch ----------------------------------------------------------------------------------------------
def locate(info, y, x):
    """Where pixel (y, x) lies in every pass geometry of a plan_info: strip, band, CTA of the cluster, warp, row of the
    warp's PR-row patch, lane and column of the lane's 4; and how far it is from the edges of its useful range."""
    if info is None:
        return 'no cluster plan (generic path)'
    parts = []
    for p in info['passes']:
        i = next(j for j, (_, u0, u1) in enumerate(p['strips']) if u0 <= x < u1)
        j = next(j for j, (_, u0, u1) in enumerate(p['bands']) if u0 <= y < u1)
        (tx0, ux0, ux1), (by0, uy0, uy1) = p['strips'][i], p['bands'][j]
        cta, r = divmod(y - by0, p['RB'])
        warp, row = divmod(r, p['PR'])
        lane, col = divmod(x - tx0, 4)
        parts.append(
            f"[{p['count']} pass(es) of {p['iters']} steps, PR={p['PR']} NW={p['NW']} cs={p['cs']}: "
            f"strip {i} of {len(p['strips'])} (tile x0 {tx0}, useful [{ux0}, {ux1}), {x - ux0} columns from its left edge, "
            f"{ux1 - 1 - x} from its right), band {j} of {len(p['bands'])} (y0 {by0}, useful [{uy0}, {uy1}), "
            f"{y - uy0} rows from its top, {uy1 - 1 - y} from its bottom), CTA {cta}, warp {warp}, patch row {row}, "
            f"lane {lane}, column {col}]")
    return ('chained ' if info.get('chained') else '') + ' '.join(parts)


def assert_exact(ours, ref, info, what):
    """`ours` equals the fp64 reference bit for bit; else the first differing pixel and its plan coordinates."""
    ours = ours.double().cpu()
    ref = ref.double().cpu()
    if torch.equal(ours, ref):
        return
    bad = ours != ref
    idx = tuple(bad.nonzero()[0].tolist())
    raise AssertionError(f'{what}: {int(bad.sum())} of {bad.numel()} differ, first at (b, c, y, x) = {idx}: '
                         f'{float(ours[idx])} instead of {float(ref[idx])}; {locate(info, idx[2], idx[3])}')


# ---- plans ------------------------------------------------------------------------------------------------------------
ENV = ('CSPN_B200_FORCE_CFG', 'CSPN_B200_FORCE_CS', 'CSPN_B200_FORCE_PASSES', 'CSPN_B200_CHAIN', 'CSPN_B200_CHAIN_GROUP',
       'CSPN_B200_BWD')


def env(cfg=None, cs=None, passes=None, chain=None, group=None):
    """Planner settings (None: unset, the planner's own choice)."""
    return dict(zip(ENV, (None if v is None else str(v) for v in (cfg, cs, passes, chain, group, None))))


def describe(e):
    return ' '.join(f'{k[len("CSPN_B200_"):]}={v}' for k, v in e.items() if v is not None) or "the planner's own plan"


def apply(monkeypatch, e):
    for k, v in e.items():
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))


def plan_of(e, B, C, H, W, n):
    """plan_info of the forward plan a call makes under settings `e` (already applied)."""
    chained = e['CSPN_B200_CHAIN'] == '1' or (e['CSPN_B200_CHAIN'] is None and
                                              'chained' in _lib.describe_plan(B, C, H, W, n, _lib.ALGO_CLUSTER))
    return _lib.plan_info(H, W, n, chained)


def rounds(info, B, C):
    """Tasks per co-resident cluster of every pass: the rounds of the persistent loop."""
    return [B * C * len(p['strips']) * len(p['bands']) / p['max_clusters'] for p in info['passes']]


def batch_for_rounds(info, C, want=3):
    """The smallest multiple of 8 images that gives every pass of `info` at least `want` rounds."""
    per_image = min(C * len(p['strips']) * len(p['bands']) / p['max_clusters'] for p in info['passes'])
    return 8 * math.ceil(want / per_image / 8)


# ---- the case matrix --------------------------------------------------------------------------------------------------
# A case: one input set (family, shapes, steps, norm, sparse) run under several planner settings, forward and (bwd) backward.
# `problem`: the forced-plan matrix problem (tests/forced_plans.py) whose plans the case runs, else None.
Case = namedtuple('Case', 'name family B C H W n gch norm sparse envs bwd problem', defaults=(None,))


def forced_case(name, family, n=None):
    """A problem of the forced-plan matrix on exact inputs: its own C, H, W, gch and plans; the directed taps as 8 images,
    with '8sum' where the problem has a backward.  At the problem's own n, 'bernoulli' sparse where the problem's is
    'signed' (which would not stay exact); with `n` given (<= 3), the problem's 'signed' sparse at n steps."""
    pb = fpl.PROBLEMS[name]
    if n is None:
        n, sparse, tag = pb.n, 'bernoulli' if pb.sparse == 'signed' else pb.sparse, ''
    else:
        assert n <= 3 and pb.sparse == 'signed'
        sparse, tag = 'signed', f'-n{n}'
    norm = '8sum' if family == 'directed' and pb.bwd else pb.norm
    return Case(f'{name}{tag}-{family}', family, 8 if family == 'directed' else pb.B, pb.C, pb.H, pb.W, n, pb.gch, norm,
                sparse, None, bool(pb.bwd), name)


# every problem at its own n, and two tall ones (PR = 5 and 2) with 'signed' sparse at n = 3
FORCED = ([forced_case(name, f) for name in sorted(fpl.PROBLEMS) for f in FAMILIES] +
          [forced_case(name, f, 3) for name in ('tall_cfg0', 'tall_cfg3') for f in FAMILIES])


# Long runs: the planner's own plan and 1, 2, 3 and an uneven number of passes (N = 80 needs two: its halo is wider
# than a strip).  516 = 4 * 128 + 4 columns; 1216 is KITTI's width; 700 rows need bands in every configuration.
LONG_PASSES = {24: (1, 2, 3, 5), 48: (1, 2, 3, 5), 80: (2, 3, 7)}
LONG_SHAPES = [('w516', 2, 48, 516, 8, '8sum', None), ('w1216', 1, 40, 1216, 9, '8sum', None),
               ('tall700', 1, 700, 260, 8, '8sum', 'bernoulli')]
LONG = [Case(f'{name}-n{n}', 'directed', 8, C, H, W, n, gch, norm, sparse,
             [env(chain=0)] + [env(passes=p, chain=0) for p in LONG_PASSES[n]], True)
        for name, C, H, W, gch, norm, sparse in LONG_SHAPES for n in (24, 48, 80)]

# Persistent rounds: B is chosen at run time (batch_for_rounds) for >= 3 tasks per co-resident cluster.  Cluster size 1 in
# configuration 0 and in the two-CTAs-per-SM configuration 4 (one CTA tall, so one band), the largest single-band cluster
# (16 CTAs of 40 rows), and KITTI under the planner's own plan.
PERSISTENT = [
    Case('cfg0-cs1', 'directed', None, 1, 40, 516, 24, 8, '8sum', 'bernoulli', [env(0, 1, 1, 0)], True),
    Case('cfg4-cs1', 'directed', None, 1, 20, 516, 24, 9, '8sum', None, [env(4, 1, 1, 0)], True),
    Case('cfg0-cs16', 'directed', None, 1, 16 * 40 - 5, 516, 24, 8, '8sum', None, [env(0, 16, 1, 0)], True),
    Case('kitti', 'directed', None, 1, 352, 1216, 24, 8, '8sum', 'bernoulli', [env()], True),
]

# Chained strips, one band of one to three CTAs: configurations 0-2, one and two passes, chain groups 1, 2, 3 and 0 (all
# image-channels in one group).
CHAIN_GROUPS = (1, 2, 3, 0)
CHAIN = [Case(f'chain-n{n}', 'directed', 8, 2, 64, 1216, n, 8, norm, 'bernoulli',
              [env(ci, math.ceil(64 / fpl.rows(ci)), passes, 1, group)
               for passes in (1, 2) for i, group in enumerate(CHAIN_GROUPS) for ci in [fpl.CHAINED[(i + passes) % 3]]],
              False)
         for n, norm in ((24, '8sum'), (31, '8sum_abs'))]

# The other routes: a long run and a ragged width (W % 4 != 0: the generic kernels); both with a ninth guidance channel
# (the host entry's per-image copy loop) and sparse, and enough images for >= 4 host chunks of 1 MB (about 1 MB per image
# at 48 x 516, 0.2 MB at 37 x 133).
ROUTES = [Case('route-long', 'directed', 8, 1, 48, 516, 48, 9, '8sum', 'bernoulli', [env()], True),
          Case('route-ragged', 'directed', 24, 2, 37, 133, 24, 9, '8sum', 'bernoulli', [env()], True)]


def inputs(case, B=None):
    return make(case.family, case.H * 7 + case.W + case.n, B or case.B, case.C, case.H, case.W, case.gch, case.sparse)
