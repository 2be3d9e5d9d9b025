"""The forced-plan matrix of the 2D cluster kernel, shared by tests/test_forced_plans_gpu.py and
tests/test_cluster_exact_gpu.py (which run it) and tests/test_plan_cpu.py (which checks, without a GPU, that the planner
honours every combination and that together they reach every configuration in every mode), plus what the 2D GPU tests
share: the special-value goldens and the forward and backward called through the C ABI under a forced plan.

Which kernels a call runs normally depends on the card: the planner picks configuration, cluster size, row bands and
passes from cudaOccupancyMaxActiveClusters and the SM count.  CSPN_B200_FORCE_CFG / _FORCE_CS / _FORCE_PASSES and
CSPN_B200_CHAIN (read on every call) pin those choices, so the suite checks every kernel whatever card it runs on.

Bit identity.  A pixel's FMA order depends only on its row inside the thread's PR-row patch and on its column inside the
lane's 4 columns.  Strip origins are multiples of 4, so the column never changes; the row does when a band starts at a
row that is not a multiple of PR.  So all plans of one problem whose band origins agree modulo PR (one band: origin 0)
must give the same bits, whatever their cluster size, strips, pass split, chaining or GENERAL kernel: see `bit_group`.
"""
import math
import warnings
from collections import namedtuple

import pytest
import torch

from cspn_b200 import _lib

import memory_contract as mc

# configs() of cspn_b200/csrc/cspn2d_cluster.cu by index: (PR rows per thread, NW warps); a CTA covers PR*NW rows x 128
CONFIGS = [(5, 8), (4, 8), (3, 8), (2, 8), (5, 4)]
CHAINED = (0, 1, 2)        # the configurations that have chained-strip forward kernels
NORMS = ('8sum', '8sum_abs')
# goldens of the reference module for 0/0, NaN fronts (next to a strip cut, in the image corner), subnormal and near-overflow
# sums of |affinity| and +-inf guidance; every one has W % 4 == 0, so the cluster kernel takes it
SPECIAL = ['nan_zero_guidance_4x8', 'nan_zero_patch_12x16_n1', 'nan_zero_patch_12x16_n2', 'nan_zero_patch_12x16_n3',
           'nan_zero_patch_40x132_n6', 'subnormal_affinity_8x8', 'huge_affinity_8x12', 'inf_guidance_8x12',
           'inf_guidance_abs_8x12']


def rows(ci):
    PR, NW = CONFIGS[ci]
    return PR * NW


# cs: forced cluster size; passes: forced pass count (None: the planner's choice); chain: CSPN_B200_CHAIN=1
Plan = namedtuple('Plan', 'cfg cs passes chain', defaults=(None, False))
Problem = namedtuple('Problem', 'B C H W n gch norm sparse fwd bwd')


def chains(plan):
    """Chaining is requested AND the configuration has chained kernels (otherwise the planner must fall back)."""
    return plan.chain and plan.cfg in CHAINED


def _tall(ci):
    """Just under 16 CTAs tall: cluster size 16 is the largest with one band, smaller clusters need several bands.
    n = 11 splits into 6 + 5 and 4 + 4 + 3 steps."""
    fwd = [Plan(ci, 16, 1), Plan(ci, 16, 2), Plan(ci, 16, 3), Plan(ci, 4, 2), Plan(ci, 1, 3), Plan(ci, 16, 1, True)]
    if ci in CHAINED:
        fwd.append(Plan(ci, 16, 2, True))
    bwd = [Plan(ci, 16, 1), Plan(ci, 16, 3), Plan(ci, 4, 2), Plan(ci, 1, 3)]
    return Problem(1, 1, 16 * rows(ci) - 5, 260, 11, 9, NORMS[ci % 2], 'signed', fwd, bwd)


# steps per pass that put every band origin of a one- or two-CTA cluster on a multiple of PR (2n % PR == 0) while
# leaving a one-CTA band at least 8 useful rows (PR*NW - 2n >= 8): banded plans then join the bit-identity group
ALIGNED_N = {0: 15, 1: 12, 2: 6, 3: 4, 4: 5}


def _short(ci):
    """Three CTAs tall, two strips, two images of two channels: cluster size 1 and 2 with several bands, 3 with one."""
    fwd = [Plan(ci, 1, 1), Plan(ci, 2, 1), Plan(ci, 3, 1), Plan(ci, 3, 2)]
    bwd = [Plan(ci, 1, 1), Plan(ci, 3, 1)]
    if ci == 4:     # 5x4x4 and 5x4x8 share PR = 5: the two warp counts must agree bit for bit
        fwd += [Plan(0, 1, 1), Plan(0, 2, 1)]
        bwd += [Plan(0, 2, 1)]
    return Problem(2, 2, 3 * rows(ci) - 2, 132, ALIGNED_N[ci], 8, NORMS[(ci + 1) % 2], None, fwd, bwd)


def _chain(ci):
    """One CTA tall and five chained strips: cluster size 1, chained and not, in one and two passes.  The norm is the
    other one of _tall's, so that both chained kernels of the configuration (8sum, 8sum_abs) run."""
    fwd = [Plan(ci, 1, 1), Plan(ci, 1, 2), Plan(ci, 1, 1, True), Plan(ci, 1, 2, True)]
    return Problem(3, 1, rows(ci) - 3, 520, 11, 8, NORMS[(ci + 1) % 2], 'bernoulli', fwd, [])


PROBLEMS = {}
for _ci in range(len(CONFIGS)):
    PROBLEMS[f'tall_cfg{_ci}'] = _tall(_ci)
    PROBLEMS[f'short_cfg{_ci}'] = _short(_ci)
    if _ci in CHAINED:
        PROBLEMS[f'chain_cfg{_ci}'] = _chain(_ci)

# the zero-affinity patch of test_cspn2d_gpu.py::test_nan_semantics_match_reference (12x16: one CTA in every configuration)
NAN_PATCH_PLANS = [Plan(ci, 1) for ci in range(len(CONFIGS))]


def special_plans(name, H):
    """Special-value goldens: every configuration at cluster size 1 and at the largest single-band cluster size;
    the golden whose NaN front crosses a strip cut also in two passes."""
    plans = []
    for ci in range(len(CONFIGS)):
        top = min(16, math.ceil(H / rows(ci)))
        plans += [Plan(ci, 1)] + ([Plan(ci, top)] if top > 1 else [])
        if name == 'nan_zero_patch_40x132_n6':
            plans.append(Plan(ci, top, 2))
    return plans


def force(monkeypatch, plan):
    """Pins `plan` for the following calls; the backward takes its default, cluster formulation."""
    monkeypatch.delenv('CSPN_B200_BWD', raising=False)
    monkeypatch.setenv('CSPN_B200_FORCE_CFG', str(plan.cfg))
    monkeypatch.setenv('CSPN_B200_FORCE_CS', str(plan.cs))
    if plan.passes:
        monkeypatch.setenv('CSPN_B200_FORCE_PASSES', str(plan.passes))
    else:
        monkeypatch.delenv('CSPN_B200_FORCE_PASSES', raising=False)
    monkeypatch.setenv('CSPN_B200_CHAIN', '1' if plan.chain else '0')


def plan_info(plan, H, W, n):
    """The plan the library will run for `plan` (call under force()): the chained one when chaining applies."""
    return _lib.plan_info(H, W, n, chains(plan))


def check_honoured(plan, info):
    """The planner gave what was forced: configuration, cluster size in every pass, pass count, chaining.
    Returns the number of launches a forward call makes (one per pass)."""
    assert info['supported'], (plan, info)
    assert info['chained'] == chains(plan), (plan, info)
    for p in info['passes']:
        assert (p['PR'], p['NW']) == CONFIGS[plan.cfg] and p['cs'] == plan.cs, (plan, p)
    n_pass = sum(p['count'] for p in info['passes'])
    if plan.passes:
        assert n_pass == plan.passes, (plan, info)
    return n_pass


def bit_group(plan, info):
    """Plans with equal keys compute every pixel with the same FMA order (module docstring): the key is PR when every
    band of every pass starts on a multiple of PR, else None (such a plan is only held against the oracle)."""
    PR = CONFIGS[plan.cfg][0]
    return PR if all(b[0] % PR == 0 for p in info['passes'] for b in p['bands']) else None


def forward(g, d, s, n, norm):
    """The C ABI on this thread (cspn_last_* are thread-local).  `out` and a workspace of exactly the queried size sit in
    sentinel-filled guarded buffers (tests/memory_contract.py): every plan must store all of `out` and nothing outside it
    or past the workspace.  Returns the workspace's interior."""
    L = _lib.lib()
    gc, dc = g.cuda().contiguous(), d.cuda().contiguous()
    sc = None if s is None else s.cuda().contiguous()
    B, C, H, W = dc.shape
    ws_bytes = L.cspn2d_workspace_bytes(B, C, H, W, n, _lib.ALGO_CLUSTER)
    ws = mc.workspace(ws_bytes)
    out = mc.guarded(dc.shape)
    rc = L.cspn2d_fwd_f32(gc.data_ptr(), dc.data_ptr(), None if sc is None else sc.data_ptr(), out.ptr(), B, C, H, W,
                          gc.shape[1], n, _lib.NORM2D[norm], _lib.ALGO_CLUSTER, ws.ptr(), ws_bytes,
                          torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'cspn2d_fwd_f32')
    torch.cuda.synchronize()
    mc.assert_written(out, 'out')
    assert ws.guards_intact(), 'a store landed past the workspace'
    return out.t.cpu(), L.cspn_last_algo(), L.cspn_last_launches(), ws.t


def chain_flags(info, B, C, H, W, ws):
    """The flag words of the last chained pass, one per (strip boundary, image-channel, CTA): the workspace layout of
    cluster2d_forward / chain_ws in cspn2d_cluster.cu (a continuation buffer when there are several passes, then the
    history blocks, then the flags).  Each is 1 once the chained kernel has finished that block."""
    BC, passes = B * C, info['passes']
    base = B * C * H * W * 4 if sum(p['count'] for p in passes) > 1 else 0
    ceil256 = lambda x: (x + 255) // 256 * 256
    hist = max(ceil256((len(p['strips']) - 1) * BC * p['cs'] * p['iters'] * p['NW'] * 8 * 4) for p in passes)
    last = passes[-1]
    blocks = (len(last['strips']) - 1) * BC * last['cs']
    return ws[base + hist:base + hist + 4 * blocks].view(torch.int32).cpu()


def refused(plan, shape):
    """The device cannot host this forced combination (cudaOccupancyMaxActiveClusters gives 0).  tests/test_plan_cpu.py
    shows the geometry of every combination is valid, so only the occupancy query can refuse it."""
    assert plan.cs > 1, f'a one-CTA cluster of configuration {plan.cfg} cannot be refused: {plan}'
    warnings.warn(f'the device refused forced plan {plan} for {shape}')


def run_forced(plan, g, d, s, n, norm):
    """Forward under `plan` (already forced): (None, None) when the device refuses it, else the output and plan_info,
    checked to come from the forced plan: the cluster algorithm, one launch per pass, a chained plan's flags all set."""
    B, C, H, W = d.shape
    info = plan_info(plan, H, W, n)
    if not info['supported']:
        with pytest.raises(_lib.CspnError, match='unsupported'):
            forward(g, d, s, n, norm)
        refused(plan, (B, C, H, W, n))
        return None, None
    n_pass = check_honoured(plan, info)
    if plan.chain and not chains(plan):       # no chained kernel in this configuration: the unchained plan runs
        assert 'chained' not in _lib.describe_plan(B, C, H, W, n, _lib.ALGO_CLUSTER)
    out, algo, launches, ws = forward(g, d, s, n, norm)
    assert _lib.ALGO_NAMES[algo] == 'cluster' and launches == n_pass, (plan, algo, launches, n_pass)
    if chains(plan):
        assert (chain_flags(info, B, C, H, W, ws) == 1).all(), f'{plan}: the chained kernel did not run'
    return out, info


def backward(g, d, s, go, n, norm):
    """The C ABI's backward called directly (ctypes, this thread): autograd would run it on the engine's worker thread,
    where the thread-local cspn_last_launches() of this thread does not see it.  Both gradients and a workspace of exactly
    the queried size sit in sentinel-filled guarded buffers (tests/memory_contract.py), checked to be fully written and
    stored within.  Returns (grad_guidance, grad_blur) in float64 on the CPU and the launch count."""
    L = _lib.lib()
    gc, dc, goc = g.cuda().contiguous(), d.cuda().contiguous(), go.cuda().contiguous()
    sc = None if s is None else s.cuda().contiguous()
    B, C, H, W = dc.shape
    gg, gd = mc.guarded(gc.shape), mc.guarded(dc.shape)
    ws_bytes = L.cspn2d_bwd_workspace_bytes(B, C, H, W, n)
    ws = mc.workspace(ws_bytes)
    rc = L.cspn2d_bwd_f32(gc.data_ptr(), dc.data_ptr(), None if sc is None else sc.data_ptr(), goc.data_ptr(), gg.ptr(),
                          gd.ptr(), B, C, H, W, gc.shape[1], n, _lib.NORM2D[norm], ws.ptr(), ws_bytes,
                          torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'cspn2d_bwd_f32')
    torch.cuda.synchronize()
    mc.assert_written(gg, 'grad_guidance')
    mc.assert_written(gd, 'grad_blur')
    assert ws.guards_intact(), 'a store landed past the workspace'
    return gg.t.double().cpu(), gd.t.double().cpu(), L.cspn_last_launches()
