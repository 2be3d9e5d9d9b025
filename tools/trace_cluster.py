"""Per-warp timeline of the 2D cluster kernel (needs a -DCSPN_TRACE build of the library):

    python -m cspn_b200.build --define CSPN_TRACE [--define CSPN_STEP=3 ...] --out tools/_build/variants/lib_trace.so
    CSPN_B200_LIB=tools/_build/variants/lib_trace.so python tools/trace_cluster.py [B H W N]

Cluster 0 stamps clock64() (lane 0 of every warp) at the phase boundaries of its 2nd..5th task and around every mbarrier
wait / publish of the step loop.  Prints where a task's cycles go and, per step, how long warps sit in the wait, how long
the wait -> publish chain is and how much work separates a publish from the next wait.  Kernels with a producer
warpgroup (warps 8..11) also print how long the producers wait for the stage and take to prepare a task.
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cspn_b200
from cspn_b200 import _lib
from cspn_b200.synth import make_inputs

B, H, W, N = [int(a) for a in sys.argv[1:5]] if len(sys.argv) > 4 else (32, 352, 1216, 24)
L = _lib.lib()
L.cspn_debug_set_trace.argtypes = [ctypes.c_void_p]
L.cspn_debug_set_trace.restype = None
NEV = L.cspn_debug_trace_events()
TASKS, CTAS, WARPS, CONSUMERS = 4, 16, 12, 8
buf = torch.zeros(TASKS * CTAS * WARPS * NEV, dtype=torch.int64, device='cuda')
g, d, s = [t.cuda() for t in make_inputs(0, min(B, 8), 1, H, W)]
if B > 8:
    rep = (B + 7) // 8
    g, d, s = [t.repeat(rep, 1, 1, 1)[:B].contiguous() for t in (g, d, s)]
for _ in range(2):
    cspn_b200.propagate2d(g, d, s, N, '8sum', _lib.ALGO_CLUSTER)
torch.cuda.synchronize()
L.cspn_debug_set_trace(buf.data_ptr())
cspn_b200.propagate2d(g, d, s, N, '8sum', _lib.ALGO_CLUSTER)
torch.cuda.synchronize()
L.cspn_debug_set_trace(None)
print(cspn_b200.describe_plan(B, 1, H, W, N, _lib.ALGO_CLUSTER))
t_all = buf.cpu().numpy().reshape(TASKS, CTAS, WARPS, NEV).astype(np.int64)
t = t_all[:, :, :CONSUMERS]
ncta = int((t[0, :, 0, 0] != 0).sum())
split = bool((t_all[:, :ncta, CONSUMERS:, 0] != 0).any())
print(f'traced {TASKS} tasks of cluster 0, {ncta} CTAs, {N} steps; cycles are SM clocks (clock64)')
if split:
    names = ['wait for producers', 'load w\' and d0', 'cluster wait', 'first publish']
else:
    names = ['load+tma wait', 'prologue', 'syncthreads', 'issue next + cluster wait']
for slot in range(TASKS):
    x = t[slot, :ncta]                      # [cta][warp][ev]
    if not x[..., 0].all():
        continue
    e = lambda i: x[..., i].astype(np.float64)
    tot = e(NEV - 1) - e(0)
    seg = dict(zip(names, [e(1) - e(0), e(2) - e(1), e(3) - e(2), e(4) - e(3)]))
    seg.update({'step loop': e(NEV - 2) - e(4), 'epilogue': e(NEV - 1) - e(NEV - 2)})
    print(f'task slot {slot}: total {tot.mean():.0f} cycles (min {tot.min():.0f} max {tot.max():.0f})  ' +
          '  '.join(f'{k} {v.mean():.0f}' for k, v in seg.items()))
    if split:
        p = t_all[slot, :ncta, CONSUMERS:].astype(np.float64)    # [cta][producer warp][ev]
        if p[..., 0].all():
            print(f'   producers: wait for stage {(p[..., 1] - p[..., 0]).mean():.0f}   prepare {(p[..., 2] - p[..., 1]).mean():.0f}   '
                  f'ready {(x[..., 1].mean() - p[..., 2].mean()):.0f} cycles before the consumers got there')
    steps = N - 1   # the last step has no publish
    w0 = np.stack([e(5 + 3 * k) for k in range(N)], -1)
    w1 = np.stack([e(6 + 3 * k) for k in range(N)], -1)
    pb = np.stack([e(7 + 3 * k) for k in range(steps)], -1)
    wait = w1 - w0
    chain = pb - w1[..., :steps]
    gap = w0[..., 1:] - pb
    period = w1[..., 1:] - w1[..., :-1]
    print(f'   per step (mean over warps/CTAs/steps): period {period.mean():.0f}   in-wait {wait.mean():.0f}   wait->publish {chain.mean():.0f}   '
          f'publish->next wait {gap.mean():.0f}')
    if slot == 1:
        print('   in-wait by warp (rows: CTA, cols: warp 0..7), mean over steps:')
        for c in range(ncta):
            print('     cta %2d: ' % c + ' '.join('%5.0f' % v for v in wait[c].mean(-1)))
        print('   in-wait by step (mean over warps of CTA %d): ' % (ncta // 2) + ' '.join('%4.0f' % v for v in wait[ncta // 2].mean(0)))
        print('   wait->publish by warp, CTA %d: ' % (ncta // 2) + ' '.join('%5.0f' % v for v in chain[ncta // 2].mean(-1)))
        print('   publish->next wait by warp, CTA %d: ' % (ncta // 2) + ' '.join('%5.0f' % v for v in gap[ncta // 2].mean(-1)))
