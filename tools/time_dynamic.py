"""Times the dynamic propagation (propagate2d_dynamic, DySPN's step, DESIGN.md section 4.23), C = 1, against the routes a
user has without it:

  - shapes: NYU's 8x1x228x304 and KITTI's 8x1x352x1216; K in {3, 5, 7}; N in {6, 24}; without samples and with a soft
    confidence on 5 % sparse samples;
  - (ours) propagate2d_dynamic;
    (a) the F.unfold + einsum composition with autograd, as a port writes it (tests/dynamic_reference.py::composition);
    (b) N single-step propagate2d_dilated calls with each step's weights formed in torch, the anchor rho * d_0 and the
        replacement added in torch;
    (c) plain propagate2d_dilated at the same K and N: what the per-step attention and the anchor cost;
  - forward under no_grad and forward + backward, as CUDA-graph device time (a replay between two events) and as eager
    time (events around the call), median of --reps; peak extra memory of one forward + backward.
    Routes are alternated shape by shape in one process.

    python tools/time_dynamic.py [--reps 10] [--json out.jsonl] [--baseline-steps 6]

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

import cspn_b200  # noqa: E402
from time_keep_sparse import card  # noqa: E402
from time_nonlocal import eager_ms, graph_ms  # noqa: E402

import dynamic_reference as yr  # noqa: E402

SHAPES = {'nyu': (8, 1, 228, 304), 'kitti': (8, 1, 352, 1216)}


def chained_dilated(aff, att, blur, s, m, K):
    """(b): one propagate2d_dilated step per t with w = a[ring] * affinity formed in torch (the centre channel then weights
    the call's blur, d_t), plus rho * d_0 and the replacement in torch."""
    NR = (K + 1) // 2
    ring = yr.rings(K, aff.device)
    d = blur
    for t in range(att.shape[1] // NR):
        w = att[:, t * NR:(t + 1) * NR][:, ring] * aff
        v = cspn_b200.propagate2d_dilated(w, d, None, None, K, 1, 1) + (1 - w.sum(1, keepdim=True)) * blur
        d = m * s + (1 - m) * v if s is not None else v
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--json')
    ap.add_argument('--shapes', default='nyu,kitti')
    ap.add_argument('--baseline-steps', default='6', help='N values at which (a) runs (it keeps N im2col tensors)')
    args = ap.parse_args()
    name, q = card()
    print(f'# {name}, power.limit, clocks.max.sm = {q}; C = 1, soft confidence on 5 % samples when with samples')
    base_n = {int(x) for x in args.baseline_steps.split(',') if x}
    rows = []
    for sname in args.shapes.split(','):
        B, C, H, W = SHAPES[sname]
        for K in (3, 5, 7):
            for N in (6, 24):
                aff, att, b, _, _ = yr.make_inputs(B, C, H, W, K, N, None, seed=K, device='cuda')
                valid = (torch.rand(B, 1, H, W, device='cuda') < 0.05).float()
                s0 = torch.rand(B, 1, H, W, device='cuda') * 10 * valid
                m0 = torch.sigmoid(torch.randn(B, 1, H, W, device='cuda')) * valid
                kern = aff.clone()
                kern[:, K * K // 2] = 0.5
                go = torch.ones(B, C, H, W, device='cuda')
                for samples in (False, True):
                    s, m = (s0, m0) if samples else (None, None)
                    routes = {'ours': (lambda a, t, bb, s=s, m=m: cspn_b200.propagate2d_dynamic(a, t, bb, s, m, K), (aff, att, b))}
                    if N in base_n:
                        routes['a_unfold_einsum'] = (lambda a, t, bb, s=s, m=m: yr.composition(a, t, bb, s, m, K), (aff, att, b))
                    routes['b_chained_dilated'] = (lambda a, t, bb, s=s, m=m: chained_dilated(a, t, bb, s, m, K), (aff, att, b))
                    routes['c_plain_dilated'] = (lambda k, bb, s=s, m=m, N=N: cspn_b200.propagate2d_dilated(k, bb, s, m, K, 1, N),
                                                 (kern, b))
                    for rname, (fn, ins) in routes.items():
                        leaves = [t.clone().requires_grad_(True) for t in ins]

                        def fwd():
                            with torch.no_grad():
                                return fn(*ins)

                        def fwd_bwd():
                            return torch.autograd.grad(fn(*leaves), leaves, go)
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                        base = torch.cuda.memory_allocated()
                        fwd_bwd()
                        torch.cuda.synchronize()
                        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                        row = dict(shape=sname, K=K, N=N, samples=samples, route=rname, fwd_eager_ms=eager_ms(fwd, args.reps),
                                   fwd_bwd_eager_ms=eager_ms(fwd_bwd, args.reps), peak_MiB=round(peak, 1))
                        try:
                            row['fwd_graph_ms'] = graph_ms(fwd, args.reps)
                            row['fwd_bwd_graph_ms'] = graph_ms(fwd_bwd, args.reps)
                        except RuntimeError as e:         # a route that cannot be captured: eager only
                            row['graph'] = str(e).splitlines()[0][:80]
                            torch.cuda.synchronize()
                        # HBM bytes one step needs at C = 1, from the shapes: K*K affinity planes, R + 1 attention planes,
                        # d_0, d_t read and d_{t+1} written (ours); K*K weight planes, d_0, d_t, d_{t+1} (c); plus m and s
                        extra = 8 if samples else 0
                        per_px = (4 * (K * K + (K - 1) // 2 + 4) if rname == 'ours' else 4 * (K * K + 3)) + extra
                        if 'fwd_graph_ms' in row and rname in ('ours', 'c_plain_dilated'):
                            row['fwd_TBps'] = round(per_px * B * H * W * N / (row['fwd_graph_ms'] * 1e-3) / 1e12, 2)
                        rows.append(row)
                        print(json.dumps(row), flush=True)
                    torch.cuda.empty_cache()
    if args.json:
        with open(args.json, 'w') as fh:
            for r in rows:
                fh.write(json.dumps(dict(r, card=name, power=q)) + '\n')


if __name__ == '__main__':
    main()
