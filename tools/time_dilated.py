"""Times the dilated propagation (propagate2d_dilated, PENet's DA-CSPN++ step, DESIGN.md section 4.22), C = 1, with a soft
confidence on 5 % sparse samples, against the routes a user has without it:

  - shapes: NYU's 8x1x228x304 and KITTI's 8x1x352x1216; K in {3, 5, 7}, dilation in {1, 2}, N in {6, 24};
  - (ours) propagate2d_dilated;  (a) PENet's F.unfold + einsum + replacement loop with autograd
    (tests/dilated_reference.py::composition);  (b) affinity_propagate at d = 1 without samples, the existing kernel
    with the same bytes per step;
  - forward under no_grad and forward + backward, as CUDA-graph device time (a replay between two events) and as eager
    time (events around the call), median of --reps; peak extra memory of one forward + backward.
    Routes are alternated shape by shape in one process.

    python tools/time_dilated.py [--reps 10] [--json out.jsonl] [--baseline-steps 6]

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

import dilated_reference as dr  # noqa: E402

SHAPES = {'nyu': (8, 1, 228, 304), 'kitti': (8, 1, 352, 1216)}


def inputs(B, C, H, W, K):
    k, b, _, _ = dr.make_inputs(B, C, H, W, K, None, seed=K, device='cuda')
    valid = (torch.rand(B, 1, H, W, device='cuda') < 0.05).float()
    s = torch.rand(B, 1, H, W, device='cuda') * 10 * valid
    m = torch.sigmoid(torch.randn(B, 1, H, W, device='cuda')) * valid
    c = K * K // 2
    gates = torch.cat([k[:, :c], k[:, c + 1:]], 1).flip(1).contiguous()
    return k, b, s, m, gates


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--json')
    ap.add_argument('--shapes', default='nyu,kitti')
    ap.add_argument('--baseline-steps', default='6', help='N values at which (a) runs (it keeps N im2col tensors)')
    args = ap.parse_args()
    name, q = card()
    print(f'# {name}, power.limit, clocks.max.sm = {q}; C = 1, soft confidence on 5 % samples')
    base_n = {int(x) for x in args.baseline_steps.split(',') if x}
    rows = []
    for sname in args.shapes.split(','):
        B, C, H, W = SHAPES[sname]
        for K in (3, 5, 7):
            k, b, s, m, gates = inputs(B, C, H, W, K)
            go = torch.ones(B, C, H, W, device='cuda')
            for dil in (1, 2):
                for N in (6, 24):
                    routes = {'ours': (lambda kk, bb, N=N, dil=dil: cspn_b200.propagate2d_dilated(kk, bb, s, m, K, dil, N), k)}
                    if N in base_n:
                        routes['a_unfold_einsum'] = (lambda kk, bb, N=N, dil=dil: dr.composition(kk, bb, s, m, K, dil, N), k)
                    if dil == 1:
                        routes['b_affinity_propagate'] = (lambda gg, bb, N=N: cspn_b200.affinity_propagate(bb, gg, K, N), gates)
                    for rname, (fn, w) in routes.items():
                        leaves = [t.clone().requires_grad_(True) for t in (w, b)]

                        def fwd():
                            with torch.no_grad():
                                return fn(w, b)

                        def fwd_bwd():
                            return torch.autograd.grad(fn(*leaves), leaves, go)
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                        base = torch.cuda.memory_allocated()
                        fwd_bwd()
                        torch.cuda.synchronize()
                        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                        row = dict(shape=sname, K=K, dilation=dil, N=N, route=rname, fwd_eager_ms=eager_ms(fwd, args.reps),
                                   fwd_bwd_eager_ms=eager_ms(fwd_bwd, args.reps), peak_MiB=round(peak, 1))
                        try:
                            row['fwd_graph_ms'] = graph_ms(fwd, args.reps)
                            row['fwd_bwd_graph_ms'] = graph_ms(fwd_bwd, args.reps)
                        except RuntimeError as e:         # a route that cannot be captured: eager only
                            row['graph'] = str(e).splitlines()[0][:80]
                            torch.cuda.synchronize()
                        # HBM bytes one step needs at C = 1, from the shapes: K*K - 1 weight planes, w_c, d_0, d_t, and
                        # m, s read, d_{t+1} written (ours); nt gate planes, d_t read, d_{t+1} written (b)
                        per_px = 4 * (K * K + 5) if rname == 'ours' else 4 * (K * K + 1)
                        if 'fwd_graph_ms' in row and rname != 'a_unfold_einsum':
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
