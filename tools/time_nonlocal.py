"""Times the non-local 2D propagation (propagate2d_nonlocal, DESIGN.md section 4.21) at NLSPN's settings, K = 3, N = 18,
C = 1, against the routes a user has without it:

  - shapes: NYU's 8x1x228x304, 8x1x240x1216 and KITTI's 8x1x352x1216; offsets of a few pixels, NLSPN-normalised
    affinities, 5 % sparse samples kept before every step;
  - (ours) propagate2d_nonlocal;  (a) torchvision's deform_conv2d once per step, NLSPN's route;  (b) the torch
    restatement of tests/nonlocal_reference.py;
  - forward under no_grad and forward + backward, as CUDA-graph device time (a replay between two events) and as eager
    time (events around the call), median of --reps; peak memory of one forward + backward.

    python tools/time_nonlocal.py [--reps 20] [--json out.jsonl]

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

import cspn_b200  # noqa: E402
from time_keep_sparse import card, event_ms  # noqa: E402

import nonlocal_reference as nr  # noqa: E402

SHAPES = {'nyu': (8, 1, 228, 304), 'wide': (8, 1, 240, 1216), 'kitti': (8, 1, 352, 1216)}
K, N = 3, 18


def routes():
    return {'ours': lambda f, o, a, s: cspn_b200.propagate2d_nonlocal(f, o, a, s, K, N),
            'a_deform_conv2d': lambda f, o, a, s: nr.propagate_torchvision(f, o, a, s, K=K, N=N),
            'b_torch': lambda f, o, a, s: nr.propagate(f, o, a, s, K=K, N=N)}


def graph_ms(fn, reps):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    graph.replay()
    torch.cuda.synchronize()
    return statistics.median(event_ms(graph.replay) for _ in range(reps))


def eager_ms(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    return statistics.median(event_ms(fn) for _ in range(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json')
    ap.add_argument('--shapes', default='nyu,wide,kitti')
    ap.add_argument('--routes', default='ours,a_deform_conv2d,b_torch')
    args = ap.parse_args()
    name, q = card()
    print(f'# {name}, power.limit, clocks.max.sm = {q}; K = {K}, N = {N}, C = 1, sparse kept before every step')
    rows = []
    for sname in args.shapes.split(','):
        B, C, H, W = SHAPES[sname]
        f, o, a, s = nr.make_inputs(B, C, H, W, K, scale=3.0, seed=1, device='cuda')
        s = torch.where(torch.rand(B, C, H, W, device='cuda') < 0.05, torch.rand(B, C, H, W, device='cuda') * 10, torch.zeros((), device='cuda'))
        go = torch.ones(B, C, H, W, device='cuda')
        for rname in args.routes.split(','):
            fn = routes()[rname]
            leaves = [t.clone().requires_grad_(True) for t in (f, o, a)]

            def fwd():
                with torch.no_grad():
                    return fn(f, o, a, s)

            def fwd_bwd():
                return torch.autograd.grad(fn(*leaves, s), leaves, go)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fwd_bwd()
            torch.cuda.synchronize()
            peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            row = dict(shape=sname, route=rname, fwd_eager_ms=eager_ms(fwd, args.reps), fwd_bwd_eager_ms=eager_ms(fwd_bwd, args.reps),
                       peak_MiB=peak)
            try:
                row['fwd_graph_ms'] = graph_ms(fwd, args.reps)
                row['fwd_bwd_graph_ms'] = graph_ms(fwd_bwd, args.reps)
            except RuntimeError as e:                     # a route that cannot be captured: eager only
                row['graph'] = str(e).splitlines()[0][:80]
                torch.cuda.synchronize()
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, 'w') as fh:
            for r in rows:
                fh.write(json.dumps(dict(r, card=name, power=q)) + '\n')


if __name__ == '__main__':
    main()
