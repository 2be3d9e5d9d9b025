"""Times the aggregation of the 2D steps (propagate2d_aggregate, DESIGN.md section 4.20) at N = 24, every step aggregated,
keep mode, against the routes a user has without it:

  - shapes: NYU's 8x1x228x304 and KITTI's 8x1x352x1216; K = 3, 5 and 7;
  - (ours) propagate2d_aggregate;  (a) the torch composition with autograd;  (b) plain propagate2d_k at N (the cost of the
    aggregation itself; K = 3 there is the cluster kernel);  (c) T separate propagate2d_k calls plus a torch sum, the
    library's only route before the op;
  - forward under no_grad and forward + backward, as CUDA-graph device time (a replay between two events) and as eager
    time (events around the call), median of --reps; peak memory of one forward + backward.

    python tools/time_aggregate.py [--reps 20] [--json out.jsonl]

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
from cspn_b200.synth import make_inputs  # noqa: E402
from time_keep_sparse import card, event_ms  # noqa: E402

import aggregate_reference as ar  # noqa: E402

SHAPES = {'nyu': (8, 1, 228, 304), 'kitti': (8, 1, 352, 1216)}
N = 24
STEPS = tuple(range(1, N + 1))


def routes(K, g, d, s, sw):
    def ours():
        return cspn_b200.propagate2d_aggregate(g, d, sw, s, K, keep_sparse=True)

    def torch_composition():
        return ar.composition(g, d, s, sw, STEPS, K, None, True)

    def plain():
        return cspn_b200.Affinity_PropagateK(N, K, keep_sparse=True)(g, d, s)

    def separate():
        m = [cspn_b200.Affinity_PropagateK(n, K, keep_sparse=True) for n in STEPS]
        return ar.aggregate([mi(g, d, s) for mi in m], sw)
    return {'ours': ours, 'a_torch': torch_composition, 'b_plain': plain, 'c_separate': separate}


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
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    return statistics.median(event_ms(fn) for _ in range(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json')
    ap.add_argument('--shapes', default='nyu,kitti')
    args = ap.parse_args()
    name, q = card()
    print(f'# {name}, power.limit, clocks.max.sm = {q}; N = {N}, every step aggregated, keep mode')
    rows = []
    for sname in args.shapes.split(','):
        B, C, H, W = SHAPES[sname]
        for K in (3, 5, 7):
            g, d, s = [t.cuda() for t in make_inputs(K, B, C, H, W, K * K - 1, 'bernoulli', 20)]
            sw = torch.softmax(torch.randn(B, N, H, W, device='cuda'), 1)
            for rname, fn in routes(K, g, d, s, sw).items():
                if rname == 'a_torch' and sname == 'kitti' and K == 7:
                    continue                                   # autograd's saved tensors of 24 x 48 shifts do not pay
                leaves = [t.clone().requires_grad_(True) for t in (g, d, sw)]
                go = torch.ones(B, C, H, W, device='cuda')

                def fwd():
                    with torch.no_grad():
                        return fn()

                def fwd_bwd():
                    gg, dd, ww = leaves
                    f = routes(K, gg, dd, s, ww)[rname]
                    return torch.autograd.grad(f(), [gg, dd, ww] if rname in ('ours', 'a_torch', 'c_separate') else [gg, dd],
                                               go, allow_unused=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                fwd_bwd()
                torch.cuda.synchronize()
                peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                row = dict(shape=sname, K=K, route=rname, fwd_eager_ms=eager_ms(fwd, args.reps),
                           fwd_bwd_eager_ms=eager_ms(fwd_bwd, args.reps), peak_MiB=peak)
                try:
                    row['fwd_graph_ms'] = graph_ms(fwd, args.reps)
                    row['fwd_bwd_graph_ms'] = graph_ms(fwd_bwd, args.reps)
                except RuntimeError as e:                     # a route that cannot be captured: eager only
                    row['graph'] = str(e).splitlines()[0][:80]
                    torch.cuda.synchronize()
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, 'w') as f:
            for r in rows:
                f.write(json.dumps(dict(r, card=name, power=q)) + '\n')


if __name__ == '__main__':
    main()
