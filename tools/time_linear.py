"""Times the linear propagation (propagate2d_linear, SPN's three-way scans, DESIGN.md section 4.24) against the routes a
user has without it, and against the byte floor:

  - shapes: 8x1x352x1216 (KITTI depth refinement) and 8x32x88x304 (a multi-channel feature map at a quarter of KITTI's
    resolution), shared gates;
  - cases: one direction (l2r, and t2b, whose lanes run along memory) and all four; forward under no_grad and forward + backward;
  - (ours) propagate2d_linear;
    (a) the torch restatement's per-column loop with autograd (tests/linear_reference.py::composition, in fp32), eager
        and as a CUDA graph;
  - device time of a CUDA-graph replay between two events, median of --reps (eager time with events around the call
    for (a) eager);
  - the byte floor from the shapes: each direction reads x and three gate planes and writes h (20 B per pixel at C = 1);
    four directions merge by reading the four planes and writing out (+20 B); the backward reads x, the gates, its
    planes and grad_out and writes grad_x and the gates' gradients.  The share is floor time at 3.35 TB/s over the
    measured time.

    python tools/time_linear.py [--reps 10] [--json out.jsonl]

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

import linear_reference as R  # noqa: E402

SHAPES = {'kitti': (8, 1, 352, 1216), 'feat': (8, 32, 88, 304)}
HBM_TBPS = 3.35


def floor_bytes(B, C, H, W, nd, backward):
    """HBM bytes the op needs at least, from the shapes (shared gates: 3 planes per image per direction)."""
    px, gate = B * C * H * W, B * H * W
    f = nd * (4 * px + 12 * gate + 4 * px)                   # x, the gates, h
    if nd > 1:
        f += 4 * nd * px + 4 * px                            # the merge reads the planes, writes out
    if backward:
        b = nd * (4 * px + 12 * gate + 4 * px + 4 * px)      # x, the gates, the plane, grad_out per direction
        b += 4 * px + 12 * nd * gate                         # grad_x and the gates' gradients written
        if nd > 1:
            b += 4 * nd * px                                 # the merge's pick re-read from the planes
        f += b
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--json')
    ap.add_argument('--shapes', default='kitti,feat')
    ap.add_argument('--no-baseline', action='store_true')
    args = ap.parse_args()
    name, q = card()
    print(f'# {name}, power.limit, clocks.max.sm = {q}; shared gates, sum |g| <= 1')
    rows = []
    for sname in args.shapes.split(','):
        B, C, H, W = SHAPES[sname]
        for dirs in (('l2r',), ('t2b',), R.DIRECTIONS):
            f, g = R.random_inputs(B, C, H, W, dirs, False, seed=1, device='cuda')
            go = torch.ones(B, C, H, W, device='cuda')
            routes = {'ours': lambda x, gt, dirs=dirs: cspn_b200.propagate2d_linear(x, gt, dirs)}
            if not args.no_baseline:
                routes['a_torch_loop'] = lambda x, gt, dirs=dirs: R.composition(x, gt, dirs)
            for rname, fn in routes.items():
                leaves = [f.clone().requires_grad_(True), g.clone().requires_grad_(True)]

                def fwd():
                    with torch.no_grad():
                        return fn(f, g)

                def fwd_bwd():
                    return torch.autograd.grad(fn(*leaves), leaves, go)
                row = dict(shape=sname, B=B, C=C, H=H, W=W, directions=len(dirs), route=rname,
                           fwd_eager_ms=eager_ms(fwd, max(2, args.reps // 3 if rname != 'ours' else args.reps)),
                           fwd_bwd_eager_ms=eager_ms(fwd_bwd, max(2, args.reps // 3 if rname != 'ours' else args.reps)))
                try:
                    row['fwd_graph_ms'] = graph_ms(fwd, args.reps)
                    row['fwd_bwd_graph_ms'] = graph_ms(fwd_bwd, args.reps)
                except RuntimeError as e:                   # a route that cannot be captured: eager only
                    row['graph'] = str(e).splitlines()[0][:80]
                    torch.cuda.synchronize()
                for key, bwd in (('fwd', False), ('fwd_bwd', True)):
                    fb = floor_bytes(B, C, H, W, len(dirs), bwd)
                    row[f'{key}_floor_B_per_px'] = round(fb / (B * H * W), 1)
                    row[f'{key}_floor_ms'] = round(fb / (HBM_TBPS * 1e12) * 1e3, 4)
                    if f'{key}_graph_ms' in row:
                        row[f'{key}_floor_share'] = round(row[f'{key}_floor_ms'] / row[f'{key}_graph_ms'], 3)
                rows.append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if args.json:
        with open(args.json, 'w') as fh:
            for r in rows:
                fh.write(json.dumps(dict(r, card=name, power=q)) + '\n')


if __name__ == '__main__':
    main()
