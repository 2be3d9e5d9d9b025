"""Times cspn_b200.affinity_propagate (the Paddle op with caller-supplied gates) against the 'paddle' path on the same inputs,
in the same process, alternating the two measurement by measurement, at N = 24:

  - 2D: 8x1x228x304 (NYU) and 8x1x352x1216 (KITTI), K = 3, 5, 7, against propagate2d_paddle / Affinity_Propagate2DPaddle;
  - 3D: 3x1x48x64x128, K = 3, 5, against propagate3d_k(..., 'paddle') / Affinity_Propagate3DK(..., 'paddle');
  - forward under no_grad and forward + backward: one pair of CUDA events around --calls back-to-back calls (a single
    call of 0.1-1 ms is too short a window for a stable number), per-call time = the interval / --calls, median of
    --reps such intervals after a warm-up;
  - the forward once more as the replay of a CUDA graph of one call: the GPU time without the host's per-call work.
  - forward + backward of affinity_propagate with the input's gradient only (the gates do not require grad).
The gates given to affinity_propagate are |g| / sum |g| of the guidance the 'paddle' path takes, computed once outside the
timed region, so both compute the same propagation; the 'paddle' path normalises inside.

    python tools/time_gates.py [--reps 15] [--calls 10] [--json out.jsonl]

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

import cspn_b200  # noqa: E402
import gates_reference as gr  # noqa: E402

N = 24
CASES = [('2d', (8, 1, 228, 304), K) for K in (3, 5, 7)] + [('2d', (8, 1, 352, 1216), K) for K in (3, 5, 7)] + \
        [('3d', (3, 1, 48, 64, 128), K) for K in (3, 5)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def per_call_ms(fn, calls):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def alternate(fns, reps, calls, warmup=3):
    """Median per-call ms of each fn, the fns measured in turn rep by rep so that clock and thermal drift hit them alike."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    times = [[] for _ in fns]
    for _ in range(reps):
        for t, fn in zip(times, fns):
            t.append(per_call_ms(fn, calls))
    return [statistics.median(t) for t in times]


def graphed(fn):
    """The replay of a CUDA graph of one call of fn (warmed up on a side stream first)."""
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        fn()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph.replay


def fwd_bwd(fn, args, go):
    leaves = [t.clone().requires_grad_(True) for t in args]

    def run():
        for t in leaves:
            t.grad = None
        fn(*leaves).backward(go)
    return run


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=15)
    ap.add_argument('--calls', type=int, default=10, help='back-to-back calls per timed interval')
    ap.add_argument('--json', help='also append one JSON line per measurement to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_gates.py measures on a CUDA device; none is present')
    torch.cuda.set_device(0)
    name, power = card()
    print(f'card: {name}, power limit {power}; N = {N}, median of {a.reps} intervals of {a.calls} calls, '
          'gates and paddle alternated')
    rows = []
    for nd, shape, K in CASES:
        nt = K ** (len(shape) - 2) - 1
        gen = torch.Generator().manual_seed(K)
        g = torch.rand(shape[0], nt, *shape[2:], generator=gen).cuda()
        x = torch.rand(*shape, generator=gen).cuda()
        go = torch.randn(*shape, generator=gen).cuda()
        gates = gr.paddle_gates(g, nt)
        if nd == '2d':
            paddle = cspn_b200.Affinity_Propagate2DPaddle(N, K)
        else:
            paddle = cspn_b200.Affinity_Propagate3DK(N, K, 'paddle')
        ours = lambda xx, gg: cspn_b200.affinity_propagate(xx, gg, K, N)
        with torch.no_grad():
            f_ours, f_pad = alternate([lambda: ours(x, gates), lambda: paddle(g, x)], a.reps, a.calls)
            gr_ours, gr_pad = alternate([graphed(lambda: ours(x, gates)), graphed(lambda: paddle(g, x))], a.reps, a.calls)
        fb_ours, fb_pad = alternate([fwd_bwd(ours, (x, gates), go), fwd_bwd(lambda xx, gg: paddle(gg, xx), (x, g), go)],
                                    a.reps, a.calls)
        xg = x.clone().requires_grad_(True)              # a model that trains the input's producer only: no gate gradient

        def input_only():
            xg.grad = None
            ours(xg, gates).backward(go)
        fbx_ours = alternate([input_only], a.reps, a.calls)[0]
        row = dict(card=name, power_limit=power, dim=nd, shape='x'.join(map(str, shape)), K=K, N=N,
                   gates_fwd_ms=round(f_ours, 3), paddle_fwd_ms=round(f_pad, 3), fwd_ratio=round(f_pad / f_ours, 2),
                   gates_fwd_graph_ms=round(gr_ours, 3), paddle_fwd_graph_ms=round(gr_pad, 3),
                   fwd_graph_ratio=round(gr_pad / gr_ours, 2),
                   gates_fwd_bwd_ms=round(fb_ours, 3), paddle_fwd_bwd_ms=round(fb_pad, 3), fwd_bwd_ratio=round(fb_pad / fb_ours, 2),
                   gates_fwd_bwd_input_only_ms=round(fbx_ours, 3))
        rows.append(row)
        print(json.dumps(row), flush=True)
        del g, x, go, gates
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'a') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')
    print("\n| shape | K | forward: gates / 'paddle' | speed-up | forward, graph replay | speed-up | "
          "fwd + bwd: gates / 'paddle' | speed-up | fwd + bwd, input gradient only |")
    print('|---|---|---|---|---|---|---|---|---|')
    for r in rows:
        print(f"| {r['shape']} | {r['K']} | {r['gates_fwd_ms']} / {r['paddle_fwd_ms']} ms | {r['fwd_ratio']}x | "
              f"{r['gates_fwd_graph_ms']} / {r['paddle_fwd_graph_ms']} ms | {r['fwd_graph_ratio']}x | "
              f"{r['gates_fwd_bwd_ms']} / {r['paddle_fwd_bwd_ms']} ms | {r['fwd_bwd_ratio']}x | "
              f"{r['gates_fwd_bwd_input_only_ms']} ms |")


if __name__ == '__main__':
    main()
