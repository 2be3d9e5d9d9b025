"""Times the keep-sparse mode against the default mode of the 2D propagation, call by call alternated, at N = 24:

  - shapes: cfg2 (32x1x352x1216, BASELINE.json configs[1]) and NYU's 8x1x228x304;
  - K = 3 (cluster kernel), 5 and 7 (the K x K launches; keep mode adds one d0' plane to the prep);
  - forward under no_grad (the functional entry) and forward + backward through Affinity_Propagate(K);
  - CUDA events around each call after a warm-up, the two modes interleaved so drift hits both; median of --reps.

    python tools/time_keep_sparse.py [--reps 20] [--json out.jsonl]

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

import torch  # noqa: E402

import cspn_b200  # noqa: E402
from cspn_b200.synth import make_inputs  # noqa: E402

SHAPES = {'cfg2': (32, 1, 352, 1216), 'nyu': (8, 1, 228, 304)}
N = 24


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def alternate(fns, reps, warmup=3):
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            times[i].append(event_ms(f))
    return [statistics.median(t) for t in times]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_keep_sparse.py measures on a CUDA device; none is available')
    name, power = card()
    print(f'card: {name}; power limit, max SM clock: {power}')
    rows = []
    for shape, (B, C, H, W) in SHAPES.items():
        for K in (3, 5, 7):
            nt = K * K - 1
            g, d, s = make_inputs(1, B, C, H, W, nt, 'signed', 500)
            g, d, s = g.cuda(), d.cuda(), s.abs().cuda()
            with torch.no_grad():
                fwd = [lambda keep=keep: cspn_b200.propagate2d_k(g, d, s, K, N, keep_sparse=keep) for keep in (False, True)]
                f_def, f_keep = alternate(fwd, a.reps)
            mods = [cspn_b200.Affinity_PropagateK(N, K, keep_sparse=keep) for keep in (False, True)]
            gl, dl, sl = g.clone().requires_grad_(True), d.clone().requires_grad_(True), s.clone().requires_grad_(True)

            def train(m):
                for t in (gl, dl, sl):
                    t.grad = None
                m(gl, dl, sl).sum().backward()

            b_def, b_keep = alternate([lambda m=m: train(m) for m in mods], max(a.reps // 2, 5))
            row = dict(shape=shape, B=B, C=C, H=H, W=W, K=K, N=N, fwd_default_ms=f_def, fwd_keep_ms=f_keep,
                       fwd_bwd_default_ms=b_def, fwd_bwd_keep_ms=b_keep, card=name, power_limit=power)
            rows.append(row)
            print(f'{shape} {B}x{C}x{H}x{W} K={K}: forward {f_def:.3f} ms default, {f_keep:.3f} ms keep '
                  f'({f_keep / f_def:.3f}x); forward+backward {b_def:.3f} ms default, {b_keep:.3f} ms keep '
                  f'({b_keep / b_def:.3f}x)', flush=True)
            del g, d, s, gl, dl, sl
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'a') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
