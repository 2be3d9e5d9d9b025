"""Times the 2D propagation with the Paddle module's own-location gates (Affinity_Propagate2DPaddle, K = 3, 5, 7) at N = 24
on the NYU (8x1x228x304) and KITTI (8x1x352x1216) batch shapes:

  - forward under no_grad and forward + backward, CUDA events, warm-up, median of --reps;
  - the torch port's eager op sequence (tests/paddle2d_reference.py::cspn2d_torch_paddle) on the same GPU as the baseline;
  - at K = 3, the cluster kernel's '8sum_abs' (Affinity_Propagate) at the same shape: what running the own-location form
    on the K x K kernels instead of the cluster kernel costs;
  - the bytes a step moves from a byte model: K*K-1 weight planes and d_t read, d_{t+1} written, (K*K-1 + 2C) * 4 B per
    pixel (40, 104, 200 B at C = 1); the rate divides N such steps by the whole forward, prep included.

    python tools/time_2d_paddle.py [--reps 20] [--baseline-reps 3] [--json out.jsonl]

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
import paddle2d_reference as pr  # noqa: E402

SHAPES = {'nyu': (8, 1, 228, 304), 'kitti': (8, 1, 352, 1216)}
N = 24


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def median_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def step_bytes(B, C, H, W, K):
    """Bytes one step moves: K*K-1 weight planes per image, d_t per channel read, d_{t+1} per channel written."""
    return 4 * B * H * W * (K * K - 1 + 2 * C)


def fwd_and_bwd(m, args, reps):
    with torch.no_grad():
        fwd = median_ms(lambda: m(*args), reps)
    leaves = [t.clone().requires_grad_(True) if i < 2 else t for i, t in enumerate(args)]
    go = torch.randn_like(args[1])

    def fb():
        for t in leaves[:2]:
            t.grad = None
        m(*leaves).backward(go)
    return fwd, median_ms(fb, reps)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--baseline-reps', type=int, default=3)
    ap.add_argument('--json', help='also append one JSON line per measurement to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_2d_paddle.py measures on a CUDA device; none is present')
    torch.cuda.set_device(0)
    name, power = card()
    print(f'card: {name}, power limit {power}; N = {N}, median of {a.reps} (baseline {a.baseline_reps})')
    rows = []
    for shape_name, (B, C, H, W) in SHAPES.items():
        for K in (3, 5, 7):
            nt = K * K - 1
            gen = torch.Generator().manual_seed(K)
            g = torch.rand(B, nt, H, W, generator=gen).cuda()
            f = torch.rand(B, C, H, W, generator=gen).cuda()
            fwd, fb = fwd_and_bwd(cspn_b200.Affinity_Propagate2DPaddle(N, K), (g, f), a.reps)
            with torch.no_grad():
                base = median_ms(lambda: pr.cspn2d_torch_paddle(g, f, N, K), a.baseline_reps, warmup=1)
            sb = step_bytes(B, C, H, W, K)
            row = dict(card=name, power_limit=power, shape=f'{B}x{C}x{H}x{W}', K=K, N=N, fwd_ms=round(fwd, 3),
                       fwd_bwd_ms=round(fb, 3), eager_port_fwd_ms=round(base, 2), speedup_fwd=round(base / fwd, 1),
                       step_bytes=sb, fwd_step_GBps=round(sb * N / (fwd * 1e-3) / 1e9))
            if K == 3:
                g8 = torch.rand(B, 8, H, W, generator=gen).cuda()
                cf, cfb = fwd_and_bwd(cspn_b200.Affinity_Propagate(N, 3, '8sum_abs'), (g8, f), a.reps)
                row.update(cluster_8sum_abs_fwd_ms=round(cf, 3), cluster_8sum_abs_fwd_bwd_ms=round(cfb, 3))
                del g8
            rows.append(row)
            print(json.dumps(row), flush=True)
            del g, f
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'a') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')
    print('\n| shape | K | forward | forward + backward | eager op sequence, forward | bytes / step | forward rate | '
          "cluster kernel '8sum_abs', forward / fwd + bwd |")
    print('|---|---|---|---|---|---|---|---|')
    for r in rows:
        cl = f"{r['cluster_8sum_abs_fwd_ms']} ms / {r['cluster_8sum_abs_fwd_bwd_ms']} ms" if r['K'] == 3 else ''
        print(f"| {r['shape']} | {r['K']} | {r['fwd_ms']} ms | {r['fwd_bwd_ms']} ms | {r['eager_port_fwd_ms']} ms | "
              f"{r['step_bytes'] / 1e6:.0f} MB | {r['fwd_step_GBps'] / 1e3:.2f} TB/s | {cl} |")


if __name__ == '__main__':
    main()
