"""Times the K x K x K 3D propagation (K = 3, 5) on cspn_paddle/demo.py's volume (3 x 1 x 48 x 64 x 128, N = 24) and,
forward only for K = 5, on the cfg4 shape (8 x 1 x 64 x 96 x 312, N = 12; its guidance alone is 7.6 GB, so its backward
is not timed on a shared card):

  - forward under no_grad and forward + backward through Affinity_Propagate3DK, every norm, CUDA events, warm-up, median
    of --reps;
  - the torch port's eager op sequence (oracle/cspn_torch_port_3d_k.py::cspn3d_torch_k) at the demo shape as the baseline;
  - the bytes a step moves, computed from shapes, and the rate that gives.

At K = 3 the demo volume's forward (W % 4 == 0) runs cspn3d.cu's raw-guidance step and its backward the K x K x K kernels at
R = 1; at K = 5 both run the K x K x K kernels.

    python tools/time_3d_k.py [--reps 10] [--baseline-reps 3] [--json out.jsonl]

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
from oracle import cspn_torch_port_3d_k as tpk  # noqa: E402

DEMO = (3, 1, 48, 64, 128, 24)
CFG4 = (8, 1, 64, 96, 312, 12)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def median_ms(fn, reps, warmup=2):
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


def step_bytes(B, C, V, K, norm):
    """HBM bytes of one forward step: 'paddle' reads K^3-1 guidance planes, d_t and writes d_{t+1}; the gathered norms read
    K^3 weight planes, d_0, d_t and write d_{t+1}.  K = 3 at W % 4 == 0 runs cspn3d.cu's raw-guidance kernels (26 guidance
    planes for every norm, plus d_0 for the gathered ones)."""
    nt = K ** 3 - 1
    if K == 3:
        return 4 * B * V * (nt + (2 if norm == 'paddle' else 3) * C)
    return 4 * B * V * ((nt + 2 * C) if norm == 'paddle' else (nt + 1 + 3 * C))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--baseline-reps', type=int, default=3)
    ap.add_argument('--json', help='also append one JSON line per measurement to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_3d_k.py measures on a CUDA device; none is present')
    torch.cuda.set_device(0)
    name, power = card()
    print(f'card: {name}, power limit {power}; median of {a.reps} (baseline {a.baseline_reps})')
    rows = []
    cases = [(DEMO, K, norm, True) for K in (3, 5) for norm in (f'{K ** 3 - 1}sum', f'{K ** 3 - 1}sum_abs', 'paddle')]
    cases += [(CFG4, 5, norm, False) for norm in ('124sum', '124sum_abs', 'paddle')]
    for (B, C, D, H, W, N), K, norm, with_bwd in cases:
        nt, V = K ** 3 - 1, D * H * W
        gen = torch.Generator(device='cuda').manual_seed(0)
        g = torch.rand(B, nt, D, H, W, device='cuda', generator=gen)
        f = torch.rand(B, C, D, H, W, device='cuda', generator=gen)
        m = cspn_b200.Affinity_Propagate3DK(N, K, norm)
        with torch.no_grad():
            fwd = median_ms(lambda: m(g, f), a.reps)
        sb = step_bytes(B, C, V, K, norm)
        row = dict(card=name, power_limit=power, shape=f'{B}x{C}x{D}x{H}x{W}', K=K, N=N, norm=norm, fwd_ms=round(fwd, 3),
                   step_bytes=sb, fwd_TBps=round(sb * N / (fwd * 1e-3) / 1e12, 2))
        if with_bwd:
            gr, fr = g.clone().requires_grad_(True), f.clone().requires_grad_(True)
            go = torch.randn_like(f)

            def fwd_bwd():
                gr.grad = fr.grad = None
                m(gr, fr).backward(go)
            row['fwd_bwd_ms'] = round(median_ms(fwd_bwd, a.reps), 2)
            del gr, fr, go
            torch.cuda.empty_cache()
            with torch.no_grad():
                base = median_ms(lambda: tpk.cspn3d_torch_k(g, f, N, K, norm), a.baseline_reps, warmup=1)
            row.update(eager_port_fwd_ms=round(base, 1), speedup_fwd=round(base / fwd, 1))
        rows.append(row)
        print(json.dumps(row), flush=True)
        del g, f
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'a') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')
    print('\n| shape | K | norm | forward ms | fwd+bwd ms | eager port fwd ms | bytes / step | forward rate |')
    print('|---|---|---|---|---|---|---|---|')
    for r in rows:
        print(f"| {r['shape']} N={r['N']} | {r['K']} | {r['norm']} | {r['fwd_ms']} | {r.get('fwd_bwd_ms', '')} | "
              f"{r.get('eager_port_fwd_ms', '')} | {r['step_bytes'] / 1e6:.0f} MB | {r['fwd_TBps']} TB/s |")


if __name__ == '__main__':
    main()
