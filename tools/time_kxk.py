"""Times the K x K 2D propagation (K = 3, 5, 7) at N = 24 on the NYU (8x1x228x304) and KITTI (8x1x352x1216) batch shapes:

  - forward under no_grad and forward + backward through Affinity_PropagateK, CUDA events, warm-up, median of --reps;
  - the torch port's eager op sequence (oracle/cspn_torch_port_k.py::cspn2d_torch_k) on the same GPU as the baseline;
  - for K = 5 / 7, the forward in launch groups sized so their weight planes fit the L2 (forced through
    CSPN_B200_KXK_GROUP) against the library's one group for the whole batch, alternated;
  - the bytes a step moves, computed from shapes, and where its weight planes come from (L2 or HBM).

    python tools/time_kxk.py [--reps 20] [--baseline-reps 5] [--json out.jsonl]

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
from oracle import cspn_torch_port_k as tpk  # noqa: E402

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


def group_images(B, K, H, W, l2):
    """Images per group whose K*K weight planes fit the L2 (at least one)."""
    return max(1, min(B, l2 // (4 * K * K * H * W)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--baseline-reps', type=int, default=5)
    ap.add_argument('--json', help='also append one JSON line per measurement to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_kxk.py measures on a CUDA device; none is present')
    torch.cuda.set_device(0)
    name, power = card()
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    print(f'card: {name}, power limit {power}, L2 {l2 / 2**20:.0f} MiB; N = {N}, median of {a.reps} (baseline {a.baseline_reps})')
    rows = []
    for shape_name, (B, C, H, W) in SHAPES.items():
        for K in (3, 5, 7):
            nt = K * K - 1
            g, d, s = [t.cuda() for t in make_inputs(0, B, C, H, W, nt)]
            m = cspn_b200.Affinity_PropagateK(N, K)
            with torch.no_grad():
                fwd = median_ms(lambda: m(g, d, s), a.reps)
            gr, dr = g.clone().requires_grad_(True), d.clone().requires_grad_(True)
            go = torch.randn_like(d)

            def fwd_bwd():
                gr.grad = dr.grad = None
                m(gr, dr, s).backward(go)
            fb = median_ms(fwd_bwd, a.reps)
            with torch.no_grad():
                base = median_ms(lambda: tpk.cspn2d_torch_k(g, d, s, N, K), a.baseline_reps, warmup=1)
            row = dict(card=name, power_limit=power, shape=f'{B}x{C}x{H}x{W}', K=K, N=N, fwd_ms=round(fwd, 3),
                       fwd_bwd_ms=round(fb, 3), eager_port_fwd_ms=round(base, 2), speedup_fwd=round(base / fwd, 1))
            HW = H * W
            if K > 3:
                G = group_images(B, K, H, W, l2)
                step_bytes = 4 * B * HW * (K * K + 3 * C)          # K*K weight planes + d_t, d_0 read + d_{t+1} written
                fits = 4 * K * K * HW <= l2
                # the library runs the batch as one group: its weight planes come from L2 only if they all fit there
                row.update(step_bytes=step_bytes, weights_from='L2' if 4 * K * K * HW * B <= l2 else 'HBM',
                           l2_group_images=G, l2_group_weights_from='L2' if fits else 'HBM',
                           fwd_step_GBps=round(step_bytes * N / (fwd * 1e-3) / 1e9))
                # launch groups sized to the L2 vs one group for the whole batch, alternated
                grouped, whole = [], []
                with torch.no_grad():
                    for _ in range(3):
                        os.environ['CSPN_B200_KXK_GROUP'] = str(G)
                        grouped.append(median_ms(lambda: m(g, d, s), max(5, a.reps // 2)))
                        os.environ.pop('CSPN_B200_KXK_GROUP', None)
                        whole.append(median_ms(lambda: m(g, d, s), max(5, a.reps // 2)))
                row.update(fwd_ms_l2_groups=round(statistics.median(grouped), 3),
                           fwd_ms_one_group=round(statistics.median(whole), 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
            del g, d, s, gr, dr, go
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'a') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')
    print('\n| shape | K | forward ms | fwd+bwd ms | eager port fwd ms | bytes/step (weights from) | fwd GB/s | '
          'forward ms in L2-sized groups (images, weights from) |')
    print('|---|---|---|---|---|---|---|---|')
    for r in rows:
        extra = (f"{r['step_bytes'] / 1e6:.0f} MB ({r['weights_from']}) | {r['fwd_step_GBps']} | "
                 f"{r['fwd_ms_l2_groups']} ({r['l2_group_images']}, {r['l2_group_weights_from']}) vs "
                 f"{r['fwd_ms_one_group']} in one group") if r['K'] > 3 else 'cluster kernel | | '
        print(f"| {r['shape']} | {r['K']} | {r['fwd_ms']} | {r['fwd_bwd_ms']} | {r['eager_port_fwd_ms']} | {extra} |")


if __name__ == '__main__':
    main()
