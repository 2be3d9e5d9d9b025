"""Times cspn_b200.affinity_atrous_pool2d against the torch composition of the same op (tests/affinity_atrous_reference.py:
per rate an F.unfold, abs, a sum, a broadcast divide, a product and a sum) on the same GPU.

    python tools/time_affinity_atrous.py [--reps 30] [--json out.json]

Shapes: PSMNet's quarter-resolution feature map with C = 128 channels and DeepLab's rates (6, 12, 18, 24): the training
crop B=4, 64x128; KITTI inference B=1, 96x312; the SceneFlow test size B=1, 136x240.  Per shape: the forward under
no_grad and forward + backward through autograd (the gradients of feat and gate from a fixed gradient of the output).
Each is timed eagerly, as a user calls it (host dispatch included), and as a CUDA graph of 10 calls replayed, which leaves
the device time alone.  CUDA events around each call, warm-up first, the sides alternated call by call, medians reported.
The byte floor counts what must cross HBM at least once over 3.35 TB/s, the H100 SXM's HBM3 bandwidth: the forward reads
feat and gate and writes the (B, L*C, H, W) output; forward + backward also reads the output's gradient and writes both
gradients, feat and gate counted once (at these shapes feat is at most 17 MB and stays in L2).  Its share is the floor
over the fused op's device time.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import cspn_b200  # noqa: E402
from cspn_b200 import torch_op  # noqa: E402
import affinity_atrous_reference as ar  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
C = 128
RATES = (6, 12, 18, 24)
SHAPES = [('training crop', 4, 64, 128), ('KITTI inference', 1, 96, 312), ('SceneFlow test', 1, 136, 240)]


def timed(fns, reps, warmup=3):
    """Median time in ms of each callable, the callables alternated call by call."""
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts[k].append(a.elapsed_time(b))
    return [statistics.median(t) for t in ts]


def graphed(f, n=10):
    """A callable that replays a CUDA graph of n calls of f; its time / n is f's device time without host dispatch."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            f()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            f()
    return g.replay


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                     # the name still comes from torch
        q = f'{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})'
    return q


def bytes_moved(B, H, W):
    """(forward, forward + backward) bytes that must cross HBM."""
    feat, gate, out = B * C * H * W * 4, B * 9 * len(RATES) * H * W * 4, B * len(RATES) * C * H * W * 4
    return feat + gate + out, 2 * (feat + gate + out)


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--json')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch_op.load()
    info = card()
    print('card:', info)
    rows = []
    for name, B, H, W in SHAPES:
        gen = torch.Generator('cuda').manual_seed(0)
        feat = torch.randn(B, C, H, W, device='cuda', generator=gen)
        gate = torch.randn(B, 9 * len(RATES), H, W, device='cuda', generator=gen)
        grad = torch.randn(B, len(RATES) * C, H, W, device='cuda', generator=gen)
        sides = {'fused': lambda f, g: cspn_b200.affinity_atrous_pool2d(f, g, RATES),
                 'torch composition': lambda f, g: ar.compose(f, g, RATES)}
        fr, gr = feat.clone().requires_grad_(True), gate.clone().requires_grad_(True)

        def fwd_of(f):
            def run():
                with torch.no_grad():
                    f(feat, gate)
            return run

        def fb_of(f):
            def run():
                fr.grad = gr.grad = None
                f(fr, gr).backward(grad)
            return run

        with torch.no_grad():
            diff = float((sides['fused'](feat, gate) - sides['torch composition'](feat, gate)).abs().max())
        fb, fbb = bytes_moved(B, H, W)
        label = f'{name} B={B} C={C} {H}x{W} r={RATES}'
        row = dict(shape=name, B=B, C=C, H=H, W=W, rates=list(RATES), max_abs_diff_vs_composition=diff)
        lines = [f'{label}: feat {feat.numel() * 4 / 1e6:.2f} MB, max |fused - composition| {diff:.3g}']
        for what, maker, nbytes in (('fwd', fwd_of, fb), ('fwd_bwd', fb_of, fbb)):
            fns = [maker(f) for f in sides.values()]
            eager = timed(fns, a.reps)
            torch.cuda.empty_cache()
            dev = [t / 10 for t in timed([graphed(f) for f in fns], max(5, a.reps // 3))]
            torch.cuda.empty_cache()
            floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
            for k, e, d in zip(sides, eager, dev):
                row[f'{what}_{k.replace(" ", "_")}_ms'] = round(e, 4)
                row[f'{what}_{k.replace(" ", "_")}_device_ms'] = round(d, 4)
            row[f'{what}_floor_ms'] = round(floor_ms, 4)
            row[f'{what}_floor_share'] = round(floor_ms / dev[0], 3)
            lines.append(f'  {what:8s} eager  ' + ' | '.join(f'{k} {e:.3f}' for k, e in zip(sides, eager)) + ' ms')
            lines.append(f'  {what:8s} device ' + ' | '.join(f'{k} {d:.3f}' for k, d in zip(sides, dev)) +
                         f' ms; byte floor {floor_ms:.4f} ms ({nbytes / 1e6:.1f} MB), fused at {floor_ms / dev[0]:.0%} of it')
        rows.append(row)
        print('\n'.join(lines), flush=True)
        del feat, gate, grad, fr, gr
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
