"""Times cspn_b200.disparity_regression against the two chains a user would otherwise write, on the same GPU:
F.interpolate(mode='trilinear', align_corners=True) -> softmax -> sum(o * p), and cspn_b200.resize_trilinear -> softmax ->
sum(o * p).

    python tools/time_disparity_regression.py [--reps 30] [--json out.json]

Shapes: the quarter-resolution cost volume of a 256x512 training crop with 192 disparities, 4x1x48x64x128 -> 192x256x512,
and KITTI inference at full resolution, 1x1x48x96x312 -> 192x384x1248.  Per shape: the forward under no_grad and
forward + backward through autograd (grad of the cost from a fixed grad_out).  Each is timed twice: eagerly, as a user calls
it (host dispatch included), and as a CUDA graph of 10 calls replayed, which leaves the device time alone.  CUDA events
around each call, warm-up first, the three sides alternated call by call, medians reported.  The peak of
torch.cuda.max_memory_allocated above the inputs is taken over one forward + backward of each side.  The card's name and
power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cspn_b200  # noqa: E402
from cspn_b200 import torch_op  # noqa: E402

SHAPES = [('training crop', (4, 1, 48, 64, 128), (192, 256, 512)), ('KITTI inference', (1, 1, 48, 96, 312), (192, 384, 1248))]


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


def regress(u):
    o = torch.arange(u.shape[2], dtype=u.dtype, device=u.device)[:, None, None]
    return (torch.softmax(u, dim=2) * o).sum(2)


def peak_mb(f):
    """max_memory_allocated above what is allocated before f, in MB."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    f()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e6


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
    for name, shape, size in SHAPES:
        x = torch.randn(*shape, device='cuda') * 3
        g = torch.randn(*shape[:2], *size[1:], device='cuda')
        xr = x.clone().requires_grad_(True)
        sides = {
            'fused': lambda t: cspn_b200.disparity_regression(t, size, align_corners=True),
            'interpolate': lambda t: regress(F.interpolate(t, size=size, mode='trilinear', align_corners=True)),
            'resize_trilinear': lambda t: regress(cspn_b200.resize_trilinear(t, size, align_corners=True)),
        }

        def fwd_of(f):
            def run():
                with torch.no_grad():
                    f(x)
            return run

        def fb_of(f):
            def run():
                xr.grad = None
                f(xr).backward(g)
            return run

        with torch.no_grad():
            ys = {k: f(x) for k, f in sides.items()}
        diff = {k: float((ys['fused'] - ys[k]).abs().max()) for k in ys if k != 'fused'}
        del ys
        peaks = {k: round(peak_mb(fb_of(f)), 2) for k, f in sides.items()}
        volume_mb = 4 * shape[0] * shape[1] * size[0] * size[1] * size[2] / 1e6
        row = dict(shape=name, input=list(shape), output=list(size), upsampled_mb=round(volume_mb, 2),
                   max_abs_diff_vs=diff, peak_fwd_bwd_mb=peaks)
        line = [f'{name} {tuple(shape)} -> {size} (upsampled volume {volume_mb:.2f} MB): max |fused - chain| {diff}',
                f'  peak max_memory_allocated of fwd+bwd above the inputs, MB: {peaks}']
        for what, maker in (('fwd', fwd_of), ('fwd_bwd', fb_of)):
            fns = [maker(f) for f in sides.values()]
            eager = timed(fns, a.reps)
            torch.cuda.empty_cache()
            dev = [t / 10 for t in timed([graphed(f) for f in fns], max(5, a.reps // 3))]
            torch.cuda.empty_cache()
            for k, e, d in zip(sides, eager, dev):
                row[f'{what}_{k}_ms'] = round(e, 4)
                row[f'{what}_{k}_device_ms'] = round(d, 4)
            line.append(f'  {what:8s} eager ' + ' | '.join(f'{k} {e:.3f}' for k, e in zip(sides, eager)) + ' ms')
            line.append(f'  {what:8s} device ' + ' | '.join(f'{k} {d:.3f}' for k, d in zip(sides, dev)) + ' ms')
        rows.append(row)
        print('\n'.join(line), flush=True)
        del x, g, xr
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
