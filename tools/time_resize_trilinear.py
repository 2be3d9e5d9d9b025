"""Times cspn_b200.resize_trilinear against F.interpolate(mode='trilinear', align_corners=True), the one mode both have, on
the same GPU.

    python tools/time_resize_trilinear.py [--reps 50] [--json out.json]

Shapes: demo.py's volume 3x1x48x64x128 upsampled x2, and a stereo cost volume 4x1x48x64x128 upsampled to 192x256x512
(403 MB of output).  Per shape: the forward under no_grad, forward + backward through autograd (grad of x from a fixed
grad_out), and the backward op alone (cspn_b200::resize_trilinear_backward against aten::upsample_trilinear3d_backward, the
zero fill and atomics of F.interpolate's backward).  Each is timed twice: eagerly, as a user calls it (host dispatch
included), and as a CUDA graph of 10 calls replayed, which leaves the device time alone.  CUDA events around each call,
warm-up first, the two sides alternated call by call, medians reported.  The byte floor is
4 * (V_in + V_out) bytes each way (read one volume, write the other), over the 3.35 TB/s of the H100 SXM data sheet; the
card's name and power limit are read in the same run."""
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

SHAPES = [('demo x2', (3, 1, 48, 64, 128), (96, 128, 256)), ('cost volume', (4, 1, 48, 64, 128), (192, 256, 512))]
HBM_TBS = 3.35


def timed(fns, reps, warmup=5):
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


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--json')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch_op.load()
    info = card()
    print('card:', info)
    rows = []
    for name, shape, size in SHAPES:
        x = torch.randn(*shape, device='cuda')
        g = torch.randn(*shape[:2], *size, device='cuda')
        xr = x.clone().requires_grad_(True)

        def ours_fwd():
            with torch.no_grad():
                cspn_b200.resize_trilinear(x, size, align_corners=True)

        def torch_fwd():
            with torch.no_grad():
                F.interpolate(x, size=size, mode='trilinear', align_corners=True)

        def ours_fb():
            xr.grad = None
            cspn_b200.resize_trilinear(xr, size, align_corners=True).backward(g)

        def torch_fb():
            xr.grad = None
            F.interpolate(xr, size=size, mode='trilinear', align_corners=True).backward(g)

        with torch.no_grad():
            diff = float((cspn_b200.resize_trilinear(x, size) - F.interpolate(x, size=size, mode='trilinear',
                                                                               align_corners=True)).abs().max())
        v_in, v_out = x.numel(), g.numel()
        floor_ms = 4 * (v_in + v_out) / (HBM_TBS * 1e12) * 1e3

        def ours_bwd():
            torch.ops.cspn_b200.resize_trilinear_backward(g, *shape[2:], True, 1)

        def torch_bwd():
            torch.ops.aten.upsample_trilinear3d_backward(g, list(size), list(shape), True)

        row = dict(shape=name, input=list(shape), output=list(size), floor_ms=round(floor_ms, 4), max_abs_diff_vs_torch=diff)
        line = [f'{name} {tuple(shape)} -> {size}: byte floor {floor_ms:.3f} ms each way, max |ours - torch| {diff:.2e}']
        for what, pair in (('fwd', (ours_fwd, torch_fwd)), ('fwd_bwd', (ours_fb, torch_fb)), ('bwd_op', (ours_bwd, torch_bwd))):
            eager = timed(list(pair), a.reps)
            dev = [t / 10 for t in timed([graphed(f) for f in pair], max(5, a.reps // 5))]
            row.update({f'{what}_ms': round(eager[0], 4), f'{what}_torch_ms': round(eager[1], 4),
                        f'{what}_device_ms': round(dev[0], 4), f'{what}_torch_device_ms': round(dev[1], 4)})
            line.append(f'  {what:8s} eager {eager[0]:.3f} ms (torch {eager[1]:.3f}) | device {dev[0]:.3f} ms '
                        f'(torch {dev[1]:.3f})')
        rows.append(row)
        print('\n'.join(line))
        del x, g, xr
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
