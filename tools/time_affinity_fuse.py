"""Times cspn_b200.affinity_fuse2d against the torch composition of the same op (tests/affinity_fuse_reference.py: abs, a
sum over the levels, a broadcast divide, F.interpolate of every level, L products and a sum) and against PSMNet's
F.interpolate of every level and torch.cat, the upsampling a fusion replaces, on the same GPU.

    python tools/time_affinity_fuse.py [--reps 30] [--json out.json]

Shapes: PSMNet's quarter-resolution feature map with C = 32 channels per level (the branch convolutions' width) and the
levels (H // p, W // p) of the pyramid p = (64, 32, 16, 8), align_corners=False, align_mode=0 (F.interpolate's rule):
the training crop B=4, 64x128; KITTI inference B=1, 96x312; the SceneFlow test size B=1, 136x240.  Per shape: the forward
under no_grad and forward + backward through autograd (the gradients of the levels and the gate from a fixed gradient of
the output; the concatenation's of the levels alone).  Each is timed eagerly, as a user calls it (host dispatch
included), and as a CUDA graph of 10 calls replayed, which leaves the device time alone.  CUDA events around each call,
warm-up first, the sides alternated call by call, medians reported.  The byte floor counts the gate, the levels and the
output once each way (forward: read the levels and gate, write out; backward: read them, out and grad_out, write both
gradients) over 3.35 TB/s, the H100 SXM's HBM3 bandwidth; its share is the floor over the fused op's device time.  The
card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import cspn_b200  # noqa: E402
from cspn_b200 import torch_op  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
C = 32
PS = (64, 32, 16, 8)
SHAPES = [('training crop', 4, 64, 128), ('KITTI inference', 1, 96, 312), ('SceneFlow test', 1, 136, 240)]


def compose(levels, gate):
    """The torch composition in fp32 with F.interpolate (align_corners=False is align_mode 0's rule)."""
    a = gate.abs()
    w = a / a.sum(dim=1, keepdim=True)
    H, W = gate.shape[2:]
    return sum(w[:, l:l + 1] * F.interpolate(x, size=(H, W), mode='bilinear', align_corners=False) for l, x in enumerate(levels))


def upsample_cat(levels, gate):
    """PSMNet: every level upsampled to the feature map and concatenated."""
    H, W = gate.shape[2:]
    return torch.cat([F.interpolate(x, size=(H, W), mode='bilinear', align_corners=False) for x in levels], 1)


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
    """(forward, backward) bytes read + written."""
    out, gate = B * C * H * W * 4, B * len(PS) * H * W * 4
    lv = B * C * sum((H // p) * (W // p) for p in PS) * 4
    return lv + gate + out, 2 * lv + 2 * gate + 2 * out


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
        levels = [torch.randn(B, C, H // p, W // p, device='cuda', generator=gen) for p in PS]
        gate = torch.randn(B, len(PS), H, W, device='cuda', generator=gen)
        grad = torch.randn(B, C, H, W, device='cuda', generator=gen)
        grad_cat = torch.randn(B, C * len(PS), H, W, device='cuda', generator=gen)
        sides = {'fused': (lambda xs, g: cspn_b200.affinity_fuse2d(xs, g, False, 0), grad),
                 'torch composition': (compose, grad),
                 'upsample+cat': (upsample_cat, grad_cat)}
        xr, gr = [x.clone().requires_grad_(True) for x in levels], gate.clone().requires_grad_(True)

        def fwd_of(f, _):
            def run():
                with torch.no_grad():
                    f(levels, gate)
            return run

        def fb_of(f, go):
            def run():
                for t in (*xr, gr):
                    t.grad = None
                f(xr, gr).backward(go)
            return run

        with torch.no_grad():
            diff = float((sides['fused'][0](levels, gate) - compose(levels, gate)).abs().max())
        fb, bb = bytes_moved(B, H, W)
        label = f'{name} B={B} C={C} {H}x{W} p={PS}'
        row = dict(shape=name, B=B, C=C, H=H, W=W, ps=list(PS), max_abs_diff_vs_composition=diff)
        lines = [f'{label}: out {B * C * H * W * 4 / 1e6:.2f} MB, max |fused - composition| {diff:.3g}']
        for what, maker, nbytes in (('fwd', fwd_of, fb), ('fwd_bwd', fb_of, fb + bb)):
            fns = [maker(f, go) for f, go in sides.values()]
            eager = timed(fns, a.reps)
            torch.cuda.empty_cache()
            dev = [t / 10 for t in timed([graphed(f) for f in fns], max(5, a.reps // 3))]
            torch.cuda.empty_cache()
            floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
            for k, e, d in zip(sides, eager, dev):
                key = k.replace(' ', '_').replace('+', '_')
                row[f'{what}_{key}_ms'] = round(e, 4)
                row[f'{what}_{key}_device_ms'] = round(d, 4)
            row[f'{what}_floor_ms'] = round(floor_ms, 4)
            row[f'{what}_floor_share'] = round(floor_ms / dev[0], 3)
            lines.append(f'  {what:8s} eager  ' + ' | '.join(f'{k} {e:.3f}' for k, e in zip(sides, eager)) + ' ms')
            lines.append(f'  {what:8s} device ' + ' | '.join(f'{k} {d:.3f}' for k, d in zip(sides, dev)) +
                         f' ms; byte floor {floor_ms:.4f} ms ({nbytes / 1e6:.1f} MB), fused at {floor_ms / dev[0]:.0%} of it')
        rows.append(row)
        print('\n'.join(lines), flush=True)
        del levels, gate, grad, grad_cat, xr, gr
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
