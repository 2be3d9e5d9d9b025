"""Times cspn_b200.build_concat_volume and build_gwc_volume against the loops a PSMNet or GwcNet port runs (a zero-filled
volume and slice writes per disparity, tests/cost_volume_reference.py), on the same GPU.

    python tools/time_cost_volume.py [--reps 30] [--json out.json]

Shapes: the quarter-resolution volumes of a 256x512 training crop, B=4, 64x128, D=48, and of KITTI inference, B=1, 96x312,
D=48; the concatenation volume with F=32 features, the group-wise correlation volume with F=320 and G=40 (GwcNet's).
Per shape and volume: the forward under no_grad and forward + backward through autograd (the gradients of both feature
maps from a fixed grad_out).  Each is timed eagerly, as a user calls it (host dispatch included), and as a CUDA graph of
10 calls replayed, which leaves the device time alone.  CUDA events around each call, warm-up first, the two sides
alternated call by call, medians reported.  The byte floor is (bytes read + bytes written) / 3.35 TB/s, the H100 SXM's
HBM3 bandwidth; its share is the floor over the fused op's device time.  The card's name and power limit are read in the
same run."""
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
import cost_volume_reference as cr  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = [('training crop', 4, 64, 128, 48), ('KITTI inference', 1, 96, 312, 48)]
VOLUMES = [('concat', 32, None), ('gwc', 320, 40)]


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


def bytes_moved(kind, B, F, H, W, D, G):
    """(forward, backward) bytes read + written: features 2*B*F*H*W floats each way, the volume once."""
    feat = 2 * B * F * H * W * 4
    vol = B * (2 * F if kind == 'concat' else G) * D * H * W * 4
    if kind == 'concat':
        return feat + vol, vol + feat                          # backward: read g, write both gradients
    return feat + vol, feat + vol + feat                       # backward: read both features and g, write both gradients


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
    for name, B, H, W, D in SHAPES:
        for kind, F, G in VOLUMES:
            gen = torch.Generator('cuda').manual_seed(0)
            L = torch.randn(B, F, H, W, device='cuda', generator=gen)
            R = torch.randn(B, F, H, W, device='cuda', generator=gen)
            if kind == 'concat':
                sides = {'fused': lambda l, r: cspn_b200.build_concat_volume(l, r, D),
                         'torch loop': lambda l, r: cr.concat_loop(l, r, D)}
                gshape = (B, 2 * F, D, H, W)
            else:
                sides = {'fused': lambda l, r: cspn_b200.build_gwc_volume(l, r, D, G),
                         'torch loop': lambda l, r: cr.gwc_loop(l, r, D, G)}
                gshape = (B, G, D, H, W)
            g = torch.randn(*gshape, device='cuda', generator=gen)
            Lr, Rr = L.clone().requires_grad_(True), R.clone().requires_grad_(True)

            def fwd_of(f):
                def run():
                    with torch.no_grad():
                        f(L, R)
                return run

            def fb_of(f):
                def run():
                    Lr.grad = Rr.grad = None
                    f(Lr, Rr).backward(g)
                return run

            with torch.no_grad():
                diff = float((sides['fused'](L, R) - sides['torch loop'](L, R)).abs().max())
            fb, bb = bytes_moved(kind, B, F, H, W, D, G)
            label = f'{name} {kind} B={B} F={F}' + (f' G={G}' if G else '') + f' {H}x{W} D={D}'
            row = dict(shape=name, volume=kind, B=B, F=F, G=G, H=H, W=W, D=D, volume_mb=round(g.numel() * 4 / 1e6, 2),
                       max_abs_diff_vs_loop=diff)
            lines = [f'{label}: volume {g.numel() * 4 / 1e6:.2f} MB, max |fused - loop| {diff:.3g}']
            for what, maker, nbytes in (('fwd', fwd_of, fb), ('fwd_bwd', fb_of, fb + bb)):
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
                             f' ms; byte floor {floor_ms:.3f} ms ({nbytes / 1e6:.1f} MB), fused at {floor_ms / dev[0]:.0%} of it')
            rows.append(row)
            print('\n'.join(lines), flush=True)
            del L, R, g, Lr, Rr
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
