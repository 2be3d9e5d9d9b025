"""Times the 3x3 2D propagation's fallback routes (the generic forward, the backward on the K x K kernels at K = 3) through
the C ABI, at N = 24:

  - AUTO on odd W (the cluster kernel declines), 8x1x228x303 and 8x1x352x1215: forward, and forward + backward;
  - CSPN_ALGO_GENERIC forward and CSPN_B200_BWD=steps backward at 8x1x228x304 (W % 4 == 0);
  - a view 4 bytes off 16-byte alignment at 8x1x228x304 (AUTO forward, default backward);
  - the keep-sparse mode at 8x1x228x303.

Each --lib is loaded side by side and the libraries are alternated --rounds times, so drift hits all of them; CUDA events
around each call after a warm-up, median of --reps.  Several libraries (say, builds of two commits) are compared on the
same inputs, and each workload also says whether their forward outputs are bit for bit equal to the first library's.

    python tools/time_3x3_fallback.py [--lib A.so --lib B.so] [--rounds 3] [--reps 20] [--json out.jsonl]

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cspn_b200 import _lib  # noqa: E402
from cspn_b200.synth import make_inputs  # noqa: E402

N = 24
# name, (B, C, H, W), algo, CSPN_B200_BWD, misaligned, keep
WORKLOADS = [
    ('odd W, NYU', (8, 1, 228, 303), _lib.ALGO_AUTO, None, False, False),
    ('odd W, KITTI', (8, 1, 352, 1215), _lib.ALGO_AUTO, None, False, False),
    ('generic / BWD=steps', (8, 1, 228, 304), _lib.ALGO_GENERIC, 'steps', False, False),
    ('misaligned view', (8, 1, 228, 304), _lib.ALGO_AUTO, None, True, False),
    ('keep, odd W', (8, 1, 228, 303), _lib.ALGO_AUTO, None, False, True),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q


def load(path):
    L = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


def tensor(t, misaligned):
    """t on the GPU; misaligned: a view 4 bytes past a 16-byte aligned base."""
    if not misaligned:
        return t.cuda().contiguous()
    buf = torch.empty(t.numel() + 1, device='cuda')
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


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


def calls(L, shape, algo, keep, t, ws, st):
    """(forward, backward) of library L on the tensors t, each raising on a failed status."""
    B, C, H, W = shape
    ptr = lambda x: None if x is None else x.data_ptr()
    g, d, s, out, go, gg, gd, gs = (ptr(t[k]) for k in ('g', 'd', 's', 'out', 'go', 'gg', 'gd', 'gs'))

    def check(rc, what):
        if rc != 0:
            raise RuntimeError(f'{what}: status {rc}: {L.cspn_last_error().decode()}')

    if keep:
        fwd = lambda: check(L.cspn2d_keep_fwd_f32(g, d, s, out, B, C, H, W, 8, 3, N, 0, algo, ws.data_ptr(), ws.numel(), st), 'fwd')
        bwd = lambda: check(L.cspn2d_keep_bwd_f32(g, d, s, go, gg, gd, gs, B, C, H, W, 8, 3, N, 0, ws.data_ptr(), ws.numel(), st),
                            'bwd')
    else:
        fwd = lambda: check(L.cspn2d_fwd_f32(g, d, s, out, B, C, H, W, 8, N, 0, algo, ws.data_ptr(), ws.numel(), st), 'fwd')
        bwd = lambda: check(L.cspn2d_bwd_f32(g, d, s, go, gg, gd, B, C, H, W, 8, N, 0, ws.data_ptr(), ws.numel(), st), 'bwd')
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', help='library to time (repeatable); default: the in-tree build')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('time_3x3_fallback: no CUDA device')
    paths = a.lib or [_lib.LIB_PATH]
    libs = [load(p) for p in paths]
    name, power = card()
    print(f'# {name}, power limit / max SM clock: {power}')
    print('# ' + ' | '.join(f'L{i} = {p}' for i, p in enumerate(paths)))
    st = torch.cuda.current_stream().cuda_stream
    rows = []
    for wname, shape, algo, bwd_env, misaligned, keep in WORKLOADS:
        B, C, H, W = shape
        g, d, s = make_inputs(0, B, C, H, W)
        go = torch.rand(B, C, H, W, generator=torch.Generator().manual_seed(1))
        t = {k: tensor(v, misaligned) for k, v in (('g', g), ('d', d), ('s', s), ('go', go))}
        for k, shp in (('out', (B, C, H, W)), ('gg', (B, 8, H, W)), ('gd', (B, C, H, W)), ('gs', (B, 1, H, W))):
            t[k] = tensor(torch.empty(shp), misaligned)
        if bwd_env:
            os.environ['CSPN_B200_BWD'] = bwd_env
        else:
            os.environ.pop('CSPN_B200_BWD', None)
        need = 0
        for L in libs:
            if keep:
                need = max(need, L.cspn2d_keep_workspace_bytes(B, C, H, W, 3, N, algo), L.cspn2d_keep_workspace_bytes(
                    B, C, H, W, 3, N, _lib.ALGO_GENERIC), L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, 3, N))
            else:
                need = max(need, L.cspn2d_workspace_bytes(B, C, H, W, N, algo), L.cspn2d_workspace_bytes(
                    B, C, H, W, N, _lib.ALGO_GENERIC), L.cspn2d_bwd_workspace_bytes(B, C, H, W, N))
        ws = torch.empty(need, dtype=torch.uint8, device='cuda')
        fns = [calls(L, shape, algo, keep, t, ws, st) for L in libs]
        times = {(i, what): [] for i in range(len(libs)) for what in ('fwd', 'fwd+bwd')}
        for _ in range(a.rounds):
            for i, (fwd, bwd) in enumerate(fns):
                times[(i, 'fwd')].append(median_ms(fwd, a.reps))
                times[(i, 'fwd+bwd')].append(median_ms(lambda: (fwd(), bwd()), a.reps))
        outs = []
        for fwd, _ in fns:   # each library's forward result, for the bit comparison
            fwd()
            outs.append(t['out'].clone())
        same = [torch.equal(outs[0], o) for o in outs]
        for what in ('fwd', 'fwd+bwd'):
            cells = []
            for i in range(len(libs)):
                ms = times[(i, what)]
                cells.append(f'L{i} {min(ms):.3f}-{max(ms):.3f} ms')
                rows.append({'workload': wname, 'shape': list(shape), 'what': what, 'lib': paths[i], 'ms': ms,
                             'out_equal_L0': same[i], 'card': name, 'power': power})
            print(f'{wname:20s} {what:8s} ' + ' | '.join(cells), flush=True)
        print(f'{wname:20s} out bit for bit equal to L0: {same}', flush=True)
    os.environ.pop('CSPN_B200_BWD', None)
    if a.json:
        with open(a.json, 'w') as fh:
            for r in rows:
                fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
