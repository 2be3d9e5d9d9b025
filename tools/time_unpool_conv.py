"""Times the guidance / depth heads (Unpool + crop + 3x3 convolution) as one cspn_b200 kernel against the reference's op
sequence (conv_transpose2d, narrow, cuDNN conv2d; torch_resnet_cspn_nyu.py:41-54, 187-205) on the same GPU.

    python tools/time_unpool_conv.py [--batch 8] [--reps 30] [--json out.json]

cudnn.benchmark = True, as train.py:166 and eval.py:118 set it, under allow_tf32 True (PyTorch's default for cuDNN
convolutions) and False.  Per shape (NYU and KITTI heads, Cout 8 and 1): the forward under no_grad, and forward + backward
(grads of x and weight); then the whole tail, both heads + Affinity_Propagate(24, 3, '8sum').  CUDA events around each
call, warm-up first, the two sides alternated call by call, medians reported.  Bytes and MACs are computed from the
shapes; the card's name and power limit are read in the same run."""
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

SHAPES = {'nyu': (64, 114, 152, 228, 304), 'kitti': (64, 176, 608, 352, 1216)}


def op_sequence(x, weight, H, W):
    C = x.shape[1]
    k = torch.zeros(C, 1, 2, 2, dtype=x.dtype, device=x.device)
    k[:, :, 0, 0] = 1
    return F.conv2d(F.conv_transpose2d(x, k, stride=2, groups=C).narrow(2, 0, H).narrow(3, 0, W), weight, padding=1)


def fused(x, weight, H, W):
    return cspn_b200.unpool_conv3x3(x, weight, H, W)


def counts(B, Cin, h, w, Cout, H, W):
    """Minimum algorithmic bytes and MACs of one head, fp32: read x and weight, write out."""
    return 4 * (B * Cin * h * w + Cout * Cin * 9 + B * Cout * H * W), B * ((H + 1) // 2) * ((W + 1) // 2) * Cin * Cout * 9


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


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                     # the name still comes from torch
        q = f'{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})'
    return q


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--json')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.backends.cudnn.benchmark = True
    info = card()
    print('card:', info)
    rows = []
    B = a.batch
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        for name, (Cin, h, w, H, W) in SHAPES.items():
            g = torch.Generator(device='cuda').manual_seed(0)
            x = torch.randn(B, Cin, h, w, device='cuda', generator=g)
            for Cout in (8, 1):
                wt = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) / 24
                nbytes, macs = counts(B, Cin, h, w, Cout, H, W)
                with torch.no_grad():
                    t_f, t_r = timed([lambda: fused(x, wt, H, W), lambda: op_sequence(x, wt, H, W)], a.reps)
                xr, wr = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
                go = torch.randn(B, Cout, H, W, device='cuda', generator=g)

                def fb(f):
                    return lambda: torch.autograd.backward(f(xr, wr, H, W), go)

                tb_f, tb_r = timed([fb(fused), fb(op_sequence)], a.reps)
                row = dict(tf32=tf32, shape=name, B=B, Cout=Cout, bytes=nbytes, macs=macs, fwd_fused_ms=t_f, fwd_ops_ms=t_r,
                           fwdbwd_fused_ms=tb_f, fwdbwd_ops_ms=tb_r)
                rows.append(row)
                print(f'tf32={tf32!s:5} {name:5} B={B} Cout={Cout}: bytes {nbytes / 1e6:7.1f} MB, MACs {macs / 1e9:6.2f} G | '
                      f'fwd fused {t_f:7.3f} ms  ops {t_r:7.3f} ms  ({t_r / t_f:5.2f}x) | fwd+bwd fused {tb_f:7.3f} ms  '
                      f'ops {tb_r:7.3f} ms  ({tb_r / tb_f:5.2f}x)', flush=True)
            # the whole tail: both heads and the propagation
            w6 = torch.randn(8, Cin, 3, 3, device='cuda', generator=g) / 24
            w5 = torch.randn(1, Cin, 3, 3, device='cuda', generator=g) / 24
            sparse = (torch.rand(B, 1, H, W, device='cuda', generator=g) < 0.01).float() * 5
            prop = cspn_b200.Affinity_Propagate(24, 3, '8sum')

            def tail(f):
                return lambda: prop(f(x, w6, H, W), f(x, w5, H, W), sparse)

            with torch.no_grad():
                tt_f, tt_r = timed([tail(fused), tail(op_sequence)], a.reps)
            rows.append(dict(tf32=tf32, shape=name, B=B, tail=True, tail_fused_ms=tt_f, tail_ops_ms=tt_r))
            print(f'tf32={tf32!s:5} {name:5} B={B} tail (both heads + Affinity_Propagate 24 steps, no_grad): fused {tt_f:7.3f} ms  '
                  f'ops {tt_r:7.3f} ms  ({tt_r / tt_f:5.2f}x)', flush=True)
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
