"""Multi-GPU check of the fused / chunked final gather (run under torchrun on 2..8 GPUs of one box):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
        tools/gather_check.py [B H W N] [--families]
    ... tools/gather_check.py --3d [B D H W N]

Every rank propagates its own images; every gather route must leave the same full batch on every rank, bit for bit equal
to each rank's own plain forward after a serial NCCL all-gather.  Prints one line per route with its time per call (CUDA
events, max over ranks).  The 3x3 operator (propagate2d) always runs; --families adds the K x K operator with K = 5 and
7 (propagate_k), the Paddle module's own-location gates (propagate_paddle, K = 5) and caller-supplied gates
(affinity_propagate, K = 5).  --3d runs the 3D routes instead, on B single-channel volumes per rank (default
2 x 1 x 64 x 96 x 312, N = 12): the 3x3x3 operator with 'paddle' and '26sum_abs' (propagate3d), the 5x5x5 one with
'paddle' (propagate3d_k) and 3x3x3 caller-supplied gates (affinity_propagate3d).  They have no chunked route."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

import cspn_b200
from cspn_b200.gather import ChunkedGather, FusedGather
from cspn_b200.sharding import gather_outputs
from cspn_b200.synth import make_inputs, make_inputs_3d

FAMILIES = '--families' in sys.argv
THREE_D = '--3d' in sys.argv
ARGS = [int(a) for a in sys.argv[1:] if a not in ('--families', '--3d')]
if THREE_D:
    B, D, H, W, N = ARGS[:5] if len(ARGS) > 4 else (2, 64, 96, 312, 12)
else:
    B, H, W, N = ARGS[:4] if len(ARGS) > 3 else (32, 352, 1216, 24)
rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)


def inputs(seed, gch):
    g, d, s = [t.to(dev) for t in make_inputs(seed, min(B, 8), 1, H, W, gch)]
    if B > 8:
        g, d, s = [t.repeat((B + 7) // 8, 1, 1, 1)[:B].contiguous() for t in (g, d, s)]
    return g, d, s


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    dist.barrier()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(b) / reps], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def report(name, ms, ok, extra=''):
    oks = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(oks, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(f'{name}: {ms:.4f} ms/call on {world} GPUs, identical on every rank: {bool(oks.item())} {extra}', flush=True)
    return bool(oks.item())


def check_routes(op, shape, plain, fused, chunked=None):
    """shape: this rank's (B, C, H, W) or (B, C, D, H, W); plain() -> this rank's result of that shape; fused(FusedGather)
    and chunked(ChunkedGather) -> the gathered batch."""
    mine = plain()
    ref = gather_outputs(mine, world * B)                   # kernel, then NCCL all_gather_into_tensor
    ok = torch.equal(ref[rank * B:(rank + 1) * B], mine)
    full = torch.empty(world * B, *shape[1:], device=dev)
    ok &= report(f'{op}: kernel only', timed(plain), True)
    ok &= report(f'{op}: serial NCCL (kernel, then all_gather_into_tensor)',
                 timed(lambda: dist.all_gather_into_tensor(full, plain())), torch.equal(full, ref))
    if chunked is not None and B % 4 == 0:
        cg = ChunkedGather(*shape, dev, n_chunks=4)
        ms = timed(lambda: chunked(cg))
        ok &= report(f'{op}: chunked NCCL (4 chunks, kernel i+1 overlaps gather i)', ms, torch.equal(cg.as_rank_major(), ref))
    for mc in (True, False):
        try:
            fg = FusedGather(*shape[:2], *shape[-2:], dev, multicast=mc, D=shape[2] if len(shape) == 5 else None)
            ms = timed(lambda: fused(fg))
            res = fused(fg)
            torch.cuda.synchronize()
            ok &= report(f'{op}: fused ({fg.mode})', ms, torch.equal(res, ref))
            if fg.mode == 'peer_stores':
                break
        except Exception as e:                                 # noqa: BLE001 -- report and go on with the other routes
            if rank == 0:
                print(f'{op}: fused (multicast={mc}) unavailable: {type(e).__name__}: {str(e)[:300]}', flush=True)
    return ok


def check_3d():
    shape = (B, 1, D, H, W)
    g, f = [t.to(dev) for t in make_inputs_3d(rank, B, 1, D, H, W)]
    ok = True
    for norm in ('paddle', '26sum_abs'):
        ok &= check_routes(f'propagate3d 3x3x3 {norm}', shape, lambda norm=norm: cspn_b200.propagate3d(g, f, N, norm),
                           lambda fg, norm=norm: fg.propagate3d(g, f, N, norm))
    g5 = torch.rand(B, 124, D, H, W, generator=torch.Generator().manual_seed(rank + 5)).to(dev)
    ok &= check_routes('propagate3d_k 5x5x5 paddle', shape, lambda: cspn_b200.propagate3d_k(g5, f, 5, N, 'paddle'),
                       lambda fg: fg.propagate3d_k(g5, f, 5, N, 'paddle'))
    gates = g / g.sum(1, keepdim=True)                          # demo.py's normalisation (g >= 0), done by the caller
    ok &= check_routes('affinity_propagate3d 3x3x3', shape, lambda: cspn_b200.affinity_propagate(f, gates, 3, N),
                       lambda fg: fg.affinity_propagate3d(f, gates, 3, N))
    return ok


if THREE_D:
    all_ok = check_3d()
else:
    g, d, s = inputs(rank, 8)
    all_ok = check_routes('propagate2d 3x3', (B, 1, H, W), lambda: cspn_b200.propagate2d(g, d, s, N, '8sum'),
                          lambda fg: fg.propagate(g, d, s, N, '8sum'), lambda cg: cg.propagate(g, d, s, N, '8sum'))
if FAMILIES and not THREE_D:
    for K in (5, 7):
        gk, dk, sk = inputs(rank + 100 * K, K * K - 1)
        all_ok &= check_routes(f'propagate2d_k {K}x{K}', (B, 1, H, W), lambda gk=gk, dk=dk, sk=sk, K=K: cspn_b200.propagate2d_k(gk, dk, sk, K, N),
                               lambda fg, gk=gk, dk=dk, sk=sk, K=K: fg.propagate_k(gk, dk, sk, K, N),
                               lambda cg, gk=gk, dk=dk, sk=sk, K=K: cg.propagate_k(gk, dk, sk, K, N))
    gp, fp, _ = inputs(rank + 1000, 24)
    all_ok &= check_routes('propagate2d_paddle 5x5', (B, 1, H, W), lambda: cspn_b200.propagate2d_paddle(gp, fp, 5, N),
                           lambda fg: fg.propagate_paddle(gp, fp, 5, N))
    gates = gp.abs() / gp.abs().sum(1, keepdim=True)            # demo.py's normalisation, done by the caller
    all_ok &= check_routes('affinity_propagate 5x5', (B, 1, H, W), lambda: cspn_b200.affinity_propagate(fp, gates, 5, N),
                           lambda fg: fg.affinity_propagate(fp, gates, 5, N))
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if all_ok else 1)
