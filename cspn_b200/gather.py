"""Data-parallel propagation with the final gather fused into the kernel (one process per GPU, torchrun).

The reference's multi-GPU story is nn.DataParallel (eval.py:117): replicas compute their slice of the batch, then the
outputs are gathered.  Images are independent, so there is no collective on the data path; the only exchange is that
gather.  Three ways to do it, all ending with the full (world * B_local, C, H, W) output, or (world * B_local, C, D, H, W)
in 3D, on every rank:

  FusedGather (this file)   the kernel stores every finished result into the gather buffers of ALL GPUs: peer pointers
                            of a CUDA symmetric-memory allocation (plain NVLink stores) or, where the fabric offers it,
                            one NVLS multicast address (a single `multimem.st`, replicated by the switch).  One forward,
                            one barrier across ranks.  `propagate` (3x3) runs `cspn2d_fwd_gather_f32`: the cluster
                            kernel's epilogue sends each tile while it goes on computing the next ones, so the transfer
                            hides behind the arithmetic.  `propagate_k` (K x K), `propagate_paddle` (the Paddle module's
                            own-location gates) and `affinity_propagate` (caller-supplied gates, 2D) run
                            `cspn2d_{k,paddle,gates}_fwd_gather_f32`: the last step kernel of the stepped forward stores
                            to every destination; the intermediate steps stay local.  Built with D=..., the buffer holds
                            volumes, and `propagate3d` (3x3x3), `propagate3d_k` (K x K x K) and `affinity_propagate3d`
                            (caller-supplied gates, 3D) do the same through `cspn3d_{,k_,gates_}fwd_gather_f32`.
  ChunkedGather             no symmetric memory needed: the local batch is cut into chunks, the kernel of chunk i+1
                            runs while NCCL all-gathers chunk i (`propagate`, 3x3, and `propagate_k`, K x K; 2D only).
  sharding.gather_outputs   kernel, then one NCCL all_gather_into_tensor (what round 1 measured: the baseline).
"""
import ctypes
import math

import torch
import torch.distributed as dist

from . import _lib
from .cspn import (_check_gates, _check_inputs_2d_k, _check_inputs_2d_paddle, _check_shapes_3d_k, _per_channel_gate_views,
                   _ptr, norm_code_2d_k, norm_code_3d_k, propagate2d, propagate2d_k)


class FusedGather:
    """Owns the symmetric gather buffer of one problem shape.  Each method mirrors the module function of its name and
    returns a view of that buffer holding all ranks' results, rank-major: out[r * B_local + i] is image (or volume) i of
    rank r.  The input to propagate (blur_depth, feat or input) must have the (B_local, C, H, W) the buffer was built for,
    or with D given, the (B_local, C, D, H, W) of the 3D methods."""

    def __init__(self, B_local, C, H, W, device, group=None, multicast=True, *, D=None):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        if self.world > 8:
            raise _lib.CspnError('FusedGather addresses at most 8 GPUs of one NVLink domain')
        self.shape = (B_local, C, H, W) if D is None else (B_local, C, D, H, W)
        self.block = math.prod(self.shape)                # floats per rank
        self.buf = symm_mem.empty((self.world * B_local, *self.shape[1:]), dtype=torch.float32, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, self.group)
        mine = self.rank * self.block * 4                 # byte offset of this rank's block inside every buffer
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.local = ptrs[self.rank] + mine
        mc = int(self.hdl.multicast_ptr) if (multicast and self.hdl.has_multicast_support) else 0
        if mc:
            self.mode = 'nvls_multicast'
            self.mc = mc + mine
            self.peers = []
        else:
            self.mode = 'peer_stores'
            self.mc = 0
            self.peers = [ptrs[r] + mine for r in range(self.world) if r != self.rank]
        self._peer_arr = (ctypes.c_void_p * max(1, len(self.peers)))(*self.peers)
        self._ws = None

    def _check_shape(self, t):
        if tuple(t.shape) != self.shape:
            raise ValueError(f'this FusedGather was built for {self.shape}, got {tuple(t.shape)}')

    def _gather(self, entry, device, inputs, dims, ws_bytes):
        """entry(*inputs, out, peer_out, n_peer, multicast_out, *dims, workspace, workspace_bytes, stream) with this
        rank's destinations and the shared workspace, then the barrier after which every rank's stores are complete."""
        if ws_bytes and (self._ws is None or self._ws.numel() < ws_bytes):
            self._ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        rc = getattr(_lib.lib(), entry)(*inputs, self.local, ctypes.cast(self._peer_arr, ctypes.c_void_p), len(self.peers),
                                        self.mc or None, *dims, None if not ws_bytes else self._ws.data_ptr(), ws_bytes,
                                        torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, entry)
        self.hdl.barrier()            # every rank's kernel (and with it its remote stores) is complete
        return self.buf

    def propagate(self, guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum', keep_sparse=False):
        """propagate2d (3x3) on the cluster kernel, which must be able to take the shape.  keep_sparse: as in propagate2d."""
        if keep_sparse:
            return self.propagate_k(guidance, blur_depth, sparse_depth, 3, prop_time, ('8sum', '8sum_abs')[_lib.NORM2D[norm_type]],
                                    keep_sparse=True)
        self._check_shape(blur_depth)
        B, C, H, W = self.shape
        g, d = guidance.contiguous(), blur_depth.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        ws_bytes = _lib.lib().cspn2d_workspace_bytes(B, C, H, W, int(prop_time), _lib.ALGO_CLUSTER)
        return self._gather('cspn2d_fwd_gather_f32', d.device, [_ptr(g), _ptr(d), _ptr(s)],
                            [B, C, H, W, g.shape[1], int(prop_time), _lib.NORM2D[norm_type]], ws_bytes)

    def propagate_k(self, guidance, blur_depth, sparse_depth=None, prop_kernel=5, prop_time=24, norm_type=None, keep_sparse=False):
        """propagate2d_k.  K = 3 is `propagate` (the cluster kernel); K = 5 and 7 take any W.  keep_sparse: as in
        propagate2d_k (cspn2d_keep_fwd_gather_f32)."""
        code = norm_code_2d_k(prop_kernel, norm_type)
        _check_inputs_2d_k(guidance, blur_depth, sparse_depth, prop_kernel)
        self._check_shape(blur_depth)
        B, C, H, W = self.shape
        g, d = guidance.contiguous(), blur_depth.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        if keep_sparse:
            ws_bytes = _lib.lib().cspn2d_keep_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time), _lib.ALGO_CLUSTER)
            return self._gather('cspn2d_keep_fwd_gather_f32', d.device, [_ptr(g), _ptr(d), _ptr(s)],
                                [B, C, H, W, g.shape[1], prop_kernel, int(prop_time), code], ws_bytes)
        ws_bytes = _lib.lib().cspn2d_k_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time))
        return self._gather('cspn2d_k_fwd_gather_f32', d.device, [_ptr(g), _ptr(d), _ptr(s)],
                            [B, C, H, W, g.shape[1], prop_kernel, int(prop_time), code], ws_bytes)

    def propagate_paddle(self, guidance, feat, prop_kernel=3, prop_time=24):
        """propagate2d_paddle; per-channel guidance (B, (K*K-1)*C, H, W) included."""
        Bi, Ci = _check_inputs_2d_paddle(guidance, feat, prop_kernel)
        self._check_shape(feat)
        H, W = feat.shape[2:]
        g, f = guidance.contiguous(), feat.contiguous()
        ws_bytes = _lib.lib().cspn2d_paddle_workspace_bytes(Bi, Ci, H, W, prop_kernel, int(prop_time))
        return self._gather('cspn2d_paddle_fwd_gather_f32', f.device, [_ptr(g), _ptr(f)],
                            [Bi, Ci, H, W, prop_kernel, int(prop_time)], ws_bytes)

    def affinity_propagate(self, input, gate_weight, kernel_size=3, prop_step=1):
        """affinity_propagate in 2D; per-channel gates (B, (K*K-1)*C, H, W) included."""
        if input.dim() == 5:
            raise ValueError('FusedGather.affinity_propagate is 2D only: 3D input goes to affinity_propagate3d')
        _, Bi, Ci = _check_gates(input, gate_weight, kernel_size, prop_step)
        self._check_shape(input)
        H, W = input.shape[2:]
        g, x = gate_weight.contiguous(), input.contiguous()
        ws_bytes = _lib.lib().cspn2d_gates_workspace_bytes(Bi, Ci, H, W, kernel_size, int(prop_step))
        return self._gather('cspn2d_gates_fwd_gather_f32', x.device, [_ptr(g), _ptr(x)],
                            [Bi, Ci, H, W, kernel_size, int(prop_step)], ws_bytes)

    def _volumes_3d_k(self, guidance, feat, prop_kernel):
        """The checked inputs of a K x K x K call as the C ABI takes them: per-channel guidance (B, (K**3-1)*C, D, H, W)
        becomes B*C single-channel volumes, as in Affinity_Propagate3DK."""
        views = _per_channel_gate_views(guidance, feat, prop_kernel ** 3 - 1)
        g, f = views if views is not None else (guidance.contiguous(), feat.contiguous())
        _check_shapes_3d_k(g, f, prop_kernel)
        self._check_shape(feat)
        return g, f

    def propagate3d(self, guidance, feat, prop_time=12, norm_type='26sum_abs'):
        """propagate3d (3x3x3); per-channel guidance (B, 26*C, D, H, W) included, as Affinity_Propagate3D takes it."""
        code = norm_code_3d_k(3, norm_type)
        g, f = self._volumes_3d_k(guidance, feat, 3)
        ws_bytes = _lib.lib().cspn3d_workspace_bytes(*f.shape, int(prop_time))
        return self._gather('cspn3d_fwd_gather_f32', f.device, [_ptr(g), _ptr(f)], [*f.shape, int(prop_time), code],
                            ws_bytes)

    def propagate3d_k(self, guidance, feat, prop_kernel=5, prop_time=12, norm_type=None):
        """propagate3d_k; per-channel guidance (B, (K**3-1)*C, D, H, W) included.  K = 3 is `propagate3d`."""
        code = norm_code_3d_k(prop_kernel, norm_type)
        g, f = self._volumes_3d_k(guidance, feat, prop_kernel)
        ws_bytes = _lib.lib().cspn3d_k_workspace_bytes(*f.shape, prop_kernel, int(prop_time))
        return self._gather('cspn3d_k_fwd_gather_f32', f.device, [_ptr(g), _ptr(f)],
                            [*f.shape, prop_kernel, int(prop_time), code], ws_bytes)

    def affinity_propagate3d(self, input, gate_weight, kernel_size=3, prop_step=1):
        """affinity_propagate in 3D; per-channel gates (B, (K**3-1)*C, D, H, W) included."""
        if input.dim() != 5:
            raise ValueError('FusedGather.affinity_propagate3d is 3D only: 2D input goes to affinity_propagate')
        _, Bi, Ci = _check_gates(input, gate_weight, kernel_size, prop_step)
        self._check_shape(input)
        D, H, W = input.shape[2:]
        g, x = gate_weight.contiguous(), input.contiguous()
        ws_bytes = _lib.lib().cspn3d_gates_workspace_bytes(Bi, Ci, D, H, W, kernel_size, int(prop_step))
        return self._gather('cspn3d_gates_fwd_gather_f32', x.device, [_ptr(g), _ptr(x)],
                            [Bi, Ci, D, H, W, kernel_size, int(prop_step)], ws_bytes)


class ChunkedGather:
    """Kernel on chunk i+1 while NCCL moves chunk i.  Result layout is CHUNK-major: out[c][r] is chunk c of rank r
    (shape (n_chunks, world, B_chunk, C, H, W)); `as_rank_major()` gives a copy in FusedGather's order."""

    def __init__(self, B_local, C, H, W, device, n_chunks=4, group=None):
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        if B_local % n_chunks:
            raise ValueError('n_chunks must divide the local batch')
        self.n_chunks, self.bc = n_chunks, B_local // n_chunks
        self.full = torch.empty(n_chunks, self.world, self.bc, C, H, W, dtype=torch.float32, device=device)
        self.local = torch.empty(B_local, C, H, W, dtype=torch.float32, device=device)

    def _chunks(self, run):
        """run(batch slice, out) for every chunk, each chunk's all-gather enqueued behind its kernel."""
        works = []
        for c in range(self.n_chunks):
            sl = slice(c * self.bc, (c + 1) * self.bc)
            oc = self.local[sl]
            run(sl, oc)
            # NCCL's stream waits for the kernel just enqueued; the next chunk's kernel does not wait for NCCL
            works.append(dist.all_gather_into_tensor(self.full[c], oc, group=self.group, async_op=True))
        for w in works:
            w.wait()
        return self.full

    def propagate(self, guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum', algo=_lib.ALGO_AUTO):
        return self._chunks(lambda sl, oc: propagate2d(guidance[sl], blur_depth[sl],
                                                       None if sparse_depth is None else sparse_depth[sl], prop_time,
                                                       norm_type, algo, out=oc))

    def propagate_k(self, guidance, blur_depth, sparse_depth=None, prop_kernel=5, prop_time=24, norm_type=None):
        return self._chunks(lambda sl, oc: propagate2d_k(guidance[sl], blur_depth[sl],
                                                         None if sparse_depth is None else sparse_depth[sl], prop_kernel,
                                                         prop_time, norm_type, out=oc))

    def as_rank_major(self):
        return self.full.permute(1, 0, 2, 3, 4, 5).reshape(self.world * self.n_chunks * self.bc, *self.full.shape[3:])
