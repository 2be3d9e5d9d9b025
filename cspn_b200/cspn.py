"""Drop-in replacement of the reference's CSPN operator module.

Mirrors /root/reference/cspn_pytorch/models/cspn.py (class Affinity_Propagate, :14-83): same
constructor, attributes, forward signature, assertion behaviour and return convention, so
`import cspn as post_process` (torch_resnet_cspn_nyu.py:12) resolves to this file when it is
placed first on sys.path (see INTEGRATION.md).  All arithmetic runs in libcspn_b200.so
(hand-written sm_90a CUDA behind the C ABI of include/cspn_b200.h); PyTorch only supplies
device memory, the current stream and autograd plumbing.  There is no CPU / eager fallback.
"""
import torch
import torch.nn as nn

import os

from . import _lib, torch_op
from ._lib import ALGO_AUTO, ALGO_CLUSTER, ALGO_GENERIC, NORM2D, NORM3D  # noqa: F401


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _check_inputs_2d(guidance, blur_depth, sparse_depth):
    if guidance.dim() != 4 or blur_depth.dim() != 4:
        raise ValueError('guidance and blur_depth must be (B,C,H,W)')
    if guidance.dtype != torch.float32 or blur_depth.dtype != torch.float32:
        # the reference raises here too: its ones-weight conv is fp32 (cspn.py:50)
        raise RuntimeError('cspn_b200 is fp32 only (as the reference, cspn.py:44-53)')
    B, C, H, W = blur_depth.shape
    if guidance.shape[0] != B or guidance.shape[2:] != (H, W) or guidance.shape[1] < 8:
        raise ValueError(f'guidance {tuple(guidance.shape)} does not match blur_depth {tuple(blur_depth.shape)} '
                         '(need (B,>=8,H,W))')
    if guidance.device != blur_depth.device:
        raise RuntimeError('guidance and blur_depth are on different devices')
    if sparse_depth is not None:
        if sparse_depth.shape != (B, 1, H, W):
            raise ValueError(f'sparse_depth must be (B,1,H,W), got {tuple(sparse_depth.shape)}')
        if sparse_depth.dtype != torch.float32 or sparse_depth.device != blur_depth.device:
            raise RuntimeError('sparse_depth must be fp32 on the device of blur_depth')


def _overlaps(a, b):
    """True when the memory of two tensors intersects.  Different storages (the normal case) are told apart at once; only
    views of one storage pay for the exact range test."""
    if a is None or b is None or a.device != b.device or a.numel() == 0 or b.numel() == 0:
        return False
    if a.untyped_storage().data_ptr() != b.untyped_storage().data_ptr():
        return False
    a0, b0 = a.data_ptr(), b.data_ptr()
    span = lambda t: (sum((n - 1) * abs(st) for n, st in zip(t.shape, t.stride())) + 1) * t.element_size()
    return a0 < b0 + span(b) and b0 < a0 + span(a)


def _check_out(out, like, *inputs):
    if out.shape != like.shape or out.dtype != like.dtype or out.device != like.device or not out.is_contiguous():
        raise ValueError('`out` must be a contiguous tensor with the shape, dtype and device of blur_depth')
    for t in (like,) + inputs:       # include/cspn_b200.h: `out` must not alias the inputs
        if _overlaps(out, t):
            raise ValueError('`out` must not alias an input tensor')


def propagate2d(guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum', algo=ALGO_AUTO, out=None):
    """Forward only, no autograd.  CUDA tensors: enqueued on the current stream of their device.
    CPU tensors: shipped through the library's chunked H2D/compute/D2H pipeline on cuda:0
    (the C ABI's host-buffer entry point) -- still the GPU kernels, never a CPU implementation.
    `out` (optional) receives the result instead of a freshly allocated tensor: same shape/dtype/device as
    blur_depth, contiguous (serving loops reuse one pinned buffer: allocating 55 MB of pinned memory costs milliseconds)."""
    _check_inputs_2d(guidance, blur_depth, sparse_depth)
    if prop_time == 0:
        if out is None:
            return blur_depth                  # cspn.py:61,83 returns the input tensor itself
        _check_out(out, blur_depth, guidance, sparse_depth)
        out.copy_(blur_depth)                  # a caller-provided result buffer always holds the result
        return out
    L = _lib.lib()
    B, C, H, W = blur_depth.shape
    g = guidance.contiguous()
    d = blur_depth.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    if not d.is_cuda:
        if not torch.cuda.is_available():
            raise _lib.CspnError('cspn_b200 needs a CUDA device (no CPU implementation exists in this package)')
        if out is None:
            out = torch.empty_like(d, pin_memory=d.is_pinned())  # pinned in -> pinned out: the D2H stays asynchronous
        _check_out(out, d, g, s)
        rc = L.cspn2d_fwd_f32_host(_ptr(g), _ptr(d), _ptr(s), _ptr(out), B, C, H, W, g.shape[1], int(prop_time),
                                   NORM2D[norm_type], algo, torch.cuda.current_device())
        _lib.check(rc, 'cspn2d_fwd_f32_host')
        return out
    if out is None:
        out = torch.empty_like(d)
    _check_out(out, d, g, s)
    if algo == ALGO_AUTO and any(t is not None and t.data_ptr() % 16 for t in (g, d, s, out)):
        algo = ALGO_GENERIC   # views at odd storage offsets: the cluster kernel's TMA / float4 accesses need 16-byte bases
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_workspace_bytes(B, C, H, W, int(prop_time), algo)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(out), B, C, H, W, g.shape[1], int(prop_time),
                              NORM2D[norm_type], algo, _ptr(ws), ws_bytes, _stream(d.device))
    _lib.check(rc, 'cspn2d_fwd_f32')
    return out


class _Propagate2dFn(torch.autograd.Function):
    """autograd seam for train.py:196-199: native forward + native adjoint (cspn2d_bwd_f32)."""

    @staticmethod
    def forward(ctx, guidance, blur_depth, sparse_depth, prop_time, norm_type, algo):
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (prop_time, norm_type)
        return propagate2d(guidance, blur_depth, sparse_depth, prop_time, norm_type, algo)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        prop_time, norm_type = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, H, W = blur_depth.shape
        g = guidance.contiguous()
        d = blur_depth.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        go = grad_out.contiguous()
        need_g, need_d = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg = torch.empty_like(g) if need_g else None
        gd = torch.empty_like(d) if need_d else None
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_bwd_workspace_bytes(B, C, H, W, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(go), _ptr(gg), _ptr(gd), B, C, H, W, g.shape[1],
                                  int(prop_time), NORM2D[norm_type], _ptr(ws), ws_bytes, _stream(d.device))
        _lib.check(rc, 'cspn2d_bwd_f32')
        return gg, gd, None, None, None, None


def _use_torch_op():
    """The dispatcher-op route is taken when libcspn_b200_torch.so exists (CSPN_B200_NO_TORCH_OP=1 forces ctypes)."""
    if os.environ.get('CSPN_B200_NO_TORCH_OP') == '1' or not torch_op.available():
        return False
    torch_op.load()
    return True


class Affinity_Propagate(nn.Module):
    """Same surface as the reference class (cspn.py:14-39): no parameters, no buffers."""

    def __init__(self, prop_time, prop_kernel, norm_type='8sum', algo=ALGO_AUTO):
        super(Affinity_Propagate, self).__init__()
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        assert prop_kernel == 3, 'this version only support 8 (3x3 - 1) neighborhood'      # cspn.py:33
        self.norm_type = norm_type
        assert norm_type in ['8sum', '8sum_abs']                                           # cspn.py:36
        self.in_feature = 1
        self.out_feature = 1
        self.algo = algo
        # torch.ops.cspn_b200.propagate2d (csrc/torch_op.cpp) when the shim is built: one dispatcher op with fake kernel
        # and autograd formula, so torch.compile / export trace through the module.  Same C ABI underneath; without the
        # shim the ctypes binding below is used (still the CUDA kernels -- there is no non-native path).
        self._use_op = _use_torch_op()

    def forward(self, guidance, blur_depth, sparse_depth=None):
        if self._use_op and blur_depth.is_cuda and self.prop_time > 0:
            sd = None if sparse_depth is None else sparse_depth.detach()   # train.py never differentiates it (:351 clones the input)
            return torch.ops.cspn_b200.propagate2d(guidance, blur_depth, sd, self.prop_time, NORM2D[self.norm_type], self.algo)
        needs_grad = torch.is_grad_enabled() and (guidance.requires_grad or blur_depth.requires_grad)
        if needs_grad and self.prop_time > 0:
            sd = None if sparse_depth is None else sparse_depth.detach()
            return _Propagate2dFn.apply(guidance, blur_depth, sd, self.prop_time, self.norm_type, self.algo)
        return propagate2d(guidance, blur_depth, sparse_depth, self.prop_time, self.norm_type, self.algo)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, norm_type={self.norm_type!r}'


def propagate3d(guidance, feat, prop_time=12, norm_type='26sum_abs'):
    """3D CSPN, guidance (B,26,D,H,W), feat (B,C,D,H,W).  See Affinity_Propagate3D."""
    if guidance.dim() != 5 or feat.dim() != 5:
        raise ValueError('guidance and feat must be (B,C,D,H,W)')
    if guidance.dtype != torch.float32 or feat.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    B, C, D, H, W = feat.shape
    if guidance.shape != (B, 26, D, H, W):
        raise ValueError(f'guidance must be (B,26,D,H,W), got {tuple(guidance.shape)} for feat {tuple(feat.shape)}')
    if guidance.device != feat.device:
        raise RuntimeError('guidance and feat are on different devices')
    if prop_time == 0:
        return feat
    L = _lib.lib()
    g, f = guidance.contiguous(), feat.contiguous()
    if not f.is_cuda:
        if not torch.cuda.is_available():
            raise _lib.CspnError('cspn_b200 needs a CUDA device (no CPU implementation exists in this package)')
        out = torch.empty_like(f, pin_memory=f.is_pinned())
        rc = L.cspn3d_fwd_f32_host(_ptr(g), _ptr(f), _ptr(out), B, C, D, H, W, int(prop_time), NORM3D[norm_type],
                                   torch.cuda.current_device())
        _lib.check(rc, 'cspn3d_fwd_f32_host')
        return out
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        ws_bytes = L.cspn3d_workspace_bytes(B, C, D, H, W, int(prop_time))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
        rc = L.cspn3d_fwd_f32(_ptr(g), _ptr(f), _ptr(out), B, C, D, H, W, int(prop_time), NORM3D[norm_type],
                              _ptr(ws), ws_bytes, _stream(f.device))
    _lib.check(rc, 'cspn3d_fwd_f32')
    return out


class _Propagate3dFn(torch.autograd.Function):
    """autograd seam of the 3D operator (the Paddle op is trained through: cspn_paddle/demo.py:72-75)."""

    @staticmethod
    def forward(ctx, guidance, feat, prop_time, norm_type):
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (prop_time, norm_type)
        return propagate3d(guidance, feat, prop_time, norm_type)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        prop_time, norm_type = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, D, H, W = feat.shape
        g, f, go = guidance.contiguous(), feat.contiguous(), grad_out.contiguous()
        gg = torch.empty_like(g) if ctx.needs_input_grad[0] else None
        gf = torch.empty_like(f) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(f.device):
            ws_bytes = L.cspn3d_bwd_workspace_bytes(B, C, D, H, W, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
            rc = L.cspn3d_bwd_f32(_ptr(g), _ptr(f), _ptr(go), _ptr(gg), _ptr(gf), B, C, D, H, W, int(prop_time),
                                  NORM3D[norm_type], _ptr(ws), ws_bytes, _stream(f.device))
        _lib.check(rc, 'cspn3d_bwd_f32')
        return gg, gf, None, None


class Affinity_Propagate3D(nn.Module):
    """3D (3x3x3, 26 neighbours) counterpart; the reference has only call sites for it
    (cspn_paddle/demo.py:20-54: CSPN.cspn(guide, feat)).  norm_type:
      '26sum' / '26sum_abs' -- the cspn.py scheme lifted to 3D (gathered affinities, centre term);
      'paddle'              -- demo.py's |guide| / sum_k |guide_k| at the voxel's own location,
                               then prop_time applications of out = sum_k gate_k * shift_k(feat).
    guidance is (B,26,D,H,W) -- one gate shared by all C feature channels (cspn_paddle/README.md:56) -- or (B,26*C,D,H,W):
    one gate per feature channel, demo.py:28-45."""

    def __init__(self, prop_time, prop_kernel=3, norm_type='26sum_abs'):
        super().__init__()
        assert prop_kernel == 3, 'only the 3x3x3 (26-neighbour) kernel is supported'      # demo.py:91 choices=[3]
        assert norm_type in NORM3D
        self.prop_time, self.prop_kernel, self.norm_type = prop_time, prop_kernel, norm_type
        self._use_op = _use_torch_op()

    def forward(self, guidance, feat):
        if feat.dim() == 5 and guidance.dim() == 5 and feat.shape[1] > 1 and guidance.shape[1] == 26 * feat.shape[1]:
            # per-channel gates, the feat.shape[1] > 1 branch of CSPN.cspn (cspn_paddle/demo.py:28-45): channel c of feat is
            # propagated with guide channels [26c, 26c+26).  In memory that IS a batch of B*C single-channel volumes with
            # 26-channel gates, so the views below cost nothing (contiguous inputs) and the same kernels run.
            B, C = feat.shape[:2]
            out = self.forward(guidance.contiguous().view(B * C, 26, *guidance.shape[2:]),
                               feat.contiguous().view(B * C, 1, *feat.shape[2:]))
            return out.view(feat.shape)
        if self._use_op and feat.is_cuda and self.prop_time > 0:
            return torch.ops.cspn_b200.propagate3d(guidance, feat, self.prop_time, NORM3D[self.norm_type])
        if torch.is_grad_enabled() and (guidance.requires_grad or feat.requires_grad) and self.prop_time > 0:
            return _Propagate3dFn.apply(guidance, feat, self.prop_time, self.norm_type)
        return propagate3d(guidance, feat, self.prop_time, self.norm_type)
