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

import ctypes
import operator
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


def propagate2d(guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum', algo=ALGO_AUTO, out=None,
                keep_sparse=False):
    """Forward only, no autograd.  CUDA tensors: enqueued on the current stream of their device.
    CPU tensors: shipped through the library's chunked H2D/compute/D2H pipeline on cuda:0
    (the C ABI's host-buffer entry point) -- still the GPU kernels, never a CPU implementation.
    `out` (optional) receives the result instead of a freshly allocated tensor: same shape/dtype/device as
    blur_depth, contiguous (serving loops reuse one pinned buffer: allocating 55 MB of pinned memory costs milliseconds).
    keep_sparse=True: the CSPN paper's replacement step, which keeps the samples in the output (DESIGN.md section 4.13;
    CUDA tensors only)."""
    if keep_sparse:
        return _propagate2d_keep(guidance, blur_depth, sparse_depth, 3, prop_time, NORM2D[norm_type], algo, out)
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


def _propagate2d_keep(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo=ALGO_AUTO, out=None):
    """The keep-sparse mode (cspn2d_keep_fwd_f32), forward only: m = 1[sparse_depth > 0], and every step sets
    d <- (1 - m) d + m sparse_depth, so the result passes through the samples.  CUDA tensors only."""
    nt = prop_kernel * prop_kernel - 1
    if guidance.dim() == 4 and guidance.shape[1] < nt:
        raise ValueError(f'a {prop_kernel}x{prop_kernel} kernel needs guidance (B,>={nt},H,W), got {tuple(guidance.shape)}')
    _check_inputs_2d(guidance, blur_depth, sparse_depth)
    if not (guidance.is_cuda and blur_depth.is_cuda and (sparse_depth is None or sparse_depth.is_cuda)):
        raise _lib.CspnError('keep_sparse takes CUDA tensors only (there is no host-buffer entry point for it)')
    if prop_time == 0:
        if out is None:
            return blur_depth
        _check_out(out, blur_depth, guidance, sparse_depth)
        out.copy_(blur_depth)
        return out
    L = _lib.lib()
    B, C, H, W = blur_depth.shape
    g, d = guidance.contiguous(), blur_depth.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    if out is None:
        out = torch.empty_like(d)
    _check_out(out, d, g, s)
    if algo == ALGO_AUTO and any(t is not None and t.data_ptr() % 16 for t in (g, d, s, out)):
        algo = ALGO_GENERIC   # views at odd storage offsets: the cluster kernel's TMA / float4 accesses need 16-byte bases
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_keep_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time), algo)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_keep_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(out), B, C, H, W, g.shape[1], prop_kernel, int(prop_time),
                                   code, algo, _ptr(ws), ws_bytes, _stream(d.device))
    _lib.check(rc, 'cspn2d_keep_fwd_f32')
    return out


class _Propagate2dKeepFn(torch.autograd.Function):
    """autograd seam of the keep-sparse mode without the torch-op shim: native forward + native adjoint
    (cspn2d_keep_bwd_f32), differentiable in guidance, blur_depth and sparse_depth."""

    @staticmethod
    def forward(ctx, guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo):
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (prop_kernel, prop_time, code)
        return _propagate2d_keep(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        prop_kernel, prop_time, code = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, H, W = blur_depth.shape
        g, d, go = guidance.contiguous(), blur_depth.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        need_g, need_d, need_s = ctx.needs_input_grad[:3]
        gg = torch.empty_like(g) if need_g else None
        gd = torch.empty_like(d) if need_d else None
        gs = torch.empty_like(s) if need_s and s is not None else None
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_keep_bwd_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_keep_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(go), _ptr(gg), _ptr(gd), _ptr(gs), B, C, H, W, g.shape[1],
                                       prop_kernel, int(prop_time), code, _ptr(ws), ws_bytes, _stream(d.device))
        _lib.check(rc, 'cspn2d_keep_bwd_f32')
        return gg, gd, gs, None, None, None, None


def _keep_forward(use_op, guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo):
    """The keep-sparse forward of the modules: the registered op, else the ctypes autograd seam; sparse_depth is not
    detached (its gradient is m * sum_c Gc_c)."""
    if prop_time == 0:
        return blur_depth
    if not blur_depth.is_cuda:
        raise _lib.CspnError('keep_sparse takes CUDA tensors only (there is no host-buffer entry point for it)')
    if use_op:
        return torch.ops.cspn_b200.propagate2d_keep(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (guidance, blur_depth, sparse_depth)):
        return _Propagate2dKeepFn.apply(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo)
    return _propagate2d_keep(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, algo)


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

    def __init__(self, prop_time, prop_kernel, norm_type='8sum', algo=ALGO_AUTO, keep_sparse=False):
        super(Affinity_Propagate, self).__init__()
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        assert prop_kernel == 3, 'this version only support 8 (3x3 - 1) neighborhood'      # cspn.py:33
        self.norm_type = norm_type
        assert norm_type in ['8sum', '8sum_abs']                                           # cspn.py:36
        self.in_feature = 1
        self.out_feature = 1
        self.algo = algo
        # keep_sparse: the CSPN paper's replacement step, d <- (1 - m) d + m sparse_depth with m = 1[sparse_depth > 0], so
        # the output passes through the samples (DESIGN.md section 4.13); the reference module replaces with blur_depth
        self.keep_sparse = keep_sparse
        # torch.ops.cspn_b200.propagate2d (csrc/torch_op.cpp) when the shim is built: one dispatcher op with fake kernel
        # and autograd formula, so torch.compile / export trace through the module.  Same C ABI underneath; without the
        # shim the ctypes binding below is used (still the CUDA kernels -- there is no non-native path).
        self._use_op = _use_torch_op()

    def forward(self, guidance, blur_depth, sparse_depth=None):
        if self.keep_sparse:
            return _keep_forward(self._use_op, guidance, blur_depth, sparse_depth, 3, self.prop_time, NORM2D[self.norm_type],
                                 self.algo)
        if self._use_op and blur_depth.is_cuda and self.prop_time > 0:
            sd = None if sparse_depth is None else sparse_depth.detach()   # train.py never differentiates it (:351 clones the input)
            return torch.ops.cspn_b200.propagate2d(guidance, blur_depth, sd, self.prop_time, NORM2D[self.norm_type], self.algo)
        needs_grad = torch.is_grad_enabled() and (guidance.requires_grad or blur_depth.requires_grad)
        if needs_grad and self.prop_time > 0:
            sd = None if sparse_depth is None else sparse_depth.detach()
            return _Propagate2dFn.apply(guidance, blur_depth, sd, self.prop_time, self.norm_type, self.algo)
        return propagate2d(guidance, blur_depth, sparse_depth, self.prop_time, self.norm_type, self.algo)

    def extra_repr(self):
        keep = ', keep_sparse=True' if self.keep_sparse else ''
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, norm_type={self.norm_type!r}{keep}'


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


def _per_channel_gate_views(guidance, feat, nt):
    """Per-channel gates, the feat.shape[1] > 1 branch of CSPN.cspn (cspn_paddle/demo.py:28-45): with guidance
    (B, nt*C, D, H, W), channel c of feat is propagated with guide channels [nt*c, nt*c+nt).  In memory that IS a batch of
    B*C single-channel volumes with nt-channel gates, so the views returned cost nothing (contiguous inputs) and the same
    kernels run.  None when the shapes are not of that form."""
    if feat.dim() == 5 and guidance.dim() == 5 and feat.shape[1] > 1 and guidance.shape[1] == nt * feat.shape[1]:
        B, C = feat.shape[:2]
        return (guidance.contiguous().view(B * C, nt, *guidance.shape[2:]),
                feat.contiguous().view(B * C, 1, *feat.shape[2:]))
    return None


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
        views = _per_channel_gate_views(guidance, feat, 26)
        if views is not None:
            return self.forward(*views).view(feat.shape)
        if self._use_op and feat.is_cuda and self.prop_time > 0:
            return torch.ops.cspn_b200.propagate3d(guidance, feat, self.prop_time, NORM3D[self.norm_type])
        if torch.is_grad_enabled() and (guidance.requires_grad or feat.requires_grad) and self.prop_time > 0:
            return _Propagate3dFn.apply(guidance, feat, self.prop_time, self.norm_type)
        return propagate3d(guidance, feat, self.prop_time, self.norm_type)


# ---- 2D with a K x K affinity kernel (K in {3, 5, 7}) ----------------------------------------------------------------
KERNEL_SIZES_2D = (3, 5, 7)


def norm_code_2d_k(prop_kernel, norm_type=None):
    """The norm names of a K x K kernel follow the 3D naming, f'{K*K-1}sum' / f'{K*K-1}sum_abs' ('8sum', '24sum',
    '48sum', ...); returns the cspn_norm2d code (0 signed, 1 abs).  Raises AssertionError for another K or name."""
    assert prop_kernel in KERNEL_SIZES_2D, f'prop_kernel must be 3, 5 or 7, got {prop_kernel}'
    nt = prop_kernel * prop_kernel - 1
    names = {f'{nt}sum': 0, f'{nt}sum_abs': 1}
    norm_type = norm_type or f'{nt}sum'
    assert norm_type in names, f'norm_type of a {prop_kernel}x{prop_kernel} kernel is one of {sorted(names)}, got {norm_type!r}'
    return names[norm_type]


def _check_inputs_2d_k(guidance, blur_depth, sparse_depth, prop_kernel):
    nt = prop_kernel * prop_kernel - 1
    if guidance.dim() == 4 and guidance.shape[1] < nt:
        raise ValueError(f'a {prop_kernel}x{prop_kernel} kernel needs guidance (B,>={nt},H,W), got {tuple(guidance.shape)}')
    _check_inputs_2d(guidance, blur_depth, sparse_depth)
    if not (guidance.is_cuda and blur_depth.is_cuda):
        raise _lib.CspnError(f'the {prop_kernel}x{prop_kernel} propagation takes CUDA tensors only '
                             '(there is no host-buffer entry point for it)')


def propagate2d_k(guidance, blur_depth, sparse_depth=None, prop_kernel=5, prop_time=24, norm_type=None, out=None,
                  keep_sparse=False):
    """2D CSPN with a K x K affinity kernel, forward only (no autograd), CUDA tensors only, enqueued on the current stream.
    guidance (B, >=K*K-1, H, W): channels 0..K*K-2 are used, shared by the C channels of blur_depth (B, C, H, W);
    norm_type f'{K*K-1}sum' (default) or f'{K*K-1}sum_abs'.  K = 3 is propagate2d itself (same kernels, same bits).
    keep_sparse=True: the samples are kept in the output, as in propagate2d."""
    code = norm_code_2d_k(prop_kernel, norm_type)
    if keep_sparse:
        return _propagate2d_keep(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, code, ALGO_AUTO, out)
    _check_inputs_2d_k(guidance, blur_depth, sparse_depth, prop_kernel)
    if prop_kernel == 3:
        return propagate2d(guidance, blur_depth, sparse_depth, prop_time, ('8sum', '8sum_abs')[code], ALGO_AUTO, out)
    if prop_time == 0:
        if out is None:
            return blur_depth
        _check_out(out, blur_depth, guidance, sparse_depth)
        out.copy_(blur_depth)
        return out
    L = _lib.lib()
    B, C, H, W = blur_depth.shape
    g, d = guidance.contiguous(), blur_depth.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    if out is None:
        out = torch.empty_like(d)
    _check_out(out, d, g, s)
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_k_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_k_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(out), B, C, H, W, g.shape[1], prop_kernel, int(prop_time),
                                code, _ptr(ws), ws_bytes, _stream(d.device))
    _lib.check(rc, 'cspn2d_k_fwd_f32')
    return out


class _Propagate2dKFn(torch.autograd.Function):
    """autograd seam of the K x K operator without the torch-op shim: native forward + native adjoint (cspn2d_k_bwd_f32)."""

    @staticmethod
    def forward(ctx, guidance, blur_depth, sparse_depth, prop_kernel, prop_time, norm_type):
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (prop_kernel, prop_time, norm_type)
        return propagate2d_k(guidance, blur_depth, sparse_depth, prop_kernel, prop_time, norm_type)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        prop_kernel, prop_time, norm_type = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, H, W = blur_depth.shape
        g, d, go = guidance.contiguous(), blur_depth.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        need_g, need_d = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg = torch.empty_like(g) if need_g else None
        gd = torch.empty_like(d) if need_d else None
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_k_bwd_workspace_bytes(B, C, H, W, prop_kernel, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_k_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(go), _ptr(gg), _ptr(gd), B, C, H, W, g.shape[1],
                                    prop_kernel, int(prop_time), norm_code_2d_k(prop_kernel, norm_type), _ptr(ws), ws_bytes,
                                    _stream(d.device))
        _lib.check(rc, 'cspn2d_k_bwd_f32')
        return gg, gd, None, None, None, None


class Affinity_PropagateK(nn.Module):
    """2D CSPN with a K x K affinity kernel, K in {3, 5, 7}: Affinity_Propagate with K*K-1 neighbours instead of 8
    (cspn.py with its pad tuples generalised; DESIGN.md section 4.8).  forward(guidance (B, >=K*K-1, H, W),
    blur_depth (B, C, H, W), sparse_depth (B, 1, H, W) or None).  norm_type defaults to f'{K*K-1}sum'; the other is
    f'{K*K-1}sum_abs'.  No parameters, no buffers; prop_time == 0 returns blur_depth itself.  Forward and backward run
    in CUDA kernels (K = 3 in those of Affinity_Propagate, with the same bits)."""

    def __init__(self, prop_time, prop_kernel, norm_type=None, keep_sparse=False):
        super().__init__()
        norm_code_2d_k(prop_kernel, norm_type)      # AssertionError for K not in {3, 5, 7} or a name that does not match K
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        self.norm_type = norm_type or f'{prop_kernel * prop_kernel - 1}sum'
        self.keep_sparse = keep_sparse              # as in Affinity_Propagate
        self._use_op = _use_torch_op()

    def forward(self, guidance, blur_depth, sparse_depth=None):
        if self.prop_time == 0:
            return blur_depth
        code = norm_code_2d_k(self.prop_kernel, self.norm_type)
        if self.keep_sparse:
            return _keep_forward(self._use_op, guidance, blur_depth, sparse_depth, self.prop_kernel, self.prop_time, code, ALGO_AUTO)
        sd = None if sparse_depth is None else sparse_depth.detach()
        if self._use_op and blur_depth.is_cuda:
            return torch.ops.cspn_b200.propagate2d_k(guidance, blur_depth, sd, self.prop_kernel, self.prop_time, code)
        if torch.is_grad_enabled() and (guidance.requires_grad or blur_depth.requires_grad):
            return _Propagate2dKFn.apply(guidance, blur_depth, sd, self.prop_kernel, self.prop_time, self.norm_type)
        return propagate2d_k(guidance, blur_depth, sparse_depth, self.prop_kernel, self.prop_time, self.norm_type)

    def extra_repr(self):
        keep = ', keep_sparse=True' if self.keep_sparse else ''
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, norm_type={self.norm_type!r}{keep}'


# ---- aggregation of the 2D steps: CSPN++'s context-aware CSPN (DESIGN.md section 4.20) ------------------------------------
def _check_aggregate(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, steps):
    """The checks of propagate2d_aggregate, every refusal of an argument before the device check; returns the steps as a
    tuple of ints (default 1..T)."""
    if step_weight.dim() != 4 or blur_depth.dim() != 4:
        raise ValueError(f'step_weight and blur_depth must be (B,T,H,W) and (B,C,H,W), got {tuple(step_weight.shape)} and '
                         f'{tuple(blur_depth.shape)}')
    B, C, H, W = blur_depth.shape
    T = step_weight.shape[1]
    if steps is None:
        steps = tuple(range(1, T + 1))
    if (isinstance(steps, (str, bytes)) or not hasattr(steps, '__len__')
            or any(isinstance(s, bool) or not isinstance(s, int) for s in steps)):
        raise ValueError(f'steps must be a sequence of ints, got {steps!r}')
    steps = tuple(steps)
    if not steps or steps[0] < 1 or any(a >= b for a, b in zip(steps, steps[1:])) or steps[-1] > 2 ** 31 - 1:
        raise ValueError(f'steps must be strictly increasing ints >= 1, got {steps}')
    if tuple(step_weight.shape) != (B, len(steps), H, W):
        raise ValueError(f'step_weight must be (B, len(steps), H, W) = {(B, len(steps), H, W)}, got {tuple(step_weight.shape)}')
    if step_weight.dtype != torch.float32 or step_weight.device != blur_depth.device:
        raise RuntimeError('step_weight must be fp32 on the device of blur_depth')
    _check_inputs_2d_k(guidance, blur_depth, sparse_depth, prop_kernel)
    return steps


def _aggregate_fwd(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, code, keep, steps):
    """Forward only (no autograd) through cspn2d_agg_fwd_f32, on the current stream."""
    L = _lib.lib()
    B, C, H, W = blur_depth.shape
    g, d, w = guidance.contiguous(), blur_depth.contiguous(), step_weight.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    out = torch.empty_like(d)
    st = _c_sizes(steps)
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_agg_workspace_bytes(B, C, H, W, prop_kernel, st, len(steps), int(keep))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_agg_fwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(w), _ptr(out), B, C, H, W, g.shape[1], prop_kernel, st, len(steps),
                                  code, int(keep), _ptr(ws), ws_bytes, _stream(d.device))
    _lib.check(rc, 'cspn2d_agg_fwd_f32')
    return out


class _Propagate2dAggregateFn(torch.autograd.Function):
    """autograd seam of propagate2d_aggregate without the torch-op shim: native forward + native adjoint
    (cspn2d_agg_bwd_f32), differentiable in guidance, blur_depth, step_weight and, in keep mode, sparse_depth."""

    @staticmethod
    def forward(ctx, guidance, blur_depth, step_weight, sparse_depth, prop_kernel, code, keep, steps):
        ctx.save_for_backward(guidance, blur_depth, step_weight, sparse_depth)
        ctx.cfg = (prop_kernel, code, keep, steps)
        return _aggregate_fwd(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, code, keep, steps)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, blur_depth, step_weight, sparse_depth = ctx.saved_tensors
        prop_kernel, code, keep, steps = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, H, W = blur_depth.shape
        g, d, w, go = guidance.contiguous(), blur_depth.contiguous(), step_weight.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        need_g, need_d, need_w, need_s = ctx.needs_input_grad[:4]
        need_s = need_s and keep
        gg = torch.empty_like(g) if need_g else None
        gd = torch.empty_like(d) if need_d else None
        gw = torch.empty_like(w) if need_w else None
        gs = torch.empty_like(s) if need_s and s is not None else None
        st = _c_sizes(steps)
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_agg_bwd_workspace_bytes(B, C, H, W, prop_kernel, st, len(steps), int(keep))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_agg_bwd_f32(_ptr(g), _ptr(d), _ptr(s), _ptr(w), _ptr(go), _ptr(gg), _ptr(gd), _ptr(gs), _ptr(gw), B, C, H, W,
                                      g.shape[1], prop_kernel, st, len(steps), code, int(keep), _ptr(ws), ws_bytes, _stream(d.device))
        _lib.check(rc, 'cspn2d_agg_bwd_f32')
        return gg, gd, gw, gs, None, None, None, None


def propagate2d_aggregate(guidance, blur_depth, step_weight, sparse_depth=None, prop_kernel=3, norm_type=None, keep_sparse=False,
                          steps=None):
    """CSPN++'s context-aware CSPN for one kernel size: a per-pixel weighted sum of the 2D propagation's iterates,
        out = sum_j step_weight[:, j] * d_{steps[j]},
    where d_0 = blur_depth and d_{t+1} is one step of propagate2d_k(..., prop_kernel, keep_sparse=keep_sparse), so the run
    is steps[-1] steps long.  guidance (B, >=K*K-1, H, W), blur_depth (B, C, H, W), sparse_depth (B, 1, H, W) or None and
    step_weight (B, T, H, W), shared by the C channels, are fp32 CUDA tensors; steps holds T strictly increasing ints >= 1
    (default 1..T).  The weights are used as given: apply CSPN++'s softmax before the call.  No iterate is stored: the
    forward keeps the running sum in the output.  Differentiable in guidance, blur_depth, step_weight and, with
    keep_sparse=True, sparse_depth.  DESIGN.md section 4.20."""
    code = norm_code_2d_k(prop_kernel, norm_type)
    steps = _check_aggregate(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, steps)
    keep = bool(keep_sparse)
    if not keep and sparse_depth is not None:
        sparse_depth = sparse_depth.detach()       # the default mode's m = sign(sparse) takes no gradient
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.propagate2d_aggregate(guidance, blur_depth, sparse_depth, step_weight, list(steps), prop_kernel,
                                                         code, keep)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (guidance, blur_depth, step_weight, sparse_depth)):
        return _Propagate2dAggregateFn.apply(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, code, keep, steps)
    return _aggregate_fwd(guidance, blur_depth, step_weight, sparse_depth, prop_kernel, code, keep, steps)


# ---- non-local 2D propagation: NLSPN's (DESIGN.md section 4.21) ----------------------------------------------------------
def _check_nonlocal(feat, offset, affinity, sparse_depth, prop_kernel, prop_time):
    """The checks of propagate2d_nonlocal; every refusal comes before anything is allocated or narrowed to int."""
    if prop_kernel not in (3, 5, 7) or isinstance(prop_kernel, bool):
        raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
    if isinstance(prop_time, bool) or not isinstance(prop_time, int) or not 0 <= prop_time <= 2 ** 31 - 1:
        raise ValueError(f'prop_time must be an int >= 0, got {prop_time!r}')
    T = prop_kernel * prop_kernel - 1
    if feat.dim() != 4 or min(feat.shape) < 1:
        raise ValueError(f'feat must be a non-empty (B,C,H,W), got {tuple(feat.shape)}')
    B, C, H, W = feat.shape
    if tuple(offset.shape) != (B, 2 * T, H, W):
        raise ValueError(f'offset must be (B, 2T, H, W) = {(B, 2 * T, H, W)}, got {tuple(offset.shape)}')
    if tuple(affinity.shape) != (B, T, H, W):
        raise ValueError(f'affinity must be (B, T, H, W) = {(B, T, H, W)}, got {tuple(affinity.shape)}')
    if sparse_depth is not None and tuple(sparse_depth.shape) != (B, C, H, W):
        raise ValueError(f'sparse_depth must have feat\'s shape {(B, C, H, W)}, got {tuple(sparse_depth.shape)}')
    ts = [t for t in (feat, offset, affinity, sparse_depth) if t is not None]
    if any(t.dtype != torch.float32 for t in ts):
        raise RuntimeError('cspn_b200 is fp32 only')
    if any(t.device != feat.device for t in ts):
        raise RuntimeError('feat, offset, affinity and sparse_depth must be on one device')
    if B > 2 ** 31 - 1 or C > 2 ** 31 - 1 or H * W * T >= 2 ** 31:
        raise _lib.CspnError(f'propagate2d_nonlocal takes B, C < 2^31 and H*W*T < 2^31, got feat {tuple(feat.shape)} at K={prop_kernel}')
    if not feat.is_cuda:
        raise _lib.CspnError('propagate2d_nonlocal takes CUDA tensors only (there is no host-buffer entry point for it)')


def _nonlocal_fwd(feat, offset, affinity, sparse_depth, prop_kernel, prop_time):
    """Forward only (no autograd) through cspn2d_nl_fwd_f32, on the current stream."""
    L = _lib.lib()
    f, o, a = feat.contiguous(), offset.contiguous(), affinity.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    B, C, H, W = f.shape
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        ws_bytes = L.cspn2d_nl_workspace_bytes(B, C, H, W, prop_kernel, prop_time)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
        rc = L.cspn2d_nl_fwd_f32(_ptr(f), _ptr(o), _ptr(a), _ptr(s), _ptr(out), B, C, H, W, prop_kernel, prop_time, _ptr(ws), ws_bytes,
                                 _stream(f.device))
    _lib.check(rc, 'cspn2d_nl_fwd_f32')
    return out


class _Propagate2dNonlocalFn(torch.autograd.Function):
    """autograd seam of propagate2d_nonlocal without the torch-op shim: native forward + native backward
    (cspn2d_nl_bwd_f32), differentiable in feat, offset, affinity and sparse_depth."""

    @staticmethod
    def forward(ctx, feat, offset, affinity, sparse_depth, prop_kernel, prop_time):
        ctx.save_for_backward(feat, offset, affinity, sparse_depth)
        ctx.cfg = (prop_kernel, prop_time)
        return _nonlocal_fwd(feat, offset, affinity, sparse_depth, prop_kernel, prop_time)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        feat, offset, affinity, sparse_depth = ctx.saved_tensors
        prop_kernel, prop_time = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        f, o, a, go = feat.contiguous(), offset.contiguous(), affinity.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        need_f, need_o, need_a, need_s = ctx.needs_input_grad[:4]
        need_s = need_s and s is not None
        gf = torch.empty_like(f) if need_f else None
        gof = torch.empty_like(o) if need_o else None
        ga = torch.empty_like(a) if need_a else None
        gs = torch.empty_like(s) if need_s else None
        B, C, H, W = f.shape
        with torch.cuda.device(f.device):
            ws_bytes = L.cspn2d_nl_bwd_workspace_bytes(B, C, H, W, prop_kernel, prop_time)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
            rc = L.cspn2d_nl_bwd_f32(_ptr(f), _ptr(o), _ptr(a), _ptr(s), _ptr(go), _ptr(gf), _ptr(gof), _ptr(ga), _ptr(gs), B, C, H, W,
                                     prop_kernel, prop_time, _ptr(ws), ws_bytes, _stream(f.device))
        _lib.check(rc, 'cspn2d_nl_bwd_f32')
        return gf, gof, ga, gs, None, None


def propagate2d_nonlocal(feat, offset, affinity, sparse_depth=None, prop_kernel=3, prop_time=18):
    """NLSPN's non-local 2D propagation (Park et al., ECCV 2020): each of a pixel's T = K*K - 1 neighbours sits at a learned,
    fractional offset from its grid position and is read by bilinear sampling (torchvision's deform_conv2d sampling).
    feat (B, C, H, W) is h_0; offset (B, 2T, H, W) holds (dy, dx) of tap k in channels 2k, 2k + 1; affinity (B, T, H, W)
    the weights a_k, used as given (normalise them before the call) and shared by the C channels; sparse_depth, of feat's
    shape, or None.  All fp32 CUDA tensors; prop_kernel K in {3, 5, 7}.  Tap k runs over (i, j) in [0, K)^2 in raster order
    without the centre, base offset (i - R, j - R), R = (K - 1) // 2: torchvision's and DCN's order, the reverse of the
    K x K propagation's (R - t, R - l).  prop_time steps of
        h_{t+1}(p) = a_c(p) h~_t(p) + sum_k a_k(p) S(h~_t, p + base_k + offset_k(p)),  a_c = 1 - sum_k a_k,
    where h~_t = (1 - m) h_t + m sparse_depth with m = 1[sparse_depth > 0] (h~_t = h_t without it); the result h_N is not
    replaced.  One step is deform_conv2d(h~_t, offset with a zero centre, ones(C, 1, K, K), padding=R, mask=affinity with
    a_c at the centre) with groups = C.  Differentiable in feat, offset, affinity and sparse_depth, with a deterministic
    backward (no floating-point atomics).  prop_time == 0 returns feat itself.  DESIGN.md section 4.21."""
    _check_nonlocal(feat, offset, affinity, sparse_depth, prop_kernel, prop_time)
    if prop_time == 0:
        return feat
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.propagate2d_nonlocal(feat, offset, affinity, sparse_depth, prop_kernel, prop_time)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (feat, offset, affinity, sparse_depth)):
        return _Propagate2dNonlocalFn.apply(feat, offset, affinity, sparse_depth, prop_kernel, prop_time)
    return _nonlocal_fwd(feat, offset, affinity, sparse_depth, prop_kernel, prop_time)


class Affinity_PropagateNonLocal(nn.Module):
    """NLSPN's non-local propagation as a module: forward(feat, offset, affinity, sparse_depth=None) is
    propagate2d_nonlocal(feat, offset, affinity, sparse_depth, prop_kernel, prop_time).  No parameters, no buffers: the
    offsets and affinities come from the caller's guidance network (INTEGRATION.md section 2f)."""

    def __init__(self, prop_time, prop_kernel=3):
        super().__init__()
        if prop_kernel not in (3, 5, 7):
            raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel

    def forward(self, feat, offset, affinity, sparse_depth=None):
        return propagate2d_nonlocal(feat, offset, affinity, sparse_depth, self.prop_kernel, self.prop_time)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}'


# ---- dilated 2D propagation with a centre weight and a learned confidence: PENet's DA-CSPN++ (DESIGN.md section 4.22) ------
def _check_dilated(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time):
    """The checks of propagate2d_dilated; every refusal comes before anything is allocated or narrowed to int."""
    if prop_kernel not in (3, 5, 7) or isinstance(prop_kernel, bool):
        raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
    if isinstance(dilation, bool) or not isinstance(dilation, int) or not 1 <= dilation <= 4:
        raise ValueError(f'dilation must be an int in [1, 4], got {dilation!r}')
    if isinstance(prop_time, bool) or not isinstance(prop_time, int) or not 0 <= prop_time <= 2 ** 31 - 1:
        raise ValueError(f'prop_time must be an int >= 0, got {prop_time!r}')
    if (sparse_depth is None) != (confidence is None):
        raise ValueError('sparse_depth and confidence come together or not at all')
    if blur_depth.dim() != 4 or min(blur_depth.shape) < 1:
        raise ValueError(f'blur_depth must be a non-empty (B,C,H,W), got {tuple(blur_depth.shape)}')
    B, C, H, W = blur_depth.shape
    KK = prop_kernel * prop_kernel
    if tuple(kernel.shape) != (B, KK, H, W):
        raise ValueError(f'kernel must be (B, K*K, H, W) = {(B, KK, H, W)}, got {tuple(kernel.shape)}')
    for name, t in (('sparse_depth', sparse_depth), ('confidence', confidence)):
        if t is not None and tuple(t.shape) != (B, 1, H, W):
            raise ValueError(f'{name} must be (B, 1, H, W) = {(B, 1, H, W)}, got {tuple(t.shape)}')
    ts = [t for t in (kernel, blur_depth, sparse_depth, confidence) if t is not None]
    if any(t.dtype != torch.float32 for t in ts):
        raise RuntimeError('cspn_b200 is fp32 only')
    if any(t.device != blur_depth.device for t in ts):
        raise RuntimeError('kernel, blur_depth, sparse_depth and confidence must be on one device')
    if B * C > 65535 or -(-H // 16) > 65535 or W > 2 ** 31 - 1:
        raise _lib.CspnError(f'propagate2d_dilated takes B*C <= 65535 and ceil(H/16) <= 65535, got blur_depth {tuple(blur_depth.shape)}')
    if not blur_depth.is_cuda:
        raise _lib.CspnError('propagate2d_dilated takes CUDA tensors only (there is no host-buffer entry point for it)')


def _dilated_fwd(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time):
    """Forward only (no autograd) through cspn2d_dil_fwd_f32, on the current stream."""
    L = _lib.lib()
    k, d = kernel.contiguous(), blur_depth.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    m = None if confidence is None else confidence.contiguous()
    B, C, H, W = d.shape
    out = torch.empty_like(d)
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_dil_workspace_bytes(B, C, H, W, prop_kernel, dilation, prop_time)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_dil_fwd_f32(_ptr(k), _ptr(d), _ptr(s), _ptr(m), _ptr(out), B, C, H, W, prop_kernel, dilation, prop_time,
                                  _ptr(ws), ws_bytes, _stream(d.device))
    _lib.check(rc, 'cspn2d_dil_fwd_f32')
    return out


class _Propagate2dDilatedFn(torch.autograd.Function):
    """autograd seam of propagate2d_dilated without the torch-op shim: native forward + native backward
    (cspn2d_dil_bwd_f32), differentiable in kernel, blur_depth, sparse_depth and confidence."""

    @staticmethod
    def forward(ctx, kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time):
        ctx.save_for_backward(kernel, blur_depth, sparse_depth, confidence)
        ctx.cfg = (prop_kernel, dilation, prop_time)
        return _dilated_fwd(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        kernel, blur_depth, sparse_depth, confidence = ctx.saved_tensors
        prop_kernel, dilation, prop_time = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        k, d, go = kernel.contiguous(), blur_depth.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        m = None if confidence is None else confidence.contiguous()
        need_k, need_d, need_s, need_m = ctx.needs_input_grad[:4]
        need_s, need_m = need_s and s is not None, need_m and m is not None
        gk = torch.empty_like(k) if need_k else None
        gd = torch.empty_like(d) if need_d else None
        gs = torch.empty_like(s) if need_s else None
        gm = torch.empty_like(m) if need_m else None
        B, C, H, W = d.shape
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_dil_bwd_workspace_bytes(B, C, H, W, prop_kernel, dilation, prop_time)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_dil_bwd_f32(_ptr(k), _ptr(d), _ptr(s), _ptr(m), _ptr(go), _ptr(gk), _ptr(gd), _ptr(gs), _ptr(gm), B, C, H, W,
                                      prop_kernel, dilation, prop_time, _ptr(ws), ws_bytes, _stream(d.device))
        _lib.check(rc, 'cspn2d_dil_bwd_f32')
        return gk, gd, gs, gm, None, None, None


def propagate2d_dilated(kernel, blur_depth, sparse_depth=None, confidence=None, prop_kernel=3, dilation=1, prop_time=6):
    """PENet's dilated and accelerated CSPN++ step (Hu et al., ICRA 2021), N = prop_time steps of
        u_t(p) = sum_{j != c} w_j(p) d_t(p + dilation*o_j) + w_c(p) d_0(p),
        d_{t+1} = m s + (1 - m) u_t   (d_{t+1} = u_t without samples),   out = d_N.
    kernel (B, K*K, H, W) holds the weights exactly as given (no abs, no normalisation, no softmax), shared by the C
    channels.  Channel j = i*K + l weights the value at p + dilation*(i - R, l - R), R = (K - 1) // 2: F.unfold's row
    order, PENet's `kernel` argument.  The centre channel c = (K*K - 1) // 2 weights d_0 = blur_depth (B, C, H, W), not the
    current iterate.  sparse_depth s and confidence m, (B, 1, H, W) and shared by the channels, come together or not at
    all and are used as given; a hard mask is confidence = (sparse_depth > 0).float().  A read outside the image is 0.
    All fp32 CUDA tensors; prop_kernel K in {3, 5, 7}, dilation in [1, 4].  Differentiable in kernel, blur_depth,
    sparse_depth and confidence, with a deterministic backward.  prop_time == 0 returns blur_depth itself.
    DESIGN.md section 4.22; INTEGRATION.md section 2g composes PENet's refinement from it."""
    _check_dilated(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time)
    if prop_time == 0:
        return blur_depth
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.propagate2d_dilated(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (kernel, blur_depth, sparse_depth, confidence)):
        return _Propagate2dDilatedFn.apply(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time)
    return _dilated_fwd(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time)


class Affinity_PropagateDilated(nn.Module):
    """PENet's DA-CSPN++ propagation as a module: forward(kernel, blur_depth, sparse_depth=None, confidence=None) is
    propagate2d_dilated(kernel, blur_depth, sparse_depth, confidence, prop_kernel, dilation, prop_time).  No parameters,
    no buffers: the weights and the confidence come from the caller's network (INTEGRATION.md section 2g)."""

    def __init__(self, prop_time, prop_kernel=3, dilation=1):
        super().__init__()
        if prop_kernel not in (3, 5, 7):
            raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
        if dilation not in (1, 2, 3, 4):
            raise ValueError(f'dilation must be in [1, 4], got {dilation!r}')
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        self.dilation = dilation

    def forward(self, kernel, blur_depth, sparse_depth=None, confidence=None):
        return propagate2d_dilated(kernel, blur_depth, sparse_depth, confidence, self.prop_kernel, self.dilation, self.prop_time)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, dilation={self.dilation}'


# ---- dynamic 2D propagation with per-step ring attention and an anchor to d_0: DySPN's step (DESIGN.md section 4.23) ------
def _check_dynamic(affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel):
    """The checks of propagate2d_dynamic; every refusal comes before anything is allocated or narrowed to int.  Returns N."""
    if prop_kernel not in (3, 5, 7) or isinstance(prop_kernel, bool):
        raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
    if (sparse_depth is None) != (confidence is None):
        raise ValueError('sparse_depth and confidence come together or not at all')
    if blur_depth.dim() != 4 or min(blur_depth.shape) < 1:
        raise ValueError(f'blur_depth must be a non-empty (B,C,H,W), got {tuple(blur_depth.shape)}')
    B, C, H, W = blur_depth.shape
    KK, NR = prop_kernel * prop_kernel, (prop_kernel + 1) // 2
    if tuple(affinity.shape) != (B, KK, H, W):
        raise ValueError(f'affinity must be (B, K*K, H, W) = {(B, KK, H, W)}, got {tuple(affinity.shape)}')
    if attention.dim() != 4 or tuple(attention.shape[::2]) != (B, H) or attention.shape[3] != W or attention.shape[1] % NR \
            or attention.shape[1] > 2 ** 31 - 1:
        raise ValueError(f'attention must be (B, N*(K+1)//2, H, W) with (K+1)//2 = {NR} and (B, H, W) = {(B, H, W)}, '
                         f'got {tuple(attention.shape)}')
    for name, t in (('sparse_depth', sparse_depth), ('confidence', confidence)):
        if t is not None and tuple(t.shape) != (B, 1, H, W):
            raise ValueError(f'{name} must be (B, 1, H, W) = {(B, 1, H, W)}, got {tuple(t.shape)}')
    ts = [t for t in (affinity, attention, blur_depth, sparse_depth, confidence) if t is not None]
    if any(t.dtype != torch.float32 for t in ts):
        raise RuntimeError('cspn_b200 is fp32 only')
    if any(t.device != blur_depth.device for t in ts):
        raise RuntimeError('affinity, attention, blur_depth, sparse_depth and confidence must be on one device')
    if B * C > 65535 or -(-H // 16) > 65535 or W > 2 ** 31 - 1:
        raise _lib.CspnError(f'propagate2d_dynamic takes B*C <= 65535 and ceil(H/16) <= 65535, got blur_depth {tuple(blur_depth.shape)}')
    if not blur_depth.is_cuda:
        raise _lib.CspnError('propagate2d_dynamic takes CUDA tensors only (there is no host-buffer entry point for it)')
    return attention.shape[1] // NR


def _dynamic_fwd(affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel, N):
    """Forward only (no autograd) through cspn2d_dyn_fwd_f32, on the current stream."""
    L = _lib.lib()
    a, at, d = affinity.contiguous(), attention.contiguous(), blur_depth.contiguous()
    s = None if sparse_depth is None else sparse_depth.contiguous()
    m = None if confidence is None else confidence.contiguous()
    B, C, H, W = d.shape
    out = torch.empty_like(d)
    with torch.cuda.device(d.device):
        ws_bytes = L.cspn2d_dyn_workspace_bytes(B, C, H, W, prop_kernel, N)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
        rc = L.cspn2d_dyn_fwd_f32(_ptr(a), _ptr(at), _ptr(d), _ptr(s), _ptr(m), _ptr(out), B, C, H, W, prop_kernel, N, _ptr(ws), ws_bytes,
                                  _stream(d.device))
    _lib.check(rc, 'cspn2d_dyn_fwd_f32')
    return out


class _Propagate2dDynamicFn(torch.autograd.Function):
    """autograd seam of propagate2d_dynamic without the torch-op shim: native forward + native backward
    (cspn2d_dyn_bwd_f32), differentiable in affinity, attention, blur_depth, sparse_depth and confidence."""

    @staticmethod
    def forward(ctx, affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel, N):
        ctx.save_for_backward(affinity, attention, blur_depth, sparse_depth, confidence)
        ctx.cfg = (prop_kernel, N)
        return _dynamic_fwd(affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel, N)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        affinity, attention, blur_depth, sparse_depth, confidence = ctx.saved_tensors
        prop_kernel, N = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        a, at, d, go = affinity.contiguous(), attention.contiguous(), blur_depth.contiguous(), grad_out.contiguous()
        s = None if sparse_depth is None else sparse_depth.contiguous()
        m = None if confidence is None else confidence.contiguous()
        need_a, need_t, need_d, need_s, need_m = ctx.needs_input_grad[:5]
        need_s, need_m = need_s and s is not None, need_m and m is not None
        ga = torch.empty_like(a) if need_a else None
        gt = torch.empty_like(at) if need_t else None
        gd = torch.empty_like(d) if need_d else None
        gs = torch.empty_like(s) if need_s else None
        gm = torch.empty_like(m) if need_m else None
        B, C, H, W = d.shape
        with torch.cuda.device(d.device):
            ws_bytes = L.cspn2d_dyn_bwd_workspace_bytes(B, C, H, W, prop_kernel, N)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=d.device) if ws_bytes else None
            rc = L.cspn2d_dyn_bwd_f32(_ptr(a), _ptr(at), _ptr(d), _ptr(s), _ptr(m), _ptr(go), _ptr(ga), _ptr(gt), _ptr(gd), _ptr(gs),
                                      _ptr(gm), B, C, H, W, prop_kernel, N, _ptr(ws), ws_bytes, _stream(d.device))
        _lib.check(rc, 'cspn2d_dyn_bwd_f32')
        return ga, gt, gd, gs, gm, None, None


def propagate2d_dynamic(affinity, attention, blur_depth, sparse_depth=None, confidence=None, prop_kernel=7):
    """DySPN's dynamic spatial propagation (Lin et al., AAAI 2022), N = attention.shape[1] // ((K + 1) // 2) steps of
        w_{t,j}(p) = a_{t,ring(j)}(p) affinity_j(p),   rho_t(p) = 1 - sum_j w_{t,j}(p),
        v_t(p) = rho_t(p) d_0(p) + sum_j w_{t,j}(p) d_t(p + o_j),
        d_{t+1} = m s + (1 - m) v_t   (d_{t+1} = v_t without samples),   out = d_N.
    affinity (B, K*K, H, W) holds all K*K taps, the centre included, exactly as given (no abs, no normalisation), shared by
    the C channels.  Channel j = i*K + l weights d_t(p + o_j), o_j = (i - R, l - R), R = (K - 1) // 2: F.unfold's row
    order.  Tap j lies on ring(j) = max(|i - R|, |l - R|): ring 0 is the centre, ring r holds 8r taps.  attention
    (B, N*(R+1), H, W) holds, in channel t*(R+1) + r, the attention of ring r at step t, used as given (the caller applies
    the sigmoid).  The weight the attention takes away goes back to d_0 = blur_depth (B, C, H, W) through rho.
    sparse_depth s and confidence m, (B, 1, H, W) and shared by the channels, come together or not at all and are used as
    given; a hard mask is confidence = (sparse_depth > 0).float().  A read outside the image is 0.  All fp32 CUDA tensors;
    prop_kernel K in {3, 5, 7}.  Differentiable in affinity, attention, blur_depth, sparse_depth and confidence, with a
    deterministic backward.  N == 0 returns blur_depth itself.
    DESIGN.md section 4.23; INTEGRATION.md section 2h composes a DySPN head from it."""
    N = _check_dynamic(affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel)
    if N == 0:
        return blur_depth
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.propagate2d_dynamic(affinity, attention, blur_depth, sparse_depth, confidence, prop_kernel)
    ts = (affinity, attention, blur_depth, sparse_depth, confidence)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts):
        return _Propagate2dDynamicFn.apply(*ts, prop_kernel, N)
    return _dynamic_fwd(*ts, prop_kernel, N)


class Affinity_PropagateDynamic(nn.Module):
    """DySPN's dynamic propagation as a module: forward(affinity, attention, blur_depth, sparse_depth=None,
    confidence=None) is propagate2d_dynamic(...) after checking that the attention has the prop_time * (K + 1) // 2
    channels prop_time implies.  No parameters, no buffers: the affinity, the attention and the confidence come from the
    caller's network (INTEGRATION.md section 2h)."""

    def __init__(self, prop_time, prop_kernel=7):
        super().__init__()
        if prop_kernel not in (3, 5, 7) or isinstance(prop_kernel, bool):
            raise ValueError(f'prop_kernel must be 3, 5 or 7, got {prop_kernel!r}')
        if isinstance(prop_time, bool) or not isinstance(prop_time, int) or prop_time < 0:
            raise ValueError(f'prop_time must be an int >= 0, got {prop_time!r}')
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel

    def forward(self, affinity, attention, blur_depth, sparse_depth=None, confidence=None):
        want = self.prop_time * ((self.prop_kernel + 1) // 2)
        if attention.dim() != 4 or attention.shape[1] != want:
            raise ValueError(f'prop_time={self.prop_time} at prop_kernel={self.prop_kernel} needs {want} attention channels, '
                             f'got attention {tuple(attention.shape)}')
        return propagate2d_dynamic(affinity, attention, blur_depth, sparse_depth, confidence, self.prop_kernel)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}'


# ---- linear three-way scans: SPN's propagation (DESIGN.md section 4.24) ------------------------------------------------
LINEAR_DIRECTIONS = ('l2r', 'r2l', 't2b', 'b2t')


def _linear_mask(directions):
    """dir_mask of a non-empty subsequence of ('l2r', 'r2l', 't2b', 'b2t')."""
    if isinstance(directions, str):
        raise ValueError(f'directions must be a sequence of direction names, got {directions!r}')
    ds = tuple(directions)
    idx = [LINEAR_DIRECTIONS.index(d) if d in LINEAR_DIRECTIONS else -1 for d in ds]
    if not ds or -1 in idx or idx != sorted(set(idx)):
        raise ValueError(f'directions must be a non-empty subsequence of {LINEAR_DIRECTIONS}, got {directions!r}')
    return sum(1 << i for i in idx)


def _check_linear(feat, gate, directions):
    """The checks of propagate2d_linear; every refusal comes before anything is allocated.  Returns (mask, gate_mode)."""
    mask = _linear_mask(directions)
    nd = len(tuple(directions))
    if feat.dim() != 4 or min(feat.shape) < 1:
        raise ValueError(f'feat must be a non-empty (B,C,H,W), got {tuple(feat.shape)}')
    B, C, H, W = feat.shape
    if gate.dim() != 4 or tuple(gate.shape[::2]) != (B, H) or gate.shape[3] != W or \
            not (gate.shape[1] == 3 * nd or (C > 1 and gate.shape[1] == 3 * nd * C)):
        raise ValueError(f'gate must be (B, 3*nd, H, W) = {(B, 3 * nd, H, W)} or, with C > 1, (B, 3*nd*C, H, W) = '
                         f'{(B, 3 * nd * C, H, W)}, got {tuple(gate.shape)}')
    if feat.dtype != torch.float32 or gate.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if gate.device != feat.device:
        raise RuntimeError('feat and gate must be on one device')
    lateral = max(H if mask & 3 else 0, W if mask & 12 else 0)
    if B * C > 2 ** 31 - 1 or lateral > 2048 or H * W > 2 ** 31 - 1:
        raise _lib.CspnError(f'propagate2d_linear takes B*C <= 2^31 - 1 and a lateral extent (H for l2r / r2l, W for t2b / b2t) '
                             f'<= 2048, got feat {tuple(feat.shape)}')
    if not feat.is_cuda:
        raise _lib.CspnError('propagate2d_linear takes CUDA tensors only (there is no host-buffer entry point for it)')
    return mask, (0 if gate.shape[1] == 3 * nd else 1)


def _linear_fwd(feat, gate, mask, mode, keep_planes):
    """Forward only (no autograd) through cspn2d_lin_fwd_f32, on the current stream.  Returns (out, planes): planes is
    None for one direction, or when keep_planes is false (they then live in a workspace)."""
    L = _lib.lib()
    x, g = feat.contiguous(), gate.contiguous()
    B, C, H, W = x.shape
    nd = sum((mask >> i) & 1 for i in range(4))
    out = torch.empty_like(x)
    planes = torch.empty((nd, B, C, H, W), dtype=x.dtype, device=x.device) if keep_planes and nd > 1 else None
    with torch.cuda.device(x.device):
        ws_bytes = 0 if planes is not None else L.cspn2d_lin_workspace_bytes(B, C, H, W, mask, mode)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
        rc = L.cspn2d_lin_fwd_f32(_ptr(x), _ptr(g), _ptr(out), _ptr(planes), B, C, H, W, mask, mode, _ptr(ws), ws_bytes,
                                  _stream(x.device))
    _lib.check(rc, 'cspn2d_lin_fwd_f32')
    return out, planes


class _Propagate2dLinearFn(torch.autograd.Function):
    """autograd seam of propagate2d_linear without the torch-op shim: native forward + native backward
    (cspn2d_lin_bwd_f32) over the saved per-direction planes, differentiable in feat and gate."""

    @staticmethod
    def forward(ctx, feat, gate, mask, mode):
        out, planes = _linear_fwd(feat, gate, mask, mode, True)
        ctx.save_for_backward(feat, gate, out if planes is None else planes)
        ctx.cfg = (mask, mode)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        feat, gate, planes = ctx.saved_tensors
        mask, mode = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        x, g, p, go = feat.contiguous(), gate.contiguous(), planes.contiguous(), grad_out.contiguous()
        need_x, need_g = ctx.needs_input_grad[:2]
        gx = torch.empty_like(x) if need_x else None
        gg = torch.empty_like(g) if need_g else None
        B, C, H, W = x.shape
        with torch.cuda.device(x.device):
            ws_bytes = L.cspn2d_lin_bwd_workspace_bytes(B, C, H, W, mask, mode)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
            rc = L.cspn2d_lin_bwd_f32(_ptr(x), _ptr(g), _ptr(p), _ptr(go), _ptr(gx), _ptr(gg), B, C, H, W, mask, mode, _ptr(ws),
                                      ws_bytes, _stream(x.device))
        _lib.check(rc, 'cspn2d_lin_bwd_f32')
        return gx, gg, None, None


def propagate2d_linear(feat, gate, directions=LINEAR_DIRECTIONS):
    """SPN's linear spatial propagation with three-way connections (Liu et al., NIPS 2017), one scan per direction and a
    node-wise max over the directions.  For 'l2r' (scan index t the column, lateral index i the row):
        h[i, t] = (1 - g0 - g1 - g2) x[i, t] + g0 h[i-1, t-1] + g1 h[i, t-1] + g2 h[i+1, t-1]
    with g_j = gate_j[i, t] at the current node, used as given (no abs, no normalisation: SPN's stability condition
    sum_j |g_j| <= 1 is the caller's to enforce), and reads outside the image 0.  'r2l' reads column t + 1, 't2b' and
    'b2t' scan rows and read row y -+ 1 at columns x - 1, x, x + 1; tap j is lateral offset j - 1 along increasing index.
    directions is a non-empty subsequence of ('l2r', 'r2l', 't2b', 'b2t').  gate is (B, 3*nd, H, W), shared by the C
    channels of feat (B, C, H, W), or (B, 3*nd*C, H, W) with C > 1, one gate per channel; direction block k (the k-th
    listed direction) is channels [3k*C', 3(k+1)*C') with C' = 1 or C, and channel c uses 3c .. 3c+2 within it, so
    gate[:, block k] is the gate of a one-direction call.  Several directions are merged node-wise by max: out is h of the
    first direction that is NaN there, else of the first attaining the maximum (torch.stack(hs).max(0)); the gradient goes
    to that direction alone.  fp32 CUDA tensors; differentiable in feat and gate with a deterministic backward.
    DESIGN.md section 4.24 states the order of every operation; INTEGRATION.md section 2i builds an SPN head from it."""
    mask, mode = _check_linear(feat, gate, directions)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.propagate2d_linear(feat, gate, mask)[0]
    if torch.is_grad_enabled() and (feat.requires_grad or gate.requires_grad):
        return _Propagate2dLinearFn.apply(feat, gate, mask, mode)
    return _linear_fwd(feat, gate, mask, mode, False)[0]


class Affinity_PropagateLinear(nn.Module):
    """SPN's linear propagation as a module: forward(feat, gate) is propagate2d_linear(feat, gate, directions).  No
    parameters, no buffers: the gates come from the caller's guidance network (INTEGRATION.md section 2i)."""

    def __init__(self, directions=LINEAR_DIRECTIONS):
        super().__init__()
        _linear_mask(directions)
        self.directions = tuple(directions)

    def forward(self, feat, gate):
        return propagate2d_linear(feat, gate, self.directions)

    def extra_repr(self):
        return f'directions={self.directions}'


# ---- 3D with a K x K x K affinity kernel (K in {3, 5}) ---------------------------------------------------------------
KERNEL_SIZES_3D = (3, 5)


def norm_code_3d_k(prop_kernel, norm_type=None):
    """The norm names of a K x K x K kernel follow the 3D naming, f'{K**3-1}sum' / f'{K**3-1}sum_abs' ('26sum', '124sum',
    ...) and 'paddle'; returns the cspn_norm3d code (0 signed, 1 abs, 2 paddle).  The default is f'{K**3-1}sum_abs', as in
    Affinity_Propagate3D.  Raises AssertionError for another K or name."""
    assert prop_kernel in KERNEL_SIZES_3D, f'prop_kernel must be 3 or 5 in 3D, got {prop_kernel}'
    nt = prop_kernel ** 3 - 1
    names = {f'{nt}sum': 0, f'{nt}sum_abs': 1, 'paddle': 2}
    norm_type = norm_type or f'{nt}sum_abs'
    assert norm_type in names, (f'norm_type of a {prop_kernel}x{prop_kernel}x{prop_kernel} kernel is one of {sorted(names)}, '
                                f'got {norm_type!r}')
    return names[norm_type]


def _check_shapes_3d_k(guidance, feat, prop_kernel):
    nt = prop_kernel ** 3 - 1
    if guidance.dim() != 5 or feat.dim() != 5:
        raise ValueError('guidance and feat must be (B,C,D,H,W)')
    if guidance.dtype != torch.float32 or feat.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    B, C, D, H, W = feat.shape
    if guidance.shape != (B, nt, D, H, W):
        raise ValueError(f'a {prop_kernel}x{prop_kernel}x{prop_kernel} kernel needs guidance (B,{nt},D,H,W) or, with C > 1 '
                         f'feature channels, (B,{nt}*C,D,H,W); got {tuple(guidance.shape)} for feat {tuple(feat.shape)}')
    if guidance.device != feat.device:
        raise RuntimeError('guidance and feat are on different devices')


def propagate3d_k(guidance, feat, prop_kernel=5, prop_time=12, norm_type=None):
    """3D CSPN with a K x K x K affinity kernel, forward only (no autograd), CUDA tensors only, enqueued on the current
    stream.  guidance (B, K**3-1, D, H, W), one gate shared by the C channels of feat (B, C, D, H, W); norm_type
    f'{K**3-1}sum', f'{K**3-1}sum_abs' (default) or 'paddle'.  K = 3 is propagate3d itself (same kernels, same bits)."""
    code = norm_code_3d_k(prop_kernel, norm_type)
    _check_shapes_3d_k(guidance, feat, prop_kernel)
    if not (guidance.is_cuda and feat.is_cuda):
        raise _lib.CspnError(f'the {prop_kernel}x{prop_kernel}x{prop_kernel} propagation takes CUDA tensors only '
                             '(there is no host-buffer entry point for it)')
    if prop_time == 0:
        return feat
    if prop_kernel == 3:
        return propagate3d(guidance, feat, prop_time, ('26sum', '26sum_abs', 'paddle')[code])
    L = _lib.lib()
    B, C, D, H, W = feat.shape
    g, f = guidance.contiguous(), feat.contiguous()
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        ws_bytes = L.cspn3d_k_workspace_bytes(B, C, D, H, W, prop_kernel, int(prop_time))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
        rc = L.cspn3d_k_fwd_f32(_ptr(g), _ptr(f), _ptr(out), B, C, D, H, W, prop_kernel, int(prop_time), code, _ptr(ws),
                                ws_bytes, _stream(f.device))
    _lib.check(rc, 'cspn3d_k_fwd_f32')
    return out


class _Propagate3dKFn(torch.autograd.Function):
    """autograd seam of the K x K x K operator without the torch-op shim: native forward + native adjoint (cspn3d_k_bwd_f32)."""

    @staticmethod
    def forward(ctx, guidance, feat, prop_kernel, prop_time, norm_type):
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (prop_kernel, prop_time, norm_type)
        return propagate3d_k(guidance, feat, prop_kernel, prop_time, norm_type)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        prop_kernel, prop_time, norm_type = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        B, C, D, H, W = feat.shape
        g, f, go = guidance.contiguous(), feat.contiguous(), grad_out.contiguous()
        gg = torch.empty_like(g) if ctx.needs_input_grad[0] else None
        gf = torch.empty_like(f) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(f.device):
            ws_bytes = L.cspn3d_k_bwd_workspace_bytes(B, C, D, H, W, prop_kernel, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
            rc = L.cspn3d_k_bwd_f32(_ptr(g), _ptr(f), _ptr(go), _ptr(gg), _ptr(gf), B, C, D, H, W, prop_kernel, int(prop_time),
                                    norm_code_3d_k(prop_kernel, norm_type), _ptr(ws), ws_bytes, _stream(f.device))
        _lib.check(rc, 'cspn3d_k_bwd_f32')
        return gg, gf, None, None, None


class Affinity_Propagate3DK(nn.Module):
    """3D CSPN with a K x K x K affinity kernel, K in {3, 5}: Affinity_Propagate3D with K**3-1 neighbours instead of 26
    (DESIGN.md section 4.9).  forward(guidance, feat (B, C, D, H, W)): guidance is (B, K**3-1, D, H, W), one gate shared by
    the C channels, or (B, (K**3-1)*C, D, H, W) with C > 1, one gate per channel (cspn_paddle/demo.py:28-45).  norm_type
    defaults to f'{K**3-1}sum_abs'; the others are f'{K**3-1}sum' and 'paddle'.  No parameters, no buffers; prop_time == 0
    returns feat itself.  Forward and backward run in CUDA kernels (K = 3 in those of Affinity_Propagate3D, same bits)."""

    def __init__(self, prop_time, prop_kernel, norm_type=None):
        super().__init__()
        norm_code_3d_k(prop_kernel, norm_type)      # AssertionError for K not in {3, 5} or a name that does not match K
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        self.norm_type = norm_type or f'{prop_kernel ** 3 - 1}sum_abs'
        self._use_op = _use_torch_op()

    def forward(self, guidance, feat):
        if self.prop_time == 0:
            return feat
        views = _per_channel_gate_views(guidance, feat, self.prop_kernel ** 3 - 1)
        if views is not None:
            return self.forward(*views).view(feat.shape)
        _check_shapes_3d_k(guidance, feat, self.prop_kernel)
        code = norm_code_3d_k(self.prop_kernel, self.norm_type)
        if self._use_op and feat.is_cuda:
            return torch.ops.cspn_b200.propagate3d_k(guidance, feat, self.prop_kernel, self.prop_time, code)
        if torch.is_grad_enabled() and (guidance.requires_grad or feat.requires_grad):
            return _Propagate3dKFn.apply(guidance, feat, self.prop_kernel, self.prop_time, self.norm_type)
        return propagate3d_k(guidance, feat, self.prop_kernel, self.prop_time, self.norm_type)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, norm_type={self.norm_type!r}'


# ---- 2D with the Paddle module's own-location gates (K in {3, 5, 7}) -------------------------------------------------
def _check_inputs_2d_paddle(guidance, feat, prop_kernel):
    """Shapes of CSPN.cspn with dim_num = 2 (cspn_paddle/demo.py:20-54).  guidance (B, K*K-1, H, W) is one gate shared by
    the C channels of feat (B, C, H, W); (B, (K*K-1)*C, H, W) with C > 1 gives channel c the guide channels
    [nt*c, nt*c+nt) (demo.py:28-45), which in memory is B*C single-channel images.  Any other channel count is a
    ValueError: demo.py normalises over every guide channel it is given.  Returns the (images, channels) of the C ABI."""
    assert prop_kernel in KERNEL_SIZES_2D, f'prop_kernel must be 3, 5 or 7, got {prop_kernel}'
    nt = prop_kernel * prop_kernel - 1
    if guidance.dim() != 4 or feat.dim() != 4:
        raise ValueError('guidance and feat must be (B,C,H,W)')
    if guidance.dtype != torch.float32 or feat.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    B, C, H, W = feat.shape
    per_channel = C > 1 and guidance.shape[1] == nt * C
    if guidance.shape[0] != B or guidance.shape[2:] != (H, W) or not (guidance.shape[1] == nt or per_channel):
        raise ValueError(f"a {prop_kernel}x{prop_kernel} 'paddle' kernel needs guidance (B,{nt},H,W) or, with C > 1 feature "
                         f'channels, (B,{nt}*C,H,W); got {tuple(guidance.shape)} for feat {tuple(feat.shape)}')
    if guidance.device != feat.device:
        raise RuntimeError('guidance and feat are on different devices')
    if not (guidance.is_cuda and feat.is_cuda):
        raise _lib.CspnError(f"the {prop_kernel}x{prop_kernel} 'paddle' propagation takes CUDA tensors only "
                             '(there is no host-buffer entry point for it)')
    return (B * C, 1) if per_channel else (B, C)


def propagate2d_paddle(guidance, feat, prop_kernel=3, prop_time=24):
    """CSPN.cspn of the Paddle module with dim_num = 2, forward only (no autograd), CUDA tensors only, enqueued on the
    current stream: w_k = |g_k| / sum_j |g_j| at each pixel's own location, then prop_time steps
    d <- sum_k w_k shift_k(d) (zero padding, no centre term).  Shapes as in Affinity_Propagate2DPaddle."""
    Bi, Ci = _check_inputs_2d_paddle(guidance, feat, prop_kernel)
    if prop_time == 0:
        return feat
    L = _lib.lib()
    H, W = feat.shape[2:]
    g, f = guidance.contiguous(), feat.contiguous()
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        ws_bytes = L.cspn2d_paddle_workspace_bytes(Bi, Ci, H, W, prop_kernel, int(prop_time))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
        rc = L.cspn2d_paddle_fwd_f32(_ptr(g), _ptr(f), _ptr(out), Bi, Ci, H, W, prop_kernel, int(prop_time), _ptr(ws), ws_bytes,
                                     _stream(f.device))
    _lib.check(rc, 'cspn2d_paddle_fwd_f32')
    return out


class _Propagate2dPaddleFn(torch.autograd.Function):
    """autograd seam of the 2D 'paddle' operator without the torch-op shim: native forward + native adjoint
    (cspn2d_paddle_bwd_f32)."""

    @staticmethod
    def forward(ctx, guidance, feat, prop_kernel, prop_time):
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (prop_kernel, prop_time)
        return propagate2d_paddle(guidance, feat, prop_kernel, prop_time)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        prop_kernel, prop_time = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        Bi, Ci = _check_inputs_2d_paddle(guidance, feat, prop_kernel)
        L = _lib.lib()
        H, W = feat.shape[2:]
        g, f, go = guidance.contiguous(), feat.contiguous(), grad_out.contiguous()
        gg = torch.empty_like(g) if ctx.needs_input_grad[0] else None
        gf = torch.empty_like(f) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(f.device):
            ws_bytes = L.cspn2d_paddle_bwd_workspace_bytes(Bi, Ci, H, W, prop_kernel, int(prop_time))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device) if ws_bytes else None
            rc = L.cspn2d_paddle_bwd_f32(_ptr(g), _ptr(f), _ptr(go), _ptr(gg), _ptr(gf), Bi, Ci, H, W, prop_kernel,
                                         int(prop_time), _ptr(ws), ws_bytes, _stream(f.device))
        _lib.check(rc, 'cspn2d_paddle_bwd_f32')
        return gg, gf, None, None


class Affinity_Propagate2DPaddle(nn.Module):
    """The 2D half of the Paddle module (cspn_paddle/demo.py --dimNum=2): CSPN.cspn(guide, feat) with dim_num = 2,
    K in {3, 5, 7} (demo.py:65, guide_chan = K*K-1).  forward(guidance, feat (B, C, H, W)): guidance (B, K*K-1, H, W), one
    gate shared by the C channels, or (B, (K*K-1)*C, H, W) with C > 1, one gate per channel.  The gates are |guidance|
    normalised over the channels at each pixel's own location; each of prop_time steps is sum_k w_k shift_k(feat), with
    zero padding, no centre term and no sparse replacement (DESIGN.md section 4.10).  No parameters, no buffers;
    prop_time == 0 returns feat itself.  Forward and backward run in CUDA kernels."""

    def __init__(self, prop_time, prop_kernel=3):
        super().__init__()
        assert prop_kernel in KERNEL_SIZES_2D, f'prop_kernel must be 3, 5 or 7, got {prop_kernel}'
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        self._use_op = _use_torch_op()

    def forward(self, guidance, feat):
        if self.prop_time == 0:
            return feat
        _check_inputs_2d_paddle(guidance, feat, self.prop_kernel)
        if self._use_op:
            return torch.ops.cspn_b200.propagate2d_paddle(guidance, feat, self.prop_kernel, self.prop_time)
        if torch.is_grad_enabled() and (guidance.requires_grad or feat.requires_grad):
            return _Propagate2dPaddleFn.apply(guidance, feat, self.prop_kernel, self.prop_time)
        return propagate2d_paddle(guidance, feat, self.prop_kernel, self.prop_time)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}'


# ---- caller-supplied gates: fluid.layers.affinity_propagate itself (2D K in {3, 5, 7}, 3D K in {3, 5}) ----------------
def _check_gates(input, gate_weight, kernel_size, prop_step):
    """Shapes of fluid.layers.affinity_propagate(input, gate_weight, kernel_size) (cspn_paddle/demo.py:41-43, 51-52): a 4-D
    input (B, C, H, W) is 2D, a 5-D one (B, C, D, H, W) is 3D.  gate_weight (B, K**d-1, ...) is one gate shared by the C
    channels; (B, (K**d-1)*C, ...) with C > 1 gives channel c the gate channels [nt*c, nt*c+nt) (demo.py:28-45), which in
    memory is B*C single-channel images.  Returns (d, images, channels) of the C ABI."""
    if input.dim() not in (4, 5):
        raise ValueError(f'input must be (B,C,H,W) or (B,C,D,H,W), got {tuple(input.shape)}')
    nd = input.dim() - 2
    sizes = KERNEL_SIZES_2D if nd == 2 else KERNEL_SIZES_3D
    assert kernel_size in sizes, f'kernel_size of a {nd}D affinity_propagate must be one of {sizes}, got {kernel_size}'
    nt = kernel_size ** nd - 1
    if gate_weight.dim() != input.dim():
        raise ValueError(f'gate_weight must have the dimensions of input, got {tuple(gate_weight.shape)} for {tuple(input.shape)}')
    if prop_step < 0:
        raise ValueError(f'prop_step must be >= 0, got {prop_step}')
    if input.dtype != torch.float32 or gate_weight.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    B, C = input.shape[:2]
    per_channel = C > 1 and gate_weight.shape[1] == nt * C
    if gate_weight.shape[0] != B or gate_weight.shape[2:] != input.shape[2:] or not (gate_weight.shape[1] == nt or per_channel):
        raise ValueError(f'a {"x".join([str(kernel_size)] * nd)} kernel needs gate_weight (B,{nt},...) or, with C > 1 input '
                         f'channels, (B,{nt}*C,...); got {tuple(gate_weight.shape)} for input {tuple(input.shape)}')
    if gate_weight.device != input.device:
        raise RuntimeError('input and gate_weight are on different devices')
    if not (input.is_cuda and gate_weight.is_cuda):
        raise _lib.CspnError('affinity_propagate takes CUDA tensors only (there is no host-buffer entry point for it)')
    return (nd,) + ((B * C, 1) if per_channel else (B, C))


def _affinity_propagate_fwd(input, gate_weight, kernel_size, prop_step):
    """Forward only (no autograd) through cspn{2,3}d_gates_fwd_f32, enqueued on the current stream."""
    nd, Bi, Ci = _check_gates(input, gate_weight, kernel_size, prop_step)
    if prop_step == 0:
        return input
    L = _lib.lib()
    g, x = gate_weight.contiguous(), input.contiguous()
    out = torch.empty_like(x)
    name = f'cspn{nd}d_gates'
    with torch.cuda.device(x.device):
        ws_bytes = getattr(L, f'{name}_workspace_bytes')(Bi, Ci, *x.shape[2:], kernel_size, int(prop_step))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
        rc = getattr(L, f'{name}_fwd_f32')(_ptr(g), _ptr(x), _ptr(out), Bi, Ci, *x.shape[2:], kernel_size, int(prop_step),
                                           _ptr(ws), ws_bytes, _stream(x.device))
    _lib.check(rc, f'{name}_fwd_f32')
    return out


class _AffinityPropagateFn(torch.autograd.Function):
    """autograd seam of affinity_propagate without the torch-op shim: native forward + native adjoint
    (cspn{2,3}d_gates_bwd_f32)."""

    @staticmethod
    def forward(ctx, input, gate_weight, kernel_size, prop_step):
        ctx.save_for_backward(input, gate_weight)
        ctx.cfg = (kernel_size, prop_step)
        return _affinity_propagate_fwd(input, gate_weight, kernel_size, prop_step)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        input, gate_weight = ctx.saved_tensors
        kernel_size, prop_step = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        nd, Bi, Ci = _check_gates(input, gate_weight, kernel_size, prop_step)
        L = _lib.lib()
        x, g, go = input.contiguous(), gate_weight.contiguous(), grad_out.contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gg = torch.empty_like(g) if ctx.needs_input_grad[1] else None
        name = f'cspn{nd}d_gates'
        with torch.cuda.device(x.device):
            ws_bytes = getattr(L, f'{name}_bwd_workspace_bytes')(Bi, Ci, *x.shape[2:], kernel_size, int(prop_step))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
            rc = getattr(L, f'{name}_bwd_f32')(_ptr(g), _ptr(x), _ptr(go), _ptr(gg), _ptr(gx), Bi, Ci, *x.shape[2:], kernel_size,
                                               int(prop_step), _ptr(ws), ws_bytes, _stream(x.device))
        _lib.check(rc, f'{name}_bwd_f32')
        return gx, gg, None, None


def affinity_propagate(input, gate_weight, kernel_size=3, prop_step=1):
    """fluid.layers.affinity_propagate(input, gate_weight, kernel_size), the op the Paddle module calls once per step
    (cspn_paddle/demo.py:41-43, 51-52), run prop_step times with the gates exactly as given:
        d_{t+1}(p) = sum_k gate_k(p) * d_t(p + off_k),   d_0 = input,
    zero padding, no centre term, no normalisation (the caller normalises: cspn_paddle/README.md:54).  A 4-D input
    (B, C, H, W) is 2D with kernel_size 3, 5 or 7; a 5-D input (B, C, D, H, W) is 3D with kernel_size 3 or 5.  gate_weight is
    (B, K**d-1, ...), shared by the C channels, or (B, (K**d-1)*C, ...) with C > 1, one gate per channel.  Taps in the raster
    order of the K x K (x K) operators (DESIGN.md section 4.11).  Differentiable in both arguments; fp32 CUDA tensors only;
    prop_step == 0 returns input itself."""
    _check_gates(input, gate_weight, kernel_size, prop_step)
    if prop_step == 0:
        return input
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        op = torch.ops.cspn_b200.affinity_propagate2d if input.dim() == 4 else torch.ops.cspn_b200.affinity_propagate3d
        return op(input, gate_weight, kernel_size, prop_step)
    if torch.is_grad_enabled() and (input.requires_grad or gate_weight.requires_grad):
        return _AffinityPropagateFn.apply(input, gate_weight, kernel_size, prop_step)
    return _affinity_propagate_fwd(input, gate_weight, kernel_size, prop_step)


# ---- the guidance and depth heads: Unpool + crop + 3x3 convolution (torch_resnet_cspn_nyu.py:41-54, 187-205) ----------
def unpool_output_size(h, w, oheight=0, owidth=0):
    """The head's output size: the crop (oheight, owidth) when both are non-zero, else the whole unpooled map (2h, 2w)
    (Simple_Gudi_UpConv_Block_Last_Layer._up_pooling, torch_resnet_cspn_nyu.py:195-200)."""
    return (oheight, owidth) if oheight != 0 and owidth != 0 else (2 * h, 2 * w)


def _check_unpool_conv(x, weight, H, W):
    if x.dim() != 4 or weight.dim() != 4 or weight.shape[1] != x.shape[1] or tuple(weight.shape[2:]) != (3, 3):
        raise ValueError(f'x must be (B,Cin,h,w) and weight (Cout,Cin,3,3), got {tuple(x.shape)} and {tuple(weight.shape)}')
    if not (1 <= H <= 2 * x.shape[2] and 1 <= W <= 2 * x.shape[3]):
        raise ValueError(f'output {H}x{W} must be at least 1x1 and within the unpooled map {2 * x.shape[2]}x{2 * x.shape[3]}')
    if x.dtype != torch.float32 or weight.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if x.device != weight.device:
        raise RuntimeError('x and weight are on different devices')
    if not x.is_cuda:
        raise _lib.CspnError('unpool_conv3x3 takes CUDA tensors only (there is no host-buffer entry point for it)')


def _unpool_conv_fwd(x, weight, H, W):
    """Forward only (no autograd) through cspn_unpool_conv3x3_fwd_f32, enqueued on the current stream."""
    L = _lib.lib()
    xc, wc = x.contiguous(), weight.contiguous()
    out = xc.new_empty((xc.shape[0], wc.shape[0], H, W))
    with torch.cuda.device(xc.device):
        rc = L.cspn_unpool_conv3x3_fwd_f32(_ptr(xc), _ptr(wc), _ptr(out), *xc.shape, wc.shape[0], H, W, _stream(xc.device))
    _lib.check(rc, 'cspn_unpool_conv3x3_fwd_f32')
    return out


class _UnpoolConv3x3Fn(torch.autograd.Function):
    """autograd seam of unpool_conv3x3 without the torch-op shim: native forward + native backward
    (cspn_unpool_conv3x3_bwd_f32)."""

    @staticmethod
    def forward(ctx, x, weight, H, W):
        ctx.save_for_backward(x, weight)
        ctx.cfg = (H, W)
        return _unpool_conv_fwd(x, weight, H, W)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        x, weight = ctx.saved_tensors
        H, W = ctx.cfg
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        L = _lib.lib()
        xc, wc, go = x.contiguous(), weight.contiguous(), grad_out.contiguous()
        gx = torch.empty_like(xc) if ctx.needs_input_grad[0] else None
        gw = torch.empty_like(wc) if ctx.needs_input_grad[1] else None
        if gx is None and gw is None:
            return None, None, None, None
        shape = (*xc.shape, wc.shape[0], H, W)
        with torch.cuda.device(xc.device):
            ws_bytes = L.cspn_unpool_conv3x3_bwd_workspace_bytes(*shape) if gw is not None else 0
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=xc.device) if ws_bytes else None
            rc = L.cspn_unpool_conv3x3_bwd_f32(_ptr(xc), _ptr(wc), _ptr(go), _ptr(gx), _ptr(gw), *shape, _ptr(ws), ws_bytes,
                                               _stream(xc.device))
        _lib.check(rc, 'cspn_unpool_conv3x3_bwd_f32')
        return gx, gw, None, None


def unpool_conv3x3(x, weight, oheight=0, owidth=0):
    """The reference head's forward in one CUDA kernel: Unpool(x) (a [1,0;0,0] conv_transpose2d, stride 2), cropped to
    (oheight, owidth) when both are non-zero, then a 3x3 convolution with zero padding and no bias:
        out(co, p) = sum_ci sum_tap weight[co, ci, ky, kx] * u(ci, p + (ky-1, kx-1)),  u(2i, 2j) = x(i, j), else x(i, j) * 0.
    x (B, Cin, h, w), weight (Cout, Cin, 3, 3) -> (B, Cout, H, W).  Only the 9 of 36 products per input channel that read a
    real cell are computed; the NaN a non-finite x or weight gives through the skipped ones is put back (DESIGN.md section
    4.12).  Differentiable in x and weight; fp32 CUDA tensors only."""
    if x.dim() != 4:
        raise ValueError(f'x must be (B,Cin,h,w), got {tuple(x.shape)}')
    H, W = unpool_output_size(x.shape[2], x.shape[3], oheight, owidth)
    _check_unpool_conv(x, weight, H, W)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.unpool_conv3x3(x, weight, H, W)
    if torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad):
        return _UnpoolConv3x3Fn.apply(x, weight, H, W)
    return _unpool_conv_fwd(x, weight, H, W)


class Simple_Gudi_UpConv_Block_Last_Layer(nn.Module):
    """Drop-in for the reference's guidance / depth head (torch_resnet_cspn_nyu.py:187-205): the same constructor, the same
    conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1, bias=False) built first (a seeded construction draws the same
    weights, and state_dict() holds conv1.weight only), and a forward that runs Unpool, crop and conv1 as one CUDA kernel,
    unpool_conv3x3(x, conv1.weight, oheight, owidth)."""

    def __init__(self, in_channels, out_channels, oheight=0, owidth=0):
        super().__init__()
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1, bias=False)
        self.oheight = oheight
        self.owidth = owidth

    def forward(self, x):
        return unpool_conv3x3(x, self.conv1.weight, self.oheight, self.owidth)

    def extra_repr(self):
        return f'oheight={self.oheight}, owidth={self.owidth}'


# ---- trilinear resampling: the Paddle module's resize_trilinear (fluid.layers.resize_trilinear) -----------------------
def resize_output_size(in_shape, out_shape=None, scale=None):
    """The output's (D, H, W): out_shape as given, or int(n * scale) per axis; exactly one of the two, every size >= 1."""
    if (out_shape is None) == (scale is None):
        raise ValueError('give exactly one of out_shape and scale')
    if out_shape is not None:
        try:
            sizes = tuple(operator.index(n) for n in out_shape if not isinstance(n, bool))
        except TypeError:
            sizes = ()
        if len(sizes) != 3 or len(tuple(out_shape)) != 3:
            raise ValueError(f'out_shape must be three ints, got {out_shape!r}')
    else:
        if isinstance(scale, bool) or not isinstance(scale, (int, float)) or not scale > 0:
            raise ValueError(f'scale must be a number > 0, got {scale!r}')
        sizes = tuple(int(n * scale) for n in in_shape)
    if min(sizes) < 1:
        raise ValueError(f'every output size must be >= 1, got {sizes}')
    return sizes


def _check_resize_sizes(in_shape, out_size):
    """The C ABI takes int sizes and < 2^31 elements per (B*C) slice: refuse what it cannot take before anything is allocated
    or narrowed to int."""
    B, C, d, h, w = in_shape
    if max(B, C) > 2 ** 31 - 1 or d * h * w >= 2 ** 31 or out_size[0] * out_size[1] * out_size[2] >= 2 ** 31:
        raise _lib.CspnError(f'resize_trilinear takes B, C < 2^31 and < 2^31 elements per (B*C) slice, got input '
                             f'{tuple(in_shape)} and output size {tuple(out_size)}')


def _resize_fwd(x, D, H, W, align_corners, align_mode):
    """Forward only (no autograd) through cspn_resize_trilinear_fwd_f32, enqueued on the current stream."""
    xc = x.contiguous()
    out = xc.new_empty((*xc.shape[:2], D, H, W))
    if out.numel():
        with torch.cuda.device(xc.device):
            rc = _lib.lib().cspn_resize_trilinear_fwd_f32(_ptr(xc), _ptr(out), *xc.shape, D, H, W, int(align_corners),
                                                          align_mode, _stream(xc.device))
        _lib.check(rc, 'cspn_resize_trilinear_fwd_f32')
    return out


def _resize_bwd(grad_out, in_size, align_corners, align_mode):
    go = grad_out.contiguous()
    gx = go.new_empty((*go.shape[:2], *in_size))
    if gx.numel():
        L = _lib.lib()
        with torch.cuda.device(go.device):
            ws_bytes = L.cspn_resize_trilinear_bwd_workspace_bytes(*in_size, *go.shape[2:])
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=go.device)
            rc = L.cspn_resize_trilinear_bwd_f32(_ptr(go), _ptr(gx), *go.shape[:2], *in_size, *go.shape[2:], int(align_corners),
                                                 align_mode, _ptr(ws), ws_bytes, _stream(go.device))
        _lib.check(rc, 'cspn_resize_trilinear_bwd_f32')
    return gx


class _ResizeTrilinearFn(torch.autograd.Function):
    """autograd seam of resize_trilinear without the torch-op shim: native forward + native gather backward.  The
    backward needs the input's size only, so no tensor is saved."""

    @staticmethod
    def forward(ctx, x, D, H, W, align_corners, align_mode):
        ctx.cfg = (tuple(x.shape[2:]), align_corners, align_mode)
        return _resize_fwd(x, D, H, W, align_corners, align_mode)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        return _resize_bwd(grad_out, *ctx.cfg), None, None, None, None, None


def resize_trilinear(input, out_shape=None, scale=None, align_corners=True, align_mode=1):
    """fluid.layers.resize_trilinear on (B, C, D, H, W) fp32 CUDA tensors, forward and a deterministic backward.
    Per axis n_in -> n_out, in fp32: r = (n_in-1)/(n_out-1) with align_corners, else n_in/n_out (0 when n_out == 1);
    source s(o) = max(r*(o+0.5) - 0.5, 0) with align_corners=False and align_mode=0, else r*o; then the trilinear blend of
    the 8 voxels around s.  Give exactly one of out_shape (three ints) or scale (n_out = int(n_in * scale)).
    align_corners=True is F.interpolate(..., align_corners=True), align_corners=False with align_mode=0 is
    F.interpolate(..., align_corners=False) (for n_out > 1); align_mode=1 has no PyTorch twin.  DESIGN.md section 4.14."""
    if input.dim() != 5:
        raise ValueError(f'input must be (B,C,D,H,W), got {tuple(input.shape)}')
    if align_mode not in (0, 1) or isinstance(align_mode, bool):
        raise ValueError(f'align_mode must be 0 or 1, got {align_mode!r}')
    if min(input.shape[2:]) < 1:
        raise ValueError(f'the input volume must not be empty, got {tuple(input.shape)}')
    D, H, W = resize_output_size(input.shape[2:], out_shape, scale)
    _check_resize_sizes(input.shape, (D, H, W))
    align_corners = bool(align_corners)
    if input.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if not input.is_cuda:
        raise _lib.CspnError('resize_trilinear takes CUDA tensors only (there is no host-buffer entry point for it)')
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.resize_trilinear(input, D, H, W, align_corners, align_mode)
    if torch.is_grad_enabled() and input.requires_grad:
        return _ResizeTrilinearFn.apply(input, D, H, W, align_corners, align_mode)
    return _resize_fwd(input, D, H, W, align_corners, align_mode)


# ---- disparity regression from a low-resolution cost volume: resize_trilinear, softmax over d, expectation ------------
def _disparity_fwd(cost, D, H, W, align_corners, align_mode):
    """Forward only (no autograd) through cspn_disparity_regression_fwd_f32, enqueued on the current stream."""
    cc = cost.contiguous()
    out = cc.new_empty((*cc.shape[:2], H, W))
    if out.numel():
        with torch.cuda.device(cc.device):
            rc = _lib.lib().cspn_disparity_regression_fwd_f32(_ptr(cc), _ptr(out), *cc.shape, D, H, W, int(align_corners),
                                                              align_mode, _stream(cc.device))
        _lib.check(rc, 'cspn_disparity_regression_fwd_f32')
    return out


def _disparity_bwd(cost, grad_out, D, H, W, align_corners, align_mode):
    cc, go = cost.contiguous(), grad_out.contiguous()
    gc = torch.empty_like(cc)
    if gc.numel():
        L = _lib.lib()
        with torch.cuda.device(cc.device):
            ws_bytes = L.cspn_disparity_regression_bwd_workspace_bytes(*cc.shape[2:], D, H, W)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cc.device)
            rc = L.cspn_disparity_regression_bwd_f32(_ptr(cc), _ptr(go), _ptr(gc), *cc.shape, D, H, W, int(align_corners),
                                                     align_mode, _ptr(ws), ws_bytes, _stream(cc.device))
        _lib.check(rc, 'cspn_disparity_regression_bwd_f32')
    return gc


class _DisparityRegressionFn(torch.autograd.Function):
    """autograd seam of disparity_regression without the torch-op shim: native forward + native gather backward.  Only
    cost is saved; the backward recomputes the softmax from it."""

    @staticmethod
    def forward(ctx, cost, D, H, W, align_corners, align_mode):
        ctx.save_for_backward(cost)
        ctx.cfg = (D, H, W, align_corners, align_mode)
        return _disparity_fwd(cost, D, H, W, align_corners, align_mode)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        cost, = ctx.saved_tensors
        return _disparity_bwd(cost, grad_out, *ctx.cfg), None, None, None, None, None


def disparity_regression(cost, out_shape=None, scale=None, align_corners=True, align_mode=1):
    """Disparity from a low-resolution cost volume (B, C, D, H, W), fp32 on CUDA, in one op:
    U = resize_trilinear(cost, (Do, Ho, Wo), align_corners, align_mode), then y[b,c,h,w] = sum_o o * softmax_o(U[b,c,:,h,w])
    over the upsampled disparities o = 0 .. Do-1 (the soft-argmin head of GC-Net / PSMNet).  (Do, Ho, Wo) follow
    resize_trilinear's out_shape / scale rules; the result is (B, C, Ho, Wo).  The upsampled volume is never stored, and
    autograd saves cost alone.  For softmin, negate cost; scale or shift the result for other disparity units.
    DESIGN.md section 4.15."""
    if cost.dim() != 5:
        raise ValueError(f'cost must be (B,C,D,H,W), got {tuple(cost.shape)}')
    if align_mode not in (0, 1) or isinstance(align_mode, bool):
        raise ValueError(f'align_mode must be 0 or 1, got {align_mode!r}')
    if min(cost.shape[2:]) < 1:
        raise ValueError(f'the cost volume must not be empty, got {tuple(cost.shape)}')
    D, H, W = resize_output_size(cost.shape[2:], out_shape, scale)
    _check_resize_sizes(cost.shape, (D, H, W))
    align_corners = bool(align_corners)
    if cost.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if not cost.is_cuda:
        raise _lib.CspnError('disparity_regression takes CUDA tensors only (there is no host-buffer entry point for it)')
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.disparity_regression(cost, D, H, W, align_corners, align_mode)
    if torch.is_grad_enabled() and cost.requires_grad:
        return _DisparityRegressionFn.apply(cost, D, H, W, align_corners, align_mode)
    return _disparity_fwd(cost, D, H, W, align_corners, align_mode)


# ---- stereo cost volumes: PSMNet's concatenation volume and GwcNet's group-wise correlation volume ----------------------
def _check_cost_volume(left, right, max_disp, num_groups=None):
    """The checks of both volume fronts; every refusal comes before anything is allocated or narrowed to int."""
    if left.dim() != 4 or right.shape != left.shape:
        raise ValueError(f'left and right must be (B,F,H,W) of one shape, got {tuple(left.shape)} and {tuple(right.shape)}')
    if isinstance(max_disp, bool) or not isinstance(max_disp, int) or max_disp < 1:
        raise ValueError(f'max_disp must be an int >= 1, got {max_disp!r}')
    B, F, H, W = left.shape
    if min(B, F, H, W) < 1:
        raise ValueError(f'the feature maps must not be empty, got {tuple(left.shape)}')
    if num_groups is not None:
        if isinstance(num_groups, bool) or not isinstance(num_groups, int) or num_groups < 1 or F % num_groups:
            raise ValueError(f'num_groups must be an int >= 1 that divides F={F}, got {num_groups!r}')
    if left.dtype != torch.float32 or right.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if left.device != right.device:
        raise RuntimeError('left and right are on different devices')
    if B > 2 ** 31 - 1 or 2 * F > 2 ** 31 - 1 or max_disp * H * W >= 2 ** 31:
        raise _lib.CspnError(f'the cost volumes take B, 2F < 2^31 and < 2^31 elements per (B, channel) slice, got features '
                             f'{tuple(left.shape)} and max_disp {max_disp}')
    if not left.is_cuda:
        raise _lib.CspnError('the cost volumes take CUDA tensors only (there is no host-buffer entry point for them)')


def _concat_fwd(left, right, D):
    """Forward only (no autograd) through cspn_concat_volume_fwd_f32, enqueued on the current stream."""
    lc, rc_ = left.contiguous(), right.contiguous()
    B, F, H, W = lc.shape
    out = lc.new_empty((B, 2 * F, D, H, W))
    with torch.cuda.device(lc.device):
        rc = _lib.lib().cspn_concat_volume_fwd_f32(_ptr(lc), _ptr(rc_), _ptr(out), B, F, H, W, D, _stream(lc.device))
    _lib.check(rc, 'cspn_concat_volume_fwd_f32')
    return out


def _concat_bwd(grad_out):
    go = grad_out.contiguous()
    B, F2, D, H, W = go.shape
    gl, gr = go.new_empty((B, F2 // 2, H, W)), go.new_empty((B, F2 // 2, H, W))
    with torch.cuda.device(go.device):
        rc = _lib.lib().cspn_concat_volume_bwd_f32(_ptr(go), _ptr(gl), _ptr(gr), B, F2 // 2, H, W, D, _stream(go.device))
    _lib.check(rc, 'cspn_concat_volume_bwd_f32')
    return gl, gr


def _gwc_fwd(left, right, D, G):
    """Forward only (no autograd) through cspn_gwc_volume_fwd_f32, enqueued on the current stream."""
    lc, rc_ = left.contiguous(), right.contiguous()
    B, F, H, W = lc.shape
    out = lc.new_empty((B, G, D, H, W))
    with torch.cuda.device(lc.device):
        rc = _lib.lib().cspn_gwc_volume_fwd_f32(_ptr(lc), _ptr(rc_), _ptr(out), B, F, H, W, D, G, _stream(lc.device))
    _lib.check(rc, 'cspn_gwc_volume_fwd_f32')
    return out


def _gwc_bwd(left, right, grad_out):
    lc, rc_, go = left.contiguous(), right.contiguous(), grad_out.contiguous()
    B, F, H, W = lc.shape
    gl, gr = torch.empty_like(lc), torch.empty_like(lc)
    with torch.cuda.device(lc.device):
        rc = _lib.lib().cspn_gwc_volume_bwd_f32(_ptr(lc), _ptr(rc_), _ptr(go), _ptr(gl), _ptr(gr), B, F, H, W, go.shape[2],
                                                go.shape[1], _stream(lc.device))
    _lib.check(rc, 'cspn_gwc_volume_bwd_f32')
    return gl, gr


class _ConcatVolumeFn(torch.autograd.Function):
    """autograd seam of build_concat_volume without the torch-op shim.  The backward reads grad_out alone: no tensor is
    saved."""

    @staticmethod
    def forward(ctx, left, right, D):
        return _concat_fwd(left, right, D)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        gl, gr = _concat_bwd(grad_out)
        return gl, gr, None


class _GwcVolumeFn(torch.autograd.Function):
    """autograd seam of build_gwc_volume without the torch-op shim: left and right are saved."""

    @staticmethod
    def forward(ctx, left, right, D, G):
        ctx.save_for_backward(left, right)
        return _gwc_fwd(left, right, D, G)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        left, right = ctx.saved_tensors
        gl, gr = _gwc_bwd(left, right, grad_out)
        return gl, gr, None, None


def build_concat_volume(left, right, max_disp):
    """PSMNet's concatenation cost volume in one kernel: left and right (B, F, H, W) fp32 CUDA features give
    (B, 2F, max_disp, H, W) with out[:, c, d, y, x] = left[:, c, y, x] and out[:, F + c, d, y, x] = right[:, c, y, x - d] for
    x >= d, +0.0 for x < d.  The values are copies (every bit kept); differentiable in both inputs, and left may be right.
    DESIGN.md section 4.16."""
    _check_cost_volume(left, right, max_disp)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.concat_volume(left, right, max_disp)
    if torch.is_grad_enabled() and (left.requires_grad or right.requires_grad):
        return _ConcatVolumeFn.apply(left, right, max_disp)
    return _concat_fwd(left, right, max_disp)


def build_gwc_volume(left, right, max_disp, num_groups):
    """GwcNet's group-wise correlation cost volume in one kernel: left and right (B, F, H, W) fp32 CUDA features give
    (B, G, max_disp, H, W) with out[:, g, d, y, x] = mean over the n = F / G channels c of group g of
    left[:, c, y, x] * right[:, c, y, x - d] for x >= d, +0.0 for x < d (products summed in ascending c, then / n).
    F % G != 0 is refused.  Differentiable in both inputs, and left may be right.  DESIGN.md section 4.16."""
    _check_cost_volume(left, right, max_disp, num_groups)
    if torch.compiler.is_compiling() or _use_torch_op():
        return torch.ops.cspn_b200.gwc_volume(left, right, max_disp, num_groups)
    if torch.is_grad_enabled() and (left.requires_grad or right.requires_grad):
        return _GwcVolumeFn.apply(left, right, max_disp, num_groups)
    return _gwc_fwd(left, right, max_disp, num_groups)


# ---- affinity pooling: the CSPN stereo network's convolutional spatial pyramid pooling --------------------------------------
def _check_affinity_pool(feat, gate, kernel_sizes):
    """The checks of affinity_pool2d; every refusal comes before anything is allocated or narrowed to int.  Returns the
    kernel sizes as a tuple of ints."""
    if feat.dim() != 4 or gate.dim() != 4:
        raise ValueError(f'feat must be (B,C,H,W) and gate (B,L,H,W), got {tuple(feat.shape)} and {tuple(gate.shape)}')
    B, C, H, W = feat.shape
    if min(B, C, H, W) < 1:
        raise ValueError(f'feat must not be empty, got {tuple(feat.shape)}')
    if (isinstance(kernel_sizes, (str, bytes)) or not hasattr(kernel_sizes, '__len__')
            or any(isinstance(p, bool) or not isinstance(p, int) for p in kernel_sizes)):
        raise ValueError(f'kernel_sizes must be a sequence of ints, got {kernel_sizes!r}')
    ks = tuple(kernel_sizes)
    if not 1 <= len(ks) <= 8:
        raise ValueError(f'kernel_sizes must hold 1 to 8 sizes, got {len(ks)}')
    if any(not 1 <= p <= min(H, W) for p in ks):
        raise ValueError(f'kernel sizes must be in [1, min(H, W) = {min(H, W)}], got {ks}')
    if tuple(gate.shape) != (B, len(ks), H, W):
        raise ValueError(f'gate must be (B, L, H, W) = {(B, len(ks), H, W)}, got {tuple(gate.shape)}')
    if feat.dtype != torch.float32 or gate.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if feat.device != gate.device:
        raise RuntimeError('feat and gate are on different devices')
    if B > 2 ** 31 - 1 or C > 2 ** 31 - 1 or H * W >= 2 ** 31:
        raise _lib.CspnError(f'affinity_pool2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got feat '
                             f'{tuple(feat.shape)}')
    if not feat.is_cuda:
        raise _lib.CspnError('affinity_pool2d takes CUDA tensors only (there is no host-buffer entry point for it)')
    return ks


def _c_sizes(ks):
    return (ctypes.c_int * len(ks))(*ks)


def _pool_fwd(feat, gate, ks):
    """Forward only (no autograd) through cspn_affinity_pool2d_fwd_f32: the packed levels, on the current stream."""
    f, g = feat.contiguous(), gate.contiguous()
    B, C, H, W = f.shape
    out = f.new_empty((B * C * sum((H // p) * (W // p) for p in ks),))
    with torch.cuda.device(f.device):
        rc = _lib.lib().cspn_affinity_pool2d_fwd_f32(_ptr(f), _ptr(g), _ptr(out), B, C, H, W, len(ks), _c_sizes(ks),
                                                      _stream(f.device))
    _lib.check(rc, 'cspn_affinity_pool2d_fwd_f32')
    return out


def _pool_bwd(feat, gate, out, grad_out, ks):
    f, g, o, go = feat.contiguous(), gate.contiguous(), out.contiguous(), grad_out.contiguous()
    B, C, H, W = f.shape
    gf, gg = torch.empty_like(f), torch.empty_like(g)
    with torch.cuda.device(f.device):
        rc = _lib.lib().cspn_affinity_pool2d_bwd_f32(_ptr(f), _ptr(g), _ptr(o), _ptr(go), _ptr(gf), _ptr(gg), B, C, H, W, len(ks),
                                                      _c_sizes(ks), _stream(f.device))
    _lib.check(rc, 'cspn_affinity_pool2d_bwd_f32')
    return gf, gg


class _AffinityPoolFn(torch.autograd.Function):
    """autograd seam of affinity_pool2d without the torch-op shim: feat, gate and the packed output are saved."""

    @staticmethod
    def forward(ctx, feat, gate, ks):
        out = _pool_fwd(feat, gate, ks)
        ctx.ks = ks
        ctx.save_for_backward(feat, gate, out)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        feat, gate, out = ctx.saved_tensors
        gf, gg = _pool_bwd(feat, gate, out, grad_out, ctx.ks)
        return gf, gg, None


def affinity_pool2d(feat, gate, kernel_sizes):
    """The CSPN stereo network's convolutional spatial pyramid pooling, every level in one launch: feat (B, C, H, W) and
    gate (B, L, H, W) fp32 CUDA tensors and L kernel sizes p_l (1 <= L <= 8, 1 <= p_l <= min(H, W), any order, repeats
    allowed) give a tuple of L tensors (B, C, H // p_l, W // p_l).  Level l pools the windows of F.avg_pool2d(x, p_l)
    (stride p_l, no padding, floor mode) with the weights w = |g_l| / sum_window |g_l| of gate channel l, shared by all
    channels: out_l[:, c, i, j] = sum_window w * feat[:, c].  A constant gate gives avg_pool2d; an all-zero window gives NaN.
    Differentiable in feat and gate, with a deterministic backward.  DESIGN.md section 4.17."""
    ks = _check_affinity_pool(feat, gate, kernel_sizes)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        flat = torch.ops.cspn_b200.affinity_pool2d(feat, gate, list(ks))
    elif torch.is_grad_enabled() and (feat.requires_grad or gate.requires_grad):
        flat = _AffinityPoolFn.apply(feat, gate, ks)
    else:
        flat = _pool_fwd(feat, gate, ks)
    B, C, H, W = feat.shape
    shapes = [(B, C, H // p, W // p) for p in ks]
    return tuple(v.view(s) for v, s in zip(flat.split([B * C * h * w for _, _, h, w in shapes]), shapes))


# ---- affinity fusion: the CSPN stereo network's spatial pyramid fusion ----------------------------------------------------------
def _check_affinity_fuse(levels, gate, align_corners, align_mode):
    """The checks of affinity_fuse2d; every refusal comes before anything is allocated or narrowed to int.  Returns the
    levels as a tuple."""
    if isinstance(levels, torch.Tensor) or not isinstance(levels, (list, tuple)):
        raise ValueError(f'levels must be a list or tuple of tensors, got {type(levels).__name__}')
    lv = tuple(levels)
    if not 1 <= len(lv) <= 8:
        raise ValueError(f'levels must hold 1 to 8 tensors, got {len(lv)}')
    if not all(isinstance(x, torch.Tensor) for x in lv) or not isinstance(gate, torch.Tensor):
        raise ValueError('levels and gate must be tensors')
    if gate.dim() != 4 or any(x.dim() != 4 for x in lv):
        raise ValueError(f'levels must be (B,C,h,w) and gate (B,L,H,W), got {[tuple(x.shape) for x in lv]} and '
                         f'{tuple(gate.shape)}')
    B, L, H, W = gate.shape
    C = lv[0].shape[1]
    if L != len(lv) or any(tuple(x.shape[:2]) != (B, C) for x in lv):
        raise ValueError(f'gate (B, L, H, W) and the L levels (B, C, h, w) must agree, got gate {tuple(gate.shape)} and levels '
                         f'{[tuple(x.shape) for x in lv]}')
    if min(B, C, H, W) < 1 or any(min(x.shape[2:]) < 1 for x in lv):
        raise ValueError(f'levels and gate must not be empty, got {[tuple(x.shape) for x in lv]} and {tuple(gate.shape)}')
    if isinstance(align_mode, bool) or align_mode not in (0, 1):
        raise ValueError(f'align_mode must be 0 or 1, got {align_mode!r}')
    if gate.dtype != torch.float32 or any(x.dtype != torch.float32 for x in lv):
        raise RuntimeError('cspn_b200 is fp32 only')
    if any(x.device != gate.device for x in lv):
        raise RuntimeError('the levels and gate are on different devices')
    if B > 2 ** 31 - 1 or C > 2 ** 31 - 1 or H * W >= 2 ** 31 or any(x.shape[2] * x.shape[3] >= 2 ** 31 for x in lv):
        raise _lib.CspnError(f'affinity_fuse2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got levels '
                             f'{[tuple(x.shape) for x in lv]} and gate {tuple(gate.shape)}')
    if not gate.is_cuda:
        raise _lib.CspnError('affinity_fuse2d takes CUDA tensors only (there is no host-buffer entry point for it)')
    return lv


def _level_args(levels):
    """The C ABI's host arrays: the level pointers and (h_0, w_0, h_1, w_1, ...)."""
    hw = [n for x in levels for n in x.shape[2:]]
    return (ctypes.c_void_p * len(levels))(*[x.data_ptr() for x in levels]), (ctypes.c_int * len(hw))(*hw)


def _fuse_fwd(levels, gate, align_corners, align_mode):
    """Forward only (no autograd) through cspn_affinity_fuse2d_fwd_f32, on the current stream."""
    xs, g = [x.contiguous() for x in levels], gate.contiguous()
    B, L, H, W = g.shape
    out = g.new_empty((B, xs[0].shape[1], H, W))
    ptrs, hw = _level_args(xs)
    with torch.cuda.device(g.device):
        rc = _lib.lib().cspn_affinity_fuse2d_fwd_f32(ptrs, hw, _ptr(g), _ptr(out), B, xs[0].shape[1], H, W, L, int(align_corners),
                                                      align_mode, _stream(g.device))
    _lib.check(rc, 'cspn_affinity_fuse2d_fwd_f32')
    return out


def _fuse_bwd(levels, gate, out, grad_out, align_corners, align_mode):
    """grad_levels (a list, one per level), grad_gate through cspn_affinity_fuse2d_bwd_f32."""
    xs, g, o, go = [x.contiguous() for x in levels], gate.contiguous(), out.contiguous(), grad_out.contiguous()
    B, L, H, W = g.shape
    C = xs[0].shape[1]
    gl, gg = [torch.empty_like(x) for x in xs], torch.empty_like(g)
    ptrs, hw = _level_args(xs)
    gptrs, _ = _level_args(gl)
    Lb = _lib.lib()
    with torch.cuda.device(g.device):
        ws_bytes = Lb.cspn_affinity_fuse2d_bwd_workspace_bytes(B, C, H, W, L, hw)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=g.device)
        rc = Lb.cspn_affinity_fuse2d_bwd_f32(ptrs, hw, _ptr(g), _ptr(o), _ptr(go), gptrs, _ptr(gg), B, C, H, W, L,
                                             int(align_corners), align_mode, _ptr(ws), ws_bytes, _stream(g.device))
    _lib.check(rc, 'cspn_affinity_fuse2d_bwd_f32')
    return gl, gg


class _AffinityFuseFn(torch.autograd.Function):
    """autograd seam of affinity_fuse2d without the torch-op shim: the levels, gate and out are saved.  A level passed twice
    gets the sum of its gradients from autograd."""

    @staticmethod
    def forward(ctx, align_corners, align_mode, gate, *levels):
        out = _fuse_fwd(levels, gate, align_corners, align_mode)
        ctx.cfg = (align_corners, align_mode)
        ctx.save_for_backward(gate, out, *levels)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        gate, out, *levels = ctx.saved_tensors
        gl, gg = _fuse_bwd(levels, gate, out, grad_out, *ctx.cfg)
        return None, None, gg, *gl


def affinity_fuse2d(levels, gate, align_corners=True, align_mode=1):
    """The CSPN stereo network's spatial pyramid fusion: one CSPN step across the levels of a feature pyramid, with the
    upsampling, in one launch.  levels is a list or tuple of L fp32 CUDA tensors (B, C, h_l, w_l), 1 <= L <= 8, of any sizes
    (a level may repeat, or be finer than the output); gate (B, L, H, W) holds level l's raw affinity in channel l, shared
    by all C channels, and sets the output size.  At every pixel w_l = |g_l| / sum_l |g_l| and
    out[:, c] = sum_l w_l * u_l[:, c], where u_l is level l resampled bilinearly to (H, W) with resize_trilinear's rule:
    align_corners=False, align_mode=0 is F.interpolate(..., mode='bilinear', align_corners=False); align_corners=True is
    F.interpolate(..., align_corners=True); the default is Paddle's align_corners=True, align_mode=1.  The upsampled levels
    are never stored.  All-zero gates at a pixel give NaN there.  Returns (B, C, H, W); differentiable in the levels and
    gate, with a deterministic backward.  DESIGN.md section 4.18."""
    lv = _check_affinity_fuse(levels, gate, align_corners, align_mode)
    align_corners = bool(align_corners)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.affinity_fuse2d(list(lv), gate, align_corners, align_mode)
    if torch.is_grad_enabled() and (gate.requires_grad or any(x.requires_grad for x in lv)):
        return _AffinityFuseFn.apply(align_corners, align_mode, gate, *lv)
    return _fuse_fwd(lv, gate, align_corners, align_mode)


# ---- atrous affinity pooling: the CSPN stereo network's atrous spatial pyramid pooling (ACSPP) ---------------------------------
def _check_affinity_atrous(feat, gate, dilations):
    """The checks of affinity_atrous_pool2d; every refusal comes before anything is allocated or narrowed to int.  Returns
    the rates as a tuple of ints."""
    if feat.dim() != 4 or gate.dim() != 4:
        raise ValueError(f'feat must be (B,C,H,W) and gate (B,9L,H,W), got {tuple(feat.shape)} and {tuple(gate.shape)}')
    B, C, H, W = feat.shape
    if min(B, C, H, W) < 1:
        raise ValueError(f'feat must not be empty, got {tuple(feat.shape)}')
    if (isinstance(dilations, (str, bytes)) or not hasattr(dilations, '__len__')
            or any(isinstance(r, bool) or not isinstance(r, int) for r in dilations)):
        raise ValueError(f'dilations must be a sequence of ints, got {dilations!r}')
    rates = tuple(dilations)
    if not 1 <= len(rates) <= 8:
        raise ValueError(f'dilations must hold 1 to 8 rates, got {len(rates)}')
    if any(not 1 <= r <= max(H, W) for r in rates):
        raise ValueError(f'dilations must be in [1, max(H, W) = {max(H, W)}], got {rates}')
    if tuple(gate.shape) != (B, 9 * len(rates), H, W):
        raise ValueError(f'gate must be (B, 9L, H, W) = {(B, 9 * len(rates), H, W)}, got {tuple(gate.shape)}')
    if feat.dtype != torch.float32 or gate.dtype != torch.float32:
        raise RuntimeError('cspn_b200 is fp32 only')
    if feat.device != gate.device:
        raise RuntimeError('feat and gate are on different devices')
    if B > 2 ** 31 - 1 or C > 2 ** 31 - 1 or H * W >= 2 ** 31:
        raise _lib.CspnError(f'affinity_atrous_pool2d takes B, C < 2^31 and < 2^31 elements per (B, channel) slice, got feat '
                             f'{tuple(feat.shape)}')
    if not feat.is_cuda:
        raise _lib.CspnError('affinity_atrous_pool2d takes CUDA tensors only (there is no host-buffer entry point for it)')
    return rates


def _atrous_fwd(feat, gate, rates):
    """Forward only (no autograd) through cspn_affinity_atrous2d_fwd_f32, on the current stream."""
    f, g = feat.contiguous(), gate.contiguous()
    B, C, H, W = f.shape
    out = f.new_empty((B, len(rates) * C, H, W))
    with torch.cuda.device(f.device):
        rc = _lib.lib().cspn_affinity_atrous2d_fwd_f32(_ptr(f), _ptr(g), _ptr(out), B, C, H, W, len(rates), _c_sizes(rates),
                                                        _stream(f.device))
    _lib.check(rc, 'cspn_affinity_atrous2d_fwd_f32')
    return out


def _atrous_bwd(feat, gate, out, grad_out, rates):
    """grad_feat, grad_gate through cspn_affinity_atrous2d_bwd_f32."""
    f, g, o, go = feat.contiguous(), gate.contiguous(), out.contiguous(), grad_out.contiguous()
    B, C, H, W = f.shape
    gf, gg = torch.empty_like(f), torch.empty_like(g)
    r = _c_sizes(rates)
    Lb = _lib.lib()
    with torch.cuda.device(f.device):
        ws_bytes = Lb.cspn_affinity_atrous2d_bwd_workspace_bytes(B, C, H, W, len(rates), r)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=f.device)
        rc = Lb.cspn_affinity_atrous2d_bwd_f32(_ptr(f), _ptr(g), _ptr(o), _ptr(go), _ptr(gf), _ptr(gg), B, C, H, W, len(rates), r,
                                               _ptr(ws), ws_bytes, _stream(f.device))
    _lib.check(rc, 'cspn_affinity_atrous2d_bwd_f32')
    return gf, gg


class _AffinityAtrousFn(torch.autograd.Function):
    """autograd seam of affinity_atrous_pool2d without the torch-op shim: feat, gate and the output are saved."""

    @staticmethod
    def forward(ctx, feat, gate, rates):
        out = _atrous_fwd(feat, gate, rates)
        ctx.rates = rates
        ctx.save_for_backward(feat, gate, out)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        if not grad_out.is_cuda:
            raise _lib.CspnError('backward needs CUDA tensors')
        feat, gate, out = ctx.saved_tensors
        gf, gg = _atrous_bwd(feat, gate, out, grad_out, ctx.rates)
        return gf, gg, None


def affinity_atrous_pool2d(feat, gate, dilations):
    """The CSPN stereo network's atrous spatial pyramid pooling (ACSPP), every level in one launch: each level is one CSPN
    step at stride 1 over the 3x3 neighbourhood dilated by its rate.  feat (B, C, H, W) and gate (B, 9L, H, W) are fp32 CUDA
    tensors and dilations holds L rates r_l (1 <= L <= 8, 1 <= r_l <= max(H, W), any order, repeats allowed).  Gate channel
    9l + t is tap t of level l, offset (t // 3 - 1, t % 3 - 1) * r_l, tap 4 the centre, shared by all C channels.  At every
    pixel w_t = |g_t| / sum_t |g_t| and out[:, l*C + c] = sum_t w_t * feat[:, c] at the tap, +0.0 outside the image (such a
    tap still counts in the sum): F.unfold(feat, 3, dilation=r, padding=r) weighted and summed.  Returns (B, L*C, H, W),
    the levels concatenated along the channels.  A constant gate gives the depthwise dilated 3x3 box filter; all-zero gates
    of a level at a pixel give NaN there.  Differentiable in feat and gate, with a deterministic backward.  DESIGN.md
    section 4.19."""
    rates = _check_affinity_atrous(feat, gate, dilations)
    if torch.compiler.is_compiling() or _use_torch_op():     # under torch.compile the op is the one traceable route
        return torch.ops.cspn_b200.affinity_atrous_pool2d(feat, gate, list(rates))
    if torch.is_grad_enabled() and (feat.requires_grad or gate.requires_grad):
        return _AffinityAtrousFn.apply(feat, gate, rates)
    return _atrous_fwd(feat, gate, rates)
