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


def propagate2d_k(guidance, blur_depth, sparse_depth=None, prop_kernel=5, prop_time=24, norm_type=None, out=None):
    """2D CSPN with a K x K affinity kernel, forward only (no autograd), CUDA tensors only, enqueued on the current stream.
    guidance (B, >=K*K-1, H, W): channels 0..K*K-2 are used, shared by the C channels of blur_depth (B, C, H, W);
    norm_type f'{K*K-1}sum' (default) or f'{K*K-1}sum_abs'.  K = 3 is propagate2d itself (same kernels, same bits)."""
    code = norm_code_2d_k(prop_kernel, norm_type)
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

    def __init__(self, prop_time, prop_kernel, norm_type=None):
        super().__init__()
        norm_code_2d_k(prop_kernel, norm_type)      # AssertionError for K not in {3, 5, 7} or a name that does not match K
        self.prop_time = prop_time
        self.prop_kernel = prop_kernel
        self.norm_type = norm_type or f'{prop_kernel * prop_kernel - 1}sum'
        self._use_op = _use_torch_op()

    def forward(self, guidance, blur_depth, sparse_depth=None):
        if self.prop_time == 0:
            return blur_depth
        sd = None if sparse_depth is None else sparse_depth.detach()
        code = norm_code_2d_k(self.prop_kernel, self.norm_type)
        if self._use_op and blur_depth.is_cuda:
            return torch.ops.cspn_b200.propagate2d_k(guidance, blur_depth, sd, self.prop_kernel, self.prop_time, code)
        if torch.is_grad_enabled() and (guidance.requires_grad or blur_depth.requires_grad):
            return _Propagate2dKFn.apply(guidance, blur_depth, sd, self.prop_kernel, self.prop_time, self.norm_type)
        return propagate2d_k(guidance, blur_depth, sparse_depth, self.prop_kernel, self.prop_time, self.norm_type)

    def extra_repr(self):
        return f'prop_time={self.prop_time}, prop_kernel={self.prop_kernel}, norm_type={self.norm_type!r}'


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
