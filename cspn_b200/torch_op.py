"""torch.ops.cspn_b200.* -- dispatcher registration of the propagation path (csrc/torch_op.cpp over the C ABI).

    from cspn_b200 import torch_op
    out = torch_op.propagate2d(guidance, blur_depth, sparse_depth, 24, '8sum')     # autograd-aware, torch.compile-able

What lives here (Python) and why: the FAKE kernels (shape/dtype propagation without touching data -- what
torch.compile, torch.export and FakeTensorMode need to trace the call the reference model makes at
/root/reference/cspn_pytorch/models/torch_resnet_cspn_nyu.py:375 as one opaque node) and the AUTOGRAD formulas
(train.py:196-199 back-propagates through the op; the backward is itself a registered op, so it is traceable too).
The CUDA kernels are registered in C++.  There is no CPU kernel: CPU tensors fail in the dispatcher.
"""
import os

import torch

from . import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
TORCH_LIB_PATH = os.path.join(HERE, '_build', 'libcspn_b200_torch.so')

_loaded = False


def available():
    # once loaded, the shim stays available: no file-system lookups on the per-call path of affinity_propagate (a stat on
    # a network file system can take longer than a small propagation)
    return _loaded or (os.path.isfile(TORCH_LIB_PATH) and os.path.isfile(_lib.LIB_PATH))


def load():
    """Loads libcspn_b200_torch.so (once) and registers the fake kernels and autograd formulas."""
    global _loaded
    if _loaded:
        return
    if not available():
        raise _lib.CspnError(f'{TORCH_LIB_PATH} is missing: build it with `python -m cspn_b200.build --torch-op`')
    _lib.lib()                                   # libcspn_b200.so first: the shim resolves its symbols from it
    torch.ops.load_library(TORCH_LIB_PATH)
    _register()
    _loaded = True


def _register():
    lib = torch.library

    @lib.register_fake('cspn_b200::propagate2d')
    def _(guidance, blur_depth, sparse_depth, prop_time, norm_type, algo):
        torch._check(guidance.dim() == 4 and blur_depth.dim() == 4, lambda: 'guidance and blur_depth must be (B,C,H,W)')
        torch._check(guidance.shape[1] >= 8, lambda: 'guidance needs >= 8 channels')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_backward')
    def _(guidance, blur_depth, sparse_depth, grad_out, prop_time, norm_type, need_guidance, need_blur):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gd = torch.empty_like(blur_depth, memory_format=torch.contiguous_format) if need_blur else blur_depth.new_empty(0)
        return gg, gd

    @lib.register_fake('cspn_b200::propagate2d_k')
    def _(guidance, blur_depth, sparse_depth, kernel_size, prop_time, norm_type):
        torch._check(guidance.dim() == 4 and blur_depth.dim() == 4, lambda: 'guidance and blur_depth must be (B,C,H,W)')
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        torch._check(guidance.shape[1] >= kernel_size * kernel_size - 1,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs >= {kernel_size * kernel_size - 1} guidance channels')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_k_backward')
    def _(guidance, blur_depth, sparse_depth, grad_out, kernel_size, prop_time, norm_type, need_guidance, need_blur):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gd = torch.empty_like(blur_depth, memory_format=torch.contiguous_format) if need_blur else blur_depth.new_empty(0)
        return gg, gd

    @lib.register_fake('cspn_b200::propagate2d_paddle')
    def _(guidance, feat, kernel_size, prop_time):
        torch._check(guidance.dim() == 4 and feat.dim() == 4, lambda: 'guidance and feat must be (B,C,H,W)')
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        nt = kernel_size * kernel_size - 1
        torch._check(guidance.shape[1] == nt or (feat.shape[1] > 1 and guidance.shape[1] == nt * feat.shape[1]),
                     lambda: f'a {kernel_size}x{kernel_size} \'paddle\' kernel needs {nt} or {nt}*C guidance channels')
        return torch.empty_like(feat, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_paddle_backward')
    def _(guidance, feat, grad_out, kernel_size, prop_time, need_guidance, need_feat):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gf = torch.empty_like(feat, memory_format=torch.contiguous_format) if need_feat else feat.new_empty(0)
        return gg, gf

    @lib.register_fake('cspn_b200::propagate3d')
    def _(guidance, feat, prop_time, norm_type):
        torch._check(guidance.dim() == 5 and feat.dim() == 5, lambda: 'guidance and feat must be (B,C,D,H,W)')
        return torch.empty_like(feat, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate3d_backward')
    def _(guidance, feat, grad_out, prop_time, norm_type, need_guidance, need_feat):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gf = torch.empty_like(feat, memory_format=torch.contiguous_format) if need_feat else feat.new_empty(0)
        return gg, gf

    @lib.register_fake('cspn_b200::propagate3d_k')
    def _(guidance, feat, kernel_size, prop_time, norm_type):
        torch._check(guidance.dim() == 5 and feat.dim() == 5, lambda: 'guidance and feat must be (B,C,D,H,W)')
        torch._check(kernel_size in (3, 5), lambda: '3D kernel_size must be 3 or 5')
        torch._check(guidance.shape[1] == kernel_size ** 3 - 1,
                     lambda: f'a {kernel_size}x{kernel_size}x{kernel_size} kernel needs {kernel_size ** 3 - 1} guidance channels')
        return torch.empty_like(feat, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate3d_k_backward')
    def _(guidance, feat, grad_out, kernel_size, prop_time, norm_type, need_guidance, need_feat):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gf = torch.empty_like(feat, memory_format=torch.contiguous_format) if need_feat else feat.new_empty(0)
        return gg, gf

    def setup2d(ctx, inputs, output):
        guidance, blur_depth, sparse_depth, prop_time, norm_type, algo = inputs
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (prop_time, norm_type)

    def backward2d(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        prop_time, norm_type = ctx.cfg
        need_g, need_d = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg, gd = torch.ops.cspn_b200.propagate2d_backward(guidance, blur_depth, sparse_depth, grad_out.contiguous(),
                                                          prop_time, norm_type, need_g, need_d)
        return (gg if need_g else None), (gd if need_d else None), None, None, None, None

    lib.register_autograd('cspn_b200::propagate2d', backward2d, setup_context=setup2d)

    def setup2d_k(ctx, inputs, output):
        guidance, blur_depth, sparse_depth, kernel_size, prop_time, norm_type = inputs
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (kernel_size, prop_time, norm_type)

    def backward2d_k(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        kernel_size, prop_time, norm_type = ctx.cfg
        need_g, need_d = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg, gd = torch.ops.cspn_b200.propagate2d_k_backward(guidance, blur_depth, sparse_depth, grad_out.contiguous(),
                                                            kernel_size, prop_time, norm_type, need_g, need_d)
        return (gg if need_g else None), (gd if need_d else None), None, None, None, None

    lib.register_autograd('cspn_b200::propagate2d_k', backward2d_k, setup_context=setup2d_k)

    def setup2d_paddle(ctx, inputs, output):
        guidance, feat, kernel_size, prop_time = inputs
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (kernel_size, prop_time)

    def backward2d_paddle(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        kernel_size, prop_time = ctx.cfg
        need_g, need_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg, gf = torch.ops.cspn_b200.propagate2d_paddle_backward(guidance, feat, grad_out.contiguous(), kernel_size, prop_time,
                                                                 need_g, need_f)
        return (gg if need_g else None), (gf if need_f else None), None, None

    lib.register_autograd('cspn_b200::propagate2d_paddle', backward2d_paddle, setup_context=setup2d_paddle)

    def setup3d(ctx, inputs, output):
        guidance, feat, prop_time, norm_type = inputs
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (prop_time, norm_type)

    def backward3d(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        prop_time, norm_type = ctx.cfg
        need_g, need_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg, gf = torch.ops.cspn_b200.propagate3d_backward(guidance, feat, grad_out.contiguous(), prop_time, norm_type,
                                                          need_g, need_f)
        return (gg if need_g else None), (gf if need_f else None), None, None

    lib.register_autograd('cspn_b200::propagate3d', backward3d, setup_context=setup3d)

    def setup3d_k(ctx, inputs, output):
        guidance, feat, kernel_size, prop_time, norm_type = inputs
        ctx.save_for_backward(guidance, feat)
        ctx.cfg = (kernel_size, prop_time, norm_type)

    def backward3d_k(ctx, grad_out):
        guidance, feat = ctx.saved_tensors
        kernel_size, prop_time, norm_type = ctx.cfg
        need_g, need_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gg, gf = torch.ops.cspn_b200.propagate3d_k_backward(guidance, feat, grad_out.contiguous(), kernel_size, prop_time,
                                                            norm_type, need_g, need_f)
        return (gg if need_g else None), (gf if need_f else None), None, None, None

    lib.register_autograd('cspn_b200::propagate3d_k', backward3d_k, setup_context=setup3d_k)

    for nd in (2, 3):
        _register_gates(lib, nd)

    @lib.register_fake('cspn_b200::unpool_conv3x3')
    def _(x, weight, H, W):
        torch._check(x.dim() == 4 and weight.dim() == 4 and weight.shape[1] == x.shape[1] and tuple(weight.shape[2:]) == (3, 3),
                     lambda: 'x must be (B,Cin,h,w) and weight (Cout,Cin,3,3)')
        torch._check(1 <= H <= 2 * x.shape[2] and 1 <= W <= 2 * x.shape[3], lambda: 'the output must lie within the unpooled map')
        return x.new_empty((x.shape[0], weight.shape[0], H, W))

    @lib.register_fake('cspn_b200::unpool_conv3x3_backward')
    def _(x, weight, grad_out, H, W, need_x, need_weight):
        gx = torch.empty_like(x, memory_format=torch.contiguous_format) if need_x else x.new_empty(0)
        gw = torch.empty_like(weight, memory_format=torch.contiguous_format) if need_weight else weight.new_empty(0)
        return gx, gw

    def setup_unpool(ctx, inputs, output):
        x, weight, H, W = inputs
        ctx.save_for_backward(x, weight)
        ctx.cfg = (H, W)

    def backward_unpool(ctx, grad_out):
        x, weight = ctx.saved_tensors
        H, W = ctx.cfg
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gx, gw = torch.ops.cspn_b200.unpool_conv3x3_backward(x, weight, grad_out.contiguous(), H, W, need_x, need_w)
        return (gx if need_x else None), (gw if need_w else None), None, None

    lib.register_autograd('cspn_b200::unpool_conv3x3', backward_unpool, setup_context=setup_unpool)


def _register_gates(lib, nd):
    """Fake kernels and autograd of affinity_propagate{nd}d (fluid.layers.affinity_propagate with the caller's gates)."""
    sizes = (3, 5, 7) if nd == 2 else (3, 5)

    @lib.register_fake(f'cspn_b200::affinity_propagate{nd}d')
    def _(input, gate_weight, kernel_size, prop_step):
        torch._check(input.dim() == nd + 2 and gate_weight.dim() == nd + 2,
                     lambda: f'input and gate_weight must have {nd + 2} dimensions')
        torch._check(kernel_size in sizes, lambda: f'kernel_size of a {nd}D affinity_propagate must be one of {sizes}')
        nt = kernel_size ** nd - 1
        torch._check(gate_weight.shape[1] == nt or (input.shape[1] > 1 and gate_weight.shape[1] == nt * input.shape[1]),
                     lambda: f'a kernel of size {kernel_size} needs {nt} or {nt}*C gate channels')
        return torch.empty_like(input, memory_format=torch.contiguous_format)

    @lib.register_fake(f'cspn_b200::affinity_propagate{nd}d_backward')
    def _(input, gate_weight, grad_out, kernel_size, prop_step, need_input, need_gate):
        gx = torch.empty_like(input, memory_format=torch.contiguous_format) if need_input else input.new_empty(0)
        gg = torch.empty_like(gate_weight, memory_format=torch.contiguous_format) if need_gate else gate_weight.new_empty(0)
        return gx, gg

    def setup(ctx, inputs, output):
        input, gate_weight, kernel_size, prop_step = inputs
        ctx.save_for_backward(input, gate_weight)
        ctx.cfg = (kernel_size, prop_step)

    def backward(ctx, grad_out):
        input, gate_weight = ctx.saved_tensors
        kernel_size, prop_step = ctx.cfg
        need_x, need_g = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        op = getattr(torch.ops.cspn_b200, f'affinity_propagate{nd}d_backward')
        gx, gg = op(input, gate_weight, grad_out.contiguous(), kernel_size, prop_step, need_x, need_g)
        return (gx if need_x else None), (gg if need_g else None), None, None

    lib.register_autograd(f'cspn_b200::affinity_propagate{nd}d', backward, setup_context=setup)


def propagate2d(guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum', algo=_lib.ALGO_AUTO):
    """The dispatcher op (CUDA tensors only).  prop_time == 0 returns blur_depth itself, as cspn.py:61,83 does."""
    if prop_time == 0:
        return blur_depth
    load()
    return torch.ops.cspn_b200.propagate2d(guidance, blur_depth, sparse_depth, int(prop_time), _lib.NORM2D[norm_type], int(algo))


def propagate3d(guidance, feat, prop_time=12, norm_type='26sum_abs'):
    if prop_time == 0:
        return feat
    load()
    return torch.ops.cspn_b200.propagate3d(guidance, feat, int(prop_time), _lib.NORM3D[norm_type])
