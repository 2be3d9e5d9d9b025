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

    @lib.register_fake('cspn_b200::propagate2d_keep')
    def _(guidance, blur_depth, sparse_depth, kernel_size, prop_time, norm_type, algo):
        torch._check(guidance.dim() == 4 and blur_depth.dim() == 4, lambda: 'guidance and blur_depth must be (B,C,H,W)')
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        torch._check(guidance.shape[1] >= kernel_size * kernel_size - 1,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs >= {kernel_size * kernel_size - 1} guidance channels')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_keep_backward')
    def _(guidance, blur_depth, sparse_depth, grad_out, kernel_size, prop_time, norm_type, need_guidance, need_blur, need_sparse):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gd = torch.empty_like(blur_depth, memory_format=torch.contiguous_format) if need_blur else blur_depth.new_empty(0)
        gs = (torch.empty_like(sparse_depth, memory_format=torch.contiguous_format) if need_sparse and sparse_depth is not None
              else blur_depth.new_empty(0))
        return gg, gd, gs

    def setup2d_keep(ctx, inputs, output):
        guidance, blur_depth, sparse_depth, kernel_size, prop_time, norm_type, algo = inputs
        ctx.save_for_backward(guidance, blur_depth, sparse_depth)
        ctx.cfg = (kernel_size, prop_time, norm_type)

    def backward2d_keep(ctx, grad_out):
        guidance, blur_depth, sparse_depth = ctx.saved_tensors
        kernel_size, prop_time, norm_type = ctx.cfg
        need_g, need_d, need_s = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gg, gd, gs = torch.ops.cspn_b200.propagate2d_keep_backward(guidance, blur_depth, sparse_depth, grad_out.contiguous(),
                                                                   kernel_size, prop_time, norm_type, need_g, need_d, need_s)
        return (gg if need_g else None), (gd if need_d else None), (gs if need_s else None), None, None, None, None

    lib.register_autograd('cspn_b200::propagate2d_keep', backward2d_keep, setup_context=setup2d_keep)

    @lib.register_fake('cspn_b200::propagate2d_aggregate')
    def _(guidance, blur_depth, sparse_depth, step_weight, steps, kernel_size, norm_type, keep):
        torch._check(guidance.dim() == 4 and blur_depth.dim() == 4, lambda: 'guidance and blur_depth must be (B,C,H,W)')
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        torch._check(guidance.shape[1] >= kernel_size * kernel_size - 1,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs >= {kernel_size * kernel_size - 1} guidance channels')
        torch._check(len(steps) >= 1 and all(s >= 1 for s in steps) and all(a < b for a, b in zip(steps, steps[1:])),
                     lambda: 'steps must be strictly increasing ints >= 1')
        torch._check(step_weight.dim() == 4 and step_weight.shape[1] == len(steps), lambda: 'step_weight must be (B, len(steps), H, W)')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_aggregate_backward')
    def _(guidance, blur_depth, sparse_depth, step_weight, grad_out, steps, kernel_size, norm_type, keep, need_guidance,
          need_blur, need_sparse, need_step_weight):
        gg = torch.empty_like(guidance, memory_format=torch.contiguous_format) if need_guidance else guidance.new_empty(0)
        gd = torch.empty_like(blur_depth, memory_format=torch.contiguous_format) if need_blur else blur_depth.new_empty(0)
        gs = (torch.empty_like(sparse_depth, memory_format=torch.contiguous_format) if need_sparse and sparse_depth is not None
              else blur_depth.new_empty(0))
        gw = torch.empty_like(step_weight, memory_format=torch.contiguous_format) if need_step_weight else step_weight.new_empty(0)
        return gg, gd, gs, gw

    def setup2d_aggregate(ctx, inputs, output):
        guidance, blur_depth, sparse_depth, step_weight, steps, kernel_size, norm_type, keep = inputs
        ctx.save_for_backward(guidance, blur_depth, sparse_depth, step_weight)
        ctx.cfg = (steps, kernel_size, norm_type, keep)

    def backward2d_aggregate(ctx, grad_out):
        guidance, blur_depth, sparse_depth, step_weight = ctx.saved_tensors
        steps, kernel_size, norm_type, keep = ctx.cfg
        need_g, need_d, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[3]
        need_s = bool(keep) and ctx.needs_input_grad[2]     # the default mode's sign(sparse) is not differentiated
        gg, gd, gs, gw = torch.ops.cspn_b200.propagate2d_aggregate_backward(
            guidance, blur_depth, sparse_depth, step_weight, grad_out.contiguous(), steps, kernel_size, norm_type, keep, need_g,
            need_d, need_s, need_w)
        return ((gg if need_g else None), (gd if need_d else None), (gs if need_s else None), (gw if need_w else None),
                None, None, None, None)

    lib.register_autograd('cspn_b200::propagate2d_aggregate', backward2d_aggregate, setup_context=setup2d_aggregate)

    @lib.register_fake('cspn_b200::propagate2d_nonlocal')
    def _(feat, offset, affinity, sparse_depth, kernel_size, prop_time):
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        nt = kernel_size * kernel_size - 1
        torch._check(feat.dim() == 4 and offset.dim() == 4 and affinity.dim() == 4, lambda: 'feat, offset and affinity must be 4D')
        torch._check(offset.shape[1] == 2 * nt and affinity.shape[1] == nt,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs offset (B,{2 * nt},H,W) and affinity (B,{nt},H,W)')
        torch._check(prop_time >= 0, lambda: 'prop_time must be >= 0')
        return torch.empty_like(feat, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_nonlocal_backward')
    def _(feat, offset, affinity, sparse_depth, grad_out, kernel_size, prop_time, need_feat, need_offset, need_affinity,
          need_sparse):
        new = lambda need, x: torch.empty_like(x, memory_format=torch.contiguous_format) if need else x.new_empty(0)
        gs = new(need_sparse, sparse_depth) if sparse_depth is not None else feat.new_empty(0)
        return new(need_feat, feat), new(need_offset, offset), new(need_affinity, affinity), gs

    def setup2d_nonlocal(ctx, inputs, output):
        feat, offset, affinity, sparse_depth, kernel_size, prop_time = inputs
        ctx.save_for_backward(feat, offset, affinity, sparse_depth)
        ctx.cfg = (kernel_size, prop_time)

    def backward2d_nonlocal(ctx, grad_out):
        feat, offset, affinity, sparse_depth = ctx.saved_tensors
        kernel_size, prop_time = ctx.cfg
        need_f, need_o, need_a = ctx.needs_input_grad[:3]
        need_s = ctx.needs_input_grad[3] and sparse_depth is not None
        gf, go, ga, gs = torch.ops.cspn_b200.propagate2d_nonlocal_backward(
            feat, offset, affinity, sparse_depth, grad_out.contiguous(), kernel_size, prop_time, need_f, need_o, need_a, need_s)
        return ((gf if need_f else None), (go if need_o else None), (ga if need_a else None), (gs if need_s else None),
                None, None)

    lib.register_autograd('cspn_b200::propagate2d_nonlocal', backward2d_nonlocal, setup_context=setup2d_nonlocal)

    @lib.register_fake('cspn_b200::propagate2d_dilated')
    def _(kernel, blur_depth, sparse_depth, confidence, kernel_size, dilation, prop_time):
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        torch._check(1 <= dilation <= 4, lambda: 'dilation must be in [1, 4]')
        torch._check(kernel.dim() == 4 and blur_depth.dim() == 4, lambda: 'kernel and blur_depth must be 4D')
        torch._check(kernel.shape[1] == kernel_size * kernel_size,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs (B,{kernel_size * kernel_size},H,W) weights')
        torch._check((sparse_depth is None) == (confidence is None), lambda: 'sparse_depth and confidence come together')
        torch._check(prop_time >= 0, lambda: 'prop_time must be >= 0')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_dilated_backward')
    def _(kernel, blur_depth, sparse_depth, confidence, grad_out, kernel_size, dilation, prop_time, need_kernel, need_blur,
          need_sparse, need_confidence):
        new = lambda need, x: torch.empty_like(x, memory_format=torch.contiguous_format) if need else blur_depth.new_empty(0)
        gs = new(need_sparse, sparse_depth) if sparse_depth is not None else blur_depth.new_empty(0)
        gm = new(need_confidence, confidence) if confidence is not None else blur_depth.new_empty(0)
        return new(need_kernel, kernel), new(need_blur, blur_depth), gs, gm

    def setup2d_dilated(ctx, inputs, output):
        kernel, blur_depth, sparse_depth, confidence, kernel_size, dilation, prop_time = inputs
        ctx.save_for_backward(kernel, blur_depth, sparse_depth, confidence)
        ctx.cfg = (kernel_size, dilation, prop_time)

    def backward2d_dilated(ctx, grad_out):
        kernel, blur_depth, sparse_depth, confidence = ctx.saved_tensors
        kernel_size, dilation, prop_time = ctx.cfg
        need_k, need_d = ctx.needs_input_grad[:2]
        need_s = ctx.needs_input_grad[2] and sparse_depth is not None
        need_m = ctx.needs_input_grad[3] and confidence is not None
        gk, gd, gs, gm = torch.ops.cspn_b200.propagate2d_dilated_backward(
            kernel, blur_depth, sparse_depth, confidence, grad_out.contiguous(), kernel_size, dilation, prop_time, need_k, need_d,
            need_s, need_m)
        return ((gk if need_k else None), (gd if need_d else None), (gs if need_s else None), (gm if need_m else None),
                None, None, None)

    lib.register_autograd('cspn_b200::propagate2d_dilated', backward2d_dilated, setup_context=setup2d_dilated)

    @lib.register_fake('cspn_b200::propagate2d_dynamic')
    def _(affinity, attention, blur_depth, sparse_depth, confidence, kernel_size):
        torch._check(kernel_size in (3, 5, 7), lambda: 'kernel_size must be 3, 5 or 7')
        torch._check(affinity.dim() == 4 and attention.dim() == 4 and blur_depth.dim() == 4,
                     lambda: 'affinity, attention and blur_depth must be 4D')
        torch._check(affinity.shape[1] == kernel_size * kernel_size,
                     lambda: f'a {kernel_size}x{kernel_size} kernel needs (B,{kernel_size * kernel_size},H,W) affinities')
        torch._check(attention.shape[1] % ((kernel_size + 1) // 2) == 0,
                     lambda: f'the attention needs a multiple of {(kernel_size + 1) // 2} channels')
        torch._check((sparse_depth is None) == (confidence is None), lambda: 'sparse_depth and confidence come together')
        return torch.empty_like(blur_depth, memory_format=torch.contiguous_format)

    @lib.register_fake('cspn_b200::propagate2d_dynamic_backward')
    def _(affinity, attention, blur_depth, sparse_depth, confidence, grad_out, kernel_size, need_affinity, need_attention, need_blur,
          need_sparse, need_confidence):
        new = lambda need, x: torch.empty_like(x, memory_format=torch.contiguous_format) if need else blur_depth.new_empty(0)
        gs = new(need_sparse, sparse_depth) if sparse_depth is not None else blur_depth.new_empty(0)
        gm = new(need_confidence, confidence) if confidence is not None else blur_depth.new_empty(0)
        return new(need_affinity, affinity), new(need_attention, attention), new(need_blur, blur_depth), gs, gm

    def setup2d_dynamic(ctx, inputs, output):
        affinity, attention, blur_depth, sparse_depth, confidence, kernel_size = inputs
        ctx.save_for_backward(affinity, attention, blur_depth, sparse_depth, confidence)
        ctx.kernel_size = kernel_size

    def backward2d_dynamic(ctx, grad_out):
        affinity, attention, blur_depth, sparse_depth, confidence = ctx.saved_tensors
        need_a, need_t, need_d = ctx.needs_input_grad[:3]
        need_s = ctx.needs_input_grad[3] and sparse_depth is not None
        need_m = ctx.needs_input_grad[4] and confidence is not None
        ga, gt, gd, gs, gm = torch.ops.cspn_b200.propagate2d_dynamic_backward(
            affinity, attention, blur_depth, sparse_depth, confidence, grad_out.contiguous(), ctx.kernel_size, need_a, need_t, need_d,
            need_s, need_m)
        return ((ga if need_a else None), (gt if need_t else None), (gd if need_d else None), (gs if need_s else None),
                (gm if need_m else None), None)

    lib.register_autograd('cspn_b200::propagate2d_dynamic', backward2d_dynamic, setup_context=setup2d_dynamic)

    @lib.register_fake('cspn_b200::propagate2d_linear')
    def _(feat, gate, dir_mask):
        torch._check(1 <= dir_mask <= 15, lambda: 'dir_mask must be 1 .. 15')
        torch._check(feat.dim() == 4 and gate.dim() == 4, lambda: 'feat and gate must be (B,C,H,W)')
        nd = sum((dir_mask >> i) & 1 for i in range(4))
        torch._check(gate.shape[1] == 3 * nd or gate.shape[1] == 3 * nd * feat.shape[1],
                     lambda: f'{nd} directions need (B,{3 * nd},H,W) or (B,{3 * nd}*C,H,W) gates')
        out = torch.empty_like(feat, memory_format=torch.contiguous_format)
        planes = feat.new_empty((nd, *feat.shape)) if nd > 1 else feat.new_empty(0)
        return out, planes

    @lib.register_fake('cspn_b200::propagate2d_linear_backward')
    def _(feat, gate, planes, grad_out, dir_mask, need_feat, need_gate):
        new = lambda need, x: torch.empty_like(x, memory_format=torch.contiguous_format) if need else x.new_empty(0)
        return new(need_feat, feat), new(need_gate, gate)

    def setup2d_linear(ctx, inputs, output):
        feat, gate, dir_mask = inputs
        out, planes = output
        ctx.mark_non_differentiable(planes)
        ctx.save_for_backward(feat, gate, planes if dir_mask & (dir_mask - 1) else out)   # one direction: its plane is out
        ctx.dir_mask = dir_mask

    def backward2d_linear(ctx, grad_out, _grad_planes):
        feat, gate, planes = ctx.saved_tensors
        need_f, need_g = ctx.needs_input_grad[:2]
        gf, gg = torch.ops.cspn_b200.propagate2d_linear_backward(feat, gate, planes, grad_out.contiguous(), ctx.dir_mask, need_f,
                                                                 need_g)
        return (gf if need_f else None), (gg if need_g else None), None

    lib.register_autograd('cspn_b200::propagate2d_linear', backward2d_linear, setup_context=setup2d_linear)

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

    @lib.register_fake('cspn_b200::resize_trilinear')
    def _(x, D, H, W, align_corners, align_mode):
        torch._check(x.dim() == 5, lambda: 'input must be (B,C,D,H,W)')
        torch._check(D >= 1 and H >= 1 and W >= 1 and align_mode in (0, 1), lambda: 'sizes >= 1 and align_mode 0 or 1')
        return x.new_empty((x.shape[0], x.shape[1], D, H, W))

    @lib.register_fake('cspn_b200::resize_trilinear_backward')
    def _(grad_out, D, H, W, align_corners, align_mode):
        torch._check(grad_out.dim() == 5, lambda: 'grad_out must be (B,C,D,H,W)')
        return grad_out.new_empty((grad_out.shape[0], grad_out.shape[1], D, H, W))

    def setup_resize(ctx, inputs, output):        # the backward needs the input's size only: no tensor is saved
        x, D, H, W, align_corners, align_mode = inputs
        ctx.cfg = (*x.shape[2:], align_corners, align_mode)

    def backward_resize(ctx, grad_out):
        return torch.ops.cspn_b200.resize_trilinear_backward(grad_out.contiguous(), *ctx.cfg), None, None, None, None, None

    lib.register_autograd('cspn_b200::resize_trilinear', backward_resize, setup_context=setup_resize)

    @lib.register_fake('cspn_b200::disparity_regression')
    def _(cost, D, H, W, align_corners, align_mode):
        torch._check(cost.dim() == 5, lambda: 'cost must be (B,C,D,H,W)')
        torch._check(D >= 1 and H >= 1 and W >= 1 and align_mode in (0, 1), lambda: 'sizes >= 1 and align_mode 0 or 1')
        return cost.new_empty((cost.shape[0], cost.shape[1], H, W))

    @lib.register_fake('cspn_b200::disparity_regression_backward')
    def _(cost, grad_out, D, H, W, align_corners, align_mode):
        torch._check(cost.dim() == 5 and grad_out.dim() == 4, lambda: 'cost must be (B,C,D,H,W) and grad_out (B,C,H,W)')
        return cost.new_empty(cost.shape)

    def setup_disparity(ctx, inputs, output):     # the backward recomputes the softmax: cost is the one saved tensor
        cost, D, H, W, align_corners, align_mode = inputs
        ctx.save_for_backward(cost)
        ctx.cfg = (D, H, W, align_corners, align_mode)

    def backward_disparity(ctx, grad_out):
        cost, = ctx.saved_tensors
        return (torch.ops.cspn_b200.disparity_regression_backward(cost, grad_out.contiguous(), *ctx.cfg),
                None, None, None, None, None)

    lib.register_autograd('cspn_b200::disparity_regression', backward_disparity, setup_context=setup_disparity)

    @lib.register_fake('cspn_b200::concat_volume')
    def _(left, right, max_disp):
        torch._check(left.dim() == 4 and left.shape == right.shape, lambda: 'left and right must be (B,F,H,W) of one shape')
        torch._check(max_disp >= 1, lambda: 'max_disp must be >= 1')
        B, F, H, W = left.shape
        return left.new_empty((B, 2 * F, max_disp, H, W))

    @lib.register_fake('cspn_b200::concat_volume_backward')
    def _(grad_out):
        torch._check(grad_out.dim() == 5 and grad_out.shape[1] % 2 == 0, lambda: 'grad_out must be (B,2F,D,H,W)')
        B, F2, D, H, W = grad_out.shape
        return grad_out.new_empty((B, F2 // 2, H, W)), grad_out.new_empty((B, F2 // 2, H, W))

    def setup_concat(ctx, inputs, output):        # the backward reads grad_out alone: no tensor is saved
        pass

    def backward_concat(ctx, grad_out):
        gl, gr = torch.ops.cspn_b200.concat_volume_backward(grad_out.contiguous())
        return gl, gr, None

    lib.register_autograd('cspn_b200::concat_volume', backward_concat, setup_context=setup_concat)

    @lib.register_fake('cspn_b200::gwc_volume')
    def _(left, right, max_disp, num_groups):
        torch._check(left.dim() == 4 and left.shape == right.shape, lambda: 'left and right must be (B,F,H,W) of one shape')
        torch._check(max_disp >= 1 and num_groups >= 1 and left.shape[1] % num_groups == 0,
                     lambda: 'max_disp >= 1 and num_groups >= 1 dividing F')
        B, F, H, W = left.shape
        return left.new_empty((B, num_groups, max_disp, H, W))

    @lib.register_fake('cspn_b200::gwc_volume_backward')
    def _(left, right, grad_out):
        torch._check(left.dim() == 4 and grad_out.dim() == 5, lambda: 'left must be (B,F,H,W) and grad_out (B,G,D,H,W)')
        return left.new_empty(left.shape), left.new_empty(left.shape)

    def setup_gwc(ctx, inputs, output):
        left, right, max_disp, num_groups = inputs
        ctx.save_for_backward(left, right)

    def backward_gwc(ctx, grad_out):
        left, right = ctx.saved_tensors
        gl, gr = torch.ops.cspn_b200.gwc_volume_backward(left, right, grad_out.contiguous())
        return gl, gr, None, None

    lib.register_autograd('cspn_b200::gwc_volume', backward_gwc, setup_context=setup_gwc)

    @lib.register_fake('cspn_b200::affinity_pool2d')
    def _(feat, gate, kernel_sizes):
        torch._check(feat.dim() == 4 and gate.dim() == 4 and 1 <= len(kernel_sizes) <= 8 and gate.shape[1] == len(kernel_sizes),
                     lambda: 'feat must be (B,C,H,W), gate (B,L,H,W) and kernel_sizes L <= 8 ints')
        B, C, H, W = feat.shape
        torch._check(all(1 <= p <= min(H, W) for p in kernel_sizes), lambda: 'kernel sizes must be in [1, min(H, W)]')
        return feat.new_empty((B * C * sum((H // p) * (W // p) for p in kernel_sizes),))

    @lib.register_fake('cspn_b200::affinity_pool2d_backward')
    def _(feat, gate, out, grad_out, kernel_sizes):
        torch._check(feat.dim() == 4 and gate.dim() == 4 and out.dim() == 1 and grad_out.shape == out.shape,
                     lambda: 'feat and gate must be 4D, out and grad_out the packed levels')
        return feat.new_empty(feat.shape), gate.new_empty(gate.shape)

    def setup_pool(ctx, inputs, output):
        feat, gate, kernel_sizes = inputs
        ctx.kernel_sizes = kernel_sizes
        ctx.save_for_backward(feat, gate, output)

    def backward_pool(ctx, grad_out):
        feat, gate, out = ctx.saved_tensors
        gf, gg = torch.ops.cspn_b200.affinity_pool2d_backward(feat, gate, out, grad_out.contiguous(), ctx.kernel_sizes)
        return gf, gg, None

    lib.register_autograd('cspn_b200::affinity_pool2d', backward_pool, setup_context=setup_pool)

    @lib.register_fake('cspn_b200::affinity_fuse2d')
    def _(levels, gate, align_corners, align_mode):
        torch._check(1 <= len(levels) <= 8 and gate.dim() == 4 and gate.shape[1] == len(levels) and align_mode in (0, 1),
                     lambda: 'levels must be 1..8 tensors (B, C, h, w) and gate (B, L, H, W)')
        torch._check(all(x.dim() == 4 and x.shape[:2] == levels[0].shape[:2] for x in levels),
                     lambda: 'every level must be (B, C, h, w) with one B and C')
        return gate.new_empty((gate.shape[0], levels[0].shape[1], gate.shape[2], gate.shape[3]))

    @lib.register_fake('cspn_b200::affinity_fuse2d_backward')
    def _(levels, gate, out, grad_out, align_corners, align_mode):
        torch._check(gate.dim() == 4 and out.shape == grad_out.shape, lambda: 'gate must be 4D and grad_out match out')
        return [x.new_empty(x.shape) for x in levels], gate.new_empty(gate.shape)

    def setup_fuse(ctx, inputs, output):
        levels, gate, align_corners, align_mode = inputs
        ctx.cfg = (align_corners, align_mode)
        ctx.save_for_backward(gate, output, *levels)

    def backward_fuse(ctx, grad_out):
        gate, out, *levels = ctx.saved_tensors
        gl, gg = torch.ops.cspn_b200.affinity_fuse2d_backward(levels, gate, out, grad_out.contiguous(), *ctx.cfg)
        return list(gl), gg, None, None

    lib.register_autograd('cspn_b200::affinity_fuse2d', backward_fuse, setup_context=setup_fuse)

    @lib.register_fake('cspn_b200::affinity_atrous_pool2d')
    def _(feat, gate, dilations):
        torch._check(feat.dim() == 4 and gate.dim() == 4 and 1 <= len(dilations) <= 8 and gate.shape[1] == 9 * len(dilations),
                     lambda: 'feat must be (B,C,H,W), gate (B,9L,H,W) and dilations L <= 8 ints')
        B, C, H, W = feat.shape
        torch._check(all(1 <= r <= max(H, W) for r in dilations), lambda: 'dilations must be in [1, max(H, W)]')
        return feat.new_empty((B, len(dilations) * C, H, W))

    @lib.register_fake('cspn_b200::affinity_atrous_pool2d_backward')
    def _(feat, gate, out, grad_out, dilations):
        torch._check(feat.dim() == 4 and gate.dim() == 4 and out.dim() == 4 and grad_out.shape == out.shape,
                     lambda: 'feat, gate and out must be 4D, and grad_out match out')
        return feat.new_empty(feat.shape), gate.new_empty(gate.shape)

    def setup_atrous(ctx, inputs, output):
        feat, gate, dilations = inputs
        ctx.dilations = dilations
        ctx.save_for_backward(feat, gate, output)

    def backward_atrous(ctx, grad_out):
        feat, gate, out = ctx.saved_tensors
        gf, gg = torch.ops.cspn_b200.affinity_atrous_pool2d_backward(feat, gate, out, grad_out.contiguous(), ctx.dilations)
        return gf, gg, None

    lib.register_autograd('cspn_b200::affinity_atrous_pool2d', backward_atrous, setup_context=setup_atrous)


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
