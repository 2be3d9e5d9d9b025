"""Device-side counterparts of what the reference computes on the HOST after every step with the propagation's output:

    utils.evaluate_error(gt_depth, pred_depth)     /root/reference/cspn_pytorch/utils.py:19-47   (train.py:204-206, eval.py:147-150)
    Wighted_L1_Loss()(pred, label)                 /root/reference/cspn_pytorch/loss.py:12-23    (train.py:197, eval.py:145)

Same names, same dictionary keys, same arithmetic (valid = gt > 1e-4, IEEE quotients for the delta thresholds), but the
tensors never leave the GPU: one CUDA pass (cspn_b200/csrc/metrics.cu, C ABI `cspn_depth_metrics_f32`) yields all sums on the
caller's stream and the values come back as 0-d CUDA tensors -- `.item()` them when (and if) a number is needed, e.g. every
500 steps as train.py:211 prints them, instead of synchronising every step.
"""
import torch
import torch.nn as nn

from . import _lib

KEYS = ('MSE', 'RMSE', 'MAE', 'ABS_REL', 'DELTA1.02', 'DELTA1.05', 'DELTA1.10', 'DELTA1.25', 'DELTA1.25^2', 'DELTA1.25^3')
_SLOT = {'MSE': 1, 'RMSE': 2, 'MAE': 3, 'ABS_REL': 4, 'DELTA1.02': 5, 'DELTA1.05': 6, 'DELTA1.10': 7, 'DELTA1.25': 8,
         'DELTA1.25^2': 9, 'DELTA1.25^3': 10}


def _stats(pred, gt):
    """-> CUDA float tensor [12]: n_valid, MSE, RMSE, MAE, ABS_REL, six deltas, reserved (metrics.cu header)."""
    if not (pred.is_cuda and gt.is_cuda):
        raise _lib.CspnError('cspn_b200.metrics works on CUDA tensors (that is its point: no host round trip)')
    if pred.shape != gt.shape or pred.dtype != torch.float32 or gt.dtype != torch.float32 or pred.device != gt.device:
        raise ValueError('pred and gt must be fp32 CUDA tensors of one shape on one device')
    L = _lib.lib()
    p, g = pred.detach().contiguous(), gt.detach().contiguous()
    out = torch.empty(12, dtype=torch.float32, device=p.device)
    ws = torch.empty(L.cspn_depth_metrics_workspace_bytes() // 8, dtype=torch.float64, device=p.device)
    with torch.cuda.device(p.device):
        rc = L.cspn_depth_metrics_f32(p.data_ptr(), g.data_ptr(), p.numel(), out.data_ptr(), ws.data_ptr(), ws.numel() * 8,
                                      torch.cuda.current_stream(p.device).cuda_stream)
    _lib.check(rc, 'cspn_depth_metrics_f32')
    return out


def evaluate_error(gt_depth, pred_depth):
    """utils.evaluate_error's dictionary (utils.py:23-26, incl. the never-filled 'LG10': 0) with 0-d CUDA tensors as values."""
    s = _stats(pred_depth, gt_depth)
    err = {k: s[i] for k, i in _SLOT.items()}
    err['LG10'] = 0
    return err


class _MaskedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, label):
        s = _stats(pred, label)
        ctx.save_for_backward(pred, label, s)
        return s[3].clone()                      # MAE over the valid pixels == loss.py:21-22

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        pred, label, s = ctx.saved_tensors
        L = _lib.lib()
        p, g = pred.contiguous(), label.contiguous()
        gl = grad_loss.contiguous().to(torch.float32)
        grad = torch.empty_like(p)
        with torch.cuda.device(p.device):
            rc = L.cspn_masked_l1_bwd_f32(p.data_ptr(), g.data_ptr(), s.data_ptr(), gl.data_ptr(), grad.data_ptr(), p.numel(),
                                          torch.cuda.current_stream(p.device).cuda_stream)
        _lib.check(rc, 'cspn_masked_l1_bwd_f32')
        return grad, None


class Wighted_L1_Loss(nn.Module):
    """Same name (typo included) and call as the reference's criterion (loss.py:12-23): mean |pred - label| over label > 1e-4.
    Forward and backward are single CUDA passes; the returned loss is a 0-d CUDA tensor.  fp32 CUDA tensors of one shape,
    any rank and layout; usable on any stream and inside a CUDA graph.

    The gradient with respect to pred is sign(pred - label) * fl(fl(1 / n_valid) * grad_loss) where label > 1e-4 (0 where
    pred == label or the difference is NaN) and 0 elsewhere; label gets none, and a second derivative is refused.  The
    count reaches the backward as a float: above 2^24 valid pixels it is rounded to even first, which moves the scale by
    at most one ulp.

    With no valid pixel the loss is 0 and its gradient all zeros.  The reference returns 0 / 0 = NaN there (the sum of an
    empty selection over a count of zero, loss.py:22); a frame without ground truth would then poison every weight of a
    training run, so this deviation is deliberate (DESIGN.md section 4.7)."""

    def forward(self, pred, label):
        return _MaskedL1.apply(pred, label)
