"""PyTorch-op port of the reference's CPU/eager path.  TEST + BASELINE INFRASTRUCTURE ONLY.

This is what `bench.py --impl reference` and bench.py's `cpu_baseline` leg time on the GPU
machine's host cores: the same ATen op sequence per iteration as the reference's
cspn_pytorch/models/cspn.py -- 8 zero-pads + cat
(cspn.py:147-172), broadcast mul + ones-weight Conv3d as the 8-way sum (cspn.py:44-53,70),
crop (cspn.py:71-72), centre term (cspn.py:76), mask replacement (cspn.py:81) -- so its cost
profile (about 25-30 small ops and two (B,8,C,H+2,W+2) temporaries per iteration) is the
reference's, minus the `.cuda()` call at cspn.py:50 that makes the original unusable on CPU.
Held bit for bit against outputs of the real module (stored under tests/golden/reference_forward/)
in tests/test_oracle.py.
Never imported by the product package.
"""
import torch
import torch.nn.functional as F

# ZeroPad2d tuples (left, right, top, bottom) in channel order, cspn.py:105-129 == 149-168
PADS = ((0, 2, 0, 2), (1, 1, 0, 2), (2, 0, 0, 2),
        (0, 2, 1, 1),               (2, 0, 1, 1),
        (0, 2, 2, 0), (1, 1, 2, 0), (2, 0, 2, 0))


def _stack_padded(t):
    """(B,C,H,W) -> (B,8,C,H+2,W+2): eight differently padded copies (cspn.py:147-172)."""
    return torch.cat([F.pad(t, p).unsqueeze(1) for p in PADS], 1)


def _sum8(t, ones):
    """8-way channel sum as a 1x1x1 Conv3d with all-ones weight (cspn.py:44-53)."""
    return F.conv3d(t, ones)


def cspn2d_torch(guidance, blur_depth, sparse_depth=None, prop_time=24, norm_type='8sum'):
    assert norm_type in ('8sum', '8sum_abs')
    ones = torch.ones(1, 8, 1, 1, 1, dtype=blur_depth.dtype, device=blur_depth.device)
    g = guidance.abs() if 'abs' in norm_type else guidance                   # cspn.py:88-89
    gate = torch.cat([F.pad(g.narrow(1, k, 1), PADS[k]).unsqueeze(1) for k in range(8)], 1)  # :91-132
    gate = gate / _sum8(gate.abs(), ones)                                    # :135-138
    gate_sum = _sum8(gate, ones).squeeze(1)[:, :, 1:-1, 1:-1]                # :139-142
    raw = blur_depth
    result = blur_depth
    mask = sparse_depth.sign() if sparse_depth is not None else None         # :63-64
    for _ in range(prop_time):                                               # :66
        nb = _sum8(gate * _stack_padded(result), ones).squeeze(1)[:, :, 1:-1, 1:-1]   # :69-72
        result = (1.0 - gate_sum) * raw + nb                                 # :76
        if mask is not None:
            result = (1 - mask) * result + mask * raw                        # :81
    return result


# ---- 3D (differentiable restatement of oracle/cspn_numpy.py::cspn3d; used as the autograd reference in tests) ----
OFFSETS_3D = tuple((1 - f, 1 - t, 1 - l) for f in range(3) for t in range(3) for l in range(3) if (f, t, l) != (1, 1, 1))


def _shift3d(a, dz, dy, dx):
    """b[..., z, y, x] = a[..., z+dz, y+dy, x+dx], zero outside."""
    D, H, W = a.shape[-3:]
    p = F.pad(a, (1, 1, 1, 1, 1, 1))
    return p[..., 1 + dz:1 + dz + D, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W]


def cspn3d_torch(guidance, feat, prop_time=12, norm_type='26sum_abs'):
    g = guidance[:, :26]
    if norm_type == 'paddle':
        a = g.abs()                                               # demo.py:24
        gate = a / a.sum(1, keepdim=True)                         # demo.py:47-49 (own location)
    else:
        if 'abs' in norm_type:
            g = g.abs()
        a = torch.stack([_shift3d(g[:, k], *o) for k, o in enumerate(OFFSETS_3D)], 1)
        gate = a / a.abs().sum(1, keepdim=True)
    gate_sum = gate.sum(1, keepdim=True)
    raw = feat
    result = feat
    for _ in range(prop_time):
        acc = 0
        for k, o in enumerate(OFFSETS_3D):
            acc = acc + gate[:, k:k + 1] * _shift3d(result, *o)
        result = acc if norm_type == 'paddle' else (1.0 - gate_sum) * raw + acc
    return result
