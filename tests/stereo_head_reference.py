"""An independent model of the CSPN stereo head (arXiv 1810.02695), built from stock torch ops only, and the comparator the
stereo-head tests judge the CUDA ops by.  TEST INFRASTRUCTURE ONLY: shared by tests/test_stereo_head_cpu.py and
tests/test_stereo_head_gpu.py; the product package never imports it.

Every op here is written from its public docstring and DESIGN.md sections 4.14 to 4.19, and from the networks it comes
from (PSMNet's and GwcNet's cost-volume loops, PSMNet's soft-argmin regression).  It imports no other file under tests/
and nothing under oracle/, so it shares no code and no convention with the per-op restatements: a convention that is wrong
the same way in a kernel and in its restatement is still caught here.

The conventions, each stated once:
- cost volumes: the matched pixel of left[..., x] at disparity d is right[..., x - d]; cells with x < d are +0.0;
- CSPP: level l pools the floor-mode windows of F.avg_pool2d(x, p_l) with w = |g_l| / sum_window |g_l|;
- ACSPP: gate channel 9l + t is tap t of level l, at offset r_l * (t // 3 - 1, t % 3 - 1), the order of F.unfold;
- fusion: w_l = |g_l| / sum_l |g_l| over the levels, each level resampled bilinearly to the output size;
- resampling, per axis n_in -> n_out: align_corners=True is F.interpolate(align_corners=True); align_corners=False with
  align_mode=0 is F.interpolate(align_corners=False); align_corners=False with align_mode=1 (Paddle's rule) samples
  s(o) = o * n_in / n_out, i0 = floor(s), i1 = min(i0 + 1, n_in - 1), lambda = s - i0, out = (1 - lambda) x[i0] + lambda x[i1].
  That rule is F.interpolate(align_corners=True) of x with its last sample repeated once, to n_out + 1 samples, with the
  last output dropped (the ratio (n_in + 1 - 1) / (n_out + 1 - 1) is n_in / n_out); the CPU tests pin it there and on the
  sizes where it is the identity or nearest-neighbour downsampling;
- 3D propagation: tap k enumerates (f, t, l) over [0, 3)^3 in raster order without the centre and reads the source voxel
  p + (1 - f, 1 - t, 1 - l); the 'paddle' gates are |g_k| / sum_j |g_j| at the voxel's own location; each step is
  d <- sum_k gate_k * d(p + off_k) with zero padding;
- disparity regression: U = the trilinear resampling of the cost volume to (Do, Ho, Wo), then sum_o o * softmax_o(U) over
  the upsampled indices o = 0 .. Do - 1, so the result is in full-resolution pixels.
"""
import copy

import torch
import torch.nn as nn
import torch.nn.functional as F

import cspn_b200

# ---- the ops --------------------------------------------------------------------------------------------------------------


def concat_volume(left, right, D):
    """PSMNet's concatenation volume: a zero-filled (B, 2F, D, H, W) volume, then two slice writes per disparity."""
    B, C, H, W = left.shape
    vol = left.new_zeros((B, 2 * C, D, H, W))
    for d in range(min(D, W)):
        vol[:, :C, d, :, d:] = left[:, :, :, d:]
        vol[:, C:, d, :, d:] = right[:, :, :, :W - d]
    return vol


def gwc_volume(left, right, D, G):
    """GwcNet's group-wise correlation volume: per disparity, the channel products averaged within each of G groups."""
    B, C, H, W = left.shape
    vol = left.new_zeros((B, G, D, H, W))
    for d in range(min(D, W)):
        prod = left[:, :, :, d:] * right[:, :, :, :W - d]
        vol[:, :, d, :, d:] = prod.view(B, G, C // G, H, W - d).mean(dim=2)
    return vol


def affinity_pool(feat, gate, kernel_sizes):
    """CSPP: a tuple of L levels (B, C, H // p, W // p), each window an affinity-weighted average of its pixels."""
    B, C, H, W = feat.shape
    outs = []
    for l, p in enumerate(kernel_sizes):
        h, w = H // p, W // p
        a = gate[:, l:l + 1, :h * p, :w * p].abs().reshape(B, 1, h, p, w, p)
        S = a.sum(dim=(3, 5), keepdim=True)
        outs.append((a / S * feat[:, :, :h * p, :w * p].reshape(B, C, h, p, w, p)).sum(dim=(3, 5)))
    return tuple(outs)


def affinity_atrous(feat, gate, rates):
    """ACSPP: (B, L*C, H, W), level l the 9 dilated taps of F.unfold weighted by |g| / sum |g| of gate[:, 9l : 9l + 9]."""
    B, C, H, W = feat.shape
    outs = []
    for l, r in enumerate(rates):
        taps = F.unfold(feat, 3, dilation=r, padding=r).view(B, C, 9, H, W)
        a = gate[:, 9 * l:9 * l + 9].abs()
        outs.append((a / a.sum(dim=1, keepdim=True)).unsqueeze(1).mul(taps).sum(dim=2))
    return torch.cat(outs, dim=1)


def _paddle_axis(x, dim, n_out):
    """Paddle's align_mode=1 rule (align_corners=False) along one axis, in x's dtype: s = o * n_in / n_out."""
    n_in = x.shape[dim]
    s = torch.arange(n_out, dtype=x.dtype, device=x.device) * (torch.tensor(n_in, dtype=x.dtype) / n_out)
    i0 = s.floor().long().clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    lam = (s - i0.to(x.dtype)).view([-1] + [1] * (x.dim() - 1 - dim))
    return (1 - lam) * x.index_select(dim, i0) + lam * x.index_select(dim, i1)


def resample(x, size, align_corners, align_mode):
    """Bilinear (4-D x) or trilinear (5-D x) resampling to `size` under the rules of the module docstring."""
    if align_corners or align_mode == 0:
        mode = 'bilinear' if x.dim() == 4 else 'trilinear'
        return F.interpolate(x, size=tuple(size), mode=mode, align_corners=bool(align_corners))
    for k, n in enumerate(size):
        x = _paddle_axis(x, 2 + k, n)
    return x


def affinity_fuse(levels, gate, align_corners, align_mode):
    """Pyramid fusion: at every pixel sum_l w_l * resample(level l), w_l = |g_l| / sum_l |g_l|."""
    a = gate.abs()
    w = a / a.sum(dim=1, keepdim=True)
    return sum(w[:, l:l + 1] * resample(x, gate.shape[2:], align_corners, align_mode) for l, x in enumerate(levels))


OFFSETS_3D = tuple((1 - f, 1 - t, 1 - l) for f in range(3) for t in range(3) for l in range(3) if (f, t, l) != (1, 1, 1))


def paddle_gates(guide):
    """The Paddle module's normalisation at the voxel's own location: |g_k| / sum_j |g_j| over the 26 channels."""
    a = guide.abs()
    return a / a.sum(dim=1, keepdim=True)


def affinity_propagate3d(feat, gates, steps):
    """fluid.layers.affinity_propagate, 3x3x3, run `steps` times with the gates as given: 26 shifted copies of the
    zero-padded volume, each weighted by its gate, summed."""
    D, H, W = feat.shape[2:]
    for _ in range(steps):
        p = F.pad(feat, (1, 1, 1, 1, 1, 1))
        acc = 0
        for k, (dz, dy, dx) in enumerate(OFFSETS_3D):
            acc = acc + gates[:, k:k + 1] * p[:, :, 1 + dz:1 + dz + D, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
        feat = acc
    return feat


def disparity_regression(cost, size, align_corners, align_mode):
    """PSMNet's soft-argmin at full resolution: resample (B, 1, D, H, W) to `size` = (Do, Ho, Wo), softmax over the
    disparities, then the expectation over o = 0 .. Do - 1.  Returns (B, 1, Ho, Wo)."""
    p = torch.softmax(resample(cost, size, align_corners, align_mode), dim=2)
    o = torch.arange(size[0], dtype=cost.dtype, device=cost.device).view(1, 1, -1, 1, 1)
    return (p * o).sum(dim=2)


# ---- the head ---------------------------------------------------------------------------------------------------------------


class StereoHead(nn.Module):
    """A small CSPN stereo head with learned layers between the ops, so that gate layouts and channel orders come out of
    convolutions as they do in a network:
      1. left and right features at a quarter of the image size (a shared 4x4, stride-4 convolution and tanh);
      2. CSPP and ACSPP branches on them, their gates from 3x3 convolutions;
      3. fusion of the CSPP levels and the ACSPP levels (each C channels of its output) under gates from a 3x3 convolution,
         then a 1x1 convolution of the features and the fused map;
      4. the group-wise correlation and concatenation volumes, concatenated, and a 1x1x1 conv3d down to one cost channel;
      5. the 3D CSPN on the cost volume, its gates from a 3x3x3 conv3d of the cost ('paddle' own-location normalisation);
      6. disparity regression to the full image size, D disparities at the features' scale becoming 4D, of the propagated
         cost times a fixed sharpness.
    Only the 3D gate convolution has a bias, 26 values: the cost volume is +0.0 where x < d, and without a bias all 26
    gates there would be 0 and their normalisation 0/0.  The other convolutions have none, so that every parameter is a
    tensor of many elements and a normwise distance per gradient is a statistic, not one number.
    forward(left, right, native) runs the cspn_b200 ops (fp32 CUDA) when native is set and the stock-torch ops above
    otherwise; `prop3d` picks the native 3D route: 'paddle' is Affinity_Propagate3D(..., 'paddle') with the normalisation
    fused, 'gates' normalises in torch and calls affinity_propagate on the 5-D volume."""

    SHARPNESS = 32.0    # the propagation smooths the cost; scaled, its softmax over 4D disparities is not flat

    def __init__(self, channels=16, kernel_sizes=(64, 32, 16, 8), rates=(6, 12, 18, 24), max_disp=48, groups=4,
                 out_channels=8, prop_steps=12, align_corners=True, align_mode=1, prop3d='paddle', seed=0):
        super().__init__()
        assert len(kernel_sizes) + len(rates) <= 8 and prop3d in ('paddle', 'gates')
        self.kernel_sizes, self.rates, self.max_disp, self.groups = tuple(kernel_sizes), tuple(rates), max_disp, groups
        self.prop_steps, self.align_corners, self.align_mode, self.prop3d = prop_steps, align_corners, align_mode, prop3d
        C = channels
        gen = torch.Generator().manual_seed(seed)
        self.stem = nn.Conv2d(3, C, 4, stride=4, bias=False)
        self.pool_gate = nn.Conv2d(C, len(kernel_sizes), 3, padding=1, bias=False)
        self.atrous_gate = nn.Conv2d(C, 9 * len(rates), 3, padding=1, bias=False)
        self.fuse_gate = nn.Conv2d(C, len(kernel_sizes) + len(rates), 3, padding=1, bias=False)
        self.mix = nn.Conv2d(2 * C, out_channels, 1, bias=False)
        self.cost = nn.Conv3d(groups + 2 * out_channels, 1, 1, bias=False)
        self.prop_gate = nn.Conv3d(1, 26, 3, padding=1)
        with torch.no_grad():
            for m in self.modules():
                if isinstance(m, (nn.Conv2d, nn.Conv3d)):
                    fan_in = m.weight[0].numel()
                    m.weight.copy_(torch.randn(m.weight.shape, generator=gen) / fan_in ** 0.5)
            self.prop_gate.bias.copy_(torch.randn(26, generator=gen))
            self.cost.weight.mul_(4.0)

    def features(self, img, ops, fuse_gate_mask=None):
        x = torch.tanh(self.stem(img))
        pooled = ops.affinity_pool(x, self.pool_gate(x), self.kernel_sizes)
        atrous = ops.affinity_atrous(x, self.atrous_gate(x), self.rates)
        levels = list(pooled) + list(atrous.chunk(len(self.rates), dim=1))
        g = self.fuse_gate(x)
        if fuse_gate_mask is not None:
            g = g * fuse_gate_mask
        fused = ops.affinity_fuse(levels, g, self.align_corners, self.align_mode)
        return self.mix(torch.cat([x, fused], dim=1))

    def forward(self, left, right, native=False, fuse_gate_mask=None, taps=None):
        """Disparity (B, 1, Hi, Wi) of the image pair (B, 3, Hi, Wi).  `fuse_gate_mask` (B, 1, Hi / 4, Wi / 4) multiplies the
        left image's fusion gates (a 0 there makes a pixel's gates all zero).  If `taps` is a dict, it receives the cost
        volume entering the 3D CSPN and the raw 3D gates, so that a caller can differentiate with respect to them."""
        ops = NativeOps(self.prop3d) if native else ReferenceOps
        fl = self.features(left, ops, fuse_gate_mask)
        fr = self.features(right, ops)
        vol = torch.cat([ops.gwc_volume(fl, fr, self.max_disp, self.groups), ops.concat_volume(fl, fr, self.max_disp)], dim=1)
        cost = self.cost(vol)
        guide = self.prop_gate(cost)
        if taps is not None:
            taps['cost'], taps['guide'] = cost, guide
        cost = ops.propagate3d(cost, guide, self.prop_steps) * self.SHARPNESS
        size = (4 * self.max_disp, left.shape[2], left.shape[3])
        return ops.disparity_regression(cost, size, self.align_corners, self.align_mode)


class ReferenceOps:
    concat_volume = staticmethod(lambda l, r, D: concat_volume(l, r, D))
    gwc_volume = staticmethod(lambda l, r, D, G: gwc_volume(l, r, D, G))
    affinity_pool = staticmethod(lambda f, g, ks: affinity_pool(f, g, ks))
    affinity_atrous = staticmethod(lambda f, g, rates: affinity_atrous(f, g, rates))
    affinity_fuse = staticmethod(lambda lv, g, ac, am: affinity_fuse(lv, g, ac, am))
    propagate3d = staticmethod(lambda cost, guide, n: affinity_propagate3d(cost, paddle_gates(guide), n))
    disparity_regression = staticmethod(lambda cost, size, ac, am: disparity_regression(cost, size, ac, am))
    # (the lambdas look the functions up at call time, so a copy of this module with a function replaced runs the copy's)


class NativeOps:
    """The same head on the cspn_b200 ops.  Each call takes its route (dispatcher op or autograd.Function) from
    CSPN_B200_NO_TORCH_OP at the time of the call."""

    def __init__(self, prop3d):
        self.cb, self.prop3d = cspn_b200, prop3d

    def concat_volume(self, l, r, D):
        return self.cb.build_concat_volume(l, r, D)

    def gwc_volume(self, l, r, D, G):
        return self.cb.build_gwc_volume(l, r, D, G)

    def affinity_pool(self, f, g, ks):
        return self.cb.affinity_pool2d(f, g, ks)

    def affinity_atrous(self, f, g, rates):
        return self.cb.affinity_atrous_pool2d(f, g, rates)

    def affinity_fuse(self, levels, g, ac, am):
        return self.cb.affinity_fuse2d(levels, g, align_corners=ac, align_mode=am)

    def propagate3d(self, cost, guide, n):
        if self.prop3d == 'paddle':
            return self.cb.Affinity_Propagate3D(n, 3, 'paddle')(guide, cost)
        return self.cb.affinity_propagate(cost, paddle_gates(guide), 3, n)

    def disparity_regression(self, cost, size, ac, am):
        return self.cb.disparity_regression(cost, size, align_corners=ac, align_mode=am)


def as_dtype(head, dtype):
    """A copy of the head with its parameters in `dtype`: the same model, another precision."""
    return copy.deepcopy(head).to(dtype)


def inputs(seed, B, Hi, Wi, max_disp, device):
    """An image pair (B, 3, Hi, Wi) and a target disparity map (B, 1, Hi, Wi) in full-resolution pixels, with PSMNet's
    validity mask target < 4 * max_disp - 1."""
    gen = torch.Generator().manual_seed(seed)
    left = torch.rand(B, 3, Hi, Wi, generator=gen)
    right = torch.rand(B, 3, Hi, Wi, generator=gen)
    target = torch.rand(B, 1, Hi, Wi, generator=gen) * (4.4 * max_disp)
    return left.to(device), right.to(device), target.to(device), (target < 4 * max_disp - 1).to(device)


def run(head, left, right, target, valid, native=False, wrt='all', fuse_gate_mask=None):
    """One training step without the update: the disparity map, and the gradients of the masked smooth-L1 loss
    sum_valid smooth_l1(y, target) / #valid, with respect to both images and every parameter (wrt='all') or to the cost
    volume entering the 3D CSPN and its raw gates (wrt='taps').  The inputs are cast to the head's dtype.  Returns a dict
    of detached tensors: 'disparity' and 'grad <name>'."""
    dtype = head.stem.weight.dtype
    left, right = (t.detach().to(dtype).requires_grad_(wrt == 'all') for t in (left, right))
    mask = None if fuse_gate_mask is None else fuse_gate_mask.to(dtype)
    taps = {}
    y = head(left, right, native, mask, taps)
    per_pixel = F.smooth_l1_loss(y, target.to(dtype), reduction='none')
    loss = torch.where(valid, per_pixel, torch.zeros_like(per_pixel)).sum() / valid.sum()
    if wrt == 'all':
        named = [('left', left), ('right', right)] + list(head.named_parameters())
    else:
        named = [('cost', taps['cost']), ('guide', taps['guide'])]
    grads = torch.autograd.grad(loss, [t for _, t in named])
    out = {'disparity': y.detach()}
    out.update({f'grad {n}': g for (n, _), g in zip(named, grads)})
    return out


# ---- the comparator ---------------------------------------------------------------------------------------------------------


def normwise(got, want):
    """||got - want|| / ||want|| over the elements where `want` is finite, in fp64."""
    m = torch.isfinite(want)
    g, w = got.detach().double()[m], want.detach().double()[m]
    return float((g - w).norm() / w.norm().clamp_min(1e-300))


def same_nonfinite(got, want):
    """The fp64 model's masks of NaN, +inf and -inf are reproduced exactly."""
    got, want = got.detach(), want.detach()
    return all(torch.equal(f(got), f(want))
               for f in (torch.isnan, lambda t: t == float('inf'), lambda t: t == float('-inf')))


def compare(ours, ref32, ref64, factor=4.0):
    """Judge a set of named results (the disparity map and gradients) against the fp64 model.  `ref32` is the same model
    evaluated in eager fp32: its distance from fp64, e32, is the error fp32 arithmetic makes on this model at these inputs,
    and ours may be at most `factor` times that, per result.  Returns (accepted, rows), one row per result:
    (name, ours' distance, e32, masks reproduced, accepted)."""
    rows = []
    for name, want in ref64.items():
        d, e32 = normwise(ours[name], want), normwise(ref32[name], want)
        masks = same_nonfinite(ours[name], want)
        rows.append((name, d, e32, masks, masks and d <= factor * e32))
    return all(r[-1] for r in rows), rows


def report(rows):
    return '\n'.join(f'  {n:>22}: ours {d:.3e}  e32 {e:.3e}  ratio {d / e if e else float("inf"):7.3f}  '
                     f'masks {"ok" if m else "DIFFER"}  {"accepted" if a else "REJECTED"}' for n, d, e, m, a in rows)
