"""fp64 restatement of the guidance / depth head (Simple_Gudi_UpConv_Block_Last_Layer,
/root/reference/cspn_pytorch/models/torch_resnet_cspn_nyu.py:187-205): Unpool (:41-54, a [1,0;0,0] conv_transpose2d with
stride 2), a crop to (H, W) (:195-200), and conv1, a 3x3 convolution with zero padding and no bias.

unpool_conv_numpy is the polyphase form the CUDA kernels compute (cspn_b200/csrc/unpool_conv.cu): output row 2i reads source
row i, row 2i+1 reads rows i and i+1 (the latter only if 2i+2 < H), and the same for columns -- 9 products per input channel
and 2x2 output block.  It then puts back what the skipped products with structural zeros give in IEEE arithmetic:
  - a non-finite x(i, j) makes the three inserted cells of its block NaN (x * 0), so every output whose 3x3 window touches
    one of them (inside the crop) is NaN, whatever the weights;
  - a non-finite weight[co, ci, tap] makes every output of channel co whose tap reads an inserted cell or the padding NaN.
op_sequence is torch's own op sequence (conv_transpose2d, narrow, conv2d) in fp64 on the CPU, the thing being restated.
Used by tests/test_unpool_conv_{cpu,gpu}.py and __graft_entry__.smoke(); the product never imports it."""
import numpy as np
import torch
import torch.nn.functional as F


def op_sequence(x, weight, H, W):
    """The reference head's forward on torch tensors (any dtype / device): Unpool, crop, conv1."""
    C = x.shape[1]
    k = torch.zeros(C, 1, 2, 2, dtype=x.dtype, device=x.device)
    k[:, :, 0, 0] = 1
    u = F.conv_transpose2d(x, k, stride=2, groups=C)
    u = u.narrow(2, 0, H).narrow(3, 0, W)
    return F.conv2d(u, weight, padding=1)


def unpool_conv_numpy(x, weight, H, W):
    """x (B, Cin, h, w), weight (Cout, Cin, 3, 3) -> (B, Cout, H, W) in fp64, polyphase, with the IEEE rule above."""
    x = np.asarray(x, dtype=np.float64)
    wt = np.asarray(weight, dtype=np.float64)
    B, Cin, h, w = x.shape
    Cout = wt.shape[0]
    hv, wv = (H + 1) // 2, (W + 1) // 2
    # the surviving source window, with one zero row / column after it: rows i+1 with 2i+2 >= H read the padding
    xs = np.zeros((B, Cin, hv + 1, wv + 1))
    xs[:, :, :hv, :wv] = x[:, :, :hv, :wv]
    s00, s01, s10, s11 = xs[:, :, :hv, :wv], xs[:, :, :hv, 1:], xs[:, :, 1:, :wv], xs[:, :, 1:, 1:]
    with np.errstate(invalid='ignore', over='ignore'):
        def conv(tap, s):
            return np.einsum('oc,bcij->boij', wt[:, :, tap // 3, tap % 3], s)
        big = np.zeros((B, Cout, 2 * hv, 2 * wv))
        big[:, :, 0::2, 0::2] = conv(4, s00)
        big[:, :, 0::2, 1::2] = conv(3, s00) + conv(5, s01)
        big[:, :, 1::2, 0::2] = conv(1, s00) + conv(7, s10)
        big[:, :, 1::2, 1::2] = conv(0, s00) + conv(2, s01) + conv(6, s10) + conv(8, s11)
    out = big[:, :, :H, :W].copy()
    # the structural zeros: which taps of each output read an inserted cell or the padding, and whose block that cell is
    bad_x = ~np.isfinite(x[:, :, :hv, :wv]).all(axis=1)                     # (B, hv, wv)
    bad_w = ~np.isfinite(wt).all(axis=1).reshape(Cout, 9)                  # (Cout, 9)
    if not bad_x.any() and not bad_w.any():
        return out
    for oy in range(H):
        for ox in range(W):
            zero_taps = np.zeros(9, bool)
            xnan = np.zeros(B, bool)
            for t in range(9):
                uy, ux = oy + t // 3 - 1, ox + t % 3 - 1
                if uy < 0 or ux < 0 or uy >= H or ux >= W:
                    zero_taps[t] = True
                elif uy % 2 or ux % 2:
                    zero_taps[t] = True
                    xnan |= bad_x[:, uy // 2, ux // 2]
            wnan = (bad_w & zero_taps).any(axis=1)                          # (Cout,)
            out[:, :, oy, ox][xnan[:, None] | wnan[None, :]] = np.nan
    return out


def bound(x, weight, H, W):
    """The a-priori bound of an fp32 evaluation of out with at most n = 4*Cin terms per output in any order:
    |fl(out) - out| <= gamma_n * (the same conv on |x|, |w|), gamma_n = n u / (1 - n u), u = 2^-24."""
    n = 4 * np.asarray(x).shape[1]
    u = 2.0 ** -24
    return n * u / (1 - n * u) * unpool_conv_numpy(np.abs(x), np.abs(weight), H, W)
