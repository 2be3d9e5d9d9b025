"""Golden of the two heads in front of the propagation: the reference's OWN model (torch_resnet_cspn_nyu.py, resnet50 with
seeded random weights, the run of make_golden_model.py) recording the input both heads receive and their conv1 weights
(gud_up_proj_layer6 -> guidance, gud_up_proj_layer5 -> blur, :372-373).

    python tests/golden/make_golden_heads.py      (needs the reference tree; CPU only)

tests/golden/model/nyu_resnet50_heads.npz: x, the bottom-right WINDOW x rows [y0, 114) x cols [x0, 152) of the heads'
input (1,64,114,152), with y0, x0; w_guidance (8,64,3,3), w_blur (1,64,3,3), oheight, owidth.  The whole input does not fit
the repository (a post-ReLU map with random mantissas: 2.1 MB compressed).  The window is enough: an output (oy, ox) with
oy >= 2*y0 and ox >= 2*x0 reads source rows >= y0 and cols >= x0 only, and the window shares the image's bottom and right
borders, so the heads run on the window give exactly the products of the full run there, in the same order.
The run must reproduce nyu_resnet50_tail.npz's `out` bit for bit (asserted), so the two files describe one forward: the
GPU test feeds the window through cspn_b200's heads and compares with the tail golden's guidance / blur over the matching
region, and propagates the golden guidance / blur with that region replaced against the tail golden's `out`.
"""
import importlib
import os
import sys

import numpy as np
import torch

REF_MODELS = '/root/reference/cspn_pytorch/models'
HERE = os.path.dirname(os.path.abspath(__file__))
WINDOW = (36, 48)            # source rows x cols kept: 64*36*48 floats, about 0.2 MB compressed


def main():
    assert os.path.isdir(REF_MODELS), 'reference tree not mounted'
    sys.path.append(REF_MODELS)
    torch.Tensor.cuda = lambda self, *a, **k: self    # Unpool's ctor and cspn.py:50 call .cuda()
    torch.manual_seed(1234)                           # the construction and input of make_golden_model.py
    model = importlib.import_module('torch_resnet_cspn_nyu')
    net = model.resnet50(pretrained=False, cspn_config={'step': 24, 'norm_type': '8sum'}).eval()
    seen = {}
    head = net.gud_up_proj_layer6
    orig = head.forward

    def spy(x):
        seen['x'] = x.clone()
        return orig(x)

    head.forward = spy
    g = torch.Generator().manual_seed(99)
    x = torch.rand(1, 4, 228, 304, generator=g)
    x[:, 3] = x[:, 3] * 10 * (torch.rand(1, 228, 304, generator=g) < 500.0 / (228 * 304))
    with torch.no_grad():
        out = net(x)
    tail = np.load(os.path.join(HERE, 'model', 'nyu_resnet50_tail.npz'))
    assert np.array_equal(out.numpy(), tail['out']), 'this run does not reproduce nyu_resnet50_tail.npz'
    g6, g5 = net.gud_up_proj_layer6, net.gud_up_proj_layer5
    assert (g6.oheight, g6.owidth) == (g5.oheight, g5.owidth) == (228, 304)
    path = os.path.join(HERE, 'model', 'nyu_resnet50_heads.npz')
    h, w = seen['x'].shape[2:]
    y0, x0 = h - WINDOW[0], w - WINDOW[1]
    np.savez_compressed(path, x=seen['x'][:, :, y0:, x0:].numpy(), y0=y0, x0=x0, w_guidance=g6.conv1.weight.detach().numpy(),
                        w_blur=g5.conv1.weight.detach().numpy(), oheight=g6.oheight, owidth=g6.owidth)
    print(path, os.path.getsize(path), 'bytes; x window', (y0, x0), 'of', tuple(seen['x'].shape))


if __name__ == '__main__':
    main()
