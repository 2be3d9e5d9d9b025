"""GPU tests of the CSPN stereo head end to end (tests/stereo_head_reference.py): the head built on the cspn_b200 ops --
cost volumes, CSPP, ACSPP, fusion, the 3D CSPN and disparity regression, with small learned layers between them -- against
the same head built from stock torch ops and evaluated in fp64 on the GPU.

The tolerance calibrates itself: e32 is the normwise distance of the stock-torch head evaluated in eager fp32 from its fp64
evaluation, and ours may be at most 4 * e32, for the disparity map and for every gradient; the fp64 model's masks of NaN
and +-inf must be reproduced.  Every leg runs each op through both Python routes (the dispatcher op, and the
autograd.Function with CSPN_B200_NO_TORCH_OP=1).  Convolutions run in true fp32 (no TF32) and deterministically, so that
our head and the eager fp32 one differ only in the ops under test.

First run, on an NVIDIA H100 80GB HBM3 at a 700 W power limit: both routes gave the same numbers in every leg, every
fp64 mask was reproduced, and the largest ratio ours / e32 was 1.77 (KITTI, align_corners=True, grad cost).  Ours / e32
per leg are in each test's docstring.
"""
import pytest
import torch
import torch.nn.functional as F

import stereo_head_reference as sh

pytestmark = pytest.mark.gpu

ALIGN = [(True, 1), (False, 0)]          # F.interpolate(align_corners=True) (Paddle's default too) and (align_corners=False)
ROUTES = [('op', '0'), ('autograd.Function', '1')]
# a reduced head for the IEEE, compile and graph legs: B = 2, 64 x 128 images, features at 16 x 32, D = 12 -> 48
SMALL = dict(channels=8, kernel_sizes=(16, 8, 4, 2), rates=(2, 3, 5, 7), max_disp=12, groups=4, out_channels=8,
             prop_steps=6)


@pytest.fixture(autouse=True)
def true_fp32_deterministic_convs():
    cudnn, matmul = torch.backends.cudnn, torch.backends.cuda.matmul
    saved = (cudnn.allow_tf32, cudnn.deterministic, cudnn.benchmark, matmul.allow_tf32)
    cudnn.allow_tf32, cudnn.deterministic, cudnn.benchmark, matmul.allow_tf32 = False, True, False, False
    yield
    cudnn.allow_tf32, cudnn.deterministic, cudnn.benchmark, matmul.allow_tf32 = saved


def _judge(label, head, args, r32, r64, monkeypatch, **kw):
    """Run the native head on both routes and compare each with the fp64 model; returns the rejected rows."""
    bad = []
    for route, flag in ROUTES:
        monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', flag)
        ok, rows = sh.compare(sh.run(head, *args, native=True, **kw), r32, r64)
        print(f'\n{label}, route {route}: {"accepted" if ok else "REJECTED"}\n{sh.report(rows)}')
        bad += [(route,) + r for r in rows if not r[-1]]
    return bad


# ---- the training crop: B = 4, 256 x 512 images, features at 64 x 128, D = 48 -> Do = 192 ------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_training_crop_matches_the_fp64_model(align_corners, align_mode, monkeypatch):
    """The disparity map and the gradients of the masked smooth-L1 loss with respect to both images and every parameter.

    First H100 run, ours / e32:
                             align_corners=True          align_corners=False, align_mode=0
      disparity              5.46e-07 / 5.16e-07         5.37e-07 / 5.06e-07
      grad left              1.93e-05 / 1.92e-05         1.10e-06 / 1.14e-06
      grad right             6.55e-06 / 6.54e-06         5.89e-07 / 6.09e-07
      grad stem.weight       1.01e-06 / 7.46e-07         1.18e-07 / 2.43e-07
      grad pool_gate.weight  3.46e-06 / 3.69e-06         3.77e-06 / 3.30e-06
      grad atrous_gate.weight 8.06e-06 / 8.04e-06        8.56e-07 / 8.09e-07
      grad fuse_gate.weight  5.92e-06 / 5.50e-06         2.27e-06 / 2.23e-06
      grad mix.weight        9.65e-07 / 7.75e-07         1.24e-07 / 2.03e-07
      grad cost.weight       1.21e-06 / 1.16e-06         8.15e-07 / 7.36e-07
      grad prop_gate.weight  1.67e-05 / 1.64e-05         8.31e-07 / 8.30e-07
      grad prop_gate.bias    2.34e-05 / 2.23e-05         5.28e-07 / 4.41e-07"""
    head = sh.StereoHead(align_corners=align_corners, align_mode=align_mode, prop3d='paddle').cuda()
    args = sh.inputs(0, 4, 256, 512, head.max_disp, 'cuda')
    r64 = sh.run(sh.as_dtype(head, torch.float64), *args)
    assert all(torch.isfinite(t).all() for t in r64.values())
    r32 = sh.run(head, *args)
    bad = _judge(f'training crop, align_corners={align_corners}, align_mode={align_mode}', head, args, r32, r64, monkeypatch)
    assert not bad, bad


# ---- KITTI inference: B = 1, features at 96 x 312, Do = 192 -> 384 x 1248 --------------------------------------------------------
@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_kitti_inference_matches_the_fp64_model(align_corners, align_mode, monkeypatch):
    """The disparity map and the gradients with respect to the cost volume entering the 3D CSPN and its raw gates, here on
    affinity_propagate with the gates normalised in torch.  One fp64 forward and one backward.

    First H100 run, ours / e32:
                  align_corners=True          align_corners=False, align_mode=0
      disparity   4.66e-07 / 4.32e-07         4.06e-07 / 3.67e-07
      grad cost   2.05e-04 / 1.16e-04         3.06e-05 / 3.01e-05
      grad guide  1.20e-03 / 6.83e-04         1.93e-04 / 1.89e-04"""
    head = sh.StereoHead(align_corners=align_corners, align_mode=align_mode, prop3d='gates').cuda()
    args = sh.inputs(1, 1, 384, 1248, head.max_disp, 'cuda')
    r64 = sh.run(sh.as_dtype(head, torch.float64), *args, wrt='taps')
    assert all(torch.isfinite(t).all() for t in r64.values())
    r32 = sh.run(head, *args, wrt='taps')
    bad = _judge(f'KITTI, align_corners={align_corners}, align_mode={align_mode}', head, args, r32, r64, monkeypatch,
                 wrt='taps')
    assert not bad, bad


# ---- IEEE: all-zero fusion gates over a patch give NaN there (affinity_fuse2d's docstring), and it spreads -----------------------
@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_zero_fusion_gates_give_the_fp64_models_nan_masks(align_corners, align_mode, monkeypatch):
    """A 2 x 3 patch of the left features has all-zero fusion gates in image 0.  The NaN spreads through the cost volumes,
    the 3D CSPN and the regression; the loss leaves out the pixels where the fp64 disparity is NaN, so the gradients
    carry NaN only where the backward reads a NaN.  cuDNN is off in this test: it may pick transform-based (Winograd,
    FFT) algorithms for fp32 and not for fp64, whose NaN footprint can reach past a convolution's window, and the masks
    would then depend on the algorithm, not on our ops.

    First H100 run: every mask reproduced (every parameter gradient is all NaN, as a sum over the NaN region); on the
    finite elements, ours / e32 for align_corners=True and for align_corners=False, align_mode=0: disparity 2.13e-07 /
    1.74e-07 and 2.04e-07 / 1.60e-07, grad left 6.07e-07 / 6.23e-07 and 6.26e-07 / 5.90e-07, grad right 1.19e-06 /
    9.79e-07 and 5.47e-07 / 7.63e-07."""
    head = sh.StereoHead(**SMALL, align_corners=align_corners, align_mode=align_mode).cuda()
    left, right, target, valid = sh.inputs(2, 2, 64, 128, head.max_disp, 'cuda')
    mask = torch.ones(2, 1, 16, 32, device='cuda')
    mask[0, :, 5:7, 20:23] = 0
    with torch.backends.cudnn.flags(enabled=False):
        h64 = sh.as_dtype(head, torch.float64)
        with torch.no_grad():
            y64 = h64(left.double(), right.double(), False, mask.double())
        nan = torch.isnan(y64)
        assert nan[0].any() and not nan[1].any() and not nan[0].all()
        args = (left, right, target, valid & ~nan)
        r64 = sh.run(h64, *args, fuse_gate_mask=mask)
        r32 = sh.run(head, *args, fuse_gate_mask=mask)
        assert torch.isnan(r64['grad left']).any() and torch.isfinite(r64['grad right']).any()
        bad = _judge(f'zero fusion gates, align_corners={align_corners}, align_mode={align_mode}', head, args, r32, r64,
                     monkeypatch, fuse_gate_mask=mask)
    assert not bad, bad


# ---- the whole head under torch.compile and in a CUDA graph: the eager bits ---------------------------------------------------------
def _step(head, left, right, target, valid):
    y = head(left, right, True)
    per_pixel = F.smooth_l1_loss(y, target, reduction='none')
    (torch.where(valid, per_pixel, torch.zeros_like(per_pixel)).sum() / valid.sum()).backward()
    return y.detach()          # no autograd node of this step outlives it (a graph capture must not meet one)


def _bits(t):
    return t.detach().view(torch.int32)


@pytest.mark.parametrize('align_corners,align_mode', ALIGN)
def test_torch_compile_of_the_whole_head_gives_the_eager_bits(align_corners, align_mode, monkeypatch):
    """fullgraph=True, forward and backward, on the dispatcher ops: every op's fake kernel and autograd registration in
    composition.  aot_eager keeps stock ops on their eager kernels, so any difference is ours.  The 3D CSPN is
    affinity_propagate here, the route a compiled caller takes."""
    monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', '0')
    head = sh.StereoHead(**SMALL, align_corners=align_corners, align_mode=align_mode, prop3d='gates').cuda()
    left, right, target, valid = sh.inputs(3, 2, 64, 128, head.max_disp, 'cuda')
    y = _step(head, left, right, target, valid)
    want = [p.grad.clone() for p in head.parameters()]
    head.zero_grad(set_to_none=True)
    compiled = torch.compile(head, fullgraph=True, backend='aot_eager')
    yc = _step(compiled, left, right, target, valid)
    assert torch.equal(_bits(yc), _bits(y))
    for (name, p), w in zip(head.named_parameters(), want):
        assert torch.equal(_bits(p.grad), _bits(w)), name


@pytest.mark.parametrize('route,flag', ROUTES)
def test_cuda_graph_of_one_training_step_gives_the_eager_bits(route, flag, monkeypatch):
    monkeypatch.setenv('CSPN_B200_NO_TORCH_OP', flag)
    head = sh.StereoHead(**SMALL, prop3d='paddle').cuda()
    left, right, target, valid = sh.inputs(4, 2, 64, 128, head.max_disp, 'cuda')
    y = _step(head, left, right, target, valid)
    want = [p.grad.clone() for p in head.parameters()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            head.zero_grad(set_to_none=True)
            _step(head, left, right, target, valid)
    torch.cuda.current_stream().wait_stream(side)
    head.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = _step(head, left, right, target, valid)
    for p in head.parameters():
        p.grad.fill_(float('nan'))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(yg), _bits(y))
    for (name, p), w in zip(head.named_parameters(), want):
        assert torch.equal(_bits(p.grad), _bits(w)), name
