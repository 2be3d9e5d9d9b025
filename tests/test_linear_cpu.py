"""CPU tests of the linear propagation (SPN's three-way scans, DESIGN.md section 4.24): the kernel-order restatement of
tests/linear_reference.py against the fp64 composition, forward and backward (within tolerance on random inputs, equal
on dyadic ones); the flip and transpose identities and the merge's tie and NaN rule on the references; the C ABI's
workspace formulas and refusals without a device; the Python refusals; the op schemas and fake kernels; no spills in
cspn2d_linear.cu; and the plan constants read from the source, with the shapes the GPU tests use to cross them.

Largest ratios observed, kernel_order's normwise error over 16 u (u = 2^-24) against fp64: output 0.081, grad_feat
0.092, grad_gate 0.101."""
import os
import re

import pytest
import torch

import linear_reference as R
from cspn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'cspn_b200', 'csrc', 'cspn2d_linear.cu')
U = 2.0 ** -24
SUBSETS = [('l2r',), ('r2l',), ('t2b',), ('b2t',), ('r2l', 'b2t'), R.DIRECTIONS]


@pytest.mark.parametrize('dirs', SUBSETS, ids=lambda d: '+'.join(d))
@pytest.mark.parametrize('per_channel', [False, True])
def test_kernel_order_against_fp64(dirs, per_channel):
    C = 3
    f, g = R.random_inputs(2, C, 6, 9, dirs, per_channel, seed=len(dirs) + 7 * per_channel, dtype=torch.float64)
    go = torch.randn(2, C, 6, 9, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    out, gf, gg = R.grads(R.composition, f, g, dirs, go)
    o2, _, gf2, gg2 = R.kernel_order(f.float(), g.float(), dirs, go.float())
    assert R.normwise(o2, out) < 16 * U
    assert R.normwise(gf2, gf) < 16 * U
    assert R.normwise(gg2, gg) < 16 * U


@pytest.mark.parametrize('dirs', SUBSETS, ids=lambda d: '+'.join(d))
@pytest.mark.parametrize('per_channel', [False, True])
def test_kernel_order_equals_fp64_on_dyadic_inputs(dirs, per_channel):
    f, g = R.dyadic_inputs(2, 3, 5, 6, dirs, per_channel, seed=3)
    go = torch.randint(-4, 5, (2, 3, 5, 6), generator=torch.Generator().manual_seed(1)).float() / 4
    out, gf, gg = R.grads(R.composition, f, g, dirs, go)
    o2, _, gf2, gg2 = R.kernel_order(f, g, dirs, go)
    assert torch.equal(o2.double(), out) and torch.equal(gf2.double(), gf) and torch.equal(gg2.double(), gg)


def test_flip_and_transpose_identities_on_the_references():
    f, g = R.random_inputs(2, 2, 5, 7, ('l2r',), True, seed=2)
    l2r = lambda x, gt: R.kernel_order(x, gt, ('l2r',))[0]
    fW, fH, T = (lambda t: t.flip(-1)), (lambda t: t.flip(-2)), (lambda t: t.transpose(-1, -2))
    assert torch.equal(R.kernel_order(f, g, ('r2l',))[0], fW(l2r(fW(f), fW(g))))
    assert torch.equal(R.kernel_order(f, g, ('t2b',))[0], T(l2r(T(f), T(g))))
    assert torch.equal(R.kernel_order(f, g, ('b2t',))[0], fH(T(l2r(T(fH(f)), T(fH(g))))))
    f64 = f.double()
    assert torch.equal(R.composition(f64, g.double(), ('b2t',)), fH(T(R.composition(T(fH(f64)), T(fH(g.double())), ('l2r',)))))


def test_merge_rule_against_torch_max():
    nan = float('nan')
    hs = [torch.tensor([1., 2., nan, 0., -0., 3., nan]), torch.tensor([1., 3., 5., nan, 0., 3., nan]),
          torch.tensor([2., 3., nan, 1., 0., 1., 4.])]
    idx = R.merge_index(hs)
    assert idx.tolist() == [2, 1, 0, 1, 0, 0, 0]                  # ties to the first, NaN wins and the first NaN
    st = torch.stack(hs)
    picked = st.gather(0, idx.unsqueeze(0)).squeeze(0)
    ref = st.max(0).values
    assert torch.equal(torch.isnan(picked), torch.isnan(ref)) and torch.equal(picked[~torch.isnan(ref)], ref[~torch.isnan(ref)])
    # on random planes with forced ties the values are torch's
    gen = torch.Generator().manual_seed(0)
    hs = [torch.randint(-3, 4, (64,), generator=gen).float() for _ in range(4)]
    st = torch.stack(hs)
    assert torch.equal(st.gather(0, R.merge_index(hs).unsqueeze(0)).squeeze(0), st.max(0).values)


def test_merge_routes_the_gradient_to_the_first_tie():
    f = torch.ones(1, 1, 1, 3, dtype=torch.float64, requires_grad=True)
    g = torch.zeros(1, 6, 1, 3, dtype=torch.float64, requires_grad=True)
    out = R.composition(f, g, ('l2r', 'r2l'))                        # zero gates: both directions give x, a tie everywhere
    gf, gg = torch.autograd.grad(out.sum(), (f, g))
    assert torch.equal(gf, torch.ones_like(gf))
    assert gg[:, 3:].abs().sum() == 0                               # r2l's gates get nothing
    _, _, gf2, gg2 = R.kernel_order(f.detach().float(), g.detach().float(), ('l2r', 'r2l'), torch.ones(1, 1, 1, 3))
    assert torch.equal(gf2.double(), gf) and torch.equal(gg2.double(), gg)


# ---- the C ABI without a device --------------------------------------------------------------------------------------------
INVALID, WORKSPACE, UNSUPPORTED = -1, -2, -4
P = 1 << 20          # fake, 4-byte aligned "device" addresses: every refusal comes before any device work


def fwd(x=P, g=2 * P, out=4 * P, planes=None, B=1, C=1, H=8, W=8, mask=15, mode=0, ws=6 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_lin_fwd_f32(x, g, out, planes, B, C, H, W, mask, mode, ws, wsb, None)


def bwd(x=P, g=2 * P, planes=3 * P, go=4 * P, gx=5 * P, gg=6 * P, B=1, C=1, H=8, W=8, mask=15, mode=0, ws=8 * P, wsb=1 << 20):
    return _lib.lib().cspn2d_lin_bwd_f32(x, g, planes, go, gx, gg, B, C, H, W, mask, mode, ws, wsb, None)


def test_workspace_formulas():
    L = _lib.lib()
    n = 2 * 3 * 7 * 9
    for mask in range(1, 16):
        nd = bin(mask).count('1')
        assert L.cspn2d_lin_workspace_bytes(2, 3, 7, 9, mask, 0) == (4 * nd * n if nd > 1 else 0)
        assert L.cspn2d_lin_bwd_workspace_bytes(2, 3, 7, 9, mask, 1) == (8 * nd * n if nd > 1 else 0)
        assert L.cspn2d_lin_bwd_workspace_bytes(2, 3, 7, 9, mask, 0) == (8 * nd * n if nd > 1 else 0) + 12 * nd * n
    assert L.cspn2d_lin_bwd_workspace_bytes(2, 1, 7, 9, 1, 0) == 0            # C = 1: a shared gate needs no channel sum
    for bad in ((0, 3, 7, 9, 15, 0), (2, 3, 7, 9, 0, 0), (2, 3, 7, 9, 16, 0), (2, 3, 7, 9, 15, 2), (2, 3, 7, -1, 15, 0)):
        assert L.cspn2d_lin_workspace_bytes(*bad) == 0 and L.cspn2d_lin_bwd_workspace_bytes(*bad) == 0


def test_abi_refusals_without_a_device():
    assert fwd(x=None) == INVALID
    assert fwd(g=None) == INVALID
    assert fwd(out=None) == INVALID
    assert fwd(mask=0) == INVALID
    assert fwd(mask=16) == INVALID
    assert fwd(mask=-1) == INVALID
    assert fwd(mode=2) == INVALID
    assert fwd(B=0) == INVALID
    assert fwd(H=0) == INVALID
    assert fwd(W=-3) == INVALID
    assert fwd(x=P + 2) == INVALID                                 # misaligned
    assert fwd(planes=8 * P, mask=1) == INVALID                    # one direction: its plane is out
    assert fwd(out=P + 64) == INVALID                              # out overlaps feat
    assert b'overlaps' in _lib.lib().cspn_last_error()
    assert fwd(out=2 * P + 64) == INVALID                          # out overlaps the gate
    assert fwd(planes=4 * P + 64, ws=None) == INVALID              # the planes overlap out
    assert fwd(ws=4 * P + 16) == INVALID                           # the workspace overlaps out
    assert fwd(ws=None) == WORKSPACE
    assert fwd(wsb=4) == WORKSPACE
    assert b'linear propagation' in _lib.lib().cspn_last_error()
    assert fwd(H=2049, mask=1, out=1 << 40, ws=None) == UNSUPPORTED           # the lateral extent of l2r is H
    assert fwd(W=2049, mask=4, out=1 << 40, ws=None) == UNSUPPORTED           # of t2b it is W
    assert fwd(B=1 << 16, C=1 << 15, mask=1, g=1 << 44, out=1 << 45, ws=None) == UNSUPPORTED   # B*C beyond gridDim.x
    assert bwd(planes=None) == INVALID
    assert bwd(go=None) == INVALID
    assert bwd(x=None) == INVALID
    assert bwd(gx=P) == INVALID                                    # grad_feat overlaps feat
    assert bwd(gg=5 * P + 8) == INVALID                            # two outputs overlap
    assert bwd(gg=3 * P + 8) == INVALID                            # grad_gate overlaps the planes
    assert bwd(mask=0) == INVALID
    assert bwd(mode=-1) == INVALID
    assert bwd(wsb=16) == WORKSPACE
    assert bwd(ws=None) == WORKSPACE
    assert bwd(W=4096, mask=8, ws=1 << 40, gx=1 << 41, gg=1 << 42) == UNSUPPORTED


def test_python_refusals():
    import cspn_b200
    f, g = R.random_inputs(1, 2, 5, 6)
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g, ('r2l', 'l2r'))            # not in canonical order
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g, ())
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g, ('l2r', 'l2r'))
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g, 'l2r')
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g, ('up',))
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g[:, :9])                     # 9 gate channels for four directions
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f, g[..., :5])
    with pytest.raises(ValueError):
        cspn_b200.propagate2d_linear(f[:, :1], torch.zeros(1, 24, 5, 6))  # per-channel gates need C > 1
    with pytest.raises(ValueError):
        cspn_b200.Affinity_PropagateLinear(('t2b', 'l2r'))
    with pytest.raises(RuntimeError):
        cspn_b200.propagate2d_linear(f.double(), g)
    with pytest.raises(_lib.CspnError):
        cspn_b200.propagate2d_linear(torch.zeros(1, 1, 2049, 4), torch.zeros(1, 3, 2049, 4), ('l2r',))
    with pytest.raises(_lib.CspnError):
        cspn_b200.propagate2d_linear(f, g)                            # CPU tensors: no host entry point
    assert cspn_b200.Affinity_PropagateLinear(('l2r', 'b2t')).directions == ('l2r', 'b2t')


def test_op_schemas_and_fake_kernels():
    from cspn_b200 import torch_op
    if not torch_op.available():
        pytest.skip('the torch op library is not built')
    torch_op.load()
    op = torch.ops.cspn_b200.propagate2d_linear.default
    assert str(op._schema) == 'cspn_b200::propagate2d_linear(Tensor feat, Tensor gate, int dir_mask) -> (Tensor, Tensor)'
    bop = torch.ops.cspn_b200.propagate2d_linear_backward.default
    assert str(bop._schema) == ('cspn_b200::propagate2d_linear_backward(Tensor feat, Tensor gate, Tensor planes, Tensor grad_out, '
                                'int dir_mask, bool need_feat, bool need_gate) -> (Tensor, Tensor)')
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        f, g = torch.empty(2, 3, 5, 7), torch.empty(2, 12, 5, 7)
        out, planes = op(f, g, 15)
        assert out.shape == f.shape and planes.shape == (4, 2, 3, 5, 7)
        out, planes = op(f, g[:, :3], 4)
        assert out.shape == f.shape and planes.numel() == 0
        assert op(f, torch.empty(2, 18, 5, 7), 3)[1].shape == (2, 2, 3, 5, 7)      # per-channel gates
        gx, gg = bop(f, g, torch.empty(4, 2, 3, 5, 7), f, 15, True, False)
        assert gx.shape == f.shape and gg.numel() == 0
        with pytest.raises(Exception):
            op(f, g[:, :11], 15)


# ---- the kernels: no spills, and the plan the shapes of the GPU tests reach ------------------------------------------------
def test_no_spills_in_the_new_translation_unit():
    log = os.path.join(ROOT, 'cspn_b200', '_build', 'ptxas.log')
    if not os.path.isfile(log):
        pytest.skip('the library is not built')
    part = open(log).read().split('== cspn2d_linear.cu')[1].split('\n== ')[0]
    for name in ('lin_fwd_kernel', 'lin_bwd_kernel', 'lin_merge_kernel', 'lin_finalize_kernel'):
        assert name in part
    spills = [int(x) for x in re.findall(r'(\d+) bytes spill stores', part)]
    stacks = [int(x) for x in re.findall(r'(\d+) bytes stack frame', part)]
    assert len(spills) == 4 and max(spills) == 0 and max(stacks) == 0


def source_constants():
    src = open(SRC).read()
    get = lambda name: int(re.search(rf'constexpr int {name} = (\d+);', src).group(1))
    return get('kHalo'), get('kLinMaxSeg'), get('kLinMaxCluster'), get('kLinTargetCtas')


def plan(B, C, H, W, dirs):
    """The scan's plan as lin_plan picks it: (cluster size, segment lanes per orientation)."""
    halo, max_seg, max_cs, target = source_constants()
    nd = len(dirs)
    horiz, vert = bool(set(dirs) & {'l2r', 'r2l'}), bool(set(dirs) & {'t2b', 'b2t'})
    L = max(H if horiz else 0, W if vert else 0)
    cs = 1
    while cs < max_cs and nd * B * C * cs * 2 <= target and L // (cs * 2) >= 2 * halo:
        cs *= 2
    cs = max(cs, -(-L // max_seg))
    return cs, (-(-H // cs) if horiz else 0), (-(-W // cs) if vert else 0)


# (B, C, H, W, directions) of the GPU seam sweep: every cluster size, segments that end inside the plane and a last
# segment that is shorter or empty, scans with a partial last chunk, and the widest lateral extent
PLAN_SHAPES = [(2, 3, 37, 29, ('l2r', 'b2t')), (1, 1, 40, 300, ('l2r',)), (1, 2, 90, 70, ('r2l', 't2b')), (1, 1, 300, 77, ('l2r', 'r2l')),
               (70, 1, 45, 67, R.DIRECTIONS), (1, 1, 2048, 3, ('r2l',)), (1, 1, 5, 1500, ('b2t',))]


def test_plan_constants_and_the_shapes_that_cross_them():
    halo, max_seg, max_cs, target = source_constants()
    assert (halo, max_seg, max_cs, target) == (8, 256, 8, 264)
    plans = [plan(*s) for s in PLAN_SHAPES]
    assert {p[0] for p in plans} >= {1, 2, 4, 8}                    # every cluster size a power of two reaches
    for (B, C, H, W, d), (cs, sh, sv) in zip(PLAN_SHAPES, plans):
        S = W if d[0] in ('l2r', 'r2l') else H
        assert S % halo != 0 or S < halo                            # the last chunk is partial (or the only one)
        for seg, L in ((sh, H), (sv, W)):
            if seg:
                assert seg <= max_seg and cs * seg >= L
                if cs > 1:
                    assert seg < L                                  # segment seams inside the plane
    assert plan(8, 1, 352, 1216, R.DIRECTIONS) == (8, 44, 152)      # the KITTI shape: 8-CTA clusters
