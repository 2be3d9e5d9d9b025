"""CPU tests of the aggregation of the 2D steps (propagate2d_aggregate; DESIGN.md section 4.20): the fp32 restatement in
the kernels' order against the fp64 op sequence and its autograd, gradcheck, the dyadic cases that fp32 computes exactly,
the workspace formulas, the Python and C ABI refusals before any device work, the argtypes, the dispatcher registration,
and the machine code of cspn2d_wide.cu (no spills; every kernel that existed before the aggregation is unchanged)."""
import ctypes
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import cspn_b200
from cspn_b200 import _lib, build

import aggregate_reference as ar
import backward_exact as be
from test_resize_trilinear_cpu import header_signature

ENTRIES = ('cspn2d_agg_workspace_bytes', 'cspn2d_agg_fwd_f32', 'cspn2d_agg_bwd_workspace_bytes', 'cspn2d_agg_bwd_f32')
HERE = os.path.dirname(os.path.abspath(__file__))


def inputs(seed, B, C, H, W, K, T, dtype=torch.float64, sparse=True):
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(B, K * K - 1, H, W, generator=gen)
    d = torch.rand(B, C, H, W, generator=gen)
    s = (torch.rand(B, 1, H, W, generator=gen) < 0.3).float() * torch.rand(B, 1, H, W, generator=gen) if sparse else None
    sw = torch.randn(B, T, H, W, generator=gen)
    go = torch.randn(B, C, H, W, generator=gen)
    return [None if t is None else t.to(dtype) for t in (g, d, s, sw, go)]


def autograd(g, d, s, sw, go, steps, K, norm, keep, dtype):
    leaves = [t.detach().to(dtype).requires_grad_(True) for t in (g, d, s, sw)]
    out = ar.composition(*leaves, steps, K, norm, keep)
    out.backward(go.to(dtype))
    return [out.detach()] + [t.grad for t in leaves]


# ---- 1. the restatement is the op sequence and its autograd ----------------------------------------------------------------
CASES = [(3, '8sum', False, (1, 2, 3, 4)), (5, '24sum_abs', True, (2, 5)), (7, '48sum', True, (3,)), (5, '24sum', False, (1, 4, 6))]


@pytest.mark.parametrize('K,norm,keep,steps', CASES)
def test_restatement_against_fp64_autograd(K, norm, keep, steps):
    B, C, H, W = 2, 3, 9, 11
    g, d, s, sw, go = inputs(K + len(steps), B, C, H, W, K, len(steps), torch.float32)
    ds = ar.iterates(g, d, s, steps, K, norm, keep)
    out64, gg, gd, gs, gw = autograd(g, d, s, sw, go, steps, K, norm, keep, torch.float64)
    ok, err, scale = ar.within(ar.aggregate(ds, sw), out64, 1e-5)
    assert ok, (err, scale)
    ok, err, scale = ar.within(ar.grad_step_weight(go, ds), gw, 1e-5)
    assert ok, (err, scale)
    # the step weights' gradient is the iterates' inner product with grad_out, and the sparse samples take a gradient in
    # keep mode only
    ds64 = ar.iterates(g.double(), d.double(), s.double(), steps, K, norm, keep)
    assert torch.allclose(gw, torch.stack([(go.double() * x).sum(1) for x in ds64], 1), rtol=1e-12, atol=1e-12)
    assert (gs is not None and gs.abs().sum() > 0) == keep or not keep and (gs is None or not gs.any())


def test_gradcheck_of_the_composition():
    g, d, s, sw, _ = inputs(3, 1, 2, 5, 6, 5, 2)
    for keep in (False, True):     # sparse stays fixed: its indicator jumps where a finite difference crosses zero
        leaves = [t.clone().requires_grad_(True) for t in (g, d, sw)]
        assert torch.autograd.gradcheck(lambda g, d, sw: ar.composition(g, d, s, sw, (1, 3), 5, '24sum', keep), leaves)


def test_steps_n_with_unit_weight_is_the_last_iterate():
    g, d, s, _, _ = inputs(4, 2, 1, 8, 7, 5, 1, torch.float32)
    for keep in (False, True):
        last = ar.iterates(g, d, s, (4,), 5, '24sum', keep)[0]
        out = ar.composition(g, d, s, torch.ones(2, 1, 8, 7), (4,), 5, '24sum', keep)
        assert torch.equal(out, last)


# ---- 2. dyadic cases: fp32 computes them exactly ----------------------------------------------------------------------------
@pytest.mark.parametrize('K,sparse,keep', [(3, 'signed', False), (5, 'bernoulli', True), (7, None, False), (5, 'signed', True)])
def test_dyadic_cases_are_exact(K, sparse, keep):
    steps = (1, 2, 4)
    g, d, s, go = be.dyadic_2d(K * 7 + keep, 1, 2, 9, 10, K, sparse)
    sw = ar.dyadic_weights(torch.Generator().manual_seed(K), (1, len(steps), 9, 10))
    s = s if s is not None else None
    r64 = autograd(g, d, s if s is not None else torch.zeros(1, 1, 9, 10), sw, go, steps, K, f'{K * K - 1}sum', keep,
                   torch.float64)
    r32 = autograd(g, d, s if s is not None else torch.zeros(1, 1, 9, 10), sw, go, steps, K, f'{K * K - 1}sum', keep,
                   torch.float32)
    unit = 4.0 ** -(steps[-1] + 1) / 2
    for a, b, name in zip(r64, r32, ('out', 'grad_guidance', 'grad_blur', 'grad_sparse', 'grad_step_weight')):
        if a is None:
            continue
        be.check_exact(a, steps[-1], name, unit)
        assert torch.equal(a, b.double()), name
    ds = ar.iterates(g, d, s, steps, K, f'{K * K - 1}sum', keep)
    assert torch.equal(ar.aggregate(ds, sw).double(), r64[0])
    assert torch.equal(ar.grad_step_weight(go, ds).double(), r64[4])


# ---- 3. the Python surface ---------------------------------------------------------------------------------------------------
def test_python_validation_and_cpu_tensors_are_refused():
    g, d, sw = torch.rand(1, 24, 6, 5), torch.rand(1, 2, 6, 5), torch.rand(1, 3, 6, 5)
    f = cspn_b200.propagate2d_aggregate
    for kw in [dict(steps=(1, 2)), dict(steps=(2, 2, 3)), dict(steps=(0, 1, 2)), dict(steps=(3, 2, 1)), dict(steps=(1, 2.0, 3)),
               dict(steps=(True, 2, 3)), dict(steps='123'), dict(steps=3), dict(step_weight=torch.rand(1, 3, 6)),
               dict(step_weight=torch.rand(2, 3, 6, 5)), dict(step_weight=torch.rand(1, 3, 5, 6)),
               dict(guidance=torch.rand(1, 8, 6, 5)), dict(sparse_depth=torch.rand(1, 2, 6, 5))]:
        args = dict(guidance=g, blur_depth=d, step_weight=sw, prop_kernel=5)
        args.update(kw)
        with pytest.raises(ValueError):
            f(**args)
    with pytest.raises(AssertionError):
        f(g, d, sw, prop_kernel=4)
    with pytest.raises(AssertionError):
        f(g, d, sw, prop_kernel=5, norm_type='8sum')
    with pytest.raises(RuntimeError, match='step_weight'):
        f(g, d, sw.double(), prop_kernel=5)
    with pytest.raises(cspn_b200.CspnError, match='CUDA'):
        f(g, d, sw, prop_kernel=5)


# ---- 4. the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    assert _lib.SIGNATURES[name] == header_signature(name)


def steps_arg(*steps):
    return (ctypes.c_int * len(steps))(*steps)


def test_workspace_formulas():
    L = _lib.lib()
    for B, C, H, W, K, steps in ((2, 3, 7, 9, 3, (1, 2)), (8, 1, 228, 304, 5, tuple(range(1, 25))), (1, 2, 5, 6, 7, (3, 9))):
        N, bk, bc = steps[-1], B * K * K * H * W, B * C * H * W
        for keep in (0, 1):
            assert L.cspn2d_agg_workspace_bytes(B, C, H, W, K, steps_arg(*steps), len(steps), keep) == 4 * (bk + (2 + keep) * bc)
            assert (L.cspn2d_agg_bwd_workspace_bytes(B, C, H, W, K, steps_arg(*steps), len(steps), keep)
                    == 4 * (bk + (2 * N + 1 + keep) * bc))
    for q in (L.cspn2d_agg_workspace_bytes, L.cspn2d_agg_bwd_workspace_bytes):
        for bad in ((0, 1, 4, 5, 5, steps_arg(1), 1, 0), (1, 1, 4, 5, 4, steps_arg(1), 1, 0), (1, 1, 4, 5, 5, steps_arg(1), 0, 0),
                    (1, 1, 4, 5, 5, None, 1, 0), (1, 1, 4, 5, 5, steps_arg(2, 2), 2, 0), (1, 1, 4, 5, 5, steps_arg(0, 1), 2, 0),
                    (1, 1, 4, 5, 5, steps_arg(1), 1, 2)):
            assert q(*bad) == 0


def test_c_abi_rejects_bad_arguments_before_any_device_work():
    L = _lib.lib()
    buf = (ctypes.c_float * 65536)()
    base = ctypes.cast(buf, ctypes.c_void_p).value

    def at(k, off=0):                                    # 4096 floats apart
        return ctypes.c_void_p(base + k * 16384 + off)

    odd = ctypes.c_void_p(base + 2)
    ok = dict(B=1, C=2, H=4, W=5)     # guidance 24*20 floats, blur 40, sparse 20, step_weight (T = 2) 40
    big = 1 << 20

    def fw(g=at(0), d=at(1), s=at(2), sw=at(3), o=at(4), gch=24, K=5, steps=(1, 3), ns=None, norm=0, keep=1, ws=at(5),
           wsb=big, **over):
        v = dict(ok, **over)
        return L.cspn2d_agg_fwd_f32(g, d, s, sw, o, *v.values(), gch, K, None if steps is None else steps_arg(*steps),
                                    len(steps or ()) if ns is None else ns, norm, keep, ws, wsb, None)

    def bw(g=at(0), d=at(1), s=at(2), sw=at(3), go=at(4), gg=at(5), gd=at(6), gs=at(7), gw=at(8), gch=24, K=5, steps=(1, 3),
           ns=None, norm=0, keep=1, ws=at(9), wsb=big, **over):
        v = dict(ok, **over)
        return L.cspn2d_agg_bwd_f32(g, d, s, sw, go, gg, gd, gs, gw, *v.values(), gch, K,
                                    None if steps is None else steps_arg(*steps), len(steps or ()) if ns is None else ns,
                                    norm, keep, ws, wsb, None)

    for call, need, opt in ((fw, ('g', 'd', 'sw', 'o'), ('s',)), (bw, ('g', 'd', 'sw', 'go'), ('s', 'gg', 'gd', 'gs', 'gw'))):
        for k in ok:
            assert call(**{k: 0}) == -1 and call(**{k: -3}) == -1
        for p in need:
            assert call(**{p: None}) == -1 and b'null' in L.cspn_last_error()
        for p in need + opt:
            assert call(**{p: odd}) == -1 and b'aligned' in L.cspn_last_error()
        assert call(K=4) == -1 and b'kernel size' in L.cspn_last_error()
        assert call(gch=23) == -1 and b'guidance channels' in L.cspn_last_error()
        assert call(norm=2) == -1 and b'norm_type' in L.cspn_last_error()
        assert call(keep=2) == -1 and b'keep' in L.cspn_last_error()
        assert call(steps=None, ns=2) == -1 and call(steps=(1,), ns=0) == -1 and b'n_steps' in L.cspn_last_error()
        for steps in ((0, 1), (2, 2), (3, 1), (-1,)):
            assert call(steps=steps) == -1 and b'strictly increasing' in L.cspn_last_error()
        assert call(B=256, C=256) == -4 and b'gridDim.z' in L.cspn_last_error()
        assert call(ws=None) == -2 and call(wsb=1) == -2 and b'workspace' in L.cspn_last_error()
    # an output may overlap neither an input nor another output; inputs may alias one another
    assert fw(o=at(1, 4 * 39)) == -1 and b'out overlaps blur' in L.cspn_last_error()
    assert fw(o=at(3, 4 * 39)) == -1 and b'out overlaps step_weight' in L.cspn_last_error()
    assert fw(ws=at(0, 4 * 479)) == -1 and b'the workspace overlaps guidance' in L.cspn_last_error()
    for over, what in ((dict(gg=at(0, 4 * 479)), b'grad_guidance overlaps guidance'), (dict(gd=at(4, 4 * 39)), b'grad_blur overlaps grad_out'),
                       (dict(gs=at(2, 4 * 19)), b'grad_sparse overlaps sparse'), (dict(gw=at(3, 4 * 39)), b'grad_step_weight overlaps step_weight'),
                       (dict(gw=at(6, 4 * 39)), b'grad_step_weight overlaps grad_blur'), (dict(ws=at(8, 4 * 39)), b'the workspace overlaps grad_step_weight')):
        assert bw(**over) == -1 and what in L.cspn_last_error(), (over, L.cspn_last_error())
    assert L.cspn_last_launches() == 0


# ---- 5. the dispatcher op ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ops():
    from cspn_b200 import torch_op
    build.build_torch_op()
    torch_op.load()
    return torch.ops.cspn_b200


def test_op_schemas_and_fake_kernels(ops):
    assert ('propagate2d_aggregate(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight, int[] steps, '
            'int kernel_size, int norm_type, bool keep) -> Tensor' in str(ops.propagate2d_aggregate.default._schema))
    assert ('propagate2d_aggregate_backward(Tensor guidance, Tensor blur_depth, Tensor? sparse_depth, Tensor step_weight, '
            'Tensor grad_out, int[] steps, int kernel_size, int norm_type, bool keep, bool need_guidance, bool need_blur, '
            'bool need_sparse, bool need_step_weight) -> (Tensor, Tensor, Tensor, Tensor)'
            in str(ops.propagate2d_aggregate_backward.default._schema))
    with FakeTensorMode():
        g = torch.empty(8, 48, 228, 304, device='cuda')
        d, s = torch.empty(8, 1, 228, 304, device='cuda'), torch.empty(8, 1, 228, 304, device='cuda')
        sw = torch.empty(8, 24, 228, 304, device='cuda')
        out = ops.propagate2d_aggregate(g, d, s, sw, list(range(1, 25)), 7, 0, True)
        assert out.shape == d.shape and out.dtype == torch.float32 and out.device == d.device
        gg, gd, gs, gw = ops.propagate2d_aggregate_backward(g, d, s, sw, out, list(range(1, 25)), 7, 0, True, True, True, True, True)
        assert gg.shape == g.shape and gd.shape == d.shape and gs.shape == s.shape and gw.shape == sw.shape
        assert cspn_b200.propagate2d_aggregate(g, d, sw, s, 7, keep_sparse=True).shape == d.shape   # the op route
        for steps in ([1, 2], [2, 1] + list(range(3, 25))):
            with pytest.raises(Exception):
                ops.propagate2d_aggregate(g, d, s, sw, steps, 7, 0, True)


# ---- 6. the machine code -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def wide_cubin(tmp_path_factory):
    """cspn2d_wide.cu compiled as the build compiles it: (ptxas -v report, {kernel: SASS}), and the recorded hashes."""
    golden = json.load(open(os.path.join(HERE, 'golden', 'cspn2d_wide_sass_sm90a.json')))
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc not found')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    if not os.path.isfile(cuobjdump):
        pytest.skip('cuobjdump not found')
    version = re.search(r'release (\S+),', subprocess.run([nvcc, '--version'], capture_output=True, text=True).stdout).group(1)
    cubin = str(tmp_path_factory.mktemp('sass') / 'wide.cubin')
    ccbin = ['-ccbin', shutil.which('g++')] if shutil.which('g++') else []
    r = subprocess.run([nvcc] + ccbin + build.NVCC_FLAGS + ['-Xptxas', '-v', '-cubin', '-o', cubin,
                                                             os.path.join(build.CSRC, 'cspn2d_wide.cu')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines(keepends=True):
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            name = re.sub(r'_GLOBAL__N__[0-9a-f]+_\d+_cspn2d_wide_cu_[0-9a-f]+', '_GLOBAL__N_', m.group(1))
            kernels[name] = ''
        elif name:
            kernels[name] += line
    return r.stderr, kernels, golden, version


def test_no_new_kernel_spills(wide_cubin):
    report, kernels, golden, _ = wide_cubin
    spills = dict(re.findall(r'Function properties for (\S+)\n\s+\d+ bytes stack frame, (\d+) bytes spill stores', report))
    norm = {re.sub(r'_GLOBAL__N__[0-9a-f]+_\d+_cspn2d_wide_cu_[0-9a-f]+', '_GLOBAL__N_', k): int(v) for k, v in spills.items()}
    new = [k for k in kernels if k not in golden['kernels']]
    assert len(new) == 10 and all(k in norm for k in new)             # 3 x (vec step, scalar step, adjoint) + gradw
    assert all(norm[k] == 0 for k in new), {k: norm[k] for k in new if norm[k]}


def test_every_pre_existing_kernel_keeps_its_machine_code(wide_cubin):
    _, kernels, golden, version = wide_cubin
    if version != golden['nvcc']:
        pytest.skip(f'the recorded machine code is from nvcc {golden["nvcc"]}, this is {version}')
    changed = [k for k, h in golden['kernels'].items() if hashlib.sha256(kernels.get(k, '').encode()).hexdigest() != h]
    assert not changed, changed
