"""The IEEE contract of the normalised 3D propagation on every route of its forward, and its backward at special sums of
|gates| (tests/ieee3d.py has the families, the references and the matrix):
  - scaled dyadic gates: `out` bit for bit against fp64 with S rounded to fp32, on every route of the 3x3x3 forward
    (raw-guidance float4 kernels, CSPN_B200_3D_PADDLE=planes, odd W, a misaligned view, ragged volume groups, B * C * D >
    65535) and both steps of the 5x5x5 one, through both modules and both call routes;
  - the same inputs backward: grad_guidance and grad_feat bit for bit at tile-crossing shapes, through both autograd routes;
  - random gates with special regions, and inf / NaN in feat: the oracle's NaN, +inf and -inf masks and parity_ok(1e-4),
    and the same masks on every route;
  - the fused gather's last step (the FAN instances of the step kernels) delivers the plain forward's bits on such inputs.
"""
import ctypes

import numpy as np
import pytest
import torch

import cspn_b200
from cspn_b200 import _lib, torch_op

import ieee3d as ie
import memory_contract as mc

pytestmark = pytest.mark.gpu

D, H = 6, 9
NORM_CODE = {'paddle': 2}


def norm_code(norm):
    return NORM_CODE.get(norm, 1 if norm.endswith('_abs') else 0)


def misaligned_copy(t):
    """The same values in a view whose data pointer is 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def set_route(monkeypatch, route, g, f, K, N):
    """The environment of `route` for inputs g, f (per-channel gates: B * C volumes of one channel)."""
    B, C = f.shape[:2]
    Bv, Cv = (B * C, 1) if g.shape[1] == (K ** 3 - 1) * C and C > 1 else (B, C)
    paddle, ws = ie.route_env(route, Bv, Cv, *f.shape[2:], N)
    for name, v in (('CSPN_B200_3D_PADDLE', paddle), ('CSPN_B200_MAX_WS3D_KB', ws)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, v)


def module(K, N, norm, api):
    cls, use_op = api.split('-')
    m = cspn_b200.Affinity_Propagate3D(N, 3, norm) if cls == 'P3D' else cspn_b200.Affinity_Propagate3DK(N, K, norm)
    if use_op == 'op':
        torch_op.load()
    m._use_op = use_op == 'op'
    return m


def forward(g, f, N, K, norm, route, api, monkeypatch):
    """out of the module on the GPU on `route`, with the launches of the call checked against the route's."""
    set_route(monkeypatch, route, g, f, K, N)
    gc, fc = g.cuda(), f.cuda()
    if route == 'misaligned':
        gc, fc = misaligned_copy(gc), misaligned_copy(fc)
    with torch.no_grad():
        out = module(K, N, norm, api)(gc, fc)
    torch.cuda.synchronize()
    assert _lib.lib().cspn_last_launches() == ie.launches(route, K, norm, N), (route, _lib.lib().cspn_last_launches())
    return out.cpu()


def case_inputs(c, seed):
    K, norm, route = c['path']
    C, pc = ie.gates_shape(c['gates'])
    B, d, h = ie.route_dims(route, D, H)
    return K, norm, route, B, C, d, h, ie.W_OF[route], pc


def assert_bits(ours, ref, what):
    a = ours.double()
    bad = a != ref
    assert not bad.any(), (what, f'{int(bad.sum())} of {bad.numel()} differ, first at {tuple(bad.nonzero()[0].tolist())}',
                           float(a.flatten()[bad.flatten()][0]), float(ref.flatten()[bad.flatten()][0]))


# ---- 1. scaled dyadic gates, forward ---------------------------------------------------------------------------------------
SCALED = ie.scaled_cases()


@pytest.mark.parametrize('i', range(len(SCALED)), ids=[ie.case_id(c) for c in SCALED])
def test_scaled_dyadic_forward_is_exact_on_every_route(i, monkeypatch):
    c = SCALED[i]
    K, norm, route, B, C, d, h, W, pc = case_inputs(c, i)
    N, e = c['N'], c['e']
    g, f, go = ie.scaled_dyadic(3000 + i, B, C, d, h, W, K, norm, e, pc)
    ref = ie.scaled_reference(g, f, go, N, K, norm, e, backward=False)[0]
    assert_bits(forward(g, f, N, K, norm, route, c['api'], monkeypatch), ref, ie.case_id(c))


# ---- 2. scaled dyadic gates, backward --------------------------------------------------------------------------------------
BACKWARD = ie.backward_cases()


@pytest.mark.parametrize('i', range(len(BACKWARD)), ids=[ie.case_id(c) for c in BACKWARD])
def test_scaled_dyadic_backward_is_exact(i, monkeypatch):
    c = BACKWARD[i]
    (K, norm), (d, h, W), N, e = c['path'], c['dhw'], c['N'], c['e']
    C, pc = ie.gates_shape(c['gates'])
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    g, f, go = ie.scaled_dyadic(4000 + i, 1, C, d, h, W, K, norm, e, pc)
    ref = ie.scaled_reference(g, f, go, N, K, norm, e)
    for use_op in (False, True):
        m = module(K, N, norm, ('P3D' if K == 3 and i % 2 else 'P3DK') + ('-op' if use_op else '-ctypes'))
        gc, fc = g.cuda().requires_grad_(True), f.cuda().requires_grad_(True)
        out = m(gc, fc)
        out.backward(go.cuda())
        for ours, r, name in zip((out.detach(), gc.grad, fc.grad), ref, ('out', 'grad_guidance', 'grad_feat')):
            assert_bits(ours.cpu(), r, (ie.case_id(c), use_op, name))


# ---- 3. special regions and non-finite feat against the oracle ---------------------------------------------------------------
SPECIALS = ie.special_cases()


def special_inputs(kind, seed, B, C, d, h, W, K, pc):
    if kind.startswith('feat'):
        return ie.nonfinite_feat(seed, C, d, h, W, K, float(kind[4:]), pc)
    return ie.special_gates(seed, B, C, d, h, W, K, kind, pc)


@pytest.mark.parametrize('i', range(len(SPECIALS)), ids=[ie.case_id(c) for c in SPECIALS])
def test_special_sums_and_nonfinite_feat_follow_the_oracle(i, monkeypatch):
    c = SPECIALS[i]
    K, norm, route, B, C, d, h, W, pc = case_inputs(c, i)
    g, f = special_inputs(c['kind'], 5000 + i, B, C, d, h, W, K, pc)
    ref = ie.oracle(g.numpy(), f.numpy(), c['N'], K, norm)
    ie.check_masks_and_parity(forward(g, f, c['N'], K, norm, route, c['api'], monkeypatch).numpy(), ref, ie.case_id(c))


# The routes that take the same inputs (W = 136, B = 3): every one must give the masks of the first.  'groups' with
# CSPN_B200_3D_PADDLE=planes makes the float4 plane step run in ragged groups; 'misaligned' the scalar one (at K = 5 too).
SAME_INPUT_ROUTES = {3: ('raw', 'planes', 'misaligned', 'planes+groups'), 5: ('vec', 'misaligned')}


@pytest.mark.parametrize('kind', ie.SPECIAL + tuple(f'feat{v}' for v in ie.NONFINITE))
@pytest.mark.parametrize('K,norm', [(K, n) for K in (3, 5) for n in ie.be.norms_3d(K)])
def test_every_route_gives_the_same_nan_and_inf_masks(K, norm, kind, monkeypatch):
    N, W = 3, 136
    g, f = special_inputs(kind, 6000 + K, 3, 2, D, H, W, K, False)
    ref = ie.oracle(g.numpy(), f.numpy(), N, K, norm)
    first = None
    for route in SAME_INPUT_ROUTES[K]:
        monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
        monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
        if route == 'planes+groups':
            monkeypatch.setenv('CSPN_B200_3D_PADDLE', 'planes')
            monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', ie.route_env('groups', 3, 2, D, H, W, N)[1])
        gc, fc = g.cuda(), f.cuda()
        if route == 'misaligned':
            gc, fc = misaligned_copy(gc), misaligned_copy(fc)
        out = cspn_b200.propagate3d_k(gc, fc, K, N, norm).cpu().numpy()
        ie.check_masks_and_parity(out, ref, (K, norm, kind, route))
        if first is None:
            first = ie.masks(out)
        assert all(np.array_equal(a, b) for a, b in zip(first, ie.masks(out))), (K, norm, kind, route)


# ---- 4. the fused gather's last step ---------------------------------------------------------------------------------------
# One case per FAN instance of a step kernel: (K, norm, W, CSPN_B200_3D_PADDLE=planes, inputs)
GATHER = [
    (3, 'paddle', 136, False, 'e127'),        # step3d_paddle_vec4_kernel: S overflows, sum |g| d overflows
    (3, 'paddle', 136, False, 'e-149'),       # the same at the smallest subnormal
    (3, 'paddle', 136, True, 'feat-inf'),     # step3d_vec4_kernel, 'paddle' without the kappa d0 term
    (3, 'paddle', 135, False, 'featnan'),     # step3d_kernel
    (3, '26sum_abs', 136, False, 'featinf'),  # step3d_gather_vec4_kernel, kappa at an infinite d0
    (3, '26sum', 136, False, 'e-128'),        # its cold path: 1 / S overflows
    (5, 'paddle', 136, False, 'e127'),        # step3k_vec_kernel
    (5, 'paddle', 135, False, 'e-140'),       # step3k_scalar_kernel
]


@pytest.mark.parametrize('K,norm,W,planes,inputs', GATHER)
def test_fused_gather_delivers_the_plain_forward_bits(K, norm, W, planes, inputs, monkeypatch):
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    if planes:
        monkeypatch.setenv('CSPN_B200_3D_PADDLE', 'planes')
    B, C, N = 2, 2, 2
    if inputs.startswith('e'):
        e = int(inputs[1:])
        g, f, go = ie.scaled_dyadic(7000 + K + W, B, C, D, H, W, K, norm, e)
        ref = ie.scaled_reference(g, f, go, N, K, norm, e, backward=False)[0]
    else:
        g, f = ie.special_gates(7000 + K + W, B, C, D, H, W, K, 'zero')
        f[0, 1, 2, 4, 6] = float(inputs[4:])
        f[1, 0, 0, 0, 0] = float(inputs[4:])
        ref = None
    gc, fc = g.cuda(), f.cuda()
    plain = cspn_b200.propagate3d_k(gc, fc, K, N, norm)
    torch.cuda.synchronize()
    launches = _lib.lib().cspn_last_launches()
    if ref is None:
        ie.check_masks_and_parity(plain.cpu().numpy(), ie.oracle(g.numpy(), f.numpy(), N, K, norm), (K, norm, W, inputs))
    else:
        assert_bits(plain.cpu(), ref, (K, norm, W, inputs))
    L = _lib.lib()
    dims = (B, C, D, H, W) + ((N,) if K == 3 else (K, N)) + (norm_code(norm),)
    ws_bytes = L.cspn3d_workspace_bytes(B, C, D, H, W, N) if K == 3 else L.cspn3d_k_workspace_bytes(B, C, D, H, W, K, N)
    ws = mc.workspace(ws_bytes)
    out, peer = mc.guarded(plain.shape), mc.guarded(plain.shape)
    arr = (ctypes.c_void_p * 1)(peer.ptr())
    entry = 'cspn3d_fwd_gather_f32' if K == 3 else 'cspn3d_k_fwd_gather_f32'
    rc = getattr(L, entry)(gc.data_ptr(), fc.data_ptr(), out.ptr(), ctypes.cast(arr, ctypes.c_void_p), 1, None, *dims,
                           ws.ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, entry)
    torch.cuda.synchronize()
    assert L.cspn_last_launches() == launches
    assert out.guards_intact() and peer.guards_intact() and ws.guards_intact()
    for buf, name in ((out, 'out'), (peer, 'peer')):
        assert torch.equal(mc.words(buf.t), mc.words(plain)), (K, norm, W, inputs, name)
