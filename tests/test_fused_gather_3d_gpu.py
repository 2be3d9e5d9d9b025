"""The fused gather of the 3D forwards (cspn3d_{,k_,gates_}fwd_gather_f32), run on one GPU.

As in tests/test_fused_gather_k_gpu.py, n_peer + 1 ranks are emulated on one GPU: slices of guarded local buffers
(tests/memory_contract.py) stand in for the other GPUs' gather buffers, since peer pointers are plain device addresses.
The call runs as the middle rank r.  Block r of every buffer must hold exactly the bits of the plain forward
(cspn3d_{,k_,gates_}fwd_f32 on the same inputs and an equally placed workspace); every other block and every guard band
must still hold the sentinel; the inputs keep their bits; the workspace has exactly the queried size and its guards stay
intact; cspn_last_launches() counts what the plain forward launches.  Bits are compared word for word.

The matrix: the families '3d' (norms 0/1/2), 'k3d' (K = 3, the delegation to '3d', and K = 5; norms 0/1/2) and 'gates3d'
(K = 3 and 5); n_peer in {0, 1, 7}; N in {1, 2, 5} (both ping-pong parities, and N = 1 without an intermediate buffer);
C = 1, C = 2 with one shared gate and C = 2 with per-channel gates; and every route of the plain forward: W % 4 == 0 with
aligned pointers (the raw-guidance and float4 kernels), odd W (the scalar and weight-plane kernels),
CSPN_B200_3D_PADDLE=planes (the 3x3x3 float4 weight-plane kernel), a workspace 4 bytes off a 16-byte boundary, and
CSPN_B200_MAX_WS3D_KB set so that B = 3 runs as launch groups of 2 + 1.  D * H * W is a multiple of 4, so every rank's
block starts 16-byte aligned.

FusedGather's 3D methods run the same way, with local buffers set in place of what the rendezvous provides.  Out of scope
here: stores to a real NVLS multicast address and between GPUs, and the symmetric-memory rendezvous of several processes;
tools/gather_check.py --3d runs those on a multi-GPU node.
"""
import ctypes

import pytest
import torch

from cspn_b200 import _lib

import memory_contract as mc

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -4
D, H = 6, 6
W_OF = {'vec': 16, 'odd': 13}


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def exact(a, b):
    return a.shape == b.shape and torch.equal(mc.words(a), mc.words(b))


class Case:
    """Inputs of one family on the GPU and its plain and gathered forward calls.  `entry` is the plain forward's name;
    `dims` its integer arguments after the pointers (the per-channel gates as B*C single-channel volumes)."""

    def __init__(self, family, K, norm, N, B, C, W, gates='shared', seed=0, special=False):
        gen = torch.Generator().manual_seed(seed * 1009 + K * 31 + N * 7 + B * C + W + norm)
        nt = K ** 3 - 1
        self.family, self.K, self.N = family, K, N
        self.shape = (B, C, D, H, W)
        feat = torch.rand(B, C, D, H, W, generator=gen) * 4 - 1
        g = torch.randn(B, nt * C if gates == 'per_channel' else nt, D, H, W, generator=gen)
        if family == 'gates3d':
            g = g * (0.5 / nt)
            if special:                 # gates >= 0 keep the inf from meeting a -inf (inf - inf = NaN)
                g = g.abs()
                g[0, 0, 2, 3, 5] = float('nan')
                g[0, nt - 1, 0, 0, 0] = float('inf')    # tap NT-1 reads (-R, -R, -R): the padding at (0, 0, 0), inf * 0
                feat[-1, -1, 3, 3, 2] = float('inf')
        elif special:                   # zero guidance around whole neighbourhoods: 0/0 weights, NaN spreading from them
            g[:, :, :, :, 3:11] = 0
        self.g, self.feat = g.cuda().contiguous(), feat.cuda().contiguous()
        Bi, Ci = (B * C, 1) if gates == 'per_channel' else (B, C)
        L = _lib.lib()
        if family == '3d':
            self.entry, self.dims = 'cspn3d_fwd_f32', [Bi, Ci, D, H, W, N, norm]
            self.ws_bytes = L.cspn3d_workspace_bytes(Bi, Ci, D, H, W, N)
        elif family == 'k3d':
            self.entry, self.dims = 'cspn3d_k_fwd_f32', [Bi, Ci, D, H, W, K, N, norm]
            self.ws_bytes = L.cspn3d_k_workspace_bytes(Bi, Ci, D, H, W, K, N)
        else:
            self.entry, self.dims = 'cspn3d_gates_fwd_f32', [Bi, Ci, D, H, W, K, N]
            self.ws_bytes = L.cspn3d_gates_workspace_bytes(Bi, Ci, D, H, W, K, N)
        self.gather_entry = self.entry.replace('_fwd_f32', '_fwd_gather_f32')
        self.n_index = 5 if family == '3d' else 6       # where N sits in dims

    def inputs(self):
        return [self.g, self.feat]

    def plain(self, out_ptr, ws_ptr):
        return getattr(_lib.lib(), self.entry)(ptr(self.g), ptr(self.feat), out_ptr, *self.dims, ws_ptr, self.ws_bytes,
                                               stream())

    def gather(self, out_ptr, peers, ws_ptr, n_peer=None, mc_ptr=None):
        arr = None if peers is None else (ctypes.c_void_p * max(len(peers), 1))(*peers)
        return getattr(_lib.lib(), self.gather_entry)(
            ptr(self.g), ptr(self.feat), out_ptr, None if arr is None else ctypes.cast(arr, ctypes.c_void_p),
            len(peers) if n_peer is None else n_peer, mc_ptr, *self.dims, ws_ptr, self.ws_bytes, stream())


def plain_forward(case, ws_off):
    """The plain forward into a guarded out: the bits the gather must deliver, and its launch count."""
    out, ws = mc.guarded(case.shape), mc.workspace(case.ws_bytes, ws_off)
    _lib.check(case.plain(out.ptr(), ws.ptr()), case.entry)
    torch.cuda.synchronize()
    mc.assert_written(out, 'plain forward')
    assert ws.guards_intact()
    return out.t.cpu(), _lib.lib().cspn_last_launches()


def gather_world(case, n_peer, ws_off, ref, launches, what):
    B = case.shape[0]
    world = n_peer + 1
    r = world // 2
    bufs = [mc.guarded((world * B, *case.shape[1:])) for _ in range(world)]
    ws = mc.workspace(case.ws_bytes, ws_off)
    before = mc.snapshot(case.inputs())
    block = lambda j: bufs[j].t[r * B:(r + 1) * B].data_ptr()
    peers = [block(j) for j in range(world) if j != r]
    _lib.check(case.gather(block(r), peers, ws.ptr()), case.gather_entry)
    torch.cuda.synchronize()
    assert _lib.lib().cspn_last_launches() == launches, what
    assert ws.guards_intact(), f'{what}: a store landed outside the workspace'
    assert mc.unchanged(before, case.inputs()), f'{what}: an input changed'
    for j, buf in enumerate(bufs):
        assert buf.guards_intact(), f'{what}: buffer {j}: a store landed outside it'
        for k in range(world):
            blk = buf.t[k * B:(k + 1) * B]
            if k == r:
                assert exact(blk.cpu(), ref), f'{what}: buffer {j} (rank {r} of {world}): the gathered block differs'
            else:
                assert mc.n_unwritten(blk) == blk.numel(), f'{what}: buffer {j}: block {k} of rank {r} was written'


def group_of_two_kb(case):
    """A CSPN_B200_MAX_WS3D_KB under which the volumes of `case` run in launch groups of 2 (cspn3d.cu's group3d)."""
    Bi, Ci = case.dims[:2]
    planes = {'3d': 27, 'k3d': case.K ** 3, 'gates3d': 0}[case.family]
    per_vol = 4 * (planes + (Ci if case.N > 1 else 0)) * D * H * case.shape[4]
    return f'{2.5 * per_vol / 1024:.3f}'


FAMILIES = [('3d', 3, n) for n in (0, 1, 2)] + [('k3d', K, n) for K in (3, 5) for n in (0, 1, 2)] + \
           [('gates3d', K, 0) for K in (3, 5)]
FAMILY_IDS = [f'{f}-K{K}' + ('' if f == 'gates3d' else f'-norm{n}') for f, K, n in FAMILIES]

# route: (B, C, gates, W kind, workspace offset, CSPN_B200_3D_PADDLE=planes, launch groups of 2)
ROUTES = {
    'vec-C1': (2, 1, 'shared', 'vec', 0, False, False),
    'odd-C2': (2, 2, 'shared', 'odd', 0, False, False),
    'vec-per-channel': (2, 2, 'per_channel', 'vec', 0, False, False),
    'odd-per-channel': (2, 2, 'per_channel', 'odd', 0, False, False),
    'planes': (2, 2, 'shared', 'vec', 0, True, False),
    'ws-off4': (2, 2, 'shared', 'vec', 4, False, False),
    'groups-odd': (3, 2, 'shared', 'odd', 0, False, True),
    'groups-vec': (3, 1, 'shared', 'vec', 0, False, True),
}


@pytest.mark.parametrize('N', [1, 2, 5])
@pytest.mark.parametrize('family, K, norm, route',
                         [(*fam, r) for fam in FAMILIES for r in ROUTES if fam[1] == 3 or not ROUTES[r][5]],
                         ids=[f'{i}-{r}' for fam, i in zip(FAMILIES, FAMILY_IDS) for r in ROUTES
                              if fam[1] == 3 or not ROUTES[r][5]])   # CSPN_B200_3D_PADDLE acts on the 3x3x3 operator only
def test_gather_delivers_the_plain_forward_bits(family, K, norm, N, route, monkeypatch):
    B, C, gates, wkind, ws_off, planes, groups = ROUTES[route]
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    if planes:
        monkeypatch.setenv('CSPN_B200_3D_PADDLE', 'planes')
    case = Case(family, K, norm, N, B, C, W_OF[wkind], gates, seed=len(route))
    ref, launches = plain_forward(case, ws_off)
    if groups:
        monkeypatch.setenv('CSPN_B200_MAX_WS3D_KB', group_of_two_kb(case))
        single = launches
        case = Case(family, K, norm, N, B, C, W_OF[wkind], gates, seed=len(route))   # the workspace query sees the cap
        ref_g, launches = plain_forward(case, ws_off)
        assert exact(ref_g, ref)
        raw = family != 'gates3d' and K == 3 and wkind == 'vec'   # the raw-guidance route runs every volume in one launch
        if not raw and not (family == 'gates3d' and N == 1):      # one gates step needs no workspace: one group
            assert launches == 2 * single, (launches, single)     # two launch groups: 2 + 1 volumes
    for n_peer in (0, 1, 7):
        gather_world(case, n_peer, ws_off, ref, launches, f'{family} K={K} norm={norm} N={N} {route} n_peer={n_peer}')


@pytest.mark.parametrize('wkind', ['vec', 'odd'])
@pytest.mark.parametrize('family, K, norm', FAMILIES, ids=FAMILY_IDS)
def test_nan_and_inf_travel_bit_for_bit(family, K, norm, wkind, monkeypatch):
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    case = Case(family, K, norm, 2, 2, 2, W_OF[wkind], seed=0, special=True)
    ref, launches = plain_forward(case, 0)
    assert torch.isnan(ref).any() and not torch.isnan(ref).all()
    if family == 'gates3d':
        assert torch.isinf(ref).any()
    gather_world(case, 7, 0, ref, launches, f'{family} K={K} norm={norm} W={W_OF[wkind]} NaN / inf')


@pytest.mark.parametrize('family, K, norm', FAMILIES, ids=FAMILY_IDS)
def test_refusals_write_nothing(family, K, norm, monkeypatch):
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    case = Case(family, K, norm, 4, 1, 2, 16)
    cases = [
        (dict(peers=['ok'], n_peer=8), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok'], n_peer=-1), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=None, n_peer=2), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok', 'null']), ERR_INVALID, 'peer_out[1] is null or not 16-byte aligned'),
        (dict(peers=['off4', 'ok']), ERR_INVALID, 'peer_out[0] is null or not 16-byte aligned'),
        (dict(peers=['ok'], mc_off=4), ERR_INVALID, 'multicast_out is not 16-byte aligned'),
        (dict(peers=['ok'], N=0), ERR_UNSUPPORTED, 'prop_time >= 1'),
    ]
    if family != '3d':
        cases.append((dict(peers=['ok'], K=7), ERR_INVALID, 'kernel size must be 3 or 5'))
    if family != 'gates3d':
        cases.append((dict(peers=['ok'], norm=3), ERR_INVALID, 'unknown 3D norm_type 3'))
    for kw, want, msg in cases:
        out = mc.guarded(case.shape)
        bufs = [mc.guarded(case.shape) for _ in range(3)]
        ws = mc.workspace(case.ws_bytes)
        addr = {'ok': bufs[0].ptr(), 'null': None, 'off4': bufs[1].ptr() + 4}
        peers = None if kw['peers'] is None else [addr[p] for p in kw['peers']]
        mc_ptr = None if 'mc_off' not in kw else bufs[2].ptr() + kw['mc_off']
        saved = list(case.dims)
        if 'N' in kw:
            case.dims[case.n_index] = kw['N']
        if 'K' in kw:
            case.dims[5] = kw['K']
        if 'norm' in kw:
            case.dims[-1] = kw['norm']
        before = mc.snapshot(case.inputs())
        rc = case.gather(out.ptr(), peers, ws.ptr(), kw.get('n_peer'), mc_ptr)
        case.dims = saved
        torch.cuda.synchronize()
        assert rc == want and msg in _lib.lib().cspn_last_error().decode(), (kw, rc)
        assert out.untouched() and all(b.untouched() for b in bufs) and ws.untouched(), kw
        assert mc.unchanged(before, case.inputs())


# ---- FusedGather's 3D methods, with local buffers in place of the symmetric-memory rendezvous -----------------------------
class _LocalBarrier:
    def barrier(self):
        torch.cuda.synchronize()


def local_fused_gather(shape, world):
    """A FusedGather as rank world // 2 of `world`, its peers' gather buffers being guarded local buffers: what __init__
    takes from the rendezvous (buffer, block pointers, barrier) set by hand, everything after it the class's own code."""
    from cspn_b200.gather import FusedGather
    B = shape[0]
    r = world // 2
    bufs = [mc.guarded((world * B, *shape[1:])) for _ in range(world)]
    block = lambda j: bufs[j].t[r * B:(r + 1) * B].data_ptr()
    fg = FusedGather.__new__(FusedGather)
    fg.world, fg.rank, fg.shape, fg.block = world, r, tuple(shape), bufs[r].t[:B].numel()
    fg.buf, fg.hdl, fg.mode, fg.mc, fg._ws = bufs[r].t, _LocalBarrier(), 'peer_stores', 0, None
    fg.local = block(r)
    fg.peers = [block(j) for j in range(world) if j != r]
    fg._peer_arr = (ctypes.c_void_p * max(1, len(fg.peers)))(*fg.peers)
    return fg, bufs, r


@pytest.mark.parametrize('W', [16, 13])
def test_fused_gather_methods_deliver_their_module_functions(W, monkeypatch):
    import cspn_b200
    monkeypatch.delenv('CSPN_B200_MAX_WS3D_KB', raising=False)
    monkeypatch.delenv('CSPN_B200_3D_PADDLE', raising=False)
    B, C, N, world = 2, 2, 3, 3
    gen = torch.Generator().manual_seed(W)
    f = (torch.rand(B, C, D, H, W, generator=gen) * 10).cuda()
    g26 = torch.randn(B, 26, D, H, W, generator=gen).cuda()
    g26c = torch.randn(B, 26 * C, D, H, W, generator=gen).cuda()          # per-channel gates
    g124 = torch.randn(B, 124, D, H, W, generator=gen).cuda()
    g124c = torch.randn(B, 124 * C, D, H, W, generator=gen).cuda()
    gates5 = g124.abs() / g124.abs().sum(1, keepdim=True)
    gates3c = g26c.abs() / g26c.abs().view(B, C, 26, D, H, W).sum(2).repeat_interleave(26, 1)
    routes = [
        ('propagate3d 26sum_abs', lambda fg: fg.propagate3d(g26, f, N, '26sum_abs'),
         lambda: cspn_b200.propagate3d(g26, f, N, '26sum_abs')),
        ('propagate3d paddle per channel', lambda fg: fg.propagate3d(g26c, f, N, 'paddle'),
         lambda: cspn_b200.Affinity_Propagate3D(N, 3, 'paddle')(g26c, f)),
        ('propagate3d_k 5x5x5 paddle', lambda fg: fg.propagate3d_k(g124, f, 5, N, 'paddle'),
         lambda: cspn_b200.propagate3d_k(g124, f, 5, N, 'paddle')),
        ('propagate3d_k 5x5x5 124sum per channel', lambda fg: fg.propagate3d_k(g124c, f, 5, N, '124sum'),
         lambda: cspn_b200.Affinity_Propagate3DK(N, 5, '124sum')(g124c, f)),
        ('propagate3d_k 3x3x3 26sum', lambda fg: fg.propagate3d_k(g26, f, 3, N, '26sum'),
         lambda: cspn_b200.propagate3d_k(g26, f, 3, N, '26sum')),
        ('affinity_propagate3d 5x5x5', lambda fg: fg.affinity_propagate3d(f, gates5, 5, N),
         lambda: cspn_b200.affinity_propagate(f, gates5, 5, N)),
        ('affinity_propagate3d 3x3x3 per channel', lambda fg: fg.affinity_propagate3d(f, gates3c, 3, N),
         lambda: cspn_b200.affinity_propagate(f, gates3c, 3, N)),
    ]
    for name, fused, plain in routes:
        with torch.no_grad():
            ref = plain().cpu()
        fg, bufs, r = local_fused_gather((B, C, D, H, W), world)
        full = fused(fg)
        assert full.data_ptr() == bufs[r].t.data_ptr() and full.shape == (world * B, C, D, H, W), name
        for j, buf in enumerate(bufs):
            assert buf.guards_intact(), (name, j)
            for k in range(world):
                blk = buf.t[k * B:(k + 1) * B]
                if k == r:
                    assert exact(blk.cpu(), ref), (name, j)
                else:
                    assert mc.n_unwritten(blk) == blk.numel(), (name, j, k)
    fg, _, _ = local_fused_gather((B, C, D, H, W), world)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate3d(g26[:1], f[:1], N)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate3d_k(g124[:1], f[:1], 5, N, 'paddle')
    with pytest.raises(ValueError, match='built for'):
        fg.affinity_propagate3d(f[:1], gates5[:1], 5, N)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate_k(torch.randn(B, 24, H, W).cuda(), f[:, :, 0], None, 5, N)
