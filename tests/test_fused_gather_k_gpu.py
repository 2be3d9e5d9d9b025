"""The fused gather of the K x K, 'paddle' and gates forwards (cspn2d_{k,paddle,gates}_fwd_gather_f32), run on one GPU.

As in tests/test_memory_contract_gpu.py, n_peer + 1 ranks are emulated on one GPU: slices of guarded local buffers
(tests/memory_contract.py) stand in for the other GPUs' gather buffers, since peer pointers are plain device addresses.
The call runs as the middle rank r.  Block r of every buffer must hold exactly the bits of the plain forward
(cspn2d_{k,paddle,gates}_fwd_f32 on the same inputs and an equally placed workspace); every other block and every guard
band must still hold the sentinel; the inputs keep their bits; the workspace has exactly the queried size and its guards
stay intact; cspn_last_launches() counts what the plain forward launches.  Bits are compared word for word, so a NaN
must arrive with its payload and can never be mistaken for the (NaN) sentinel.

The matrix: the three families x K in {3, 5, 7}; n_peer in {0, 1, 7}; N in {1, 2, 5} (both ping-pong parities, and N = 1
without an intermediate buffer); C = 1, C = 3 with one shared gate and, for 'paddle' and gates, C = 3 with per-channel
gates; W % 4 == 0 (the float4 step kernel) and odd W (the scalar one), and a workspace 4 bytes off a 16-byte boundary,
which also moves the call to the scalar kernel; CSPN_B200_KXK_GROUP = 1 and 2 with B = 3.  K = 3 of the K x K family
is the 3x3 operator's cluster-kernel gather, which refuses odd W.

FusedGather's methods run the same way, with local buffers set in place of what the rendezvous provides.  Out of scope
here: stores to a real NVLS multicast address and between GPUs, and the symmetric-memory rendezvous of several processes;
tools/gather_check.py --families runs those on a multi-GPU node.
"""
import ctypes

import pytest
import torch

from cspn_b200 import _lib

import memory_contract as mc

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -4
H = 12                  # H * W % 4 == 0 for any W: every rank's block starts 16-byte aligned
W_OF = {'vec': 64, 'odd': 37}


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


def exact(a, b):
    return a.shape == b.shape and torch.equal(mc.words(a), mc.words(b))


class Case:
    """Inputs of one family on the GPU and its plain and gathered forward calls."""

    def __init__(self, family, K, N, B, C, W, gates='shared', seed=0, special=False):
        gen = torch.Generator().manual_seed(seed * 1009 + K * 31 + N * 7 + B * C + W)
        nt = K * K - 1
        self.family, self.K, self.N = family, K, N
        self.shape = (B, C, H, W)
        feat = torch.rand(B, C, H, W, generator=gen) * 4 - 1
        s = None
        if family == 'k':
            gch = nt + (seed % 2)
            g = torch.randn(B, gch, H, W, generator=gen)
            if C > 1:
                s = torch.where(torch.rand(B, 1, H, W, generator=gen) < 0.3, torch.randn(B, 1, H, W, generator=gen),
                                torch.zeros(()))
            if special:                 # zero guidance around whole 7x7 neighbourhoods: 0/0 weights, NaN spreading from them
                g[:, :, 2:10, 4:14] = 0
        else:
            g = torch.randn(B, nt * C if gates == 'per_channel' else nt, H, W, generator=gen)
            if family == 'gates':
                g = g * (0.5 / nt)
            if special and family == 'paddle':
                g[:, :, 2:10, 4:14] = 0
            if special and family == 'gates':  # gates >= 0 keep the inf of image 1 from meeting a -inf (inf - inf = NaN)
                g = g.abs()
                g[0, 0, 5, 7] = float('nan')
                g[0, nt - 1, 0, 0] = float('inf')       # tap NT-1 reads (-R, -R): the padding at (0, 0), inf * 0
                feat[-1, -1, 7, 2] = float('inf')
        self.g, self.feat, self.s = [None if t is None else t.cuda().contiguous() for t in (g, feat, s)]
        L = _lib.lib()
        if family == 'k':
            self.norm = seed % 2
            self.dims = [B, C, H, W, gch, K, N, self.norm]
            self.ws_bytes = L.cspn2d_k_workspace_bytes(B, C, H, W, K, N)
        else:
            Bi, Ci = (B * C, 1) if gates == 'per_channel' else (B, C)
            self.dims = [Bi, Ci, H, W, K, N]
            self.ws_bytes = getattr(L, f'cspn2d_{family}_workspace_bytes')(Bi, Ci, H, W, K, N)

    def inputs(self):
        return [self.g, self.feat, self.s]

    def _head(self):
        return [ptr(self.g), ptr(self.feat)] + ([ptr(self.s)] if self.family == 'k' else [])

    def plain(self, out_ptr, ws_ptr):
        return getattr(_lib.lib(), f'cspn2d_{self.family}_fwd_f32')(*self._head(), out_ptr, *self.dims, ws_ptr,
                                                                   self.ws_bytes, stream())

    def gather(self, out_ptr, peers, ws_ptr, n_peer=None, mc_ptr=None):
        arr = None if peers is None else (ctypes.c_void_p * max(len(peers), 1))(*peers)
        return getattr(_lib.lib(), f'cspn2d_{self.family}_fwd_gather_f32')(
            *self._head(), out_ptr, None if arr is None else ctypes.cast(arr, ctypes.c_void_p),
            len(peers) if n_peer is None else n_peer, mc_ptr, *self.dims, ws_ptr, self.ws_bytes, stream())


def plain_forward(case, ws_off):
    """The plain forward into a guarded out: the bits the gather must deliver, and its launch count."""
    out, ws = mc.guarded(case.shape), mc.workspace(case.ws_bytes, ws_off)
    _lib.check(case.plain(out.ptr(), ws.ptr()), f'cspn2d_{case.family}_fwd_f32')
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
    _lib.check(case.gather(block(r), peers, ws.ptr()), f'cspn2d_{case.family}_fwd_gather_f32')
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


# (B, C, gates, CSPN_B200_KXK_GROUP, workspace offset)
VARIANTS = [
    (2, 1, 'shared', None, 0),
    (3, 3, 'shared', 2, 4),            # a group of 2 does not divide B = 3; a misaligned workspace
    (3, 3, 'per_channel', 1, 0),       # the K x K family has no per-channel guidance: C = 3 shared, signed norm, sparse
]


@pytest.mark.parametrize('wkind', ['vec', 'odd'])
@pytest.mark.parametrize('N', [1, 2, 5])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('family', ['k', 'paddle', 'gates'])
def test_gather_delivers_the_plain_forward_bits(family, K, N, wkind, monkeypatch):
    W = W_OF[wkind]
    for v, (B, C, gates, group, ws_off) in enumerate(VARIANTS):
        if group is None:
            monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
        else:
            monkeypatch.setenv('CSPN_B200_KXK_GROUP', str(group))
        case = Case(family, K, N, B, C, W, gates, seed=v)
        if family == 'k' and K == 3 and wkind == 'odd':
            continue                   # the cluster kernel's gather refuses odd W: test_3x3_gather_refuses_odd_w
        ref, launches = plain_forward(case, ws_off)
        for n_peer in (0, 1, 7):
            gather_world(case, n_peer, ws_off, ref, launches,
                         f'{family} K={K} N={N} W={W} B={B} C={C} {gates} group={group} ws+{ws_off} n_peer={n_peer}')


@pytest.mark.parametrize('wkind', ['vec', 'odd'])
@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('family', ['k', 'paddle', 'gates'])
def test_nan_and_inf_travel_bit_for_bit(family, K, wkind, monkeypatch):
    monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
    W = W_OF[wkind]
    if family == 'k' and K == 3 and wkind == 'odd':
        pytest.skip('the cluster kernel gather refuses odd W (test_3x3_gather_refuses_odd_w)')
    case = Case(family, K, 3, 2, 2, W, seed=0, special=True)
    ref, launches = plain_forward(case, 0)
    assert torch.isnan(ref).any() and not torch.isnan(ref).all()
    if family == 'gates':
        assert torch.isinf(ref).any()
    gather_world(case, 7, 0, ref, launches, f'{family} K={K} W={W} NaN / inf')


def test_3x3_gather_refuses_odd_w(monkeypatch):
    monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
    for norm_seed in (0, 1):
        case = Case('k', 3, 4, 1, 2, 37, seed=norm_seed)
        out, peer, ws = mc.guarded(case.shape), mc.guarded(case.shape), mc.workspace(case.ws_bytes)
        rc = case.gather(out.ptr(), [peer.ptr()], ws.ptr())
        torch.cuda.synchronize()
        assert rc == ERR_UNSUPPORTED and "cluster kernel's epilogue" in _lib.lib().cspn_last_error().decode()
        assert out.untouched() and peer.untouched() and ws.untouched()


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('family', ['k', 'paddle', 'gates'])
def test_refusals_write_nothing(family, K, monkeypatch):
    monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
    case = Case(family, K, 4, 1, 2, 64)
    cases = [
        (dict(peers=['ok'], n_peer=8), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok'], n_peer=-1), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=None, n_peer=2), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=['ok', 'null']), ERR_INVALID, 'peer_out[1] is null or not 16-byte aligned'),
        (dict(peers=['off4', 'ok']), ERR_INVALID, 'peer_out[0] is null or not 16-byte aligned'),
        (dict(peers=['ok'], mc_off=4), ERR_INVALID, 'multicast_out is not 16-byte aligned'),
        (dict(peers=['ok'], N=0), ERR_UNSUPPORTED, 'prop_time >= 1'),
    ]
    for kw, want, msg in cases:
        out = mc.guarded(case.shape)
        bufs = [mc.guarded(case.shape) for _ in range(3)]
        ws = mc.workspace(case.ws_bytes)
        addr = {'ok': bufs[0].ptr(), 'null': None, 'off4': bufs[1].ptr() + 4}
        peers = None if kw['peers'] is None else [addr[p] for p in kw['peers']]
        mc_ptr = None if 'mc_off' not in kw else bufs[2].ptr() + kw['mc_off']
        saved = list(case.dims)
        if 'N' in kw:
            case.dims[5 if family != 'k' else 6] = kw['N']
        before = mc.snapshot(case.inputs())
        rc = case.gather(out.ptr(), peers, ws.ptr(), kw.get('n_peer'), mc_ptr)
        case.dims = saved
        torch.cuda.synchronize()
        assert rc == want and msg in _lib.lib().cspn_last_error().decode(), (kw, rc)
        assert out.untouched() and all(b.untouched() for b in bufs) and ws.untouched(), kw
        assert mc.unchanged(before, case.inputs())


# ---- FusedGather's methods, with local buffers in place of the symmetric-memory rendezvous --------------------------------
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
    fg.world, fg.rank, fg.shape, fg.block = world, r, tuple(shape), B * shape[1] * shape[2] * shape[3]
    fg.buf, fg.hdl, fg.mode, fg.mc, fg._ws = bufs[r].t, _LocalBarrier(), 'peer_stores', 0, None
    fg.local = block(r)
    fg.peers = [block(j) for j in range(world) if j != r]
    fg._peer_arr = (ctypes.c_void_p * max(1, len(fg.peers)))(*fg.peers)
    return fg, bufs, r


@pytest.mark.parametrize('W', [64, 37])
def test_fused_gather_methods_deliver_their_module_functions(W, monkeypatch):
    import cspn_b200
    monkeypatch.delenv('CSPN_B200_KXK_GROUP', raising=False)
    B, C, N, world = 2, 3, 4, 3
    gen = torch.Generator().manual_seed(W)
    d = (torch.rand(B, C, H, W, generator=gen) * 10).cuda()
    s = torch.where(torch.rand(B, 1, H, W, generator=gen) < 0.2, torch.rand(B, 1, H, W, generator=gen), torch.zeros(())).cuda()
    g24 = torch.randn(B, 25, H, W, generator=gen).cuda()
    g8c = torch.randn(B, 8 * C, H, W, generator=gen).cuda()            # per-channel gates
    g48 = torch.randn(B, 48, H, W, generator=gen).cuda()
    gates = g48.abs() / g48.abs().sum(1, keepdim=True)
    routes = [
        ('propagate_k 5x5', lambda fg: fg.propagate_k(g24, d, s, 5, N, '24sum_abs'),
         lambda: cspn_b200.propagate2d_k(g24, d, s, 5, N, '24sum_abs')),
        ('propagate_paddle 3x3 per channel', lambda fg: fg.propagate_paddle(g8c, d, 3, N),
         lambda: cspn_b200.propagate2d_paddle(g8c, d, 3, N)),
        ('affinity_propagate 7x7', lambda fg: fg.affinity_propagate(d, gates, 7, N),
         lambda: cspn_b200.affinity_propagate(d, gates, 7, N)),
    ]
    if W % 4 == 0:
        routes.append(('propagate_k 3x3', lambda fg: fg.propagate_k(g24, d, s, 3, N),
                       lambda: cspn_b200.propagate2d_k(g24, d, s, 3, N)))
    for name, fused, plain in routes:
        ref = plain().cpu()
        fg, bufs, r = local_fused_gather((B, C, H, W), world)
        full = fused(fg)
        assert full.data_ptr() == bufs[r].t.data_ptr() and full.shape == (world * B, C, H, W), name
        for j, buf in enumerate(bufs):
            assert buf.guards_intact(), (name, j)
            for k in range(world):
                blk = buf.t[k * B:(k + 1) * B]
                if k == r:
                    assert exact(blk.cpu(), ref), (name, j)
                else:
                    assert mc.n_unwritten(blk) == blk.numel(), (name, j, k)
    fg, _, _ = local_fused_gather((B, C, H, W), world)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate_k(g24[:1], d[:1], s[:1], 5, N)
