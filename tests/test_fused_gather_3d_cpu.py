"""CPU tests of the fused gather of the 3D forwards (cspn3d_{,k_,gates_}fwd_gather_f32): the ctypes signatures against the
header, the argument errors the C ABI returns before it touches a device, the 5-D buffer of FusedGather(..., D=...) and
the 2D methods' refusal of it, and that the gather module still does not import the oracle."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from cspn_b200 import _lib
from cspn_b200.gather import FusedGather

from test_fused_gather_k_cpu import header_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ('cspn3d_fwd_gather_f32', 'cspn3d_k_fwd_gather_f32', 'cspn3d_gates_fwd_gather_f32')
ERR_INVALID, ERR_UNSUPPORTED = -1, -4


@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    res, args = _lib.SIGNATURES[name]
    assert res is ctypes.c_int and args == header_params(name)
    # the plain forward's parameters with peer_out, n_peer, multicast_out inserted after `out`
    plain = header_params(name.replace('_gather', ''))
    assert args == plain[:3] + [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p] + plain[3:]


def _buf():
    b = (ctypes.c_float * 64)()
    return b, ctypes.addressof(b)


def call(name, ptr, peers=(), n_peer=None, mc=None, K=3, iters=3, norm=1, null_inputs=False, **shape):
    """One gather call on host addresses (never dereferenced: every case fails its checks first)."""
    dims = dict(B=1, C=1, D=2, H=4, W=8)
    dims.update(shape)
    arr = None if peers is None else (ctypes.c_void_p * max(len(peers), 1))(*peers)
    arr_p = None if arr is None else ctypes.cast(arr, ctypes.c_void_p)
    n = len(peers) if n_peer is None else n_peer
    inp = None if null_inputs else ptr
    L = _lib.lib()
    head = [inp, ptr, ptr, arr_p, n, mc, dims['B'], dims['C'], dims['D'], dims['H'], dims['W']]
    if name == 'cspn3d_fwd_gather_f32':
        return L.cspn3d_fwd_gather_f32(*head, iters, norm, None, 0, None)
    if name == 'cspn3d_k_fwd_gather_f32':
        return L.cspn3d_k_fwd_gather_f32(*head, K, iters, norm, None, 0, None)
    return L.cspn3d_gates_fwd_gather_f32(*head, K, iters, None, 0, None)


def last_error():
    return _lib.lib().cspn_last_error().decode()


@pytest.mark.parametrize('name, K', [(ENTRIES[0], 3)] + [(e, K) for e in ENTRIES[1:] for K in (3, 5)])
def test_argument_errors_before_any_device_work(name, K):
    keep, p = _buf()
    keep2, q = _buf()
    a16 = (p + 15) // 16 * 16          # 16-byte aligned addresses inside the buffers
    b16 = (q + 15) // 16 * 16
    cases = [
        (dict(peers=[a16], n_peer=8), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=[a16], n_peer=-1), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=None, n_peer=2), ERR_INVALID, 'n_peer must be 0..7'),
        (dict(peers=[a16, None]), ERR_INVALID, 'peer_out[1] is null or not 16-byte aligned'),
        (dict(peers=[b16 + 4, a16]), ERR_INVALID, 'peer_out[0] is null or not 16-byte aligned'),
        (dict(peers=[a16], mc=b16 + 4), ERR_INVALID, 'multicast_out is not 16-byte aligned'),
        (dict(peers=[a16], iters=0), ERR_UNSUPPORTED, 'prop_time >= 1'),
        (dict(peers=[a16], null_inputs=True), ERR_INVALID, 'null tensor pointer'),
        (dict(peers=[a16], iters=-1), ERR_INVALID, '>= 0'),
        (dict(peers=[a16], D=0), ERR_INVALID, 'non-positive shape'),
    ]
    if name != 'cspn3d_fwd_gather_f32':
        cases.append((dict(peers=[a16], K=7), ERR_INVALID, 'kernel size must be 3 or 5'))
    if name != 'cspn3d_gates_fwd_gather_f32':
        cases.append((dict(peers=[a16], norm=3), ERR_INVALID, 'unknown 3D norm_type 3'))
    for kw, want, msg in cases:
        kw.setdefault('K', K)
        rc = call(name, a16, **kw)
        assert rc == want and msg in last_error(), (kw, rc, last_error())


class _FakeSymm:
    """Stand-in for torch.distributed._symmetric_memory on the CPU: one rank, no multicast."""

    @staticmethod
    def empty(shape, dtype, device):
        return torch.empty(shape, dtype=dtype, device=device)

    @staticmethod
    def rendezvous(buf, group):
        class H:
            buffer_ptrs = [buf.data_ptr()]
            multicast_ptr = 0
            has_multicast_support = False
        return H()


@pytest.fixture
def one_rank_fused_gather(monkeypatch):
    """FusedGather's own __init__ on the CPU, as rank 0 of a world of 1 (no process group, no GPU)."""
    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm_mem
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 1)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: 0)
    monkeypatch.setattr(dist, 'group', type('G', (), {'WORLD': None}))
    monkeypatch.setattr(symm_mem, 'empty', _FakeSymm.empty)
    monkeypatch.setattr(symm_mem, 'rendezvous', _FakeSymm.rendezvous)
    return lambda *a, **kw: FusedGather(*a, device='cpu', **kw)


def test_init_builds_a_5d_buffer_with_depth_and_a_4d_one_without(one_rank_fused_gather):
    fg = one_rank_fused_gather(2, 3, 5, 8, D=4)
    assert fg.shape == (2, 3, 4, 5, 8) and fg.block == 2 * 3 * 4 * 5 * 8
    assert tuple(fg.buf.shape) == (2, 3, 4, 5, 8)
    fg2 = one_rank_fused_gather(2, 3, 5, 8)
    assert fg2.shape == (2, 3, 5, 8) and fg2.block == 2 * 3 * 5 * 8 and tuple(fg2.buf.shape) == (2, 3, 5, 8)


def test_2d_methods_reject_a_5d_buffer(one_rank_fused_gather):
    fg = one_rank_fused_gather(1, 2, 6, 8, D=3)
    # (propagate_k and propagate_paddle refuse CPU tensors before their shape check; the GPU tests cover them)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate(torch.rand(1, 8, 6, 8), torch.rand(1, 2, 6, 8), None, 2)
    with pytest.raises(ValueError, match='2D only.*3D'):
        fg.affinity_propagate(torch.rand(1, 2, 3, 6, 8), torch.rand(1, 26, 3, 6, 8), 3, 2)


def test_3d_methods_reject_other_shapes(one_rank_fused_gather):
    fg = one_rank_fused_gather(1, 2, 6, 8, D=3)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate3d(torch.rand(2, 26, 3, 6, 8), torch.rand(2, 2, 3, 6, 8), 2)
    with pytest.raises(ValueError, match='built for'):
        fg.propagate3d_k(torch.rand(1, 124, 4, 6, 8), torch.rand(1, 2, 4, 6, 8), 5, 2, 'paddle')
    with pytest.raises(ValueError, match=r'\(B,C,D,H,W\)'):
        fg.propagate3d(torch.rand(1, 8, 6, 8), torch.rand(1, 2, 6, 8), 2)
    with pytest.raises(ValueError, match='3D only'):
        fg.affinity_propagate3d(torch.rand(1, 2, 6, 8), torch.rand(1, 8, 6, 8), 3, 2)
    with pytest.raises(AssertionError):
        fg.propagate3d_k(torch.rand(1, 342, 3, 6, 8), torch.rand(1, 2, 3, 6, 8), 7, 2)


def test_gather_module_does_not_import_the_oracle():
    code = ('import sys, cspn_b200, cspn_b200.gather; '
            'bad = [m for m in sys.modules if m == "oracle" or m.startswith("oracle.")]; '
            'assert not bad, bad')
    subprocess.run([sys.executable, '-s', '-c', code], cwd=ROOT, check=True, env=dict(os.environ, PYTHONPATH=ROOT))
