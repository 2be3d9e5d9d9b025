"""CPU tests of the fused gather of the K x K, 'paddle' and gates forwards (cspn2d_{k,paddle,gates}_fwd_gather_f32): the
ctypes signatures against the header, the argument errors the C ABI returns before it touches a device, the 2D-only
guard of FusedGather.affinity_propagate, and that the product package still does not import the oracle."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

from cspn_b200 import _lib
from cspn_b200.gather import FusedGather

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ('cspn2d_k_fwd_gather_f32', 'cspn2d_paddle_fwd_gather_f32', 'cspn2d_gates_fwd_gather_f32')
ERR_INVALID, ERR_UNSUPPORTED = -1, -4


def header_params(name):
    """The ctypes type of every parameter of `name` as include/cspn_b200.h declares it."""
    text = open(os.path.join(ROOT, 'include', 'cspn_b200.h')).read()
    m = re.search(r'CSPN_API\s+int\s+' + name + r'\s*\(([^)]*)\)', text)
    assert m, f'{name} is not declared'
    types = []
    for prm in m.group(1).split(','):
        prm = ' '.join(prm.split())
        if '*' in prm or prm.startswith('cspn_stream_t'):
            types.append(ctypes.c_void_p)
        elif prm.startswith('size_t'):
            types.append(ctypes.c_size_t)
        else:
            assert prm.startswith('int '), prm
            types.append(ctypes.c_int)
    return types


@pytest.mark.parametrize('name', ENTRIES)
def test_argtypes_match_the_header(name):
    res, args = _lib.SIGNATURES[name]
    assert res is ctypes.c_int and args == header_params(name)
    # the plain forward's parameters with peer_out, n_peer, multicast_out inserted after `out`
    plain = header_params(name.replace('_gather', ''))
    n_in = 4 if name.startswith('cspn2d_k_') else 3
    assert args == plain[:n_in] + [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p] + plain[n_in:]


def _buf():
    b = (ctypes.c_float * 64)()
    return b, ctypes.addressof(b)


def call(name, ptr, peers=(), n_peer=None, mc=None, K=5, iters=3, null_inputs=False, **shape):
    """One gather call on host addresses (never dereferenced: every case fails its checks first)."""
    dims = dict(B=1, C=1, H=4, W=8)
    dims.update(shape)
    arr = None if peers is None else (ctypes.c_void_p * max(len(peers), 1))(*peers)
    arr_p = None if arr is None else ctypes.cast(arr, ctypes.c_void_p)
    n = len(peers) if n_peer is None else n_peer
    inp = None if null_inputs else ptr
    L = _lib.lib()
    B, C, H, W = dims['B'], dims['C'], dims['H'], dims['W']
    if name == 'cspn2d_k_fwd_gather_f32':
        return L.cspn2d_k_fwd_gather_f32(inp, ptr, None, ptr, arr_p, n, mc, B, C, H, W, K * K - 1, K, iters, 0, None, 0, None)
    return getattr(L, name)(inp, ptr, ptr, arr_p, n, mc, B, C, H, W, K, iters, None, 0, None)


def last_error():
    return _lib.lib().cspn_last_error().decode()


@pytest.mark.parametrize('K', [3, 5, 7])
@pytest.mark.parametrize('name', ENTRIES)
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
        (dict(peers=[a16], K=4), ERR_INVALID, 'kernel size must be 3, 5 or 7'),
        (dict(peers=[a16], iters=-1), ERR_INVALID, '>= 0'),
        (dict(peers=[a16], W=0), ERR_INVALID, 'non-positive shape'),
    ]
    for kw, want, msg in cases:
        kw.setdefault('K', K)
        rc = call(name, a16, **kw)
        assert rc == want and msg in last_error(), (kw, rc, last_error())


def test_fused_gather_affinity_propagate_is_2d_only():
    fg = FusedGather.__new__(FusedGather)      # the 5-D check comes before anything that needs a process group
    fg.shape = (1, 2, 3, 6, 6)
    with pytest.raises(ValueError, match='2D only.*3D'):
        fg.affinity_propagate(torch.rand(1, 2, 3, 6, 6), torch.rand(1, 26, 3, 6, 6), 3, 2)


def test_gather_module_does_not_import_the_oracle():
    code = ('import sys, cspn_b200, cspn_b200.gather; '
            'bad = [m for m in sys.modules if m == "oracle" or m.startswith("oracle.")]; '
            'assert not bad, bad')
    subprocess.run([sys.executable, '-s', '-c', code], cwd=ROOT, check=True, env=dict(os.environ, PYTHONPATH=ROOT))
