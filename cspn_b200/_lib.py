"""ctypes binding of libcspn_b200.so (include/cspn_b200.h).  Fails loudly when the library is absent:
there is no CPU or eager-PyTorch fallback anywhere in this package."""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('CSPN_B200_LIB') or os.path.join(HERE, '_build', 'libcspn_b200.so')   # env: developer hook for tuning builds

OK = 0
ALGO_AUTO, ALGO_GENERIC, ALGO_CLUSTER = 0, 1, 2
ALGO_NAMES = {0: 'auto', 1: 'generic', 2: 'cluster'}
NORM2D = {'8sum': 0, '8sum_abs': 1}
NORM3D = {'26sum': 0, '26sum_abs': 1, 'paddle': 2}

_lib = None

# name -> (restype, argtypes); must list every symbol include/cspn_b200.h declares
_vp, _i, _sz, _cp = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p
SIGNATURES = {
    'cspn2d_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_fwd_f32': (_i, [_vp] * 4 + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn2d_fwd_f32_host': (_i, [_vp] * 4 + [_i] * 9),
    'cspn2d_fwd_gather_f32': (_i, [_vp] * 5 + [_i, _vp] + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn2d_bwd_workspace_bytes': (_sz, [_i] * 5),
    'cspn2d_bwd_f32': (_i, [_vp] * 6 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn2d_k_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_k_fwd_f32': (_i, [_vp] * 4 + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn2d_k_fwd_gather_f32': (_i, [_vp] * 5 + [_i, _vp] + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn2d_k_bwd_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_k_bwd_f32': (_i, [_vp] * 6 + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn2d_paddle_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_paddle_fwd_f32': (_i, [_vp] * 3 + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn2d_paddle_fwd_gather_f32': (_i, [_vp] * 4 + [_i, _vp] + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn2d_paddle_bwd_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_paddle_bwd_f32': (_i, [_vp] * 5 + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn2d_gates_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_gates_fwd_f32': (_i, [_vp] * 3 + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn2d_gates_fwd_gather_f32': (_i, [_vp] * 4 + [_i, _vp] + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn2d_gates_bwd_workspace_bytes': (_sz, [_i] * 6),
    'cspn2d_gates_bwd_f32': (_i, [_vp] * 5 + [_i] * 6 + [_vp, _sz, _vp]),
    'cspn3d_gates_workspace_bytes': (_sz, [_i] * 7),
    'cspn3d_gates_fwd_f32': (_i, [_vp] * 3 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_gates_fwd_gather_f32': (_i, [_vp] * 4 + [_i, _vp] + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_gates_bwd_workspace_bytes': (_sz, [_i] * 7),
    'cspn3d_gates_bwd_f32': (_i, [_vp] * 5 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_workspace_bytes': (_sz, [_i] * 6),
    'cspn3d_fwd_f32': (_i, [_vp] * 3 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_fwd_gather_f32': (_i, [_vp] * 4 + [_i, _vp] + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_fwd_f32_host': (_i, [_vp] * 3 + [_i] * 8),
    'cspn3d_bwd_workspace_bytes': (_sz, [_i] * 6),
    'cspn3d_bwd_f32': (_i, [_vp] * 5 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn3d_k_workspace_bytes': (_sz, [_i] * 7),
    'cspn3d_k_fwd_f32': (_i, [_vp] * 3 + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn3d_k_fwd_gather_f32': (_i, [_vp] * 4 + [_i, _vp] + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn3d_k_bwd_workspace_bytes': (_sz, [_i] * 7),
    'cspn3d_k_bwd_f32': (_i, [_vp] * 5 + [_i] * 8 + [_vp, _sz, _vp]),
    'cspn_depth_metrics_workspace_bytes': (_sz, []),
    'cspn_depth_metrics_f32': (_i, [_vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    'cspn_masked_l1_bwd_f32': (_i, [_vp] * 5 + [_sz, _vp]),
    'cspn_unpool_conv3x3_fwd_f32': (_i, [_vp] * 3 + [_i] * 7 + [_vp]),
    'cspn_unpool_conv3x3_bwd_workspace_bytes': (_sz, [_i] * 7),
    'cspn_unpool_conv3x3_bwd_f32': (_i, [_vp] * 5 + [_i] * 7 + [_vp, _sz, _vp]),
    'cspn_host_alloc': (_vp, [_sz]),
    'cspn_host_free': (None, [_vp]),
    'cspn_last_error': (_cp, []),
    'cspn_version': (_i, []),
    'cspn_last_algo': (_i, []),
    'cspn_last_launches': (_i, []),
    'cspn2d_describe_plan': (_i, [_i] * 6 + [_cp, _i]),
    'cspn2d_plan_json': (_i, [_i] * 3 + [_cp, _i]),
    'cspn2d_plan_json_chained': (_i, [_i] * 3 + [_cp, _i]),
}


class CspnError(RuntimeError):
    pass


def lib():
    """Loads (once) the in-tree shared library.  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise CspnError(
                f'{LIB_PATH} is missing: build it with `python -m cspn_b200.build` '
                '(cspn_b200 has no CPU / eager fallback by design)')
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc, what):
    if rc != OK:
        msg = lib().cspn_last_error().decode(errors='replace')
        if rc == -1:
            raise ValueError(f'{what}: {msg}')
        raise CspnError(f'{what} failed (status {rc}): {msg}')


def describe_plan(B, C, H, W, iters, algo=ALGO_AUTO):
    buf = ctypes.create_string_buffer(1024)
    lib().cspn2d_describe_plan(B, C, H, W, iters, algo, buf, len(buf))
    return buf.value.decode()


def plan_info(H, W, iters, chained=False):
    """The cluster path's plan for an HxW image and `iters` steps as a dict (see cspn2d_plan_json[_chained])."""
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    (lib().cspn2d_plan_json_chained if chained else lib().cspn2d_plan_json)(H, W, iters, buf, len(buf))
    return json.loads(buf.value.decode())
