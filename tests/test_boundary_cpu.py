"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the header
declares, the nn.Module mirrors the reference's surface, and nothing silently falls back to a CPU path."""
import ctypes
import os
import re

import pytest
import torch

import cspn_b200
from cspn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, 'include', 'cspn_b200.h')).read()
    return sorted(set(re.findall(r'CSPN_API\s+[\w\s\*]+?\b(cspn\w+)\s*\(', text)))


def test_library_is_built_and_exports_every_declared_symbol():
    from cspn_b200 import build
    build.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(L, s), f'{s} declared in include/cspn_b200.h but not exported'
    assert sorted(_lib.SIGNATURES) == syms      # the Python binding covers the whole ABI


def test_abi_rejects_bad_arguments_without_a_gpu():
    L = _lib.lib()
    assert L.cspn_version() >= 100
    # null pointers / bad enums are caught before any CUDA call
    assert L.cspn2d_fwd_f32(None, None, None, None, 1, 1, 4, 4, 8, 1, 0, 0, None, 0, None) == -1
    assert b'null' in L.cspn_last_error()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert L.cspn2d_fwd_f32(p, p, None, p, 1, 1, 4, 4, 7, 1, 0, 0, None, 0, None) == -1       # < 8 guidance channels
    assert L.cspn2d_fwd_f32(p, p, None, p, 1, 1, 4, 4, 8, 1, 5, 0, None, 0, None) == -1       # unknown norm
    assert L.cspn2d_fwd_f32(p, p, None, p, 1, 1, 4, 4, 8, -1, 0, 0, None, 0, None) == -1      # negative iters
    assert L.cspn2d_workspace_bytes(2, 1, 10, 15, 3, _lib.ALGO_GENERIC) == 4 * (2 * 9 * 150 + 2 * 150)
    assert L.cspn3d_workspace_bytes(2, 1, 3, 4, 5, 2) == 2 * 4 * (27 * 60 + 60)   # both volumes form one launch group
    assert isinstance(cspn_b200.describe_plan(32, 1, 352, 1216, 24), str)


def test_module_surface_matches_reference():
    m = cspn_b200.Affinity_Propagate(24, 3, '8sum_abs')
    assert (m.prop_time, m.prop_kernel, m.norm_type, m.in_feature, m.out_feature) == (24, 3, '8sum_abs', 1, 1)
    assert list(m.parameters()) == [] and list(m.buffers()) == [] and m.state_dict() == {}
    with pytest.raises(AssertionError):
        cspn_b200.Affinity_Propagate(24, 5)                  # cspn.py:33
    with pytest.raises(AssertionError):
        cspn_b200.Affinity_Propagate(24, 3, '4sum')          # cspn.py:36
    # a checkpoint written by the reference carries an extra sum_conv.weight (SURVEY section 5): ignorable
    missing, unexpected = m.load_state_dict({'sum_conv.weight': torch.ones(1, 8, 1, 1, 1)}, strict=False)
    assert missing == [] and unexpected == ['sum_conv.weight']
    d = torch.rand(1, 1, 4, 4)
    assert cspn_b200.Affinity_Propagate(0, 3)(torch.randn(1, 8, 4, 4), d) is d    # prop_time=0 -> same tensor


def test_input_validation():
    m = cspn_b200.Affinity_Propagate(2, 3)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 8, 4, 4).double(), torch.rand(1, 1, 4, 4).double())       # fp32 only, like the reference
    with pytest.raises(ValueError):
        m(torch.randn(1, 7, 4, 4), torch.rand(1, 1, 4, 4))
    with pytest.raises(ValueError):
        m(torch.randn(1, 8, 4, 5), torch.rand(1, 1, 4, 4))
    with pytest.raises(ValueError):
        m(torch.randn(1, 8, 4, 4), torch.rand(1, 1, 4, 4), torch.rand(1, 2, 4, 4))


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU behaviour')
def test_no_silent_cpu_fallback():
    m = cspn_b200.Affinity_Propagate(2, 3)
    with pytest.raises(cspn_b200.CspnError):
        m(torch.randn(1, 8, 4, 4), torch.rand(1, 1, 4, 4))
    with pytest.raises(cspn_b200.CspnError):
        cspn_b200.Affinity_Propagate3D(2)(torch.rand(1, 26, 2, 4, 4), torch.rand(1, 1, 2, 4, 4))


def test_product_package_never_imports_the_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's baseline legs may touch oracle/."""
    pkg = os.path.join(ROOT, 'cspn_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(('.py', '.cu', '.cuh', '.h')):
                continue
            text = open(os.path.join(dirpath, f)).read()
            assert not re.search(r'^\s*(from|import)\s+oracle', text, re.M), f'{f} imports the oracle'
            assert 'libcspn_oracle' not in text and 'c_oracle' not in text, f'{f} loads the oracle library'


def test_c_consumer_of_the_abi_compiles_and_runs_without_a_gpu(tmp_path):
    """examples/c_abi_demo.c: a plain-C front-end (dlopen + the header) sees the same contract as the ctypes binding."""
    import shutil
    import subprocess
    cc = '/usr/bin/gcc' if os.path.isfile('/usr/bin/gcc') else shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / 'c_abi_demo')
    subprocess.check_call([cc, '-Wall', '-Werror', '-I', os.path.join(root, 'include'),
                           os.path.join(root, 'examples', 'c_abi_demo.c'), '-o', exe, '-ldl'])
    out = subprocess.run([exe, _lib.LIB_PATH], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'cluster: patch 3x4' in out.stdout and 'status -1' in out.stdout   # the H100 plan of the bench shape
