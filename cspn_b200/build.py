"""Build libcspn_b200.so (the C-ABI product library) in-tree with nvcc for sm_90a (H100).

    python -m cspn_b200.build [--force]

Output: cspn_b200/_build/libcspn_b200.so (a build product, kept out of git).
No torch headers are involved: the library is plain CUDA C++ behind include/cspn_b200.h.
"""
import glob
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT_DIR = os.path.join(HERE, '_build')
LIB = os.path.join(OUT_DIR, 'libcspn_b200.so')
STAMP = os.path.join(OUT_DIR, 'sources.sha256')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-std=c++17', '-lineinfo',
    '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden',
    '--expt-relaxed-constexpr',
]


def _nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError('nvcc not found')


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _digest():
    h = hashlib.sha256()
    for f in _sources() + sorted(glob.glob(os.path.join(CSRC, '*.cuh'))) + \
            [os.path.join(os.path.dirname(HERE), 'include', 'cspn_b200.h')]:
        h.update(f.encode())
        with open(f, 'rb') as fh:
            h.update(fh.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def up_to_date():
    return (os.path.isfile(LIB) and os.path.isfile(STAMP)
            and open(STAMP).read().strip() == _digest())


def build(force=False, verbose=False, defines=(), out=None):
    """Compiles every .cu under csrc/ (separately, in parallel) and links the shared library.

    `defines` / `out` build an experimental variant (e.g. -DCSPN_EARLY_PUBLISH) into another file, to be loaded with
    CSPN_B200_LIB=<out>; the product library and its stamp are not touched."""
    variant = bool(defines) or out is not None
    lib = os.path.abspath(out) if out else LIB
    obj_dir = os.path.join(os.path.dirname(lib), os.path.basename(lib) + '.obj') if variant else OUT_DIR
    if not variant and not force and up_to_date():
        return LIB
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = _nvcc()
    env = dict(os.environ)
    # the image exports CC=/opt/gcc/bin/gcc; nvcc wants the system g++ as host compiler
    ccbin = ['-ccbin', '/usr/bin/g++'] if os.path.isfile('/usr/bin/g++') else []
    procs = []
    objs = []
    for src in _sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [nvcc] + ccbin + NVCC_FLAGS + [f'-D{d}' for d in defines] + ['-Xptxas', '-v', '-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, env=env, text=True)))
    log = []
    for src, p in procs:
        out_text, _ = p.communicate()
        log.append(f'== {os.path.basename(src)}\n{out_text}')
        if p.returncode != 0:
            sys.stderr.write('\n'.join(log))
            raise RuntimeError(f'nvcc failed on {src}')
    with open(os.path.join(obj_dir, 'ptxas.log'), 'w') as fh:
        fh.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    link = [nvcc] + ccbin + ['-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', lib] + objs
    subprocess.check_call(link, env=env)
    if not variant:
        with open(STAMP, 'w') as fh:
            fh.write(_digest())
    return lib


TORCH_LIB = os.path.join(OUT_DIR, 'libcspn_b200_torch.so')
TORCH_STAMP = os.path.join(OUT_DIR, 'torch_op.sha256')


def _torch_digest():
    import torch
    h = hashlib.sha256()
    for f in (os.path.join(CSRC, 'torch_op.cpp'), os.path.join(os.path.dirname(HERE), 'include', 'cspn_b200.h')):
        with open(f, 'rb') as fh:
            h.update(fh.read())
    h.update(torch.__version__.encode())
    return h.hexdigest()


def build_torch_op(force=False):
    """Compiles csrc/torch_op.cpp (TORCH_LIBRARY registration, a shim over the C ABI) with the host compiler against
    this interpreter's torch headers and links it to libcspn_b200.so (found at run time through $ORIGIN).
    Output: cspn_b200/_build/libcspn_b200_torch.so, loaded with torch.ops.load_library by cspn_b200/torch_op.py."""
    build()
    if (not force and os.path.isfile(TORCH_LIB) and os.path.isfile(TORCH_STAMP)
            and open(TORCH_STAMP).read().strip() == _torch_digest()):   # dynamic link: a rebuilt libcspn_b200.so needs no relink
        return TORCH_LIB
    import torch
    from torch.utils import cpp_extension as ce
    cxx = '/usr/bin/g++' if os.path.isfile('/usr/bin/g++') else (shutil.which('g++') or 'g++')
    cuda_home = os.environ.get('CUDA_HOME') or '/usr/local/cuda'
    torch_lib = ce.library_paths()[0]
    cmd = [cxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden',
           f'-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}',
           os.path.join(CSRC, 'torch_op.cpp'), '-o', TORCH_LIB]
    cmd += [f'-I{d}' for d in ce.include_paths()] + [f'-I{os.path.join(cuda_home, "include")}']
    cmd += [f'-L{torch_lib}', '-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch', f'-L{OUT_DIR}', '-lcspn_b200',
            '-Wl,-rpath,$ORIGIN', f'-Wl,-rpath,{torch_lib}', '-Wl,--no-as-needed']
    env = dict(os.environ)
    env.pop('CC', None)
    env.pop('CXX', None)
    subprocess.check_call(cmd, env=env)
    with open(TORCH_STAMP, 'w') as fh:
        fh.write(_torch_digest())
    return TORCH_LIB


if __name__ == '__main__':
    import argparse
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--force', action='store_true')
    ap.add_argument('-v', dest='verbose', action='store_true')
    ap.add_argument('--define', action='append', default=[], help='extra -D for an experimental variant (repeatable)')
    ap.add_argument('--out', help='output .so of the variant (use with CSPN_B200_LIB)')
    ap.add_argument('--torch-op', action='store_true', help='also build the TORCH_LIBRARY shim (libcspn_b200_torch.so)')
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose, defines=tuple(a.define), out=a.out))
    if a.torch_op:
        print(build_torch_op(force=a.force))
