"""In-tree build of libr3dp_b200.so (nvcc, sm_90a only).  `python -m real3dportrait_b200.build [--force]`.

The library is plain CUDA C++ behind a C ABI (include/r3dp_b200.h): no torch headers, no pybind.  nvcc cross-compiles
without a GPU, so the library can be built on a machine without one."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, 'csrc')
LIB_DIR = os.path.join(PKG, 'lib')
LIB = os.path.join(LIB_DIR, 'libr3dp_b200.so')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
    '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr',
]


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError('nvcc not found')


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(ROOT, 'include', '*.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu under csrc/ into lib/libr3dp_b200.so; returns the library path."""
    if not force and not _stale():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIB_DIR, os.path.basename(src)[:-3] + '.o')
        cmd = [_nvcc(), *NVCC_FLAGS, '-c', src, '-o', obj] + (['-Xptxas', '-v'] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{out}')
        if verbose and out:
            print(out)
    link = [_nvcc(), '-shared', '-o', LIB, *objs, '-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart_static', '-ldl', '-lrt', '-lpthread']
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'link failed:\n{r.stdout}')
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
