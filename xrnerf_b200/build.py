"""Builds xrnerf_b200/lib/libxrnerf_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m xrnerf_b200.build [--force]

The .so is a build product (git-ignored). Sources: xrnerf_b200/csrc/*.cu.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libxrnerf_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC'] + os.environ.get('XRB_NVCC_DEFINES', '').split()   # e.g. -DXRB_FUSED_TIMERS (developer builds)


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ['../../include/xrnerf_b200.h']:
        with open(os.path.join(CSRC, f), 'rb') as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, '.stamp')
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB  # machine without a toolkit: use the library built earlier in this tree
        raise RuntimeError('nvcc not found and no prebuilt libxrnerf_b200.so')
    objs = []

    def compile_one(src):
        obj = os.path.join(LIBDIR, src[:-3] + '.o')
        cmd = [NVCC] + FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            print(' '.join(cmd), flush=True)
        subprocess.check_call(cmd)
        return obj
    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, _sources()))
    subprocess.check_call([NVCC, '-shared'] + ARCH + ['-o', LIB] + objs + ['-cudart', 'static'])
    for o in objs:
        os.remove(o)
    with open(stamp, 'w') as fh:
        fh.write(digest)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
