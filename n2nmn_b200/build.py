"""Builds csrc/ into n2nmn_b200/lib/libn2nmn_b200.so with nvcc for sm_90a (in-tree, so the
binary travels to the GPU box with the repo snapshot). Also builds nothing else: the oracle is
pure numpy."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libn2nmn_b200.so')
SOURCES = ['capi.cu', 'seq2seq.cu', 'schedule.cpp', 'pool.cpp', 'util.cpp']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '--shared', '-x', 'cu', '-Xptxas', '-v']


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(os.path.dirname(HERE), 'include', 'n2nmn_b200.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    cmd = [NVCC] + FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ['-o', LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    with open(os.path.join(LIBDIR, 'build.log'), 'w') as f:
        f.write(' '.join(cmd) + '\n' + log)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + log[-6000:])
    if verbose:
        print(log)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
