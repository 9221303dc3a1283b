"""Build libcouncil_b200.so in-tree with nvcc for sm_90a (no torch dependency, plain C ABI)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libcouncil_b200.so')
SOURCES = ['api.cu', 'conv_simt.cu', 'conv_tc.cu', 'norm.cu', 'pointwise.cu', 'losses.cu', 'head_fused.cu', 'conv_small.cu', 'augment.cu', 'vgg.cu', 'pad.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '--use_fast_math=false', '-Xcompiler', '-fPIC']


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return 'nvcc'


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'council_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every .cu into objects (parallel) and link the shared library."""
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if not f.startswith('--use_fast_math')]
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc] + flags + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, out))
        if verbose:
            print(out)
        objs.append(obj)
    cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
