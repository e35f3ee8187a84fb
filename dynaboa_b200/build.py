"""In-tree build of libdynaboa_b200.so (nvcc, sm_90a only) and of the CPU-side test helpers.

``python -m dynaboa_b200.build`` or ``__graft_entry__.build()``.  The shared object is written next to the
sources, so the package imports from the repository tree without an install step.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libdynaboa_b200.so')
HOSTMATH_LIB = os.path.join(HERE, 'libdboa_hostmath.so')
CUDA_SOURCES = ['conv.cu', 'conv_tc.cu', 'stem_wgrad.cu', 'groupnorm.cu', 'gn_fused.cu', 'norm_pool.cu', 'head.cu', 'smpl.cu', 'losses.cu', 'eval.cu', 'dataprocess.cu', 'optim.cu', 'hmr_plan.cu', 'render.cu', 'cabi.cu']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
              '--expt-relaxed-constexpr', '-Xptxas', '-v']


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a and link the shared library (parallel per file)."""
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.h', '.cuh'))]
    headers.append(os.path.join(HERE, '..', 'include', 'dynaboa_b200.h'))
    procs, objs = [], []
    for src in CUDA_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace('.cu', '.o'))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [NVCC] + NVCC_FLAGS + ['-c', s, '-o', o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append((src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f'nvcc failed on {src}')
        if verbose:
            print(out)
    if procs or force or _stale(LIB, objs):
        cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout)
            raise RuntimeError('link failed')
    with open(os.path.join(objdir, 'ptxas.log'), 'a') as f:
        for src, out in log:
            f.write(f'==== {src}\n{out}\n')
    return LIB


def build_hostmath(force=False):
    """CPU instantiation of csrc/rotmath.cuh for tests/test_hostmath.py (test infrastructure)."""
    src = os.path.join(CSRC, 'hostmath.cpp')
    if force or _stale(HOSTMATH_LIB, [src, os.path.join(CSRC, 'rotmath.cuh')]):
        subprocess.check_call(['g++', '-O2', '-shared', '-fPIC', '-o', HOSTMATH_LIB, src])
    return HOSTMATH_LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
    print(build_hostmath())
