"""Build libp2s_b200.so in-tree with nvcc for sm_90a (H100) (no torch dependency, no JIT cache).

    python -m points2surf_b200.build            # incremental
    python -m points2surf_b200.build --force
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, 'build')
LIB = os.path.join(HERE, 'libp2s_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '--extended-lambda', '-Xptxas', '-v']


def _newer(src, dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(p) > t for p in [src] + deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh')]
    hdrs.append(os.path.join(os.path.dirname(HERE), 'include', 'p2s_b200.h'))
    jobs = []
    for s in srcs:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + '.o')
        if force or _newer(src, obj, hdrs):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC] + FLAGS + ['-c', src, '-o', obj], capture_output=True, text=True)
        with open(obj + '.log', 'w') as f:
            f.write(r.stdout + r.stderr)
        return src, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        for src, r in ex.map(compile_one, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError('nvcc failed on %s' % src)
    objs = [os.path.join(OBJ, s[:-3] + '.o') for s in srcs]
    if force or jobs or not os.path.exists(LIB):
        r = subprocess.run([NVCC, '-shared', '-o', LIB] + objs + ['-lcudart'], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError('link failed')
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
