"""Build libnrgbd.so (in-tree) with nvcc for sm_90a.

    python -m neuralrgbd_b200.build [--force]

Every csrc/*.cu / *.cpp is compiled with
    nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3
into neuralrgbd_b200/_build/*.o and linked into neuralrgbd_b200/libnrgbd.so. nvcc
cross-compiles without a GPU; the .so is git-ignored but travels to the GPU box.
"""
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, '_build')
LIB = os.path.join(HERE, 'libnrgbd.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '-I', os.path.join(os.path.dirname(HERE), 'include'), '-I', CSRC]


def _newer(src, dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(p) > t for p in [src] + deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cpp')))
    hdrs = glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(CSRC, '*.h')) + \
        glob.glob(os.path.join(os.path.dirname(HERE), 'include', '*.h'))
    jobs = []
    objs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s) + '.o')
        objs.append(o)
        if force or _newer(s, o, hdrs):
            jobs.append([NVCC] + FLAGS + (['-x', 'cu'] if s.endswith('.cpp') else []) + ['-c', s, '-o', o])

    def run(cmd):
        if verbose:
            print(' '.join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed:\n%s\n%s' % (' '.join(cmd), r.stdout + r.stderr))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or not os.path.exists(LIB) or force:
        run([NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart'])
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
