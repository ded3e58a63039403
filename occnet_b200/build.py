"""Build libocc_b200.so in-tree with nvcc for sm_90a (H100; no torch headers, no JIT cache).

    python -m occnet_b200.build            # incremental
    python -m occnet_b200.build --force

The library is a plain C-ABI shared object (include/occ_b200.h), git-ignored.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'lib', 'obj')
LIB = os.path.join(HERE, 'lib', 'libocc_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
         '--expt-relaxed-constexpr', '--expt-extended-lambda', '-Xptxas', '-v']


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _newest_header():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hs.append(os.path.join(os.path.dirname(HERE), 'include', 'occ_b200.h'))
    return max(os.path.getmtime(h) for h in hs)


def _compile(src, force, log):
    obj = os.path.join(OBJ, src[:-3] + '.o')
    spath = os.path.join(CSRC, src)
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(spath), _newest_header()):
        return obj, False
    cmd = [NVCC] + FLAGS + ['-c', spath, '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(OBJ, src[:-3] + '.ptxas.log'), 'w') as f:
        f.write(r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f'nvcc failed for {src}:\n{r.stderr[-4000:]}')
    if log:
        print(f'[build] compiled {src}')
    return obj, True


def build(force=False, log=True):
    os.makedirs(OBJ, exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, force, log), srcs))
    objs = [r[0] for r in res]
    if force or any(r[1] for r in res) or not os.path.exists(LIB):
        cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n' + r.stderr[-4000:])
        if log:
            print(f'[build] linked {LIB}')
    return LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv)
