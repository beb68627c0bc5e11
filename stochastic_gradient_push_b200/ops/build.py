"""
In-tree build of the sm_90a extension (no JIT cache: the .so must travel with
the source tree to the GPU box).

    python -m stochastic_gradient_push_b200.ops.build [--force] [--verbose]

nvcc compiles the kernels (no torch headers -> seconds), g++ compiles the
bindings against the torch headers, and both are linked into
``stochastic_gradient_push_b200/_C*.so``.  Works on a host without a GPU.
"""

from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
PKG = os.path.dirname(HERE)
OBJ_DIR = os.path.join(HERE, '_obj')
EXT_NAME = '_C'

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-lineinfo', '-O3', '-std=c++17', '--use_fast_math',
    '-Xcompiler', '-fPIC', '-Xptxas', '-v',
]
# --use_fast_math would turn the push-sum division into an approximate one;
# the kernels only multiply by explicit reciprocals, but keep IEEE division:
NVCC_FLAGS.remove('--use_fast_math')


def so_path() -> str:
    suffix = sysconfig.get_config_var('EXT_SUFFIX') or '.so'
    return os.path.join(PKG, EXT_NAME + suffix)


def _cuda_home() -> str:
    for cand in (os.environ.get('CUDA_HOME'), os.environ.get('CUDA_PATH'), '/usr/local/cuda'):
        if cand and os.path.exists(os.path.join(cand, 'bin', 'nvcc')):
            return cand
    raise RuntimeError('nvcc not found (set CUDA_HOME)')


def _sources():
    cu = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith('.cu')]
    cpp = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith('.cpp')]
    hdr = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))
           if f.endswith(('.cuh', '.h'))]
    return cu, cpp, hdr


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in paths:
        with open(p, 'rb') as f:
            h.update(f.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _run(cmd, verbose):
    if verbose:
        print(' '.join(cmd), flush=True)
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError('build step failed:\n%s\n%s' % (' '.join(cmd), res.stdout))
    return res.stdout


def build(force: bool = False, verbose: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    cu, cpp, hdr = _sources()
    stamp = os.path.join(OBJ_DIR, 'stamp.txt')
    digest = _digest(cu + cpp + hdr) + torch.__version__
    out = so_path()
    if (not force and os.path.exists(out) and os.path.exists(stamp)
            and open(stamp).read().strip() == digest):
        return out

    os.makedirs(OBJ_DIR, exist_ok=True)
    cuda = _cuda_home()
    nvcc = os.path.join(cuda, 'bin', 'nvcc')
    inc = ['-I' + p for p in ce.include_paths()] + [
        '-I' + os.path.join(cuda, 'include'), '-I' + CSRC,
        '-I' + sysconfig.get_paths()['include']]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx = os.environ.get('CXX', 'g++')

    # one compiler process per translation unit, all at once (the units are independent; the
    # torch-header-heavy bindings dominate, so the wall-clock is ~ the slowest unit)
    jobs = []
    for src in cu:
        obj = os.path.join(OBJ_DIR, os.path.basename(src) + '.o')
        jobs.append((obj, [nvcc] + NVCC_FLAGS + ['-I', CSRC, '-c', src, '-o', obj]))
    for src in cpp:
        obj = os.path.join(OBJ_DIR, os.path.basename(src) + '.o')
        jobs.append((obj, [cxx, '-O2', '-std=c++17', '-fPIC', '-DTORCH_EXTENSION_NAME=' + EXT_NAME,
                           '-DTORCH_API_INCLUDE_EXTENSION_H', '-D_GLIBCXX_USE_CXX11_ABI=%d' % abi,
                           '-Wno-deprecated-declarations'] + inc + ['-c', src, '-o', obj]))
    from concurrent.futures import ThreadPoolExecutor
    workers = max(1, min(len(jobs), os.cpu_count() or 1, int(os.environ.get('SGP_B200_BUILD_JOBS', '8'))))
    with ThreadPoolExecutor(max_workers=workers) as pool:
        outs = list(pool.map(lambda job: _run(job[1], verbose), jobs))    # re-raises the first failure
    objs = [obj for obj, _ in jobs]
    log = outs[:len(cu)]                                                  # ptxas -v output of the kernels

    torch_lib = os.path.join(os.path.dirname(torch.__file__), 'lib')
    link = [cxx, '-shared', '-o', out] + objs + [
        '-L' + torch_lib, '-L' + os.path.join(cuda, 'lib64'),
        '-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch_cuda', '-ltorch', '-ltorch_python',
        '-lcudart', '-Wl,-rpath,' + torch_lib, '-Wl,-rpath,' + os.path.join(cuda, 'lib64')]
    _run(link, verbose)
    with open(os.path.join(OBJ_DIR, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    with open(stamp, 'w') as f:
        f.write(digest)
    return out


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
