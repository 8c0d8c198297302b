"""In-tree build of the native pieces (no JIT cache: the built .so files travel with the repo snapshot).

    python -m ppq_b200.build [--force] [--no-torch]

  ppq_b200/_lib/libppq_b200.so   C-ABI library (include/ppq_b200.h): hand-written sm_90a kernels, CUDA runtime only.
  ppq_b200/_C.so                 torch/pybind layer exporting the reference's 20 names (csrc/torch_binding.cc).

nvcc cross-compiles for sm_90a without a GPU.  Flags of record:
  -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false
(-fmad=false: every fused multiply-add in the kernels is written explicitly with __fmaf_rn; nothing else may contract,
 which is part of the bit-exactness contract with the reference.)
"""
import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, '_build')
LIBDIR = os.path.join(HERE, '_lib')
LIB = os.path.join(LIBDIR, 'libppq_b200.so')
EXT = os.path.join(HERE, '_C.so')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')

NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-fmad=false',
              '--expt-relaxed-constexpr', '--expt-extended-lambda',
              '-Xcompiler', '-fPIC,-fvisibility=hidden,-ffp-contract=off,-Wall', '-I', INCLUDE]
CU_SOURCES = ['fakequant.cu', 'fakequant_tma.cu', 'collectors.cu', 'search.cu', 'select.cu', 'train.cu', 'host.cc']
HEADERS = ['common.cuh', 'ops.cuh', 'half.cuh', 'variants.h', os.path.join(INCLUDE, 'ppq_b200.h')]


def _newest(paths):
    return max(os.path.getmtime(p if os.path.isabs(p) else os.path.join(CSRC, p)) for p in paths)


def _stamp(flags):
    return hashlib.sha1(' '.join(flags).encode()).hexdigest()[:12]


def build_lib(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    sources = [s for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    hdr_time = _newest(HEADERS)
    stamp = _stamp(NVCC_FLAGS)
    jobs = []
    objs = []
    for s in sources:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, f'{os.path.splitext(s)[0]}.{stamp}.o')
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_time):
            cmd = [NVCC] + NVCC_FLAGS + (['-x', 'cu'] if s.endswith('.cu') else []) + ['-c', src, '-o', obj]
            jobs.append(cmd)

    def run(cmd):
        if verbose:
            print(' '.join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + r.stdout + r.stderr)
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for out in ex.map(run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(o) for o in objs):
        # link under a temporary name, then rename: a copy of the tree taken meanwhile never sees a half-written library
        run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-shared', '-o', LIB + '.tmp'] + objs + ['-cudart', 'shared', '-Xlinker', '--no-undefined'])
        os.replace(LIB + '.tmp', LIB)
    return LIB


def build_ext(force=False, verbose=False):
    """The torch layer: one translation unit, g++ against the torch headers, linked to libppq_b200.so via $ORIGIN rpath."""
    import torch
    from torch.utils import cpp_extension
    src = os.path.join(CSRC, 'torch_binding.cc')
    if not force and os.path.exists(EXT) and os.path.getmtime(EXT) >= max(os.path.getmtime(src), os.path.getmtime(LIB),
                                                                         os.path.getmtime(os.path.join(INCLUDE, 'ppq_b200.h'))):
        return EXT
    inc = cpp_extension.include_paths(device_type='cuda') if 'device_type' in cpp_extension.include_paths.__code__.co_varnames \
        else cpp_extension.include_paths(cuda=True)
    torch_lib = os.path.join(os.path.dirname(torch.__file__), 'lib')
    cxx = os.environ.get('CXX', 'g++')
    cmd = [cxx, '-O2', '-std=c++17', '-fPIC', '-shared', '-fvisibility=hidden', '-DTORCH_EXTENSION_NAME=_C',
           '-DTORCH_API_INCLUDE_EXTENSION_H', f'-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}',
           '-I', INCLUDE, '-I', sysconfig.get_paths()['include'], '-I', '/usr/local/cuda/include']
    for p in inc:
        cmd += ['-isystem', p]
    cmd += [src, '-o', EXT + '.tmp', '-L', LIBDIR, '-lppq_b200', '-L', torch_lib, '-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch_cuda',
            '-ltorch', '-ltorch_python', '-L', '/usr/local/cuda/lib64', '-lcudart',
            '-Wl,-rpath,$ORIGIN/_lib', f'-Wl,-rpath,{torch_lib}']
    if verbose:
        print(' '.join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('g++ failed:\n' + ' '.join(cmd) + '\n' + r.stdout + r.stderr)
    os.replace(EXT + '.tmp', EXT)
    return EXT


def build_all(force=False, verbose=False, with_torch=True):
    lib = build_lib(force=force, verbose=verbose)
    ext = build_ext(force=force, verbose=verbose) if with_torch else None
    return lib, ext


if __name__ == '__main__':
    print(build_all(force='--force' in sys.argv, verbose=True, with_torch='--no-torch' not in sys.argv))
