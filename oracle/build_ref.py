"""Recipe: compile the *unmodified* reference hot-path sources, where they lie under
/root/reference, into oracle/_ref/ (git-ignored; travels to the GPU box with gpurun).

TEST INFRASTRUCTURE ONLY.  Nothing in ppq_b200/ may import or load anything built here.

Two artefacts:
  oracle/_ref/hist_mse_ref.so      g++ build of ppq/csrc/cpu/hist_mse.cc (pure C++, no torch) behind a
                                   3-line extern "C" shim (oracle/ref_shim_hist_mse.cc, ours).
  oracle/_ref/PPQ_Cuda_Impls_ref*.so
                                   the reference's own torch extension (export.cc + cuda/{linear,sort,train,
                                   floating}.cu + cpu/hist_mse.cc: exactly the source list of
                                   ppq/core/ffi.py:31-38) compiled for sm_90a with the local nvcc/torch.
                                   With PPQ_RECORD_REFERENCE set, the GPU tests call it and record what it returns
                                   (tests/refcuda.py, tests/golden/ref_cuda_calls.json.gz).

We do NOT run the reference's build system (its JIT writes into the read-only package dir); the
compile lines are ours (torch.utils.cpp_extension.load pointed at a writable build dir).
No reference source is copied into this repository.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('PPQ_REFERENCE_ROOT', '/root/reference')
OUT = os.path.join(HERE, '_ref')
CSRC = os.path.join(REF, 'ppq', 'csrc')


def have_reference() -> bool:
    return os.path.isfile(os.path.join(CSRC, 'export.cc'))


def build_hist_mse(force: bool = False) -> str:
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, 'hist_mse_ref.so')
    if os.path.exists(so) and not force:
        return so
    cmd = ['g++', '-O3', '-shared', '-fPIC', '-std=c++17',
           '-I', os.path.join(CSRC, 'cpu'),
           os.path.join(CSRC, 'cpu', 'hist_mse.cc'),
           os.path.join(HERE, 'ref_shim_hist_mse.cc'),
           '-o', so]
    subprocess.check_call(cmd)
    return so


def build_cuda_ext(force: bool = False) -> str:
    """~3 min (4 nvcc translation units that include torch/extension.h)."""
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, 'PPQ_Cuda_Impls_ref.so')
    if os.path.exists(so) and not force:
        return so
    os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0a'
    os.environ.setdefault('MAX_JOBS', '6')
    from torch.utils.cpp_extension import load
    load(name='PPQ_Cuda_Impls_ref',
         sources=[os.path.join(CSRC, 'export.cc'),
                  os.path.join(CSRC, 'cuda', 'linear.cu'),
                  os.path.join(CSRC, 'cuda', 'sort.cu'),
                  os.path.join(CSRC, 'cuda', 'train.cu'),
                  os.path.join(CSRC, 'cuda', 'floating.cu'),
                  os.path.join(CSRC, 'cpu', 'hist_mse.cc')],
         build_directory=OUT, with_cuda=True, extra_cflags=['-O3'],
         extra_cuda_cflags=['-lineinfo'], is_python_module=False, verbose=True)
    # drop the object files: only the shared object is used
    for f in os.listdir(OUT):
        if f.endswith('.o'):
            os.remove(os.path.join(OUT, f))
    return so


if __name__ == '__main__':
    if not have_reference():
        print('reference sources not present at', REF, '- nothing to build (prebuilt files are used as-is)')
        sys.exit(0)
    print(build_hist_mse(force='--force' in sys.argv))
    if '--no-cuda' not in sys.argv:
        print(build_cuda_ext(force='--force' in sys.argv))
