"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/ppq_b200.h declares,
the torch extension loads and exports the reference's names, product code never touches oracle/, host logic agrees with the
reference's golden vectors.  No kernels are launched here."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, cases_of, load_golden

LIB = os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so')


@pytest.fixture(scope='module')
def built():
    from ppq_b200 import build
    build.build_all()
    return True


def declared_symbols():
    hdr = open(os.path.join(ROOT, 'include', 'ppq_b200.h')).read()
    return sorted(set(re.findall(r'PPQ_B200_API[^;(]*?\b(ppq_b200_\w+)\s*\(', hdr)))


def test_c_abi_exports_every_declared_symbol(built):
    syms = declared_symbols()
    assert len(syms) >= 20
    lib = ctypes.CDLL(LIB)
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing
    lib.ppq_b200_abi_version.restype = ctypes.c_int
    assert lib.ppq_b200_abi_version() >= 1
    lib.ppq_b200_error_string.restype = ctypes.c_char_p
    assert lib.ppq_b200_error_string(0) == b'success'
    # no torch / python symbols leak into the C ABI library
    deps = subprocess.run(['ldd', LIB], capture_output=True, text=True).stdout
    assert 'libtorch' not in deps and 'libpython' not in deps and 'libc10' not in deps


def test_header_is_plain_c_and_a_c_program_links(built, tmp_path):
    """The boundary is a C ABI: the header compiles as C99 and a C translation unit that only knows the header links against the
    library and runs its host-side entry points (no GPU needed: version, error strings, argument validation, host MSE loss)."""
    hdr = os.path.join(ROOT, 'include', 'ppq_b200.h')
    assert subprocess.run(['gcc', '-std=c99', '-Wall', '-Wextra', '-Werror', '-fsyntax-only', '-x', 'c', hdr]).returncode == 0
    src = tmp_path / 'client.c'
    src.write_text('''
#include <stdio.h>
#include <stdint.h>
#include "ppq_b200.h"
int main(void) {
    int64_t hist[8] = {5, 4, 3, 2, 1, 0, 0, 7};
    if (ppq_b200_abi_version() < 1) return 1;
    /* null pointers / empty tensors are rejected before any launch */
    if (ppq_b200_linear_quant_t(0, 0, 0, 0, 0, -128, 127, 0, 0) == 0) return 2;
    if (ppq_b200_histogram_t(0, 16, 1.0f, 1, 0, 4096, 0) == 0) return 3;
    printf("%s|%.9g\\n", ppq_b200_error_string(1), (double)ppq_b200_compute_mse_loss(hist, 8, 1, 2, 5));
    return 0;
}
''')
    exe = tmp_path / 'client'
    cc = subprocess.run(['gcc', '-std=c99', '-Wall', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe),
                         '-L', os.path.dirname(LIB), '-lppq_b200', '-Wl,-rpath,' + os.path.dirname(LIB)], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)
    msg, loss = run.stdout.strip().split('|')
    assert 'invalid' in msg.lower()
    from oracle import compute_mse_loss
    assert np.float32(float(loss)) == np.float32(compute_mse_loss([5, 4, 3, 2, 1, 0, 0, 7], 1, 2, 5))


def test_library_contains_sm90a_code_only(built):
    out = subprocess.run(['cuobjdump', '-lelf', LIB], capture_output=True, text=True).stdout
    archs = set(re.findall(r'sm_\d+a?', out))
    assert archs == {'sm_90a'}, archs


def test_extension_loads_and_exports_reference_names(built):
    from ppq_b200.ffi import CUDA, extension
    ext = extension()
    # the complete reference table (ppq/csrc/export.cc:9-33): 20 names
    table = ['Quantile_T', 'Histogram_T', 'Histogram_Asymmetric_T', 'Histogram_C', 'QuantizeTensor_LT', 'QuantizeTensor_LC',
             'QuantizeTensor_LT_B', 'QuantizeTensor_LC_B', 'QuantizeTensor_FT', 'QuantizeTensor_FC', 'QuantizeTensor_FT_B',
             'QuantizeTensor_FC_B', 'TensorClip_T', 'TensorClip_C', 'RoundingLoss_LT', 'RoundingLoss_LC', 'RoundingLoss_LT_B',
             'RoundingLoss_LC_B', 'Isotone_T', 'compute_mse_loss']
    assert len(table) == 20
    for name in table:
        assert hasattr(ext, name), name
    for name in ['LinearQuantize_T', 'LinearQuantize_C', 'Histogram_T', 'Histogram_Asymmetric_T', 'Histogram_C', 'Quantile',
                 'compute_mse_loss', 'FloatingQuantize_T', 'FloatingQuantize_C', 'LinearQuantize_T_B', 'LinearQuantize_C_B',
                 'TensorClip_T', 'TensorClip_C', 'RoundingLoss_LT', 'RoundingLoss_LC', 'RoundingLoss_LT_B', 'RoundingLoss_LC_B',
                 'FloatingQuantize_T_B', 'FloatingQuantize_C_B', 'Sync']:
        assert hasattr(CUDA, name), name


def test_host_compute_mse_loss_matches_reference_cpp(built):
    from ppq_b200.ffi import CUDA
    g = load_golden('mse_loss.npz')
    for h, (nb, start, step, end), want in zip(g['hists'], g['args'], g['vals']):
        assert np.float32(CUDA.compute_mse_loss(h[:nb].tolist(), int(start), int(step), int(end))) == want


def test_host_mse_search_matches_reference(built):
    """Host MSE grid search over the native compute_mse_loss: same (start, end) choice as the reference's CPU pipeline.
    (The golden run used the Python-double loss twin; the C++ fp32 loss ranks these candidates identically.)"""
    from ppq_b200.search import mse_search_host
    g = load_golden('hist_search.npz')
    for c in cases_of(g, 'mse_cases'):
        sym = c['sym']
        qmin, qmax = (-128, 127) if sym else (0, 255)
        s, o = mse_search_host(g[f"mse_hist{c['j']}"].tolist(), c['hist_scale'], c['vmin'], qmin, qmax, sym, False, 1e-8)
        assert np.float32(s) == np.float32(c['scale']) and float(o) == c['offset'], c


def test_cpu_tensors_fail_loudly(built):
    import torch
    from ppq_b200 import LinearQuantizationConfig, QuantizationStates
    from ppq_b200.qfunction import PPQuantFunction
    cfg = LinearQuantizationConfig()
    cfg.scale, cfg.offset, cfg.state = torch.tensor(0.1), torch.tensor(0.0), QuantizationStates.ACTIVATED
    with pytest.raises((PermissionError, RuntimeError)):
        PPQuantFunction(torch.zeros(8), cfg)
    cfg.state = QuantizationStates.INITIAL                     # not activated -> passthrough, like the reference
    x = torch.zeros(8)
    assert PPQuantFunction(x, cfg) is x


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'ppq_b200')
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.cc', '.h', '.inc')):
                src = open(os.path.join(dirpath, f), errors='ignore').read()
                if re.search(r'^\s*(from|import)\s+oracle\b', src, re.M) or 'libppq_oracle' in src or 'oracle/_ref' in src:
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders
