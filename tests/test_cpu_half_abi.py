"""C ABI of the fp16 / bf16 entry points, checked without a device: the element-type codes, the descriptor sizes and the ABI version a
C99 client sees, and the refusal of an unknown element-type code before any launch."""
import ctypes
import os
import subprocess

import pytest

from conftest import ROOT

LIB = os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so')


@pytest.fixture(scope='module')
def built():
    from ppq_b200 import build
    build.build_all()
    return True


def test_c99_client_sees_codes_struct_sizes_and_abi_version(built, tmp_path):
    src = tmp_path / 'client.c'
    src.write_text('''
#include <stdio.h>
#include <stdint.h>
#include "ppq_b200.h"
int main(void) {
    printf("%d %d %d %d %d %d %d\\n", PPQ_B200_F32, PPQ_B200_F16, PPQ_B200_BF16, (int)sizeof(ppq_b200_tensor_desc),
           (int)sizeof(ppq_b200_lc_desc), (int)sizeof(ppq_b200_lt_desc), ppq_b200_abi_version());
    /* an unknown element type is refused before anything touches the (fake) pointers */
    if (ppq_b200_minmax_t_dt((const void *)16, 3, 8, (float *)16, 0) != 1) return 2;
    return 0;
}
''')
    exe = tmp_path / 'client'
    cc = subprocess.run(['gcc', '-std=c99', '-Wall', '-Wextra', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe),
                         '-L', os.path.dirname(LIB), '-lppq_b200', '-Wl,-rpath,' + os.path.dirname(LIB)], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)
    assert run.stdout.split() == ['0', '1', '2', '24', '56', '40', '2']


def test_unknown_dtype_codes_are_refused_before_a_launch(built):
    lib = ctypes.CDLL(LIB)
    V, I, L, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    p = V(16)                                                           # never dereferenced: the code is checked first
    calls = {
        'ppq_b200_linear_quant_t_dt': ([V, I, V, L, V, V, I, I, I, V], lambda c: (p, c, p, 8, p, p, -128, 127, 0, None)),
        'ppq_b200_linear_quant_c_dt': ([V, I, V, L, L, I, V, V, I, I, I, V], lambda c: (p, c, p, 8, 2, 4, p, p, -128, 127, 0, None)),
        'ppq_b200_linear_quant_t_toint_dt': ([V, I, V, I, L, V, V, I, I, I, V], lambda c: (p, c, p, 8, 8, p, p, -128, 127, 0, None)),
        'ppq_b200_linear_quant_c_toint_dt': ([V, I, V, I, L, L, I, V, V, I, I, I, V], lambda c: (p, c, p, 8, 8, 2, 4, p, p, -128, 127, 0, None)),
        'ppq_b200_float_quant_t_dt': ([V, I, V, L, V, V, I, I, F, F, I, V], lambda c: (p, c, p, 8, p, p, 4, 3, -448.0, 448.0, 0, None)),
        'ppq_b200_float_quant_c_dt': ([V, I, V, L, L, I, V, V, I, I, F, F, I, V], lambda c: (p, c, p, 8, 2, 4, p, p, 4, 3, -448.0, 448.0, 0, None)),
        'ppq_b200_minmax_t_dt': ([V, I, L, V, V], lambda c: (p, c, 8, p, None)),
        'ppq_b200_minmax_c_dt': ([V, I, L, L, I, V, V, V], lambda c: (p, c, 8, 2, 4, p, p, None)),
        'ppq_b200_histogram_asym_t_dt': ([V, I, L, F, F, I, V, L, V], lambda c: (p, c, 8, -1.0, 1.0, 1, p, 2048, None)),
        'ppq_b200_histogram_t_dscale_dt': ([V, I, L, V, I, V, L, V], lambda c: (p, c, 8, p, 1, p, 2048, None)),
        'ppq_b200_quantile_t_dt': ([V, I, L, F, V, V, V, V], lambda c: (p, c, 8, 0.99, p, p, None, None)),
    }
    for name, (argtypes, args) in calls.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, ctypes.c_int
        for code in (-1, 3, 4, 1 << 20):
            assert fn(*args(code)) == 1, (name, code)                   # cudaErrorInvalidValue
