"""The half-precision descriptor tables, checked without a device: the four `_dt` table entries of the C ABI exist, refuse an unknown
element-type code before anything touches their pointers, and compile into a C99 client; the host side groups a mixed set of tensors
into one table per dtype without losing a slot."""
import ctypes
import os
import subprocess
from types import SimpleNamespace

import pytest
import torch

from conftest import ROOT

LIB = os.path.join(ROOT, 'ppq_b200', '_lib', 'libppq_b200.so')
V, I, L, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
P = V(16)                                                               # never dereferenced: the code is checked first
TABLE_ENTRIES = {
    'ppq_b200_multi_minmax_t_dt': ([V, I, L, I, V, V], lambda c: (P, 2, 8, c, P, None)),
    'ppq_b200_multi_histogram_t_dt': ([V, I, L, I, V, I, V, L, V], lambda c: (P, 2, 8, c, P, 1, P, 2048, None)),
    'ppq_b200_multi_quantile_t_dt': ([V, I, L, I, F, V, L, V, L, V, V], lambda c: (P, 2, 8, c, 0.99, P, 2, P, 1 << 16, None, None)),
    'ppq_b200_multi_linear_quant_c_dt': ([V, I, L, I, I, I, I, V], lambda c: (P, 2, 8, c, -128, 127, 0, None)),
}


@pytest.fixture(scope='module')
def lib():
    from ppq_b200 import build
    build.build_all()
    return ctypes.CDLL(LIB)


def test_table_entries_exist_and_refuse_unknown_dtype_codes_before_a_launch(lib):
    for name, (argtypes, args) in TABLE_ENTRIES.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, ctypes.c_int
        for code in (-1, 3, 4, 1 << 20):
            assert fn(*args(code)) == 1, (name, code)                   # cudaErrorInvalidValue


def test_c99_client_compiles_against_the_table_entries(lib, tmp_path):
    src = tmp_path / 'client.c'
    src.write_text('''
#include <stdint.h>
#include "ppq_b200.h"
int main(void) {
    const ppq_b200_tensor_desc *t = (const ppq_b200_tensor_desc *)16;
    const ppq_b200_lc_desc *w = (const ppq_b200_lc_desc *)16;
    /* the descriptors keep their layout: the element type is an argument of the call, not a field */
    if (sizeof(ppq_b200_tensor_desc) != 24 || sizeof(ppq_b200_lc_desc) != 56 || ppq_b200_abi_version() != 2) return 3;
    if (ppq_b200_multi_minmax_t_dt(t, 1, 8, 3, (float *)16, 0) != 1) return 4;
    if (ppq_b200_multi_histogram_t_dt(t, 1, 8, -1, (const float *)16, 1, (int32_t *)16, 2048, 0) != 1) return 5;
    if (ppq_b200_multi_quantile_t_dt(t, 1, 8, 4, 0.99f, (float *)16, 2, (void *)16, 65536, 0, 0) != 1) return 6;
    if (ppq_b200_multi_linear_quant_c_dt(w, 1, 8, 3, -128, 127, 0, 0) != 1) return 7;
    return 0;
}
''')
    exe = tmp_path / 'client'
    cc = subprocess.run(['gcc', '-std=c99', '-Wall', '-Wextra', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe),
                         '-L', os.path.dirname(LIB), '-lppq_b200', '-Wl,-rpath,' + os.path.dirname(LIB)], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)


def fake(dtype, ptr, n):
    return SimpleNamespace(dtype=dtype, data_ptr=lambda: ptr, numel=lambda: n)


def test_rows_are_grouped_by_dtype_with_their_slots_in_a_stable_order():
    from ppq_b200.calibration import descriptor_rows_by_dtype
    f32, f16, bf16 = torch.float32, torch.float16, torch.bfloat16
    tensors = [fake(bf16, 1000, 5), fake(f32, 2000, 6), fake(bf16, 3000, 7), fake(f16, 4000, 8), fake(f32, 5000, 9), fake(bf16, 1000, 5)]
    groups = descriptor_rows_by_dtype(tensors, [4, 0, 2, 9, 1, 4])
    assert list(groups) == [bf16, f32, f16]                             # in the order each dtype is first met
    assert groups[bf16] == ((1000, 5, 4), (3000, 7, 2), (1000, 5, 4))   # rows keep the order of the tensors; a repeated slot stays repeated
    assert groups[f32] == ((2000, 6, 0), (5000, 9, 1))
    assert groups[f16] == ((4000, 8, 9),)
    assert sorted(r[2] for rows in groups.values() for r in rows) == [0, 1, 2, 4, 4, 9]
    # one dtype: one group, i.e. one launch -- what an all-fp32 or an all-half forward gives
    assert list(descriptor_rows_by_dtype([tensors[0], tensors[2], tensors[5]], range(3))) == [bf16]
    # real tensors describe themselves the same way
    a, b = torch.zeros(3, dtype=bf16), torch.zeros(4)
    assert descriptor_rows_by_dtype([a, b], [1, 0]) == {bf16: ((a.data_ptr(), 3, 1),), f32: ((b.data_ptr(), 4, 0),)}
