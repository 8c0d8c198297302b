"""Every binding name that launches device work has a stream-contract case (tests/test_gpu_stream_contract.py), and every case names a binding
that is still exported.  A new entry point cannot land without the side-stream gate and the graph-replay checks."""
import os
import re

from conftest import ROOT

CSRC = os.path.join(ROOT, 'ppq_b200', 'csrc')


def exported_names():
    names = []
    for f in ('torch_binding.cc', 'torch_binding_more.inc'):
        names += re.findall(r'\bm\.def\(\s*"(\w+)"', open(os.path.join(CSRC, f)).read())
    assert len(names) == len(set(names)), 'a name is exported twice'
    return set(names)


def test_every_launching_binding_has_a_stream_case():
    import test_gpu_stream_contract as sc
    names = exported_names()
    assert sc.HOST_ONLY <= names, f'host-only names no longer exported: {sorted(sc.HOST_ONLY - names)}'
    launching = names - sc.HOST_ONLY
    missing = sorted(launching - set(sc.CASES))
    stale = sorted(set(sc.CASES) - launching)
    assert not missing, f'bindings without a stream-contract case: {missing}'
    assert not stale, f'stream-contract cases for names that are not exported (or are host-only): {stale}'
    for name in sorted(launching):
        print(f'{name}: {", ".join(sc.CASES[name])}')


def test_case_table_import_touches_no_cuda():
    """The table is built at import from plain Python: no tensor, stream or device query until a test runs a builder."""
    import torch
    import test_gpu_stream_contract as sc
    assert all(callable(fn) and (kn is None or (isinstance(kn[0], str) and isinstance(kn[1], int))) and isinstance(params, dict)
               for variants in sc.CASES.values() for fn, kn, params in variants.values())
    if not torch.cuda.is_available():
        assert not torch.cuda.is_initialized()
