"""The reference's own CUDA kernels, as the GPU tests compare against them -- test infrastructure only.

The reference extension (upstream ppq/csrc, built unmodified by oracle/build_ref.py) is not part of this repository, so what its
kernels returned for the tests' seeded inputs is stored in tests/golden/ref_cuda_calls.json.gz, per test and per call: a digest of
the inputs and, per output, its exact bits when it is small (quantiles, scale gradients, losses) or a digest when it is large (those
are always compared bit for bit).  `reference(nodeid)` replays these records behind the reference's interface: a call runs our
extension's function of the same name (the two share the reference's table of names and argument orders), checks that the inputs
are the recorded ones, and returns the reference's recorded values, or our output where its digest equals the reference's.  Where it
does not, the output is poisoned (NaN / INT_MIN), so the test's own comparison fails.

    PPQ_RECORD_REFERENCE=<dir> pytest -m gpu tests     (with oracle/_ref/PPQ_Cuda_Impls_ref.so built)

calls the real extension instead and writes <dir>/ref_cuda_calls.json.gz.
"""
import atexit
import base64
import gzip
import hashlib
import importlib.util
import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_cuda_calls.json.gz')
REF_SO = os.path.join(ROOT, 'oracle', '_ref', 'PPQ_Cuda_Impls_ref.so')
SMALL = 1024                                  # outputs up to this many elements are stored as values (per-channel scale gradients)

_records = None
_recorded = {}


def _digest(v):
    h = hashlib.sha1()
    if isinstance(v, list) and any(isinstance(a, torch.Tensor) for a in v):
        h.update(''.join(_digest(a) for a in v).encode())
    elif isinstance(v, torch.Tensor):
        h.update(f'{v.dtype}{tuple(v.shape)}'.encode())
        h.update(v.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes())
    else:
        h.update(repr(v).encode())
    return h.hexdigest()[:20]


def _outputs(ret, args):
    rets = list(ret) if isinstance(ret, (tuple, list)) else [ret]
    return rets + [a for a in args if isinstance(a, torch.Tensor)]


def _record_of(v):
    if isinstance(v, torch.Tensor):
        r = {'d': _digest(v)}
        if v.numel() <= SMALL:
            r['v'] = base64.b64encode(v.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).decode()
        return r
    return {'d': _digest(v), 'py': v}


class _Recorder:
    def __init__(self, module, nodeid):
        self.module, self.calls = module, _recorded.setdefault(nodeid, [])

    def __getattr__(self, name):
        fn = getattr(self.module, name)

        def call(*args):
            entry = [name, _digest(list(args))]
            ret = fn(*args)
            entry.append([_record_of(v) for v in _outputs(ret, args)])
            self.calls.append(entry)
            return ret
        return call


def _poison(t):
    t.fill_(float('nan') if t.is_floating_point() else torch.iinfo(t.dtype).min)


class _Replay:
    def __init__(self, ext, nodeid):
        self.ext, self.nodeid, self.calls, self.k = ext, nodeid, _load().get(nodeid), 0
        assert self.calls is not None, f'no recorded reference calls for {nodeid} in {GOLDEN}'

    def __getattr__(self, name):
        fn = getattr(self.ext, name)

        def call(*args):
            assert self.k < len(self.calls), f'{self.nodeid}: more reference calls than recorded'
            rec_name, rec_in, rec_out = self.calls[self.k]
            self.k += 1
            assert rec_name == name and rec_in == _digest(list(args)), \
                f'{self.nodeid}: call {self.k - 1} ({name}) has other inputs than the recorded reference call ({rec_name})'
            ret = fn(*args)
            outs = _outputs(ret, args)
            assert len(outs) == len(rec_out)
            for i, (v, r) in enumerate(zip(outs, rec_out)):
                if not isinstance(v, torch.Tensor):
                    outs[i] = r['py']
                elif 'v' in r:
                    v.view(-1).copy_(torch.frombuffer(bytearray(base64.b64decode(r['v'])), dtype=v.dtype).to(v.device))
                elif _digest(v) != r['d']:
                    _poison(v)
            n_ret = len(outs) - sum(isinstance(a, torch.Tensor) for a in args)
            if isinstance(ret, (tuple, list)):
                return type(ret)(outs[:n_ret])
            return outs[0]
        return call


def _load():
    global _records
    if _records is None:
        with gzip.open(GOLDEN, 'rt') as f:
            _records = json.load(f)
    return _records


def _write(path):
    with gzip.open(os.path.join(path, 'ref_cuda_calls.json.gz'), 'wt') as f:
        json.dump(_recorded, f, sort_keys=True)


def reference(nodeid):
    """The reference's kernels for the test `nodeid`: the real build when recording, the recorded calls otherwise."""
    out_dir = os.environ.get('PPQ_RECORD_REFERENCE')
    if out_dir:
        spec = importlib.util.spec_from_file_location('PPQ_Cuda_Impls_ref', REF_SO)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        if not _recorded:
            os.makedirs(out_dir, exist_ok=True)
            atexit.register(_write, out_dir)
        return _Recorder(m, nodeid)
    from ppq_b200.ffi import extension
    return _Replay(extension(), nodeid)
