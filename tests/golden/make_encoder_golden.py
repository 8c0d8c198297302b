"""Encoder golden fixture: the UNMODIFIED reference pipeline (TRT_INT8 quantizer -> its own build_quant_pipeline pass list; CPU / torch path,
USING_CUDA_KERNEL = False) on a programmatically built one-block post-LN BERT encoder (tests/netspec_encoder.py), exactly as
make_graph_golden.py does for the CNN graphs.

    python tests/golden/make_encoder_golden.py        # rewrites tests/golden/graph_pipeline_encoder.npz

Stored, for kl, minmax, percentile and mse: every TensorQuantizationConfig's state / dominator / scale / offset right after
RuntimeCalibrationPass and after the last pass, the quantised graph's output on the first batch and the baked Gemm weights.  Weights and
token matrices are regenerated from seeds by tests/netspec_encoder.py.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import numpy as np
import torch

import netspec_encoder as enc
import refppq

METHODS = ('kl', 'minmax', 'percentile', 'mse')
PARAM_SEED, DATA_SEED, STEPS = 7, 11, 8
OUT = os.path.join(HERE, 'graph_pipeline_encoder.npz')


def generate(ppq):
    spec = enc.ENCODER
    params = enc.make_params(spec, PARAM_SEED)
    data = enc.make_data(DATA_SEED, STEPS)
    arrays = {}
    meta = dict(net='encoder', param_seed=PARAM_SEED, data_seed=DATA_SEED, steps=STEPS, batch=enc.B, seq=enc.S, hidden=enc.H, heads=enc.HEADS,
                ffn=enc.FFN, methods={})
    for method in METHODS:
        res = enc.run_reference_pipeline(ppq, spec, params, data, method)
        entry = {'passes': res['passes']}
        for stage in ('calibrated', 'final'):
            rows = []
            for i, row in enumerate(res[stage]):
                r = {k: row[k] for k in ('op', 'var', 'state', 'algo', 'dominator')}
                for k in ('scale', 'offset'):
                    if row[k] is not None:
                        key = f'{method}.{stage}.{i}.{k}'
                        arrays[key] = row[k].astype(np.float32)
                        r[k] = key
                rows.append(r)
            entry[stage] = rows
        arrays[f'{method}.output'] = res['output']
        for k, v in res['baked'].items(): arrays[f'{method}.baked.{k}'] = v
        meta['methods'][method] = entry
    arrays['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), 'bytes;', {m: sum(r['state'] == 'ACTIVATED' for r in meta['methods'][m]['calibrated']) for m in METHODS})


def main():
    ppq = refppq.load()
    assert ppq is not None and refppq.root() == '/root/reference', 'generate fixtures from the read-only reference checkout'
    from ppq.core import PPQ_CONFIG
    assert PPQ_CONFIG.USING_CUDA_KERNEL is False
    torch.set_num_threads(1)                                   # deterministic reductions
    generate(ppq)


if __name__ == '__main__':
    main()
