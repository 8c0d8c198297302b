"""Layerwise-analysis golden fixture: the UNMODIFIED reference pipeline (TRT_INT8 quantizer and its own pass list, minmax calibration, CPU /
torch path) on tinyres and tinycat, then the reference's own layerwise_error_analyse (ppq/quantization/analyse/layerwise.py:15-134) on the
quantised graph for 'snr', 'mse' and 'cosine', with steps=8 over the 8 calibration batches and with steps=1 over the first three batches
(two batches measured: the reference breaks after the update of batch `steps`).

    python tests/golden/make_layerwise_golden.py          # rewrites tests/golden/layerwise_ref.npz

Stored: every TensorQuantizationConfig's state / dominator / scale / offset after the last pass (as make_graph_golden.py stores them) and,
per (net, method, steps), the operation names in the reference's order and their values.  Weights and data are regenerated from seeds by
tests/netspec.py.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import numpy as np
import torch

import netspec
import refppq

NETS = ('tinyres', 'tinycat')
PARAM_SEED, DATA_SEED, STEPS, BATCH = 7, 11, 8, 4
RUNS = [('snr', 8, 8), ('mse', 8, 8), ('cosine', 8, 8), ('snr', 1, 3), ('mse', 1, 3), ('cosine', 1, 3)]     # (method, steps, batches given)


def quantised_graph(ppq, spec, params, batches):
    """netspec.run_reference_pipeline's pass list with the 'minmax' setting, returning the graph."""
    import ppq.lib as PFL
    from ppq import TargetPlatform, TorchExecutor
    from ppq.api.setting import QuantizationSettingFactory
    graph = netspec.build_ppq_graph(ppq, spec, params)
    qz = PFL.Quantizer(platform=TargetPlatform.TRT_INT8, graph=graph)
    table = PFL.Dispatcher(graph=graph).dispatch(quant_types=qz.quant_operation_types)
    for op in list(graph.operations.values()):
        qz.quantize_operation(op_name=op.name, platform=table[op.name])
    ex = TorchExecutor(graph=graph, device='cpu')
    ex.tracing_operation_meta(inputs=batches[0])
    ex.load_graph(graph=graph)
    setting = QuantizationSettingFactory.default_setting()
    setting.quantize_activation_setting.calib_algorithm = 'minmax'
    for p in qz.build_quant_pipeline(setting):
        p.optimize(graph=graph, dataloader=batches, executor=ex, verbose=False, calib_steps=len(batches), collate_fn=None)
    return graph


def generate(ppq, net, arrays, meta):
    from ppq.quantization.analyse import layerwise_error_analyse
    spec = netspec.SPECS[net]
    params = netspec.make_params(spec, PARAM_SEED)
    batches = [torch.from_numpy(x) for x in netspec.make_data(net, DATA_SEED, STEPS, BATCH)]
    graph = quantised_graph(ppq, spec, params, batches)
    rows = []
    for i, row in enumerate(netspec.snapshot(graph)):
        r = {k: row[k] for k in ('op', 'var', 'state', 'algo', 'dominator')}
        for k in ('scale', 'offset'):
            if row[k] is not None:
                key = f'{net}.final.{i}.{k}'
                arrays[key] = row[k].astype(np.float32)
                r[k] = key
        rows.append(r)
    entry = {'final': rows, 'runs': []}
    for method, steps, given in RUNS:
        res = layerwise_error_analyse(graph=graph, dataloader=batches[:given], running_device='cpu', method=method, steps=steps, verbose=False)
        key = f'{net}.{method}.{steps}'
        arrays[key] = np.array(list(res.values()), dtype=np.float64)
        entry['runs'].append({'method': method, 'steps': steps, 'batches': given, 'ops': list(res), 'values': key})
    meta['nets'][net] = entry


def main():
    ppq = refppq.load()
    assert ppq is not None, 'generate fixtures from an unmodified reference checkout (PPQ_REFERENCE_ROOT)'
    from ppq.core import PPQ_CONFIG
    assert PPQ_CONFIG.USING_CUDA_KERNEL is False
    torch.set_num_threads(1)                                   # deterministic reductions
    arrays, meta = {}, dict(param_seed=PARAM_SEED, data_seed=DATA_SEED, steps=STEPS, batch=BATCH, calibration='minmax', nets={})
    for net in NETS: generate(ppq, net, arrays, meta)
    arrays['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    out = os.path.join(HERE, 'layerwise_ref.npz')
    np.savez_compressed(out, **arrays)
    print(out, os.path.getsize(out), 'bytes')


if __name__ == '__main__':
    main()
