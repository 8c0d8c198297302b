"""oracle/cpu_pipeline.py's CPU restatement of the reference pipeline, extended to transformer blocks -- TEST INFRASTRUCTURE.

CpuPipeline hooks the module kinds of the CNN graphs it is pinned on.  EncoderCpuPipeline also hooks the executor's opt-in transformer
modules and the activations a BERT block uses:
  * ppq_b200.executor.MatMul     -> 'MatMul'             (computing: two activation inputs, no weight config),
  * ppq_b200.executor.Reshape    -> 'Reshape'            (passive),
  * ppq_b200.executor.Transpose  -> 'Transpose'          (passive),
  * ppq_b200.executor.LayerNorm  -> 'LayerNormalization' (input 0 and output configs; gamma / beta FP32, so no weight config),
  * nn.GELU -> 'Gelu' (fuses with a preceding Gemm), nn.Softmax -> 'Softmax'.
The topology passes, observers, alignment and baking are CpuPipeline's, unchanged: they already know these kinds by name
(COMPUTING, PASSIVE, ACTIVATIONS).  The executor's modules are matched by class name and module, so the oracle never imports the product.

PINNED: tests/test_cpu_encoder_parity.py checks that it reproduces, bit for bit, what the UNMODIFIED reference pipeline produced on a
one-block post-LN BERT encoder (tests/golden/graph_pipeline_encoder.npz, tests/golden/make_encoder_golden.py).
"""
import torch

from oracle import cpu_pipeline

_EXECUTOR_KINDS = {'MatMul': 'MatMul', 'Reshape': 'Reshape', 'Transpose': 'Transpose', 'LayerNorm': 'LayerNormalization'}
_TORCH_KINDS = {torch.nn.GELU: 'Gelu', torch.nn.Softmax: 'Softmax'}


def encoder_kind(m):
    """The reference operator type of a module: the transformer kinds above first, then CpuPipeline's own table."""
    for t in type(m).__mro__:
        if t.__module__ == 'ppq_b200.executor' and t.__name__ in _EXECUTOR_KINDS: return _EXECUTOR_KINDS[t.__name__]
        if t in _TORCH_KINDS: return _TORCH_KINDS[t]
    return cpu_pipeline._kind(m)


class EncoderCpuPipeline(cpu_pipeline.CpuPipeline):
    def __init__(self, model, example, fuse_bn=False):
        # the modules only encoder_kind() knows get their hooks here; CpuPipeline.__init__ hooks the rest and traces the network
        for m in model.modules():
            if cpu_pipeline._kind(m) is None and encoder_kind(m) is not None:
                m.register_forward_pre_hook(self._pre); m.register_forward_hook(self._post)
        super().__init__(model, example, fuse_bn=fuse_bn)

    def _op(self, m, n_in=1):
        key = (id(m), self.calls.get(id(m), 0))
        if key not in self.by_call:
            op = cpu_pipeline.Op(f'{self.names[id(m)]}#{key[1]}', m, encoder_kind(m), n_in)
            self.by_call[key] = op; self.ops.append(op)
        return self.by_call[key]
