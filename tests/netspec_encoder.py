"""A one-block post-LN BERT encoder in the neutral spec format of tests/netspec.py, and its two builders:
  * the REFERENCE's BaseGraph with ONNX operator types (Gemm, Reshape, Transpose, MatMul, Softmax, Add, LayerNormalization, Gelu), and
  * a torch.nn.Module whose sub-modules are ppq_b200.executor's operator kinds (one module per operation, named like the spec),
so that the same weights and token matrices go through the unmodified reference pipeline and through ours.
Test infrastructure: imported by tests/ and tests/golden/make_encoder_golden.py only.

The block works on a token matrix [B*S, H]: Q, K, V from Gemm (1/sqrt(d) folded into the Q weights and bias, so no Mul), heads by Reshape /
Transpose, MatMul(Q, K^T) -> Softmax -> MatMul(., V), Transpose / Reshape back, output Gemm, Add residual, LayerNormalization, then Gemm ->
Gelu -> Gemm, Add residual, LayerNormalization.  The leading Reshape dimension is -1, so any number of sequences of length S fits.
"""
import numpy as np
import torch

import netspec

B, S, H, HEADS, FFN = 4, 8, 32, 4, 64


def encoder_spec(seq=S, hidden=H, heads=HEADS, ffn=FFN, prefix=''):
    d = hidden // heads
    p = prefix
    x = f'{p}x' if prefix else 'x'

    def gemm(name, src, cout, cin):
        return dict(op='Gemm', name=p + name, inputs=[src], out=f'{p}{name}.o', cout=cout, cin=cin)

    def op(kind, name, inputs, **kw):
        return dict(op=kind, name=p + name, inputs=[p + i if i != x else i for i in inputs], out=f'{p}{name}.o', **kw)

    return [
        gemm('q', x, hidden, hidden), gemm('k', x, hidden, hidden), gemm('v', x, hidden, hidden),
        op('Reshape', 'q_heads', ['q.o'], shape=[-1, seq, heads, d]), op('Transpose', 'q_t', ['q_heads.o'], perm=[0, 2, 1, 3]),
        op('Reshape', 'k_heads', ['k.o'], shape=[-1, seq, heads, d]), op('Transpose', 'k_t', ['k_heads.o'], perm=[0, 2, 3, 1]),
        op('Reshape', 'v_heads', ['v.o'], shape=[-1, seq, heads, d]), op('Transpose', 'v_t', ['v_heads.o'], perm=[0, 2, 1, 3]),
        op('MatMul', 'scores', ['q_t.o', 'k_t.o']),
        op('Softmax', 'probs', ['scores.o'], axis=-1),
        op('MatMul', 'context', ['probs.o', 'v_t.o']),
        op('Transpose', 'ctx_t', ['context.o'], perm=[0, 2, 1, 3]), op('Reshape', 'ctx_flat', ['ctx_t.o'], shape=[-1, hidden]),
        gemm('attn_out', p + 'ctx_flat.o', hidden, hidden),
        op('Add', 'res1', ['attn_out.o', x]),
        op('LayerNormalization', 'ln1', ['res1.o'], dim=hidden),
        gemm('ffn1', p + 'ln1.o', ffn, hidden),
        op('Gelu', 'gelu', ['ffn1.o']),
        gemm('ffn2', p + 'gelu.o', hidden, ffn),
        op('Add', 'res2', ['ffn2.o', 'ln1.o']),
        op('LayerNormalization', 'ln2', ['res2.o'], dim=hidden),
    ]


ENCODER = encoder_spec()


def make_params(spec, seed, heads=HEADS):
    """Gemm weights from netspec.make_params (same generator), the Q weights and bias times 1/sqrt(d) in fp32, LayerNorm gamma / beta near 1 / 0
    from a second seeded generator."""
    p = netspec.make_params(spec, seed)
    r = np.random.RandomState(seed + 1)
    for o in spec:
        if o['op'] == 'Gemm' and o['name'].endswith('q'):
            f = np.float32(1.0 / np.sqrt(o['cout'] // heads))
            p[o['name'] + '.w'] = p[o['name'] + '.w'] * f
            p[o['name'] + '.b'] = p[o['name'] + '.b'] * f
        elif o['op'] == 'LayerNormalization':
            p[o['name'] + '.gamma'] = (1.0 + 0.1 * r.standard_normal(o['dim'])).astype(np.float32)
            p[o['name'] + '.beta'] = (0.1 * r.standard_normal(o['dim'])).astype(np.float32)
    return p


def make_data(seed, steps, batch=B, seq=S, hidden=H):
    """`steps` token matrices [batch*seq, hidden], standard normal (embedding-like)."""
    r = np.random.RandomState(seed)
    return [r.standard_normal((batch * seq, hidden)).astype(np.float32) for _ in range(steps)]


# ------------------------------------------------------------------------------------------------ torch.nn.Module (our executor)
class EncoderNet(torch.nn.Module):
    """Executes the spec with one sub-module per operation, names = the spec's names."""

    def __init__(self, spec, params):
        super().__init__()
        from ppq_b200 import executor as E
        self.spec = spec
        for o in spec:
            kind = o['op']
            if kind == 'Gemm': m = netspec.RefGemm(o['cin'], o['cout'])
            elif kind == 'Reshape': m = E.Reshape(o['shape'])
            elif kind == 'Transpose': m = E.Transpose(o['perm'])
            elif kind == 'MatMul': m = E.MatMul()
            elif kind == 'Softmax': m = torch.nn.Softmax(dim=o['axis'])
            elif kind == 'Add': m = E.Add()
            elif kind == 'LayerNormalization': m = E.LayerNorm(o['dim'])
            elif kind == 'Gelu': m = torch.nn.GELU()
            else: raise NotImplementedError(kind)
            with torch.no_grad():
                if kind == 'Gemm':
                    m.weight.copy_(torch.from_numpy(params[o['name'] + '.w'])); m.bias.copy_(torch.from_numpy(params[o['name'] + '.b']))
                elif kind == 'LayerNormalization':
                    m.weight.copy_(torch.from_numpy(params[o['name'] + '.gamma'])); m.bias.copy_(torch.from_numpy(params[o['name'] + '.beta']))
            self.add_module(o['name'].replace('.', '_'), m)

    def forward(self, x):
        v = {self.spec[0]['inputs'][0]: x}
        for o in self.spec:
            v[o['out']] = getattr(self, o['name'].replace('.', '_'))(*[v[i] for i in o['inputs']])
        return v[self.spec[-1]['out']]


def stacked_encoder(layers, seq, hidden, heads, ffn, seed=0):
    """`layers` encoder blocks in a row (BERT-base shape with 12, 128, 768, 12, 3072): one module per operation, block l's names prefixed `l<l>.`."""
    spec = []
    for layer in range(layers):
        block = encoder_spec(seq, hidden, heads, ffn, prefix=f'l{layer}.')
        if layer:                                                          # block l reads block l-1's output
            src, prev = block[0]['inputs'][0], spec[-1]['out']
            for o in block: o['inputs'] = [prev if i == src else i for i in o['inputs']]
        spec += block
    return EncoderNet(spec, make_params(spec, seed, heads=heads))


# ------------------------------------------------------------------------------------------------ the reference's BaseGraph
def build_ppq_graph(ppq, spec, params):
    """The spec as a reference BaseGraph: Reshape's shape is an int64 parameter input (ONNX), LayerNormalization takes gamma and beta as
    parameter inputs 1 and 2, Softmax / Transpose / LayerNormalization carry axis / perm / epsilon attributes."""
    from ppq import BaseGraph, NetworkFramework
    g = BaseGraph(name='encoder', built_from=NetworkFramework.ONNX)
    var = {}

    def v(name, value=None):
        if name not in var:
            var[name] = g.create_variable(name=name, value=None if value is None else torch.from_numpy(value.copy()), is_parameter=value is not None)
        return var[name]

    for o in spec:
        ins, attrs = [v(i) for i in o['inputs']], {}
        if o['op'] == 'Gemm':
            ins += [v(o['name'] + '.w', params[o['name'] + '.w']), v(o['name'] + '.b', params[o['name'] + '.b'])]
            attrs = {'alpha': 1.0, 'beta': 1.0, 'transB': 1}
        elif o['op'] == 'Reshape':
            ins.append(v(o['name'] + '.shape', np.asarray(o['shape'], dtype=np.int64)))
        elif o['op'] == 'Transpose':
            attrs = {'perm': list(o['perm'])}
        elif o['op'] == 'Softmax':
            attrs = {'axis': o['axis']}
        elif o['op'] == 'LayerNormalization':
            ins += [v(o['name'] + '.gamma', params[o['name'] + '.gamma']), v(o['name'] + '.beta', params[o['name'] + '.beta'])]
            attrs = {'axis': -1, 'epsilon': 1e-5}
        g.create_operation(o['op'], name=o['name'], inputs=ins, outputs=[v(o['out'])], attributes=attrs)
    g.mark_variable_as_graph_input(var[spec[0]['inputs'][0]])
    g.mark_variable_as_graph_output(var[spec[-1]['out']])
    return g


def run_reference_pipeline(ppq, spec, params, data, method, **kw):
    """netspec.run_reference_pipeline (the TRT_INT8 quantizer and its own pass list, snapshots, output, baked Gemm weights) on the encoder graph."""
    saved = netspec.build_ppq_graph
    netspec.build_ppq_graph = build_ppq_graph
    try:
        return netspec.run_reference_pipeline(ppq, spec, params, data, method, **kw)
    finally:
        netspec.build_ppq_graph = saved
