"""Executor: the slice of TorchExecutor that the hot path lives in (/root/reference/ppq/executor/torch.py:457-577, 610-652)
for a torch.nn.Module network -- no graph IR, no ONNX (neither is part of the path, SURVEY.md §8).

What is mirrored, with the reference's semantics (pinned against the unmodified reference pipeline on a programmatically built
BaseGraph: tests/golden/graph_pipeline.npz, tests/test_cpu_graph_parity.py, tests/test_gpu_graph_parity.py):
  * every quantable operation (a call site of a Conv2d / Linear / ReLU / pooling / Add / Flatten ... module) owns one
    TensorQuantizationConfig per tensor input, one for its weight and one for its output, with the TensorRT-INT8 policy of
    ppq/quantization/quantizer/TensorRTQuantizer.py:12-105: per-tensor symmetric INT8 activations ('percentile' by default),
    per-channel symmetric INT8 weights on axis 0 ('minmax'), bias FP32;
  * the topology passes that decide WHICH tensors are observed and quantised, in the reference's order
    (quantizer/base.py:249-350):  QuantizeFusionPass (optim/refine.py:91-306: computing op -> activation, passive operations,
    anything -> Relu/Clip) then QuantizeSimplifyPass (refine.py:17-88: an input config whose tensor was already quantised by the
    producer's output config with the same scheme is OVERLAPPED), on the union-find `dominated_by` links of the configs;
  * forward(inputs, hooks): for each operation call quantize_function on every input and parameter (weights are re-quantised
    on EVERY forward until baked: torch.py:516-518), run pre-forward hooks with (fp32, quantised) values, run the op, quantise
    the outputs, run post-forward hooks (torch.py:526-553).  Only ACTIVATED / PASSIVE configs quantise (core/quant.py:357-359);
  * ParameterQuantizePass (optim/parameters.py:172-215), QuantAlignmentPass for element-wise ops (refine.py:309-546, 'Align to
    Large' + force_overlap, the default setting: api/setting.py:251-256) and ParameterBakingPass (optim/baking.py:34-47,
    IR/quantize.py:98-111).
Conv / Gemm execution itself stays in torch (cuDNN / cuBLAS), as in the reference.

Functional calls inside a network (`out += identity`, torch.flatten) are invisible to module hooks.  A tensor that reaches an
operation without a visible producer gets its own INITIAL input config (what the reference does for an input coming from a
non-quantable operation), except: a view of a known tensor shares its producer's config (Reshape / Flatten / Transpose are
passive operations upstream), and a Relu / Clip fed by an invisible operation fuses with it (refine.py:293-306).  Use the
`Add` / `Concat` modules of this file when element-wise ops must be quantised and aligned like the reference's graph.

H100-native addition: `collect=True` makes the executor hand the observed fp32 tensors of a whole forward to an ArenaCalibrator
(one multi-tensor launch per phase) instead of firing one observer launch per tensor.
"""
from typing import Dict, List, Optional

import torch

from .core import LinearQuantizationConfig, QuantizationStates, TensorQuantizationConfig
from .qfunction import PPQuantFunction


class Add(torch.nn.Module):
    """Element-wise sum as a module, so that the executor sees it as the reference sees an ONNX `Add`."""

    def forward(self, a, b):
        return a + b


class Concat(torch.nn.Module):
    def __init__(self, dim: int = 1):
        super().__init__()
        self.dim = dim

    def forward(self, *tensors):
        return torch.cat(tensors, dim=self.dim)


_KINDS = {torch.nn.Conv2d: 'Conv', torch.nn.ConvTranspose2d: 'ConvTranspose', torch.nn.Linear: 'Gemm', torch.nn.ReLU: 'Relu',
          torch.nn.ReLU6: 'Clip', torch.nn.MaxPool2d: 'MaxPool', torch.nn.AdaptiveAvgPool2d: 'GlobalAveragePool',
          torch.nn.AvgPool2d: 'AveragePool', torch.nn.Flatten: 'Flatten', torch.nn.Sigmoid: 'Sigmoid', torch.nn.GELU: 'Gelu',
          torch.nn.Hardswish: 'HardSwish', torch.nn.Softmax: 'Softmax', torch.nn.LeakyReLU: 'LeakyRelu', Add: 'Add', Concat: 'Concat',
          # x * sigmoid(x) as ONE module: fuses with its convolution exactly like the Conv - Sigmoid - Mul pattern upstream (refine.py:210-239),
          # where only the Mul's output keeps a live config
          torch.nn.SiLU: 'Swish', torch.nn.Upsample: 'Resize'}


def kind_of(module: torch.nn.Module) -> Optional[str]:
    """The reference operator type a module stands for (exact type first, then base classes, so that a subclass of nn.Linear is a Gemm)."""
    for t in type(module).__mro__:
        if t in _KINDS: return _KINDS[t]
    return None


COMPUTING_OP = {'Conv', 'Gemm', 'ConvTranspose', 'MatMul'}                              # core/common.py:55
# core/common.py:51-53 -- as written upstream, where a missing comma makes 'Dropout' 'Slice' one string: neither is passive
PASSIVE_OPERATIONS = {'MaxPool', 'GlobalMaxPool', 'Reshape', 'Flatten', 'Identity', 'DropoutSlice', 'Pad', 'Split', 'Transpose',
                      'Interp', 'Squeeze', 'Unsqueeze'}
ACTIVATION_FUSION_TYPES = {'Relu', 'Clip', 'Swish', 'SoftPlus', 'Sigmoid', 'Gelu'}     # TensorRTQuantizer.py:103-104
ELEMENTWISE_ALIGNMENT_TYPES = {'Add', 'Sub', 'Sum'}                                     # core/common.py:60-63
OUTPUT_ALIGNMENT_TYPES = {'Concat', 'Resize'}                                           # align_concat_to / align_resize_to: "Align to Output" 


def fuse_conv_bn(model: torch.nn.Module) -> torch.nn.Module:
    """PPQ folds BatchNorm into the preceding convolution when it loads a graph (core/common.py:41 FORMATTER_FUSE_BN)."""
    from torch.nn.utils.fusion import fuse_conv_bn_eval
    model.eval()

    def walk(mod):
        prev_name, prev = None, None
        for name, child in list(mod.named_children()):
            if isinstance(child, torch.nn.BatchNorm2d) and isinstance(prev, torch.nn.Conv2d):
                setattr(mod, prev_name, fuse_conv_bn_eval(prev, child))
                setattr(mod, name, torch.nn.Identity())
                prev_name, prev = None, None
                continue
            walk(child)
            prev_name, prev = name, child
    walk(model)
    return model


class QuantableOperation:
    """One call site of a quantable module.  `input_configs()` / `output_configs()` are what OperationObserver walks
    (observer/__init__.py:92-113).  `sources[i]` is the operation that produced tensor input i (None: graph input or invisible)."""

    def __init__(self, name: str, module: torch.nn.Module, kind: str, num_inputs: int):
        self.name, self.module, self.kind = name, module, kind
        act = dict(symmetrical=True, quant_min=-128, quant_max=127, calibration='percentile')
        self.input_cfgs: List[TensorQuantizationConfig] = [LinearQuantizationConfig(**act) for _ in range(num_inputs)]
        self.sources: List[Optional['QuantableOperation']] = [None] * num_inputs
        self.invisible_source: List[bool] = [False] * num_inputs       # the tensor was modified in place after its producer ran
        self.weight_cfg: Optional[TensorQuantizationConfig] = None
        if kind in ('Conv', 'Gemm', 'ConvTranspose'):
            self.weight_cfg = LinearQuantizationConfig(symmetrical=True, quant_min=-128, quant_max=127, calibration='minmax',
                                                       channel_axis=1 if kind == 'ConvTranspose' else 0)
        self.output_cfg: TensorQuantizationConfig = LinearQuantizationConfig(**act)
        self.consumers: List[tuple] = []                               # (operation, input index)
        self.stored_weight: Optional[torch.Tensor] = None              # QuantableVariable.stored_value: the fp32 weight behind a baked one

    @property
    def input_cfg(self) -> Optional[TensorQuantizationConfig]:
        return self.input_cfgs[0] if self.input_cfgs else None

    def input_configs(self):
        for i, c in enumerate(self.input_cfgs): yield (f'{self.name}:in{i}', c, False)
        if self.weight_cfg is not None: yield (self.name + ':weight', self.weight_cfg, True)

    def output_configs(self):
        yield (self.name + ':out', self.output_cfg)


class TorchExecutor:
    def __init__(self, model: torch.nn.Module, example_input: torch.Tensor, fuse_bn: bool = True, channels_last: bool = False):
        """channels_last=True runs the torch network in NHWC (cuDNN's native tensor-core layout).  The hot path does not care: per-tensor
        collectors and fake-quant are order-independent and read dense tensors in storage order; axis-0 weight rows stay contiguous."""
        self.model = fuse_conv_bn(model) if fuse_bn else model.eval()
        self._channels_last = channels_last
        if channels_last:
            self.model = self.model.to(memory_format=torch.channels_last)
            if example_input.dim() == 4: example_input = example_input.contiguous(memory_format=torch.channels_last)
        self.operations: Dict[str, QuantableOperation] = {}
        self._order: List[str] = []
        self._calls: Dict[int, int] = {}
        self._names = {id(m): n for n, m in self.model.named_modules()}
        self._hooks, self._collect, self._collected, self._sink = None, False, None, None
        self._tracing, self._wq, self._swapped, self._bypass = True, {}, {}, False
        self._mw = {}                                                    # weight dtype -> (signature, MultiWeightQuantizer, module ids)
        self._dequantized = None                                       # [(config, stored state)] while dequantize() is in effect
        self._only = None                                              # the operation quantize_only() runs quantised
        self._produced = {}                                            # id(tensor) -> (operation, tensor, version at production)
        self._quant_fn = PPQuantFunction
        for m in self.model.modules():
            if kind_of(m) is not None:
                m.register_forward_pre_hook(self._pre)
                m.register_forward_hook(self._post)
        with torch.no_grad():
            self._begin()
            self.model(example_input)
        self._tracing = False
        self._produced = {}
        self._fusion_pass()
        self._simplify_pass()

    # -- graph view used by the calibration pass
    def quantable_operations(self):
        return [(n, self.operations[n]) for n in self._order]

    def quantize_function(self, tensor: torch.Tensor, config: Optional[TensorQuantizationConfig]) -> torch.Tensor:
        """torch.py:610-613."""
        if config is None or not QuantizationStates.is_activated(config.state): return tensor
        return self._quant_fn(tensor, config)

    # -- QuantizeFusionPass + QuantizeSimplifyPass on the traced topology ---------------------------------------------------------
    def _upstream(self, op: QuantableOperation):
        return [s for s in op.sources if s is not None]

    def _fuse_into_activation(self, producer: QuantableOperation, act: QuantableOperation):
        if len(producer.consumers) == 1 and len(self._upstream(act)) == 1:                     # refine.py:203-208, 301-306
            producer.output_cfg.dominated_by = act.output_cfg
            act.input_cfgs[0].dominated_by = act.output_cfg

    def _fusion_pass(self):
        ops = [self.operations[n] for n in self._order]
        for op in ops:                                                  # computing op -> activation (refine.py:186-208)
            if op.kind in COMPUTING_OP:
                for act, idx in op.consumers:
                    if act.kind in ACTIVATION_FUSION_TYPES and idx == 0: self._fuse_into_activation(op, act)
        for op in ops:                                                  # passive operations share their first input's config (:278-291)
            if op.kind in PASSIVE_OPERATIONS and op.input_cfgs and op.sources[0] is not None:
                op.output_cfg.dominated_by = op.input_cfgs[0]
        for op in ops:                                                  # anything -> Relu / Clip (:293-306)
            for act, idx in op.consumers:
                if act.kind in ('Relu', 'Clip') and idx == 0: self._fuse_into_activation(op, act)
        for op in ops:                                                  # Relu / Clip fed by an invisible (functional / in-place) operation
            if op.kind in ('Relu', 'Clip') and op.input_cfgs and op.sources[0] is None and op.invisible_source[0]:
                op.input_cfgs[0].dominated_by = op.output_cfg

    def _simplify_pass(self):
        for n in self._order:                                           # refine.py:64-88
            src = self.operations[n]
            if src.output_cfg.state == QuantizationStates.FP32: continue
            for dst, idx in src.consumers:
                cfg = dst.input_cfgs[idx]
                if cfg.state == QuantizationStates.INITIAL and cfg.is_same_scheme(src.output_cfg):
                    cfg.dominated_by = src.output_cfg

    # -- forward -----------------------------------------------------------------------------------------------------------------
    def _begin(self):
        self._calls.clear()
        self._collected = []
        self._restore_weights()
        self._wq = self._quantize_all_weights() if not self._tracing else {}

    def _restore_weights(self):
        """An operation that raised between its pre- and post-hook leaves the fake-quantised buffer in module.weight: put the fp32 data back."""
        for module, fp32 in list(self._swapped.items()): module.weight.data = fp32
        self._swapped.clear()

    def _quantize_all_weights(self):
        """All activated per-channel linear weight configs that share (axis, range, rounding) are fake-quantised by ONE multi-tensor launch
        at the start of the forward (the per-module results are what the pre-forward hooks hand to the operations) -- one table, and one
        launch, per weight dtype present (fp32, fp16, bf16).  Falls back to one launch per weight for anything else (FP8 weights, mixed
        policies)."""
        from .calibration import TABLE_DTYPES, MultiWeightQuantizer
        from .core import QuantizationProperty as P
        ops = [self.operations[n] for n in self._order]
        tabled = [op for op in ops if op.weight_cfg is not None and QuantizationStates.is_activated(op.weight_cfg.state)
                  and op.weight_cfg.policy.has_property(P.LINEAR) and op.weight_cfg.policy.has_property(P.PER_CHANNEL)
                  and not op.weight_cfg.policy.has_property(P.DYNAMIC) and self._quant_fn is PPQuantFunction]
        out = {}
        for dtype in TABLE_DTYPES:
            todo = [op for op in tabled if op.module.weight.dtype == dtype]
            if len(todo) < 2: continue
            c0 = todo[0].weight_cfg
            key0 = (c0.channel_axis, c0.quant_min, c0.quant_max, c0.rounding)
            todo = [op for op in todo if (op.weight_cfg.channel_axis, op.weight_cfg.quant_min, op.weight_cfg.quant_max, op.weight_cfg.rounding) == key0]
            sig = tuple((id(op.module), op.module.weight.data_ptr(), op.weight_cfg.scale.data_ptr(), op.weight_cfg.offset.data_ptr()) for op in todo)
            if self._mw.get(dtype, (None,))[0] != sig:
                dev = todo[0].module.weight.device
                mw = MultiWeightQuantizer([op.module.weight.data for op in todo], [op.weight_cfg.scale.to(dev) for op in todo],
                                          [op.weight_cfg.offset.to(dev) for op in todo], channel_axis=c0.channel_axis,
                                          quant_min=c0.quant_min, quant_max=c0.quant_max,
                                          rounding=c0.rounding.value if hasattr(c0.rounding, 'value') else int(c0.rounding),
                                          half_inputs=dtype != torch.float32)
                # the quantizer keeps its own references to scale/offset: the signature is what it was built from
                self._mw[dtype] = (sig, mw, [id(op.module) for op in todo])
            _, mw, ids = self._mw[dtype]
            out.update(zip(ids, mw()))
        return out

    def _op_of(self, module, num_inputs: int = 1) -> QuantableOperation:
        idx = self._calls.get(id(module), 0)
        name = f'{self._names[id(module)]}#{idx}'
        if self._tracing and name not in self.operations:
            self.operations[name] = QuantableOperation(name, module, kind_of(module), num_inputs)
            self._order.append(name)
        return self.operations[name]

    def _trace_inputs(self, op: QuantableOperation, tensors: List[torch.Tensor]):
        for i, x in enumerate(tensors):
            hit, holder = self._produced.get(id(x)), x
            if hit is None and x._base is not None:                     # a view: passive, shares the producer (and its version counter)
                hit, holder = self._produced.get(id(x._base)), x._base
            if hit is None: continue
            src, _, version = hit
            if holder._version != version:
                op.invisible_source[i] = True                          # overwritten in place since (torchvision: `out += identity`)
                continue
            op.sources[i] = src
            src.consumers.append((op, i))

    def _pre(self, module, args):
        if self._bypass: return None                                      # plain fp32 forward of the network (bench breakdown)
        tensors = [a for a in args if isinstance(a, torch.Tensor)]
        op = self._op_of(module, len(tensors))
        if self._tracing:
            self._trace_inputs(op, tensors)
            return None
        hook = self._hooks.get(op.name) if self._hooks else None
        inputs, qinputs, cfgs = [], [], []
        for x, cfg in zip(tensors, op.input_cfgs):
            inputs.append(x); qinputs.append(self.quantize_function(x, cfg)); cfgs.append(cfg)
            if self._collect and cfg.state == QuantizationStates.INITIAL: self._emit(x)
        changed = any(q is not x for q, x in zip(qinputs, tensors))
        if op.weight_cfg is not None:
            w = module.weight
            wd = w.data                                                  # (`.data` makes a new tensor object on every access)
            wq = self._wq.get(id(module))                                # re-quantised every forward (torch.py:516-518): multi-tensor launch
            if wq is None: wq = self.quantize_function(wd, op.weight_cfg)
            inputs.append(wd); qinputs.append(wq); cfgs.append(op.weight_cfg)
            if wq is not wd:                                             # BAKED / FP32 configs hand the parameter through untouched
                self._swapped[module] = wd
                w.data = wq
        if hook is not None: hook.pre_forward_hook(inputs=inputs, quant_inputs=qinputs, quant_configs=cfgs)
        if changed:
            it = iter(qinputs)
            return tuple(next(it) if isinstance(a, torch.Tensor) else a for a in args)
        return None

    def _post(self, module, args, output):
        if self._bypass: return None
        op = self._op_of(module)
        self._calls[id(module)] = self._calls.get(id(module), 0) + 1
        if self._tracing:
            self._produced[id(output)] = (op, output, output._version)
            return None
        fp32 = self._swapped.pop(module, None)
        if fp32 is not None: module.weight.data = fp32
        qout = self.quantize_function(output, op.output_cfg)
        hook = self._hooks.get(op.name) if self._hooks else None
        if hook is not None: hook.post_forward_hook(outputs=[output], quant_outputs=[qout], quant_configs=[op.output_cfg])
        if self._collect and op.output_cfg.state == QuantizationStates.INITIAL: self._emit(output)
        return qout if qout is not output else None

    def _emit(self, tensor: torch.Tensor):
        # sink(k, tensor) observes the k-th observed tensor of this forward immediately; unless it returns False the tensor is consumed
        consumed = self._sink is not None and self._sink(len(self._collected), tensor) is not False
        self._collected.append(None if consumed else tensor)

    @torch.no_grad()
    def forward(self, inputs: torch.Tensor, hooks: Optional[dict] = None, collect: bool = False, sink=None):
        """torch.py:365-410.  `collect=True` returns (output, observed fp32 tensors) for a deferred multi-tensor launch -- only
        valid for tensors the network does not overwrite in place; `sink(k, tensor)` observes the k-th tensor immediately (a sink that
        returns False leaves the tensor in the collected list instead)."""
        self._hooks, self._collect, self._sink = hooks, collect or sink is not None, sink
        if self._channels_last and inputs.dim() == 4: inputs = inputs.contiguous(memory_format=torch.channels_last)
        self._begin()
        try:
            out = self.model(inputs)
        finally:
            self._restore_weights()                                       # an op that raised must not leave a fake-quantised weight behind
        collected, self._collected, self._sink = self._collected, None, None
        return (out, collected) if collect else out

    def observed_configs(self) -> List[TensorQuantizationConfig]:
        """Configs in the order `collect=True` returns their tensors."""
        cfgs = []
        for n in self._order:
            op = self.operations[n]
            cfgs += [c for c in op.input_cfgs if c.state == QuantizationStates.INITIAL]
            if op.output_cfg.state == QuantizationStates.INITIAL: cfgs.append(op.output_cfg)
        return cfgs

    def observed_configs_all(self) -> List[TensorQuantizationConfig]:
        """All activation configs that take part in calibration, whatever their current state (same order as observed_configs())."""
        cfgs = []
        for n in self._order:
            op = self.operations[n]
            cfgs += [c for c in op.input_cfgs if c.state != QuantizationStates.OVERLAPPED]
            if op.output_cfg.state != QuantizationStates.OVERLAPPED: cfgs.append(op.output_cfg)
        return cfgs

    @torch.no_grad()
    def quantize_parameters(self):
        """ParameterQuantizePass (optim/parameters.py:172-215): per-channel min/max observers on the weights, rendered to
        scale/offset by the on-device search."""
        from .observer import TensorObserverFactroy
        for n in self._order:
            op = self.operations[n]
            if op.weight_cfg is not None and op.weight_cfg.state == QuantizationStates.INITIAL:
                ob = TensorObserverFactroy.build_observer(n + ':weight', op.weight_cfg)
                ob.observe(op.module.weight.data)
                ob.render_quantization_config()

    @torch.no_grad()
    def align_quantization(self, force_overlap: bool = True):
        """QuantAlignmentPass with the default setting (optim/refine.py:443-546; api/setting.py:251-256: element-wise 'Align to Large', concat
        'Align to Output', pooling 'None', force_alignment_overlap = True).
        Element-wise (Add / Sub / Sum): the first input config becomes the PASSIVE master of the op's inputs with the scale of the widest input
        range.  Concat / Resize: the output config is the master, every input config is slaved to it.  With force_overlap (or a single consumer) the
        producers' output configs are slaved to the master as well, so the tensors are quantised once, with the shared scale, where they are
        produced."""
        from .core import QuantizationProperty as P
        ext = self._ext()
        for n in self._order:
            op = self.operations[n]
            if not op.input_cfgs: continue
            if op.kind in ELEMENTWISE_ALIGNMENT_TYPES:
                master = op.input_cfgs[0]
                los, his = [], []
                for cfg in op.input_cfgs:
                    if cfg.state == QuantizationStates.FP32 or cfg.policy.has_property(P.FLOATING): continue
                    assert cfg.policy.has_property(P.PER_TENSOR), 'Quant Alignment can only happen with per tensor quantization.'
                    s, o = cfg.scale.float().reshape(()), cfg.offset.float().reshape(())
                    los.append(s * (cfg.quant_min - o)); his.append(s * (cfg.quant_max - o))     # fp32 products, as upstream's tensors
                zero = torch.zeros((), dtype=torch.float32, device=master.scale.device)
                lo = torch.minimum(torch.stack(los).min(), zero).reshape(1)                     # global_min / global_max start from 0
                hi = torch.maximum(torch.stack(his).max(), zero).reshape(1)
                scale, offset = ext.MinMax_To_Scale_Offset(lo, hi, 1, master.quant_min, master.quant_max, master.policy.has_property(P.SYMMETRICAL),
                                                           master.policy.has_property(P.POWER_OF_2), _min_scale_of(master))
                master._dominator = master
                master.state = QuantizationStates.PASSIVE
                master.scale, master.offset = scale.squeeze(0), offset.squeeze(0)
                for slave in op.input_cfgs[1:]:
                    slave.master_by = master
            elif op.kind in OUTPUT_ALIGNMENT_TYPES:                                            # align_to_output (refine.py:484-496)
                master = op.output_cfg
                for slave in op.input_cfgs:
                    if slave.policy.has_property(P.FLOATING) or slave.state == QuantizationStates.FP32: continue
                    slave.master_by = master
            else:
                continue
            for src in self._upstream(op):                                                      # override the producers' configs (:537-546)
                if len(src.consumers) != 1 and not force_overlap: continue
                if any(dst is op for dst, _ in src.consumers): src.output_cfg.master_by = master

    @staticmethod
    def _ext():
        from .ffi import CUDA_COMPLIER
        return CUDA_COMPLIER.CUDA_EXTENSION

    @torch.no_grad()
    def bake_parameters(self):
        """ParameterBakingPass (optim/baking.py:34-47, IR/quantize.py:98-111): every ACTIVATED / PASSIVE parameter is replaced IN PLACE by its
        fake-quantised value and its config becomes BAKED / PASSIVE_BAKED, so that later forwards use the value as is.  The fp32 value stays
        behind as the operation's `stored_weight` (QuantableVariable.stored_value upstream): dequantize() swaps it back in."""
        for n in self._order:
            op = self.operations[n]
            cfg = op.weight_cfg
            if cfg is None or cfg.state not in (QuantizationStates.ACTIVATED, QuantizationStates.PASSIVE): continue
            op.stored_weight = op.module.weight.data
            baked = self._quant_fn(op.stored_weight, cfg)
            if self._channels_last and baked.dim() == 4: baked = baked.contiguous(memory_format=torch.channels_last)
            op.module.weight.data = baked
            cfg.state = QuantizationStates.BAKED if cfg.state == QuantizationStates.ACTIVATED else QuantizationStates.PASSIVE_BAKED

    def dequantize(self):
        """QuantableOperation.dequantize for every operation (IR/quantize.py:118-141): every config's state is stored and set to FP32, baked
        parameters are swapped with their stored fp32 values -- the network runs as the original fp32 network."""
        if self._dequantized is not None: return self
        self._restore_weights()
        self._dequantized = []
        for n in self._order:
            op = self.operations[n]
            for cfg in op.input_cfgs + ([op.weight_cfg] if op.weight_cfg is not None else []) + [op.output_cfg]:
                self._dequantized.append((cfg, cfg.state)); cfg.state = QuantizationStates.FP32
            if op.stored_weight is not None: op.module.weight.data, op.stored_weight = op.stored_weight, op.module.weight.data
        return self

    def restore_quantize_state(self):
        """IR/quantize.py:143-160."""
        if self._dequantized is None: return self
        self._restore_weights()
        for cfg, state in self._dequantized: cfg.state = state
        for n in self._order:
            op = self.operations[n]
            if op.stored_weight is not None: op.module.weight.data, op.stored_weight = op.stored_weight, op.module.weight.data
        self._dequantized = None
        return self

    def quantize_only(self, name: Optional[str]):
        """While dequantize() is in effect: operation `name` alone runs quantised -- its configs get their stored states back and its baked
        weight is swapped in (QuantableOperation.restore_quantize_state of that one operation, IR/quantize.py:143-160), every other config stays
        FP32.  quantize_only(None) returns that operation to FP32, and must precede restore_quantize_state()."""
        if self._dequantized is None: raise RuntimeError('quantize_only: call dequantize() first')
        self._restore_weights()
        if self._only is not None:
            op = self.operations[self._only]
            for cfg in self._configs_of(op): cfg.state = QuantizationStates.FP32
            if op.stored_weight is not None: op.module.weight.data, op.stored_weight = op.stored_weight, op.module.weight.data
            self._only = None
        if name is not None:
            op = self.operations[name]
            stored = {id(cfg): state for cfg, state in self._dequantized}
            for cfg in self._configs_of(op): cfg.state = stored[id(cfg)]
            if op.stored_weight is not None: op.module.weight.data, op.stored_weight = op.stored_weight, op.module.weight.data
            self._only = name
        return self

    @staticmethod
    def _configs_of(op: QuantableOperation) -> List[TensorQuantizationConfig]:
        return op.input_cfgs + ([op.weight_cfg] if op.weight_cfg is not None else []) + [op.output_cfg]


def _min_scale_of(cfg) -> float:
    from .core import OBSERVER_MIN_SCALE, OBSERVER_MIN_SCALE_MANUL_OVERRIDE
    return cfg.detail.get(OBSERVER_MIN_SCALE_MANUL_OVERRIDE, OBSERVER_MIN_SCALE)


# ------------------------------------------------------------------------------------------------------------------ calibration drivers
class DeviceBatchRing:
    """Two persistent device buffers and one persistent copy stream per device for the calibration inputs: batch k+1 is copied host->device on the
    copy stream into the slot batch k-1 has been consumed from, while batch k runs.  Nothing is allocated per batch and nothing crosses streams
    inside the caching allocator (the first version allocated every batch on a fresh side stream and handed it over with `record_stream`)."""
    _rings = {}

    def __init__(self, device):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.slots = [None, None]
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.consumed = [None, None]

    @classmethod
    def of(cls, device):
        device = torch.device(device)
        key = (device.type, torch.cuda.current_device() if device.index is None else device.index)
        ring = cls._rings.get(key)
        if ring is None: ring = cls._rings[key] = cls(device)
        return ring

    def put(self, slot: int, x: torch.Tensor):
        buf = self.slots[slot]
        if buf is None or buf.shape != x.shape or buf.dtype != x.dtype:
            buf = self.slots[slot] = torch.empty(x.shape, dtype=x.dtype, device=self.device)   # allocated on the caller's stream, kept
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
        if self.consumed[slot] is not None: self.stream.wait_event(self.consumed[slot])
        with torch.cuda.stream(self.stream):
            buf.copy_(x, non_blocking=True)
            self.ready[slot].record(self.stream)
        return buf

    def release(self, slot: int):
        ev = self.consumed[slot]
        if ev is None: ev = self.consumed[slot] = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))


def prefetch_to_device(batches, to_device, device):
    """Yield every batch on the device with the copy of batch k+1 enqueued on a side stream before batch k is handed out, so the host->device
    transfer of the next calibration batch (19 MB for 32 images) overlaps the forward of the current one.
    to_device='ring': the batches are host tensors (pinned for a truly asynchronous copy); they go through the device's DeviceBatchRing -- the
    yielded tensor is valid until the next one is requested.  A callable to_device keeps the generic path (whatever it returns is allocated on a
    side stream and handed to the consumer's stream)."""
    it = iter(batches)
    if isinstance(to_device, str):
        if to_device != 'ring': raise ValueError(f"to_device must be a callable or 'ring', got {to_device!r}")
        ring = DeviceBatchRing.of(device)
        main = torch.cuda.current_stream(device)
        x = next(it, None)
        ahead = None if x is None else ring.put(0, x)
        k = 0
        while ahead is not None:
            y, slot = ahead, k % 2
            main.wait_event(ring.ready[slot])
            x = next(it, None)
            ahead = None if x is None else ring.put((k + 1) % 2, x)
            yield y
            ring.release(slot)                                           # everything the consumer enqueued for batch k precedes this event
            k += 1
        return
    copy_stream = DeviceBatchRing.of(device).stream

    def fetch():
        x = next(it, None)
        if x is None: return None
        with torch.cuda.stream(copy_stream):
            y = to_device(x)
            done = torch.cuda.Event(); done.record(copy_stream)
        return y, done

    ahead = fetch()
    while ahead is not None:
        y, done = ahead
        main = torch.cuda.current_stream(device)
        main.wait_event(done)
        if isinstance(y, torch.Tensor): y.record_stream(main)            # allocated on the copy stream, consumed on the main stream
        ahead = fetch()
        yield y


def arena_settings(cfgs, method: str) -> dict:
    """The ArenaCalibrator arguments that every observed config asks for, read the way the per-config observers read them
    (ppq_b200.observer): range, bits, symmetry, power-of-two, OBSERVER_MIN_SCALE_MANUL_OVERRIDE, the KL bin override and the percentile
    override.  One calibrator serves all tensors, so configs that differ in any of these -- or per-channel ones -- are refused."""
    from .core import (OBSERVER_KL_HIST_BINS, OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE, OBSERVER_MSE_HIST_BINS, OBSERVER_PERCENTILE,
                       OBSERVER_PERCENTILE_MANUL_OVERRIDE, QuantizationProperty as P)
    found = {}
    for c in cfgs:
        if not c.policy.has_property(P.PER_TENSOR):
            raise ValueError('calibrate_arena serves per-tensor activation configs only; use RuntimeCalibrationPass for per-channel ones')
        if method == 'kl': bins = c.detail.get(OBSERVER_KL_HIST_BINS_MANUL_OVERRIDE, OBSERVER_KL_HIST_BINS)
        else: bins = OBSERVER_MSE_HIST_BINS if method == 'mse' else None
        key = dict(quant_min=c.quant_min, quant_max=c.quant_max, num_of_bits=c.num_of_bits, symmetrical=c.policy.has_property(P.SYMMETRICAL),
                   power_of_2=c.policy.has_property(P.POWER_OF_2), min_scale=_min_scale_of(c),
                   bins=bins, percentile=c.detail.get(OBSERVER_PERCENTILE_MANUL_OVERRIDE, OBSERVER_PERCENTILE) if method == 'percentile' else OBSERVER_PERCENTILE)
        found.setdefault(tuple(key.items()), key)
    if len(found) > 1:
        raise ValueError('calibrate_arena: the observed configs differ in ' +
                         ', '.join(k for k in next(iter(found.values())) if len({f[k] for f in found.values()}) > 1) +
                         '; one arena serves one setting -- use RuntimeCalibrationPass for mixed configs')
    return next(iter(found.values())) if found else {}


@torch.no_grad()
def calibrate_arena(executor: TorchExecutor, batches, method: str = 'kl', group=None, to_device=None, deferred='auto',
                    graphs: bool = False, prefetch: bool = True, trace: list = None, half_inputs: bool = False):
    """Two-phase calibration of every observed activation through one ArenaCalibrator (statistics arena, one all-reduce per
    phase, on-device scale search).  `batches` is this rank's share of the calibration set (sample-sharded by the caller).
    deferred=False observes each tensor as the forward produces it (one launch per tensor);
    deferred=True keeps all tensors alive and issues ONE multi-tensor launch per forward (only valid when nothing is overwritten in place);
    deferred='auto' (default) finds out during the first forward which observed tensors the network later overwrites in place
    (torchvision adds residuals with `out += identity`), observes those immediately and everything else in one multi-tensor launch;
    graphs=True captures one forward per phase -- network kernels, per-forward weight fake-quant and the collectors -- into a CUDA
    graph and replays it for every batch (fixed batch shape).  Capture + instantiate
    costs more than it saves at 8-16 batches per phase, so it is off by default; it pays off for long
    calibration sets or when the same graph is reused across calls.
    The observed configs must agree in range, bits, symmetry, power-of-two, minimum scale and bin / percentile overrides and be per-tensor
    (`arena_settings`); asymmetric 'kl' raises PermissionError as upstream, asymmetric 'mse' and more than 12287 KL bins raise ValueError --
    all before the first batch.
    half_inputs=True calibrates fp16 / bf16 activations through the *_Half table kernels (scales and offsets are the fp32 ones on the upcasts): a
    network cast to half, or an fp32 network when the caller wraps this call in torch.autocast -- its activations then arrive in both dtypes
    and every deferred launch becomes one per dtype present.
    to_device: a callable applied to every batch, or 'ring' for host tensors staged through the device's persistent DeviceBatchRing.
    trace: a list that receives (phase, batch index, host time, CUDA event, thread CPU time) before every batch and at the end of a phase --
    bench.py's e2e uses it to say whether a slow calibration was slow on the host or on the device, and where."""
    import time
    half = sorted({str(p.dtype) for p in executor.model.parameters() if p.dtype != torch.float32})
    if half and not half_inputs:
        raise TypeError(f'calibrate_arena: the multi-tensor collectors read fp32 tensors, this network has {", ".join(half)} parameters; '
                        'calibrate it with RuntimeCalibrationPass (per-observer collectors, which take fp16 / bf16).')
    from .calibration import ArenaCalibrator, is_dense
    cfgs = executor.observed_configs()
    if graphs and method == 'percentile': raise ValueError('graphs=True needs static statistics buffers; the percentile observer keeps one row per batch')
    dev = next(executor.model.parameters()).device
    cal = ArenaCalibrator(len(cfgs), dev, method=method, group=group, half_inputs=half_inputs, **arena_settings(cfgs, method))
    for c in cfgs: c.observer_algorithm = method
    if iter(batches) is batches: batches = list(batches)                  # a one-shot iterator would leave phase 2 without data
    static_in = None
    mutated = None                                                        # slots whose tensors are overwritten later in the forward
    phase = 0
    while True:
        graph = None
        phase += 1
        overlapped = prefetch and to_device is not None and not graphs and dev.type == 'cuda'
        for index, x in enumerate(prefetch_to_device(batches, to_device, dev) if overlapped else batches):
            if trace is not None:
                ev = torch.cuda.Event(enable_timing=True); ev.record(torch.cuda.current_stream(dev))
                trace.append((phase, index, time.perf_counter(), ev, time.thread_time()))
            cal.begin_batch()
            if graphs:
                if static_in is None:
                    static_in = torch.empty(x.shape, dtype=x.dtype if half_inputs else torch.float32, device=dev)
                static_in.copy_(x, non_blocking=True)
                if graph is None:
                    # eager run on a side stream first (cuDNN autotuning, lazy initialisation), statistics restored afterwards:
                    # min/max are idempotent under re-observation, histogram counts are not
                    keep_mm, keep_h = cal.minmax.clone(), cal.hist.clone()
                    side = torch.cuda.Stream(device=dev)
                    side.wait_stream(torch.cuda.current_stream(dev))
                    with torch.cuda.stream(side):
                        executor.forward(static_in, sink=cal.observe_one)
                    torch.cuda.current_stream(dev).wait_stream(side)
                    cal.minmax.copy_(keep_mm); cal.hist.copy_(keep_h)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        executor.forward(static_in, sink=cal.observe_one)
                    cal.minmax.copy_(keep_mm); cal.hist.copy_(keep_h)      # capture does not execute, but stay safe
                graph.replay()
                continue
            if to_device is not None and not overlapped: x = x.to(dev, non_blocking=True) if isinstance(to_device, str) else to_device(x)
            if deferred is True:
                _, tensors = executor.forward(x, collect=True)
                cal.observe([t if is_dense(t) else t.contiguous() for t in tensors])
                del tensors
            elif deferred == 'auto':
                if mutated is None:                                       # probe forward: observe immediately, remember versions
                    seen = []

                    def probe(k, t):
                        cal.observe_one(k, t); seen.append((t, t._version))
                    executor.forward(x, sink=probe)
                    mutated = {k for k, (t, v) in enumerate(seen) if t._version != v or not is_dense(t)}
                    del seen
                else:
                    def sink(k, t):
                        if k in mutated:
                            cal.observe_one(k, t); return True
                        return False
                    _, tensors = executor.forward(x, collect=True, sink=sink)
                    rest = [(k, t) for k, t in enumerate(tensors) if t is not None]
                    cal.observe([t for _, t in rest], [k for k, _ in rest])
                    del tensors, rest
            else:
                executor.forward(x, sink=cal.observe_one)
        if trace is not None:
            ev = torch.cuda.Event(enable_timing=True); ev.record(torch.cuda.current_stream(dev))
            trace.append((phase, len(batches), time.perf_counter(), ev, time.thread_time()))
        if cal.end_phase(): break
    if trace is not None:
        ev = torch.cuda.Event(enable_timing=True); ev.record(torch.cuda.current_stream(dev))
        trace.append((phase + 1, 0, time.perf_counter(), ev, time.thread_time()))
    for i, c in enumerate(cfgs):
        c.scale, c.offset, c.state = cal.scale[i], cal.offset[i], QuantizationStates.ACTIVATED
    return cal


@torch.no_grad()
def graphwise_error_analyse(executor: TorchExecutor, batches, to_device=None, graphs: bool = False, fetchs: Optional[int] = None,
                            seed: int = 10086) -> Dict[str, float]:
    """The evaluation loop where fake-quant throughput shows up in user wall-clock (ppq/quantization/analyse/graphwise.py:64-183): run every batch
    through the network twice -- all configs dequantised (fp32) and all configs active -- and report, per quantable operation, the SNR
    mean((q - f)^2) / mean(f^2) per sample, averaged (torch_snr_error, ppq/quantization/measure/norm.py:52-93).  Every activation goes through
    QuantizeTensor_LT and every weight through the multi-tensor QuantizeTensor_LC on each quantised forward.
    graphs=True captures the fp32 forward and the quantised forward (network kernels + ~100 small fake-quant launches + the hooks' bookkeeping)
    into two CUDA graphs on the first batch and replays them for the others (fixed batch shape): the per-call host cost of the drop-in flow
    (python -> binding -> allocator -> launch, 4.5-5 us x every config x every forward) disappears from the loop.
    fetchs=None measures on whole tensors, every quantable operation.  fetchs=4096 follows the reference to the letter: computing operations
    only (graphwise.py:112-113), `fetchs` elements per sample picked by the reference's seeded linear congruential indexer
    (utils/fetch.py:4-23, seed 10086) -- pinned against the real function on the GPU (tests/test_gpu_graph_parity.py)."""
    names = [n for n, op in executor.quantable_operations() if fetchs is None or op.kind in COMPUTING_OP]
    acc = {n: None for n in names}
    count = 0
    indexers: Dict[tuple, torch.Tensor] = {}

    def sample(t: torch.Tensor) -> torch.Tensor:
        t = t.flatten(1)
        if fetchs is None: return t
        key = (t.shape[-1], t.device)
        if key not in indexers:
            idx, sd = [], seed
            for _ in range(fetchs):
                idx.append(sd % t.shape[-1]); sd = (0x343FD * sd + 0x269EC3) % (2 << 31)
            indexers[key] = torch.tensor(idx, dtype=torch.long, device=t.device)
        return t.index_select(-1, indexers[key])

    class Tap:
        def __init__(self, name, store): self.name, self.store = name, store
        def pre_forward_hook(self, **kw): pass
        def post_forward_hook(self, outputs, quant_outputs, quant_configs): self.store[self.name] = quant_outputs[0]

    def both(x, fp, qt):
        executor.dequantize(); executor.forward(x, hooks={n: Tap(n, fp) for n in names})                   # graphwise.py:131-146
        executor.restore_quantize_state(); executor.forward(x, hooks={n: Tap(n, qt) for n in names})       # :148-165

    def snr_all(fp, qt):
        out = []
        for n in names:
            f, q = sample(fp[n]).float(), sample(qt[n]).float()            # fp16 / bf16 activations: the SNR is accumulated in fp32
            out.append((torch.pow(q - f, 2).sum(dim=-1) / (torch.pow(f, 2).sum(dim=-1) + 1e-7)).mean())
        return torch.stack(out)

    static_in, graph, fp, qt, static_snr = None, None, {}, {}, None
    try:
        for x in batches:
            if to_device is not None: x = x.to(next(executor.model.parameters()).device, non_blocking=True) if isinstance(to_device, str) else to_device(x)
            if not graphs:
                fp, qt = {}, {}
                both(x, fp, qt)
                snr = snr_all(fp, qt)
            else:
                if graph is None:
                    static_in = x.clone()
                    dev = static_in.device
                    side = torch.cuda.Stream(device=dev)
                    side.wait_stream(torch.cuda.current_stream(dev))
                    with torch.cuda.stream(side):                         # eager first: lazy initialisation (descriptor tables, cuDNN plans, indexers)
                        wf, wq_ = {}, {}
                        both(static_in, wf, wq_); snr_all(wf, wq_)
                        del wf, wq_
                    torch.cuda.current_stream(dev).wait_stream(side)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        both(static_in, fp, qt)
                        static_snr = snr_all(fp, qt)
                else:
                    static_in.copy_(x, non_blocking=True)
                graph.replay()
                snr = static_snr.clone()
            acc_t = snr if count == 0 else acc_t + snr                     # noqa: F821 (defined on the first iteration)
            count += 1
    finally:
        executor.restore_quantize_state()
    if count == 0: return {n: 0.0 for n in names}
    vals = (acc_t / count).tolist()
    del acc
    return dict(zip(names, vals))


@torch.no_grad()
def layerwise_error_analyse(executor: TorchExecutor, batches, interested_outputs=None, method: str = 'snr', steps: int = 8,
                            to_device=None) -> Dict[str, float]:
    """Which operation causes the quantisation error (ppq/quantization/analyse/layerwise.py:15-134): for every computing operation (Conv, Gemm,
    ConvTranspose, MatMul, in executor order), the error of the interested outputs when that operation alone is quantised -- its configs with
    their stored states and its baked weight, every other config FP32 (TorchExecutor.quantize_only) -- against the fp32 network.
    Returns {operation name: measure}, measure = 'snr' (noise / signal power), 'mse' or 'cosine' per sample, averaged over the samples of a
    batch and then over the updates as the reference's MeasureRecorder(reduce='mean') does: one update per (batch, interested output) weighted
    by the output's shape[0], running mean (m n + r b) / (n + b) in Python doubles, batch by batch.
    interested_outputs: None = the network's return value (a tensor, or every tensor of a tuple / list, in order); a name or a list of
    operation names = those operations' outputs as the executor hands them on.  steps: the reference breaks after the update of batch
    `steps`, so min(len(batches), steps + 1) batches are measured.
    The loop is batch-outer: one fp32 forward per batch, kept on the device and measured against each operation's quantised forward of that
    batch, (K + 1)(S + 1) forwards instead of the reference's 2 K (S + 1); the result is the reference's whenever the forward is deterministic
    (deterministic cuDNN).  Each quantised forward's outputs go to one Multi_Paired_Moments launch; the per-sample measures and batch means
    are fp64 on the device, and one copy to the host at the end feeds the running means.  The measure is the value in exact arithmetic
    rounded once per fp64 addition, where the reference sums in fp32 (fp16 / bf16 outputs: their exact upcasts) -- DESIGN.md §2.
    Every config's state, scale and offset and every weight are as before the call, also when a batch raises."""
    import itertools

    from .measure import MEASURES, batch_measures
    if method not in MEASURES: raise ValueError(f"Unsupported measurement {method!r}: 'snr', 'mse' and 'cosine' are supported")
    names = [n for n, op in executor.quantable_operations() if op.kind in COMPUTING_OP]
    if isinstance(interested_outputs, str): interested_outputs = [interested_outputs]
    if interested_outputs is not None:
        unknown = [n for n in interested_outputs if n not in executor.operations]
        if unknown: raise KeyError(f'layerwise_error_analyse: no operation named {", ".join(unknown)}')

    class Tap:
        def __init__(self, store): self.store = store
        def pre_forward_hook(self, **kw): pass
        def post_forward_hook(self, outputs, quant_outputs, quant_configs): self.store.append(quant_outputs[0].clone())

    def run(x) -> List[torch.Tensor]:
        if interested_outputs is None:
            out = executor.forward(x)
            outs = list(out) if isinstance(out, (tuple, list)) else [out]
            if not all(isinstance(t, torch.Tensor) for t in outs): raise TypeError('layerwise_error_analyse: the network must return tensors')
            return outs
        taps = {n: [] for n in interested_outputs}
        executor.forward(x, hooks={n: Tap(taps[n]) for n in interested_outputs})
        return [taps[n][-1] for n in interested_outputs]

    dev = next(executor.model.parameters()).device
    res, weights = [], []                                                 # per batch: [K, outputs] fp64 on the device
    executor.dequantize()
    try:
        for x in itertools.islice(batches, steps + 1):                   # read once: a one-shot iterator is enough
            if to_device is not None: x = x.to(dev, non_blocking=True) if isinstance(to_device, str) else to_device(x)
            real = run(x)
            res.append(torch.empty(len(names), len(real), dtype=torch.float64, device=dev))
            weights.append([int(t.shape[0]) for t in real])
            for k, n in enumerate(names):
                executor.quantize_only(n)
                pred = run(x)
                executor.quantize_only(None)
                batch_measures(pred, real, method, out=res[-1][k])
            del real
    finally:
        if executor._dequantized is not None: executor.quantize_only(None)
        executor.restore_quantize_state()
    results = {n: 0.0 for n in names}
    if not weights: return results
    vals = torch.stack(res).cpu().tolist()                                # [batches, K, outputs]
    for k, n in enumerate(names):                                         # MeasureRecorder.update (analyse/util/__init__.py:32-47)
        m, cnt = 0.0, 0
        for b, ws in enumerate(weights):
            for j, e in enumerate(ws):
                m = m * cnt + vals[b][k][j] * e
                cnt += e
                m /= cnt
        results[n] = m
    return results


def e2e_calibration_benchmark(batch: int, batches: int, steps: int, warmup: int, device, world: int = 1, seed: int = 0, graphs: bool = False,
                              channels_last: bool = False, model: torch.nn.Module = None, image=(3, 224, 224), distinct_host_batches: int = 16):
    """bench.py's `e2e`: a network (default: torchvision ResNet-50; random init, BN folded) calibrated end to end through the public API -- `batches`
    x `batch` images in pinned host memory (this rank's share of the calibration set), H2D copy of every batch inside the timed region (both
    phases), torch forward with per-forward weight fake-quant, multi-tensor collectors, the two all-reduces, on-device KL search and a D2H read of
    the resulting scales.  One step = one whole calibration; `steps` of them are timed after warm-up calibrations at the timed shape have
    converged (two consecutive ones within 5 %: cuDNN autotuning, allocator growth, descriptor caches and clocks all settle there, not in a
    2-batch dry run)."""
    import torch.distributed as dist
    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = True
    if model is None:
        import torchvision
        model = torchvision.models.resnet50(weights=None)
    model = model.eval()
    ex = TorchExecutor(model.to(device), torch.zeros((2,) + tuple(image), device=device), channels_last=channels_last)
    ex.quantize_parameters()
    g = torch.Generator().manual_seed(1000 + seed)                         # every rank calibrates its OWN shard of the sample set
    distinct = [torch.rand((batch,) + tuple(image), generator=g).pin_memory() for _ in range(min(batches, distinct_host_batches))]
    host = [distinct[k % len(distinct)] for k in range(batches)]            # big inputs (3x640x640): a few pinned batches cycled; every batch is still copied
    stream = torch.cuda.current_stream()
    act_cfgs = ex.observed_configs()
    to_dev = lambda x: x.to(device, non_blocking=True)                     # noqa: E731  (raw copy, for the breakdown's H2D line)

    def reset():
        for c in act_cfgs: c.state = QuantizationStates.INITIAL

    traces = []

    def run():
        traces.append([])
        cal = calibrate_arena(ex, host, method='kl', to_device='ring', graphs=graphs, trace=traces[-1])
        s = cal.scale.cpu()                                               # D2H of the result (synchronises)
        reset()
        return s

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(stream); out = fn(); b.record(stream); torch.cuda.synchronize()
        return a.elapsed_time(b), out

    warm = []
    while len(warm) < max(warmup, 2) or (len(warm) < 8 and abs(warm[-1] - warm[-2]) > 0.05 * warm[-1]):
        warm.append(timed(run)[0])
    # A full (generation-2) collection of the cyclic garbage collector walks every container object of the process -- 100-200 ms here, i.e. a
    # whole calibration -- and lands on one step in ten at random (round-2 runs: steps of 137 / 143 / 304 ms).  Collect now, keep the collector
    # off inside the timed region (a long-running calibration service would do the same), restore afterwards.
    import gc
    gc_was_enabled = gc.isenabled()
    gc.collect(); gc.disable()
    if world > 1: dist.barrier()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per_step = []
    del traces[:]
    t0.record(stream)
    def alloc_counters():
        m = torch.cuda.memory_stats(device)
        return [m.get('num_device_alloc', 0), m.get('num_device_free', 0), m.get('num_alloc_retries', 0), m.get('reserved_bytes.all.current', 0)]

    counters = [alloc_counters()]
    for _ in range(steps):
        a = torch.cuda.Event(enable_timing=True); a.record(stream)
        scales = run()
        b = torch.cuda.Event(enable_timing=True); b.record(stream)
        per_step.append((a, b)); counters.append(alloc_counters())
    t1.record(stream)
    if world > 1: dist.barrier()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1)
    if gc_was_enabled: gc.enable()
    if world > 1:
        t = torch.tensor([ms], device=device); dist.all_reduce(t, op=dist.ReduceOp.MAX); ms = t.item()
    assert bool(torch.isfinite(scales).all()) and bool((scales > 0).all())
    timed_traces = traces[:steps]

    # ---- breakdown (untimed, after the measurement): where a calibration batch's time goes
    def forwards(bypass):
        for _ in range(2):                                                # two passes over the set, like the two phases
            for x in prefetch_to_device(host, 'ring', device):
                if bypass:
                    ex._bypass = True
                    try: ex.model(x.contiguous(memory_format=torch.channels_last) if channels_last else x)
                    finally: ex._bypass = False
                else:
                    ex.forward(x, sink=lambda k, t: True)                 # hooks + per-forward weight fake-quant, no collector launch
    with torch.no_grad():
        pure = min(timed(lambda: forwards(True))[0] for _ in range(2))
        hooked = min(timed(lambda: forwards(False))[0] for _ in range(2))
        h2d = min(timed(lambda: [to_dev(x) for x in host for _ in range(2)])[0] for _ in range(2))
    nb2 = 2.0 * batches
    step_ms = [a.elapsed_time(b) for a, b in per_step]
    # the slowest timed calibration, batch by batch: the largest gap between two consecutive batch marks on the host clock (time to ENQUEUE a
    # batch: Python, hooks, launches, allocator) and on the device clock (time to EXECUTE it), and where it fell
    slow = timed_traces[max(range(len(step_ms)), key=lambda i: step_ms[i])]
    gaps = [(slow[i + 1][2] - slow[i][2]) * 1e3 for i in range(len(slow) - 1)]
    dgaps = [slow[i][3].elapsed_time(slow[i + 1][3]) for i in range(len(slow) - 1)]
    hi, di = max(range(len(gaps)), key=gaps.__getitem__), max(range(len(dgaps)), key=dgaps.__getitem__)
    where = lambda i: f'phase {slow[i][0]} batch {slow[i][1]}' if slow[i][1] < batches else f'phase {slow[i][0]} end (exchange / search)'   # noqa: E731
    worst = max(range(len(step_ms)), key=lambda i: step_ms[i])
    cpu_in_gap = (slow[hi + 1][4] - slow[hi][4]) * 1e3                       # CPU time the enqueueing thread burnt inside its longest gap: ~gap = busy, ~0 = blocked / descheduled
    slowest = {'ms': round(max(step_ms), 3), 'host_enqueue_gap_ms': {'median': round(sorted(gaps)[len(gaps) // 2], 3), 'max': round(gaps[hi], 3), 'at': where(hi),
                                                                     'thread_cpu_ms_inside': round(cpu_in_gap, 3)},
               'gaps_over_3x_median': sum(1 for g_ in gaps if g_ > 3 * sorted(gaps)[len(gaps) // 2]),
               'allocator': {'cudaMalloc_calls': counters[worst + 1][0] - counters[worst][0], 'cudaFree_calls': counters[worst + 1][1] - counters[worst][1],
                             'alloc_retries': counters[worst + 1][2] - counters[worst][2], 'reserved_gb': round(counters[worst + 1][3] / 2**30, 2),
                             'cudaMalloc_calls_all_steps': counters[-1][0] - counters[0][0]},
               'device_gap_ms': {'median': round(sorted(dgaps)[len(dgaps) // 2], 3), 'max': round(dgaps[di], 3), 'at': where(di)}}
    total = ms / steps
    return {'value': round(world * steps * batches * batch / (ms * 1e-3), 1), 'unit': 'imgs/s',
            'h2d_bytes_per_step': 2 * batches * int(host[0].numel()) * 4, 'd2h_bytes_per_step': int(scales.numel() * 4),
            'ms_per_step': round(total, 3), 'steps': steps, 'step': f'one whole calibration: {batches} batches x {batch} images, both phases',
            'step_ms': {'min': round(min(step_ms), 3), 'median': round(sorted(step_ms)[len(step_ms) // 2], 3), 'max': round(max(step_ms), 3)},
            'warmup_calibrations_ms': [round(w, 2) for w in warm], 'slowest_step': slowest,
            'observed_tensors': int(scales.numel()), 'cuda_graphs': graphs, 'channels_last': channels_last, 'python_gc': 'collected before, disabled inside the timed region',
            'breakdown_ms_per_batch_pass': {'forward_fp32_cudnn': round(pure / nb2, 3), 'hooks_and_weight_fakequant': round((hooked - pure) / nb2, 3),
                                            'collectors_exchange_search': round((total - hooked) / nb2, 3),
                                            'h2d_copy_overlapped': round(h2d / nb2, 3), 'total': round(total / nb2, 3)},
            'what': f'pinned-host images -> H2D -> torch {type(ex.model).__name__} forward (fp32, cuDNN) with per-forward INT8 per-channel weight fake-quant '
                    '-> multi-tensor min/max (phase 1) / histogram (phase 2) -> all-reduce -> on-device KL search -> scales D2H'}
