"""Weight-only int8 for the LLaMA decoder: one fp32 scale per output row, for inference.

    model = MM_LLMs.build_random(cfg, dtype=torch.float16)   # or from_pretrained(...), then .cuda()
    model.quantize_llm_int8()                                # in place, one layer at a time

The seven projections of every decoder layer (q, k, v, o, gate, up, down) become `Int8Linear` modules holding `weight`
(int8, (N, K)) and `weight_scale` (fp32, (N,)); their 16-bit weights and every engine-derived copy of them are freed.
lm_head, embed_tokens (the alignment attention reads it as keys and values), the norms, the alignment blocks, the encoders
and the transform / project layers stay 16-bit.

The rule, per row of W:  s = fp32(max_k |W[k]|) / 127 (IEEE division),  q = clamp(rint(fp32(W) / s), -127, 127) with
ties to even,  and q = 0 where s = 0.  It runs on the device (mm_quantize_rows_int8).

How a quantized model runs (engine.py):
  * a decode step streams the int8 weights through mm_gemm_w8_thin, which reads the fused [q; k; v] / [gate | up] rows in
    place and applies the RMSNorm gain to the few activation rows; the split-K tail is the 16-bit path's mm_thin_fused;
  * a prefill (and the eval forward) dequantizes one layer at a time into a scratch buffer, round16(fp32(fp32(q s) g)), and
    runs the 16-bit GEMMs: bit-identical to the engine on a model whose decoder weights are the fp32 values q s.

Refused with RuntimeError: quantizing a model that carries LoRA adapters (merge_lora() first), quantizing twice, quantizing a
model on the CPU, add_lora on a quantized model, and a train()-mode forward (training an int8 base is not supported).
"""
from __future__ import annotations

import torch
from torch import nn

PROJECTIONS = (("self_attn", "q_proj"), ("self_attn", "k_proj"), ("self_attn", "v_proj"), ("self_attn", "o_proj"),
               ("mlp", "gate_proj"), ("mlp", "up_proj"), ("mlp", "down_proj"))


class Int8Linear(nn.Module):
    """A bias-free linear layer with per-row int8 weights: y = x (q * scale[:, None])^T.  Computed by the engine's kernels
    only; `weight_scale` stays fp32 when the model is cast to another dtype."""

    def __init__(self, weight: torch.Tensor, weight_scale: torch.Tensor):
        super().__init__()
        if weight.dtype != torch.int8 or weight.dim() != 2 or weight_scale.dtype != torch.float32 \
                or tuple(weight_scale.shape) != (weight.shape[0],):
            raise TypeError("Int8Linear: weight must be int8 (N, K) and weight_scale fp32 (N,)")
        self.out_features, self.in_features = weight.shape
        self.weight = nn.Parameter(weight, requires_grad=False)
        self.weight_scale = nn.Parameter(weight_scale, requires_grad=False)

    def _apply(self, fn, recurse=True):
        scale = self.weight_scale.data
        super()._apply(fn, recurse)
        if self.weight_scale.dtype != torch.float32:  # a dtype cast (model.to(dtype), .half()): the scale stays fp32
            self.weight_scale.data = scale.to(self.weight_scale.device)
        return self

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for name, dt in (("weight", torch.int8), ("weight_scale", torch.float32)):
            t = state_dict.get(prefix + name)
            if t is not None and t.dtype != dt:
                error_msgs.append(f"{prefix}{name}: an int8-quantized layer loads {dt} values, got {t.dtype} "
                                  f"(load the 16-bit checkpoint before quantize_llm_int8())")
                return
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def dequantized(self) -> torch.Tensor:
        """The fp32 weight q * scale the layer stands for."""
        return self.weight.float() * self.weight_scale[:, None]

    def forward(self, x):
        raise RuntimeError("Int8Linear runs inside the MM_LLMs engine only; call the model, not the layer")

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, int8 per-row scales"


def is_quantized(model) -> bool:
    layers = model.llm.model.layers
    return len(layers) > 0 and isinstance(layers[0].self_attn.q_proj, Int8Linear)


def quantize_llm_int8(model) -> None:
    """Quantize the decoder projections of `model` (an MM_LLMs on a CUDA device) in place, one layer at a time."""
    from . import lora, ops

    if is_quantized(model):
        raise RuntimeError("quantize_llm_int8: the decoder is already quantized")
    if lora.adapted_modules(model):
        raise RuntimeError("quantize_llm_int8: the model carries LoRA adapters; call merge_lora() first")
    layers = model.llm.model.layers
    for l in layers:
        for parent, name in PROJECTIONS:
            lin = getattr(getattr(l, parent), name)
            if not lin.weight.is_cuda:
                raise RuntimeError("quantize_llm_int8: the decoder lives on the CPU; move the model to a CUDA device first "
                                   "(there is no CPU quantization path)")
            if lin.bias is not None:
                raise NotImplementedError(f"quantize_llm_int8: {name} has a bias; LLaMA projections have none")
    eng = model.engine
    eng.drop_derived()  # the fused 16-bit copies go first, so the peak stays at one layer's weights
    model.__dict__.pop("_train_step", None)
    dev = layers[0].self_attn.q_proj.weight.device
    with torch.no_grad(), torch.cuda.device(dev):
        for l in layers:
            for parent, name in PROJECTIONS:
                mod = getattr(l, parent)
                q, s = ops.quantize_rows_int8(getattr(mod, name).weight.detach())
                setattr(mod, name, Int8Linear(q, s))
    eng.drop_derived()
