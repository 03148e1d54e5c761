"""Weight-only int8, and FP8 (e4m3) weights and activations, for the LLaMA decoder: one fp32 scale per row, for inference.

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

FP8 (`model.quantize_llm_fp8()`): the same seven projections become `Fp8Linear` modules, `weight` float8_e4m3fn (N, K) and
`weight_scale` fp32 (N,), with the same lifecycle and refusals (either format refuses the other).  The rule, per row, for
weights and for activation rows alike:  s = fp32(max_k |v[k]|) / 448 (IEEE division),  q = e4m3(fp32(v) / s) rounded to
nearest even and saturated to +-448,  q = 0 where s = 0 (mm_quantize_rows_e4m3).  Weights are quantized without the
RMSNorm gain; the engine applies the gain to an activation row before quantizing it:
  * prefill, the eval forward and decode steps above 64 samples quantize the four GEMM inputs of each layer (x g1, the
    attention output, x g2, the SwiGLU output) and run mm_gemm_e4m3_fwd with the 16-bit path's epilogues;
  * decode steps with up to 64 samples run mm_gemm_e4m3_thin (the int8 decode kernel on e4m3 weights, activations not
    quantized) ahead of the same mm_thin_fused tails.
"""
from __future__ import annotations

import torch
from torch import nn

PROJECTIONS = (("self_attn", "q_proj"), ("self_attn", "k_proj"), ("self_attn", "v_proj"), ("self_attn", "o_proj"),
               ("mlp", "gate_proj"), ("mlp", "up_proj"), ("mlp", "down_proj"))


class _RowQuantLinear(nn.Module):
    """A bias-free linear layer with per-row quantized weights: y = x (q * scale[:, None])^T.  Computed by the engine's
    kernels only; `weight_scale` stays fp32 when the model is cast to another dtype."""

    QDTYPE = None   # the weight's storage dtype
    FMT = ""        # its name in messages
    QUANTIZE = ""   # the model method that makes such layers

    def __init__(self, weight: torch.Tensor, weight_scale: torch.Tensor):
        super().__init__()
        if weight.dtype != self.QDTYPE or weight.dim() != 2 or weight_scale.dtype != torch.float32 \
                or tuple(weight_scale.shape) != (weight.shape[0],):
            raise TypeError(f"{type(self).__name__}: weight must be {self.FMT} (N, K) and weight_scale fp32 (N,)")
        self.out_features, self.in_features = weight.shape
        self.weight = nn.Parameter(weight, requires_grad=False)
        self.weight_scale = nn.Parameter(weight_scale, requires_grad=False)

    def _apply(self, fn, recurse=True):
        data = {"weight": self.weight.data, "weight_scale": self.weight_scale.data}
        super()._apply(fn, recurse)
        for name, dt in (("weight", self.QDTYPE), ("weight_scale", torch.float32)):
            p = getattr(self, name)
            if p.dtype != dt:  # a dtype cast (model.to(dtype), .half()): the quantized tensors keep their formats
                p.data = data[name].to(p.device)
        return self

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for name, dt in (("weight", self.QDTYPE), ("weight_scale", torch.float32)):
            t = state_dict.get(prefix + name)
            if t is not None and t.dtype != dt:
                error_msgs.append(f"{prefix}{name}: an {self.FMT}-quantized layer loads {dt} values, got {t.dtype} "
                                  f"(load the 16-bit checkpoint before {self.QUANTIZE}())")
                return
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def dequantized(self) -> torch.Tensor:
        """The fp32 weight q * scale the layer stands for."""
        return self.weight.float() * self.weight_scale[:, None]

    def forward(self, x):
        raise RuntimeError(f"{type(self).__name__} runs inside the MM_LLMs engine only; call the model, not the layer")

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, {self.FMT} per-row scales"


class Int8Linear(_RowQuantLinear):
    """Per-row int8 weights (quantize_llm_int8)."""

    QDTYPE, FMT, QUANTIZE = torch.int8, "int8", "quantize_llm_int8"


class Fp8Linear(_RowQuantLinear):
    """Per-row e4m3 weights (quantize_llm_fp8): `weight` float8_e4m3fn (N, K), `weight_scale` fp32 (N,)."""

    QDTYPE, FMT, QUANTIZE = torch.float8_e4m3fn, "e4m3", "quantize_llm_fp8"


def quant_format(model):
    """"int8", "fp8" or None: how the decoder projections of `model` are stored."""
    layers = model.llm.model.layers
    if len(layers) == 0:
        return None
    q = layers[0].self_attn.q_proj
    return "int8" if isinstance(q, Int8Linear) else "fp8" if isinstance(q, Fp8Linear) else None


def is_quantized(model) -> bool:
    return quant_format(model) is not None


def quantize_llm_int8(model) -> None:
    """Quantize the decoder projections of `model` (an MM_LLMs on a CUDA device) in place, one layer at a time."""
    from . import ops

    _quantize(model, "quantize_llm_int8", ops.quantize_rows_int8, Int8Linear)


def quantize_llm_fp8(model) -> None:
    """Per-row e4m3 weights for the decoder projections of `model` (an MM_LLMs on a CUDA device), in place, one layer at
    a time; the engine then also quantizes each GEMM's activation rows (engine.py)."""
    from . import ops

    _quantize(model, "quantize_llm_fp8", ops.quantize_rows_e4m3, Fp8Linear)


def _quantize(model, what, quantize_rows, cls) -> None:
    from . import lora

    if is_quantized(model):
        raise RuntimeError(f"{what}: the decoder is already quantized")
    if lora.adapted_modules(model):
        raise RuntimeError(f"{what}: the model carries LoRA adapters; call merge_lora() first")
    layers = model.llm.model.layers
    for l in layers:
        for parent, name in PROJECTIONS:
            lin = getattr(getattr(l, parent), name)
            if not lin.weight.is_cuda:
                raise RuntimeError(f"{what}: the decoder lives on the CPU; move the model to a CUDA device first "
                                   "(there is no CPU quantization path)")
            if lin.bias is not None:
                raise NotImplementedError(f"{what}: {name} has a bias; LLaMA projections have none")
    eng = model.engine
    eng.drop_derived()  # the fused 16-bit copies go first, so the peak stays at one layer's weights
    model.__dict__.pop("_train_step", None)
    dev = layers[0].self_attn.q_proj.weight.device
    with torch.no_grad(), torch.cuda.device(dev):
        for l in layers:
            for parent, name in PROJECTIONS:
                mod = getattr(l, parent)
                q, s = quantize_rows(getattr(mod, name).weight.detach())
                setattr(mod, name, cls(q, s))
    eng.drop_derived()
