"""Low-rank adaptation (LoRA) of the LLaMA decoder, with PEFT's configuration, initialisation and adapter file layout.

Reference: run_clm_llms.py:498-508 wraps the decoder with
    LoraConfig(r=8, lora_alpha=16, lora_dropout=0.05, bias="none", task_type="CAUSAL_LM", target_modules=[...])
    model.llm = get_peft_model(model.llm, lora_config)
and run_clm_llms_inference.py:73, 88-94 loads adapters with PeftModel / the adapter state-dict helpers.

Here the adapters are registered as children of the adapted nn.Linear modules (`q_proj.lora_A`, `q_proj.lora_B`) and
`model.llm` is NOT wrapped: `model.llm.model.embed_tokens` and every base state_dict key keep their names.  The adapted
linear computes PEFT's `Linear.forward`:  y = x W^T + s * drop(x) A^T B^T,  s = lora_alpha / r.

    cfg = LoraConfig(r=8, lora_alpha=16, lora_dropout=0.05, target_modules=["q_proj", "v_proj"])
    model.add_lora(cfg)                  # get_peft_model(model.llm, cfg): base frozen, A kaiming-uniform, B zeros
    ...train...
    model.save_lora("out/")              # adapter_config.json + adapter_model.bin, PEFT's keys
    model.load_lora("out/")              # PeftModel.from_pretrained(model.llm, "out/")
    model.merge_lora()                   # merge_and_unload(): W <- round(W + s B A), adapters removed

The training step runs the adapters on kernels of their own (csrc/lora.cu, `ops.lora_*`); evaluation and generation fold
them into the engine's derived weights through `merged_weight`, the same function `merge_lora` uses.
"""
from __future__ import annotations

import json
import math
import os
import re
from typing import Dict, List, Optional, Sequence

import torch
from torch import nn

# modules LoRA can adapt, by their name inside model.llm; the index is the adapter's Philox stream offset in its layer
TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
LM_HEAD = "lm_head"
PEFT_LLAMA_DEFAULT = ("q_proj", "v_proj")  # PEFT's TRANSFORMERS_MODELS_TO_LORA_TARGET_MODULES_MAPPING["llama"]

# Philox stream ids of the adapters' input dropout (csrc/philox.cuh: SID_LORA_LM_HEAD, SID_LORA0)
SID_LORA_LM_HEAD = 24
SID_LORA0 = 32


def lora_sid(layer: Optional[int], target: str) -> int:
    """Stream id of the dropout mask of one adapter: decoder layer `layer`, projection `target` (layer None: lm_head)."""
    if target == LM_HEAD:
        return SID_LORA_LM_HEAD
    return SID_LORA0 + 8 * int(layer) + TARGETS.index(target)


class LoraConfig:
    """PEFT's LoraConfig restricted to what this package implements (plain LoRA on nn.Linear, no bias training).

    r            rank: a multiple of 8 in [8, 64] (16-byte aligned gradient views, the kernels' tiling)
    lora_alpha   scaling = lora_alpha / r (PEFT without rsLoRA)
    lora_dropout dropout probability on the adapter's input, in [0, 1)
    target_modules  module-name suffixes inside model.llm (a list), or one regular expression the full module name must
                 match (a string), as PEFT reads them; None = PEFT's LLaMA default ("q_proj", "v_proj").  Names
                 matching no module are ignored, as PEFT ignores them; `embed_tokens` is refused
    bias         "none" only
    task_type    "CAUSAL_LM" (or None), the reference's value; it is written to adapter_config.json
    Any other PEFT field is refused with NotImplementedError naming it."""

    def __init__(self, r: int = 8, lora_alpha: float = 16, lora_dropout: float = 0.0,
                 target_modules: Optional[Sequence[str]] = None, bias: str = "none", task_type: Optional[str] = "CAUSAL_LM",
                 **unsupported):
        for name in unsupported:
            raise NotImplementedError(f"macaw_b200 LoRA: LoraConfig.{name} is not supported (fields: r, lora_alpha, "
                                      f"lora_dropout, target_modules, bias='none', task_type='CAUSAL_LM')")
        if isinstance(r, bool) or int(r) != r or not (8 <= r <= 64 and r % 8 == 0):
            raise ValueError(f"macaw_b200 LoRA: r must be a multiple of 8 in [8, 64], got {r!r}")
        if bias != "none":
            raise NotImplementedError(f"macaw_b200 LoRA: LoraConfig.bias = {bias!r} is not supported (only 'none')")
        if task_type not in (None, "CAUSAL_LM"):
            raise NotImplementedError(f"macaw_b200 LoRA: LoraConfig.task_type = {task_type!r} is not supported "
                                      "(only 'CAUSAL_LM')")
        if not 0.0 <= float(lora_dropout) < 1.0:
            raise ValueError(f"macaw_b200 LoRA: lora_dropout must be in [0, 1), got {lora_dropout!r}")
        if not float(lora_alpha) > 0:
            raise ValueError(f"macaw_b200 LoRA: lora_alpha must be > 0, got {lora_alpha!r}")
        self.r, self.lora_alpha, self.lora_dropout = int(r), lora_alpha, float(lora_dropout)
        if target_modules is None:
            target_modules = PEFT_LLAMA_DEFAULT
        self.target_modules = target_modules if isinstance(target_modules, str) else list(target_modules)
        self.bias, self.task_type = bias, task_type

    @property
    def scaling(self) -> float:
        return self.lora_alpha / self.r

    def to_dict(self) -> dict:
        """The adapter_config.json fields PEFT writes and reads for this adapter."""
        tm = self.target_modules if isinstance(self.target_modules, str) else list(self.target_modules)
        return dict(peft_type="LORA", task_type=self.task_type or "CAUSAL_LM", r=self.r, lora_alpha=self.lora_alpha,
                    lora_dropout=self.lora_dropout, target_modules=tm, bias=self.bias, fan_in_fan_out=False)

    # adapter_config.json fields of PEFT that change the adapter's arithmetic or layout, with the value under which this
    # package computes what PEFT computes; any other value is refused.  Other keys (base_model_name_or_path, revision,
    # inference_mode, init_lora_weights, peft_version, ...) do not affect a loaded adapter.
    _PEFT_DEFAULTS = {"fan_in_fan_out": False, "use_rslora": False, "use_dora": False, "rank_pattern": {},
                      "alpha_pattern": {}, "layers_to_transform": None, "layers_pattern": None, "modules_to_save": None,
                      "layer_replication": None, "megatron_config": None, "loftq_config": {}, "exclude_modules": None,
                      "lora_bias": False, "use_qalora": False, "target_parameters": None, "trainable_token_indices": None}

    @classmethod
    def from_dict(cls, d: dict) -> "LoraConfig":
        """The config of a PEFT adapter_config.json; a field that would make PEFT compute something else is refused."""
        if d.get("peft_type", "LORA") != "LORA":
            raise NotImplementedError(f"macaw_b200 LoRA: peft_type {d.get('peft_type')!r} is not supported")
        for name, default in cls._PEFT_DEFAULTS.items():
            v = d.get(name, default)
            if v != default and not (v in (None, {}, [], False) and default in (None, {}, [], False)):
                raise NotImplementedError(f"macaw_b200 LoRA: adapter_config.json {name} = {v!r} is not supported")
        return cls(r=d["r"], lora_alpha=d["lora_alpha"], lora_dropout=d.get("lora_dropout", 0.0),
                   target_modules=d.get("target_modules"), bias=d.get("bias", "none"), task_type=d.get("task_type"))

    def __repr__(self) -> str:
        return (f"LoraConfig(r={self.r}, lora_alpha={self.lora_alpha}, lora_dropout={self.lora_dropout}, "
                f"target_modules={self.target_modules!r}, bias={self.bias!r})")


def resolve_targets(llm: nn.Module, config: LoraConfig) -> Dict[str, nn.Linear]:
    """{name inside model.llm: nn.Linear} of the modules `config.target_modules` selects, matched by name suffix as PEFT
    matches them (the full name, or a suffix after a '.').  Raises for `embed_tokens`, for a matched module that is not a
    supported projection, and when no name matches anything."""
    wanted = config.target_modules

    def selected(name: str) -> bool:
        if isinstance(wanted, str):  # PEFT: a string is a regular expression over the full module name
            return re.fullmatch(wanted, name) is not None
        return any(name == t or name.endswith("." + t) for t in wanted)

    if selected("model.embed_tokens") or (not isinstance(wanted, str) and "embed_tokens" in wanted):
        raise NotImplementedError("macaw_b200 LoRA: target 'embed_tokens' is not supported (the alignment attention reads "
                                  "embed_tokens.weight; an embedding adapter would change only the gathered rows)")
    out = {}
    for name, mod in llm.named_modules():
        if not name or not selected(name):
            continue
        leaf = name.rsplit(".", 1)[-1]
        if leaf not in TARGETS + (LM_HEAD,) or not isinstance(mod, nn.Linear):
            raise ValueError(f"macaw_b200 LoRA: module {name!r} ({type(mod).__name__}) cannot be adapted; supported: "
                             f"{', '.join(TARGETS + (LM_HEAD,))}")
        out[name] = mod
    if not out:
        raise ValueError(f"macaw_b200 LoRA: target_modules {wanted} match no module of the decoder")
    return out


def is_adapted(lin: nn.Module) -> bool:
    return isinstance(lin, nn.Linear) and "lora_A" in lin._modules


def adapted_modules(model) -> Dict[str, nn.Linear]:
    """{name inside model.llm: nn.Linear} of the modules carrying an adapter."""
    return {n: m for n, m in model.llm.named_modules() if n and is_adapted(m)}


def merged_weight(lin: nn.Linear) -> torch.Tensor:
    """The effective weight of a linear layer in fp32: W + scaling * B A for an adapted one (product and sum in fp32),
    W itself otherwise.  `merge_lora` rounds it into W; the engine folds it into its derived weights."""
    w = lin.weight.detach().float()
    if is_adapted(lin):
        w = w + lin.lora_scaling * (lin.lora_B.weight.detach().float() @ lin.lora_A.weight.detach().float())
    return w


def weight_params(lin: nn.Linear) -> List[torch.Tensor]:
    """The parameters `merged_weight(lin)` depends on (the engine's weight cache is keyed on their versions)."""
    if is_adapted(lin):
        return [lin.weight, lin.lora_A.weight, lin.lora_B.weight]
    return [lin.weight]


def add_lora(model, config: LoraConfig) -> Dict[str, nn.Linear]:
    """get_peft_model(model.llm, config) without the wrapper: registers lora_A (nn.Linear(in, r)) and lora_B
    (nn.Linear(r, out)) under every targeted linear, on its device and in its dtype, A kaiming-uniform(a = sqrt(5)) and
    B zeros as PEFT initialises them; freezes every base parameter of model.llm (the alignment modules and
    video_long_self_attention stay trainable, the encoders are frozen as in the reference).  -> the adapted modules."""
    if not isinstance(config, LoraConfig):
        raise TypeError(f"add_lora: expected a LoraConfig, got {type(config).__name__}")
    if adapted_modules(model):
        raise RuntimeError("add_lora: the model already carries adapters (merge_lora() first; one adapter at a time)")
    from .quant import quant_format

    fmt = quant_format(model)
    if fmt is not None:
        raise RuntimeError(f"add_lora: the decoder is {'int8' if fmt == 'int8' else 'FP8'}-quantized; LoRA needs the 16-bit "
                           "base weights")
    targets = resolve_targets(model.llm, config)
    from .training import freeze_like_reference

    for p in model.llm.parameters():
        p.requires_grad_(False)
    freeze_like_reference(model)
    for name, lin in targets.items():
        w = lin.weight
        A = nn.Linear(lin.in_features, config.r, bias=False, device=w.device, dtype=w.dtype)
        Bm = nn.Linear(config.r, lin.out_features, bias=False, device=w.device, dtype=w.dtype)
        with torch.no_grad():
            nn.init.kaiming_uniform_(A.weight, a=math.sqrt(5))
            nn.init.zeros_(Bm.weight)
        lin.lora_A, lin.lora_B = A, Bm
        lin.lora_scaling = config.scaling
    model.__dict__["_lora_config"] = config
    _drop_grad_buffer(model)
    return targets


def _drop_grad_buffer(model) -> None:
    """The trainable set changed: the next backward builds a new gradient buffer."""
    ts = model.__dict__.get("_train_step")
    if ts is not None:
        ts.llama.grads = None


def lora_config(model) -> Optional[LoraConfig]:
    return model.__dict__.get("_lora_config") if adapted_modules(model) else None


def lora_state_dict(model) -> Dict[str, torch.Tensor]:
    """The adapter weights under PEFT's keys: base_model.model.<name inside model.llm>.lora_{A,B}.weight."""
    out = {}
    for name, lin in adapted_modules(model).items():
        out[f"base_model.model.{name}.lora_A.weight"] = lin.lora_A.weight.detach()
        out[f"base_model.model.{name}.lora_B.weight"] = lin.lora_B.weight.detach()
    return out


def save_lora(model, directory: str) -> None:
    """PEFT's save_pretrained layout: adapter_config.json and adapter_model.bin (torch.save of lora_state_dict)."""
    cfg = lora_config(model)
    if cfg is None:
        raise RuntimeError("save_lora: the model carries no adapters")
    os.makedirs(directory, exist_ok=True)
    with open(os.path.join(directory, "adapter_config.json"), "w") as f:
        json.dump(cfg.to_dict(), f, indent=2, sort_keys=True)
    torch.save({k: v.cpu().clone() for k, v in lora_state_dict(model).items()}, os.path.join(directory, "adapter_model.bin"))


def load_lora(model, directory: str) -> None:
    """PeftModel.from_pretrained(model.llm, directory): adds adapters with the stored config when the model has none,
    then copies the stored weights in.  Every stored key must name an adapter of the model and the other way round."""
    with open(os.path.join(directory, "adapter_config.json")) as f:
        cfg = LoraConfig.from_dict(json.load(f))
    if not adapted_modules(model):
        add_lora(model, cfg)
    else:
        have = lora_config(model)
        if (have.r, float(have.lora_alpha)) != (cfg.r, float(cfg.lora_alpha)):
            raise ValueError(f"load_lora: the stored adapter has r={cfg.r}, lora_alpha={cfg.lora_alpha}; the model's has "
                             f"r={have.r}, lora_alpha={have.lora_alpha}")
    sd = torch.load(os.path.join(directory, "adapter_model.bin"), map_location="cpu", weights_only=True)
    mine = {f"base_model.model.{n}.{ab}.weight": getattr(lin, ab).weight
            for n, lin in adapted_modules(model).items() for ab in ("lora_A", "lora_B")}
    if set(sd) != set(mine):
        raise ValueError(f"load_lora: adapter keys differ: missing {sorted(set(mine) - set(sd))[:4]}, "
                         f"unexpected {sorted(set(sd) - set(mine))[:4]}")
    with torch.no_grad():
        for k, p in mine.items():
            if tuple(sd[k].shape) != tuple(p.shape):
                raise ValueError(f"load_lora: {k} has shape {tuple(sd[k].shape)}, the model's is {tuple(p.shape)}")
            p.copy_(sd[k])


def merge_lora(model) -> None:
    """merge_and_unload(): W <- round(W + scaling * B A) (fp32 product and sum, one rounding into W's format) and the
    adapters are removed.  The base parameters keep their requires_grad flags."""
    with torch.no_grad():
        for lin in adapted_modules(model).values():
            lin.weight.copy_(merged_weight(lin).to(lin.weight.dtype))
            del lin.lora_A, lin.lora_B
            del lin.lora_scaling
    model.__dict__.pop("_lora_config", None)
    _drop_grad_buffer(model)
