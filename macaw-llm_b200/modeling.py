"""Drop-in class surface of the reference's `modeling.py` for the forward hot path.

  MM_LLMs_Config (alias MM_LLMsConfig)   reference modeling.py:807-861
  MM_LLMs                                reference modeling.py:863-1093
  LlamaForCausalLM / LlamaModel          parameter containers + engine-backed forward for modeling.py:345-659

Constructor kwargs, attribute names and `state_dict()` keys match the reference (SURVEY.md §8b), so
`MM_LLMs(config).load_state_dict(reference_model.state_dict())` is the checkpoint-compatibility mechanism.  The
modules defined here only HOLD parameters; all arithmetic runs through `engine.Engine` on hand-written sm_90a
kernels.  There is no CPU path: calling forward with parameters on the CPU raises.
"""
from __future__ import annotations

import copy
import math
from typing import Optional

import torch
from torch import nn
from transformers import CLIPConfig, CLIPModel, LlamaConfig, WhisperConfig, WhisperModel
from transformers import GenerationConfig, PretrainedConfig, PreTrainedModel
from transformers.modeling_outputs import CausalLMOutputWithPast

from .engine import Engine

# GenerationConfig fields that would add a logits processor, a stopping criterion or another search to HF generate,
# with the test that they are set.  The generate branch implements greedy search and multinomial sampling with
# repetition penalty / temperature / top-k / top-p only, so these are refused rather than ignored.
_UNSUPPORTED_GENERATION = {
    "num_beams": lambda v: v > 1, "num_beam_groups": lambda v: v > 1, "diversity_penalty": lambda v: v != 0.0,
    "num_return_sequences": lambda v: v > 1, "penalty_alpha": lambda v: v is not None,
    "dola_layers": lambda v: v is not None, "guidance_scale": lambda v: v != 1, "constraints": lambda v: bool(v),
    "force_words_ids": lambda v: bool(v), "min_length": lambda v: v > 0, "min_new_tokens": lambda v: v > 0,
    "no_repeat_ngram_size": lambda v: v > 0, "encoder_no_repeat_ngram_size": lambda v: v > 0,
    "encoder_repetition_penalty": lambda v: v != 1.0, "typical_p": lambda v: v < 1.0, "min_p": lambda v: True,
    "top_h": lambda v: True, "epsilon_cutoff": lambda v: v > 0.0, "eta_cutoff": lambda v: v > 0.0,
    "bad_words_ids": lambda v: True, "suppress_tokens": lambda v: True, "begin_suppress_tokens": lambda v: True,
    "sequence_bias": lambda v: True, "forced_bos_token_id": lambda v: True, "forced_eos_token_id": lambda v: True,
    "remove_invalid_values": lambda v: bool(v), "exponential_decay_length_penalty": lambda v: True,
    "renormalize_logits": lambda v: bool(v), "watermarking_config": lambda v: True, "stop_strings": lambda v: True,
    "max_time": lambda v: True, "token_healing": lambda v: bool(v), "prompt_lookup_num_tokens": lambda v: True,
}


def generation_settings(generation_config) -> dict:
    """Decoding keyword arguments of Engine.generate from an HF GenerationConfig, resolved as HF generate resolves them:
    an unset (None) field takes the installed transformers' default (GenerationConfig._get_default_generation_params()).
    A field that would change the search or add another logits processor raises NotImplementedError naming it."""
    defaults = GenerationConfig._get_default_generation_params()

    def get(name):
        v = getattr(generation_config, name, None)
        return defaults.get(name) if v is None else v

    for name, is_set in _UNSUPPORTED_GENERATION.items():
        v = get(name)
        if v is not None and is_set(v):
            raise NotImplementedError(f"macaw_b200: generation_config.{name} = {v!r} is not supported by the generate "
                                      f"branch (greedy search or sampling with repetition_penalty / temperature / "
                                      f"top_k / top_p only)")
    return dict(do_sample=bool(get("do_sample")), temperature=float(get("temperature")), top_k=int(get("top_k") or 0),
                top_p=float(get("top_p")), repetition_penalty=float(get("repetition_penalty")))


# ---------------------------------------------------------------------------------------------------- config
class MM_LLMs_Config(PretrainedConfig):
    """Composite configuration (reference modeling.py:807-861): nested CLIP / Whisper / LLaMA configs plus the
    alignment hyper-parameters.  `hidden_size` is the max of the sub-model widths, as in the reference (:827)."""

    model_type = "mm_llms"
    is_composition = True

    def __init__(self, n_frames=6, attention_heads=8, image_conv_kernel=48, image_conv_stride=36,
                 video_conv_kernel=36, video_conv_stride=30, audio_conv_kernel=240, audio_conv_stride=220,
                 clip_config=None, whisper_config=None, llm_config=None, **kwargs):
        self.image_config = clip_config
        self.audio_config = whisper_config
        self.llm_config = llm_config
        self.n_frames = n_frames
        self.attention_heads = attention_heads
        self.image_conv_kernel, self.image_conv_stride = image_conv_kernel, image_conv_stride
        self.video_conv_kernel, self.video_conv_stride = video_conv_kernel, video_conv_stride
        self.audio_conv_kernel, self.audio_conv_stride = audio_conv_kernel, audio_conv_stride
        if clip_config is not None and whisper_config is not None and llm_config is not None:
            self.hidden_size = max(llm_config.hidden_size, clip_config.projection_dim, whisper_config.d_model)
        kwargs.pop("hidden_size", None)
        kwargs.pop("image_config", None)
        kwargs.pop("audio_config", None)
        super().__init__(**kwargs)

    _NESTED = ("image_config", "audio_config", "llm_config")

    def to_dict(self):
        out = {k: copy.deepcopy(v) for k, v in self.__dict__.items() if k not in self._NESTED}
        for k in self._NESTED:
            sub = getattr(self, k, None)
            out[k] = sub.to_dict() if sub is not None else None
        out["model_type"] = self.__class__.model_type
        return out

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, **kwargs):
        """Reference modeling.py:853-861, plus the `return_unused_kwargs` contract of PretrainedConfig.from_pretrained
        that `PreTrainedModel.from_pretrained(dir)` (no `config=`) relies on: it then expects `(config, unused_kwargs)`."""
        return_unused = bool(kwargs.pop("return_unused_kwargs", False))
        d, kwargs = cls.get_config_dict(pretrained_model_name_or_path, **kwargs)
        names = ("n_frames", "attention_heads", "image_conv_kernel", "image_conv_stride", "video_conv_kernel",
                 "video_conv_stride", "audio_conv_kernel", "audio_conv_stride")
        hyper = {k: d[k] for k in names if k in d}
        unused = {}
        for k, v in kwargs.items():  # explicit overrides of our own hyper-parameters are applied, the rest handed back
            if k in names:
                hyper[k] = v
            else:
                unused[k] = v
        cfg = cls(clip_config=CLIPConfig.from_dict(d["image_config"]),
                  whisper_config=WhisperConfig.from_dict(d["audio_config"]),
                  llm_config=LlamaConfig.from_dict(d["llm_config"]), **hyper)
        if return_unused:
            return cfg, unused
        for k, v in unused.items():  # reference behaviour: remaining kwargs become config attributes (PretrainedConfig(**kwargs))
            setattr(cfg, k, v)
        return cfg


MM_LLMsConfig = MM_LLMs_Config  # BASELINE.json spells it this way


# ---------------------------------------------------------------------------------------------------- LLaMA containers
class _RotaryEmbedding(nn.Module):
    """Holds the persistent `inv_freq` buffer (reference modeling.py:94-98) so state_dict keys match."""

    def __init__(self, dim, base=10000):
        super().__init__()
        self.register_buffer("inv_freq", 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim)))


class _RMSNormWeight(nn.Module):
    def __init__(self, hidden_size, eps):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps


class _LlamaAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        E, H = config.hidden_size, config.num_attention_heads
        if E % H != 0:
            raise ValueError(f"hidden_size must be divisible by num_heads (got `hidden_size`: {E} and `num_heads`: {H}).")
        self.q_proj = nn.Linear(E, E, bias=False)
        self.k_proj = nn.Linear(E, E, bias=False)
        self.v_proj = nn.Linear(E, E, bias=False)
        self.o_proj = nn.Linear(E, E, bias=False)
        self.rotary_emb = _RotaryEmbedding(E // H)


class _LlamaMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.gate_proj = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)
        self.down_proj = nn.Linear(config.intermediate_size, config.hidden_size, bias=False)
        self.up_proj = nn.Linear(config.hidden_size, config.intermediate_size, bias=False)


class _LlamaDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self_attn = _LlamaAttention(config)
        self.mlp = _LlamaMLP(config)
        self.input_layernorm = _RMSNormWeight(config.hidden_size, config.rms_norm_eps)
        self.post_attention_layernorm = _RMSNormWeight(config.hidden_size, config.rms_norm_eps)


class _LlamaPreTrained(PreTrainedModel):
    config_class = LlamaConfig
    base_model_prefix = "model"
    _no_split_modules = ["_LlamaDecoderLayer"]

    def _init_weights(self, module):
        std = getattr(self.config, "initializer_range", 0.02)
        if isinstance(module, nn.Linear):
            nn.init.normal_(module.weight, mean=0.0, std=std)
            if module.bias is not None:
                nn.init.zeros_(module.bias)
        elif isinstance(module, nn.Embedding):
            nn.init.normal_(module.weight, mean=0.0, std=std)


class LlamaModel(_LlamaPreTrained):
    def __init__(self, config):
        super().__init__(config)
        self.padding_idx = config.pad_token_id
        self.vocab_size = config.vocab_size
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, self.padding_idx)
        self.layers = nn.ModuleList([_LlamaDecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = _RMSNormWeight(config.hidden_size, config.rms_norm_eps)
        self.post_init()

    def get_input_embeddings(self):
        return self.embed_tokens

    def set_input_embeddings(self, value):
        self.embed_tokens = value


class _EngineRef:
    """Weak handle from the LLaMA container to the owning MM_LLMs engine that copies / pickles as an EMPTY handle (the
    copy's owner attaches its own engine)."""

    def __init__(self, eng=None):
        import weakref

        self._r = weakref.ref(eng) if eng is not None else None

    def __call__(self):
        return self._r() if self._r is not None else None

    def __deepcopy__(self, memo):
        return _EngineRef()

    def __reduce__(self):
        return (_EngineRef, ())


class LlamaForCausalLM(_LlamaPreTrained):
    """Parameter container with the reference's names; `forward(inputs_embeds=..., attention_mask=..., labels=...)`
    runs on the owning MM_LLMs engine (reference modeling.py:555-622)."""

    def __init__(self, config):
        super().__init__(config)
        self.model = LlamaModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self._engine_ref = _EngineRef()
        self.post_init()
        # read by MM_LLMs' generate branch as HF generate reads it (this class is not a GenerationMixin, so transformers
        # leaves the attribute None); assignable, e.g. from a checkpoint's generation_config.json
        self.generation_config = GenerationConfig.from_model_config(config)

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def get_output_embeddings(self):
        return self.lm_head

    def set_output_embeddings(self, new_embeddings):
        self.lm_head = new_embeddings

    def forward(self, input_ids=None, attention_mask=None, inputs_embeds=None, labels=None, **unused):
        eng = self._engine_ref()
        if eng is None:
            raise RuntimeError("LlamaForCausalLM must be owned by an MM_LLMs module to run (engine not attached)")
        from . import ops

        if (input_ids is None) == (inputs_embeds is None):
            raise ValueError("You have to specify exactly one of input_ids or inputs_embeds")
        with torch.no_grad():
            eng.set_format()
            if inputs_embeds is None:
                table = eng.w(self.model.embed_tokens.weight, "llm.embed")
                B, L = input_ids.shape
                inputs_embeds = ops.embed_gather(table, input_ids.to(table.device)).view(B, L, -1)
            elif inputs_embeds.dtype != ops.ACT():
                inputs_embeds = inputs_embeds.to(ops.ACT())
            logits = eng.llama_forward(inputs_embeds, attention_mask)
            loss = None
            if labels is not None:
                loss = ops.ce_loss(logits, labels.to(logits.device).to(torch.int64).contiguous())
        return CausalLMOutputWithPast(loss=loss, logits=logits)


# ---------------------------------------------------------------------------------------------------- MM_LLMs
class MM_LLMs(PreTrainedModel):
    """Reference modeling.py:863-1093.  Same sub-module / parameter names (including the parameters the reference
    creates but never reaches from forward: temporal_self_attention, temporal_position_embeddings, logit_scale,
    layer_norm), same `forward(inputs)` contract, same return type."""

    config_class = MM_LLMs_Config
    base_model_prefix = "mm_llms"

    def __init__(self, config):
        super().__init__(config)
        self.config = config
        P = config.image_config.projection_dim
        E = config.llm_config.hidden_size
        A = config.audio_config.d_model

        self.temporal_position_embeddings = nn.Embedding(config.n_frames, P)
        self.image_encoder = CLIPModel(config.image_config)
        self.video_encoder = CLIPModel(config.image_config)
        self.audio_encoder = WhisperModel(config.audio_config)
        self.llm = LlamaForCausalLM(config.llm_config)

        def mha(dim, heads):
            return nn.MultiheadAttention(dim, heads, dropout=0.1, add_bias_kv=True, add_zero_attn=True)

        self.temporal_self_attention = mha(P, config.attention_heads)
        self.video_align_attention = mha(E, config.attention_heads * 2)
        self.audio_align_attention = mha(E, config.attention_heads * 2)
        self.image_align_attention = mha(E, config.attention_heads * 2)
        self.video_long_self_attention = mha(P, config.attention_heads)

        self.transform_video_to_hidden = nn.Linear(P, E)
        self.transform_audio_to_hidden = nn.Linear(A, E)
        self.transform_image_to_hidden = nn.Linear(P, E)

        self.project_image = nn.Conv1d(P, P, kernel_size=config.image_conv_kernel, stride=config.image_conv_stride)
        self.project_video = nn.Conv1d(P, P, kernel_size=config.video_conv_kernel, stride=config.video_conv_stride)
        self.project_audio = nn.Conv1d(A, A, kernel_size=config.audio_conv_kernel, stride=config.audio_conv_stride)

        self.logit_scale = nn.Parameter(torch.ones([]) * math.log(1 / 0.07))
        self.layer_norm = nn.LayerNorm(P)

        self._attach_engine()
        self.post_init()

    # the engine is not a sub-module and must not be (de)serialised or deep-copied with the parameters: a copy of the
    # model gets its OWN engine (weight caches and CUDA graphs are keyed by the parameters of the owning module)
    @property
    def engine(self) -> Engine:
        return self._engine

    def _attach_engine(self):
        self.__dict__["_engine"] = Engine(self)
        self.llm._engine_ref = _EngineRef(self._engine)

    def __deepcopy__(self, memo):
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k not in ("_engine", "_train_step"):
                new.__dict__[k] = copy.deepcopy(v, memo)
        new._attach_engine()
        return new

    def __getstate__(self):
        st = dict(self.__dict__)
        st.pop("_engine", None)
        st.pop("_train_step", None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self._attach_engine()

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Conv1d, nn.Conv2d)):
            nn.init.normal_(module.weight, mean=0.0, std=0.02)
            if module.bias is not None:
                nn.init.zeros_(module.bias)
        elif isinstance(module, nn.Embedding):
            nn.init.normal_(module.weight, mean=0.0, std=0.02)
        elif isinstance(module, nn.LayerNorm):
            nn.init.ones_(module.weight)
            nn.init.zeros_(module.bias)

    # ---- reference-facing API -------------------------------------------------------------------------------
    def forward(self, inputs=None):
        """inputs: dict with images (B,3,H,W) | None, audios (B,80,3000) | None, videos (B,F,3,H,W) | None,
        input_ids (B,L), optional attention_mask (B,L), labels (B,L) | None, {image,audio,video}_{starts,ends} (B,),
        optional `inference: True` (generation, returns token ids; `max_new_tokens` defaults to the reference's 128;
        greedy or sampled as `self.llm.generation_config` says) (reference modeling.py:941-963, llm_trainer.py:366-381)."""
        if inputs.get("inference") is True:
            # generate branch (reference modeling.py:954-960): greedy or sampled decode, returns the new token ids
            # (B, <= 128); every other decoding parameter comes from llm.generation_config, as in HF generate
            return self._engine.generate(inputs, max_new_tokens=int(inputs.get("max_new_tokens", 128)),
                                         eos_token_id=2, pad_token_id=32006,
                                         **generation_settings(self.llm.generation_config))
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return self._forward_train(inputs)
        loss, logits, _, _, _ = self._engine.forward(inputs)
        return CausalLMOutputWithPast(loss=loss, logits=logits)

    def _forward_train(self, inputs):
        """train() mode with gradients enabled (reference llm_trainer.py:184-188: `loss = model(**inputs)[0]`, then
        `loss.backward()`): the loss is produced by the kernel-library training step (training.py) and carries a grad_fn
        whose backward runs the hand-written backward pass.  Logits are not returned in this mode (they are consumed in
        place by the cross-entropy backward)."""
        from .quant import quant_format
        from .training import TrainStep

        fmt = quant_format(self)
        if fmt == "int8":
            raise RuntimeError("macaw_b200: the decoder is int8-quantized (quantize_llm_int8) and cannot be trained; call "
                               "model.eval() / torch.no_grad() for inference")
        if fmt == "fp8":
            raise RuntimeError("macaw_b200: the decoder is FP8-quantized (quantize_llm_fp8) and cannot be trained; call "
                               "model.eval() / torch.no_grad() for inference")
        if "_train_step" not in self.__dict__:
            self.__dict__["_train_step"] = TrainStep(self)
        if inputs.get("labels") is None:
            raise ValueError("macaw_b200: a train()-mode forward needs `labels` (the differentiated quantity is the loss); "
                             "call model.eval() / torch.no_grad() for logits")
        loss = self.__dict__["_train_step"](inputs)
        return CausalLMOutputWithPast(loss=loss, logits=None)

    @property
    def train_step(self):
        from .training import TrainStep

        if "_train_step" not in self.__dict__:
            self.__dict__["_train_step"] = TrainStep(self)
        return self.__dict__["_train_step"]

    # ---- LoRA adapters on the decoder (lora.py; reference run_clm_llms.py:498-508, run_clm_llms_inference.py:88-94) ----
    def add_lora(self, config):
        """`get_peft_model(model.llm, config)`: adapters on the targeted decoder projections, base decoder frozen."""
        from . import lora

        return lora.add_lora(self, config)

    def save_lora(self, directory: str) -> None:
        """PEFT's adapter layout: adapter_config.json + adapter_model.bin."""
        from . import lora

        lora.save_lora(self, directory)

    def load_lora(self, directory: str) -> None:
        """`PeftModel.from_pretrained(model.llm, directory)` (adds the adapters first when the model has none)."""
        from . import lora

        lora.load_lora(self, directory)

    def merge_lora(self) -> None:
        """`merge_and_unload()`: the adapters are folded into the base weights and removed."""
        from . import lora

        lora.merge_lora(self)

    # ---- int8 decoder weights (quant.py) ----
    def quantize_llm_int8(self) -> None:
        """Weight-only int8 for the seven projections of every decoder layer (per-row fp32 scales), in place; inference
        only.  lm_head, embed_tokens, the norms, the alignment blocks and the encoders stay 16-bit."""
        from . import quant

        quant.quantize_llm_int8(self)

    def quantize_llm_fp8(self) -> None:
        """Per-row e4m3 weights for the seven projections of every decoder layer, in place; the prefill GEMMs then run on
        FP8 tensor cores with per-row e4m3 activations.  Inference only; what stays 16-bit is as for quantize_llm_int8."""
        from . import quant

        quant.quantize_llm_fp8(self)

    def enable_int8_kv_cache(self, flag: bool = True) -> None:
        """Generate with an int8 KV cache (per-(token, head) fp32 scales; Engine.enable_int8_kv_cache), or with the
        16-bit cache again (flag=False).  Affects `inputs['inference'] = True` only; off by default."""
        self._engine.enable_int8_kv_cache(flag)

    def prepare_inputs_for_generation(self, inputs):
        return self._engine.prepare_inputs(inputs)

    def encode_image(self, images):
        eng = self._engine
        dev = eng.w(self.llm.model.embed_tokens.weight, "llm.embed").device
        return eng.clip_tokens(eng._to_dev_bf16(images, dev), "image_encoder")

    def encode_audio(self, audios):
        eng = self._engine
        dev = eng.w(self.llm.model.embed_tokens.weight, "llm.embed").device
        return eng.whisper_encode(eng._to_dev_bf16(audios, dev))

    def encode_video_long(self, videos):
        eng = self._engine
        dev = eng.w(self.llm.model.embed_tokens.weight, "llm.embed").device
        return eng.encode_video_long(eng._to_dev_bf16(videos, dev))

    # ---- construction helper for benchmarks ----------------------------------------------------------------
    @classmethod
    def build_random(cls, config, device="cuda", dtype=torch.bfloat16, seed: int = 0, std: float = 0.02):
        """Random-init model materialised directly on `device` in `dtype` (no 28 GB fp32 CPU detour).  Norm weights
        are 1, biases 0, everything else N(0, std) from a device generator — the same family the reference's
        `init_weights()` draws from; used by bench.py / smoke() where no checkpoint exists."""
        try:
            from transformers.initialization import no_init_weights
        except ImportError:  # older transformers
            from transformers.modeling_utils import no_init_weights

        prev = torch.get_default_dtype()
        torch.set_default_dtype(dtype)
        try:
            with torch.device(device), no_init_weights():
                model = cls(config)
        finally:
            torch.set_default_dtype(prev)
        g = torch.Generator(device=device).manual_seed(seed)
        with torch.no_grad():
            for name, p in model.named_parameters():
                if p.dim() == 0:
                    p.fill_(math.log(1 / 0.07))
                elif p.dim() == 1 and (("norm" in name.lower() and name.endswith("weight")) or "layrnorm.weight" in name):
                    p.fill_(1.0)
                elif p.dim() == 1:
                    p.zero_()
                else:
                    p.normal_(0.0, std, generator=g)
            for name, b in model.named_buffers():
                if name.endswith("inv_freq"):
                    hd = b.numel() * 2
                    b.copy_(1.0 / (10000 ** (torch.arange(0, hd, 2, device=b.device).float() / hd)))
                elif name.endswith("position_ids"):
                    b.copy_(torch.arange(b.shape[-1], device=b.device).expand_as(b))
        return model.eval()
