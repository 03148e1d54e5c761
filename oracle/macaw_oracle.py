"""CPU oracle for the MM_LLMs forward hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` leg may import this module; the
product path (macaw-llm_b200/) never does and fails loudly when its CUDA library is missing.

What it is: a plain-torch fp32 restatement, on CPU, of the arithmetic the reference executes for
`MM_LLMs.forward` (/root/reference/modeling.py), written as pure functions over a `state_dict` so that it does not
depend on the transformers version for its *arithmetic* (CLIP / Whisper encoder math is restated here too).
Each function cites the reference lines (or the third-party lines the reference delegates to) it follows.

Pin: the reference ships no tests or golden vectors (SURVEY.md §4, §8c).  The pin is therefore the reference ITSELF,
imported in-process in the build container by tests/golden/make_golden.py (which cannot travel to the GPU box):
that script runs the unmodified /root/reference/modeling.py on seeded tiny configurations, checks this oracle
against it (run in fp64; measured max |d| 2e-9 on embeds / 7e-7 on logits — the reference softmaxes in fp32 even in fp64
mode — asserted at 1e-6 / 1e-5) and commits inputs/outputs as fixtures under tests/golden/.  tests/test_oracle.py re-checks
the oracle against those fixtures everywhere, and against the live reference when /root/reference exists.

Third-party arithmetic the reference delegates to (absent from /root/reference):
  torch == 2.0.0 (requirements.txt:1)           nn.MultiheadAttention, Conv1d, Linear, Embedding, CrossEntropyLoss
  transformers == 4.29.0 (requirements.txt:24)  CLIPModel.vision_model / visual_projection, WhisperModel.encoder
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# ------------------------------------------------------------------------------------------------ hyper-parameters
def hp_from_config(cfg) -> dict:
    """Flatten an MM_LLMs_Config-like object (modeling.py:807-829) into plain numbers."""
    ic, ac, lc = cfg.image_config, cfg.audio_config, cfg.llm_config
    vc = ic.vision_config
    return dict(
        n_frames=cfg.n_frames, attention_heads=cfg.attention_heads,
        image_conv=(cfg.image_conv_kernel, cfg.image_conv_stride),
        video_conv=(cfg.video_conv_kernel, cfg.video_conv_stride),
        audio_conv=(cfg.audio_conv_kernel, cfg.audio_conv_stride),
        clip=dict(hidden=vc.hidden_size, layers=vc.num_hidden_layers, heads=vc.num_attention_heads,
                  patch=vc.patch_size, image_size=vc.image_size, eps=vc.layer_norm_eps, act=vc.hidden_act,
                  proj=ic.projection_dim),
        whisper=dict(d_model=ac.d_model, layers=ac.encoder_layers, heads=ac.encoder_attention_heads,
                     act=ac.activation_function, max_pos=ac.max_source_positions),
        llama=dict(hidden=lc.hidden_size, layers=lc.num_hidden_layers, heads=lc.num_attention_heads,
                   eps=lc.rms_norm_eps, vocab=lc.vocab_size),
    )


def _act(name: str):
    if name == "quick_gelu":
        return lambda x: x * torch.sigmoid(1.702 * x)
    if name == "gelu":
        return F.gelu
    if name in ("silu", "swish"):
        return F.silu
    raise ValueError(f"oracle: unsupported activation {name}")


class _SD:
    """state_dict view that upcasts on access (so bf16 checkpoints can be consumed layer by layer)."""

    def __init__(self, sd: Dict[str, Tensor], dtype=torch.float32, prefix: str = "", keep_graph: bool = False):
        self.sd, self.dtype, self.prefix, self.keep_graph = sd, dtype, prefix, keep_graph

    def __call__(self, name: str) -> Tensor:
        t = self.sd[self.prefix + name]
        if self.keep_graph:  # gradient oracle: the tensors are autograd leaves (already on the CPU in the working dtype)
            return t
        return t.detach().to("cpu").to(self.dtype)

    def has(self, name: str) -> bool:
        return (self.prefix + name) in self.sd

    def sub(self, prefix: str) -> "_SD":
        return _SD(self.sd, self.dtype, self.prefix + prefix, self.keep_graph)


# ------------------------------------------------------------------------------------------------ torch MHA restatement
def mha_forward(query: Tensor, key: Tensor, value: Tensor, w: _SD, num_heads: int,
                dropout_mult: Optional[Tensor] = None) -> Tensor:
    """nn.MultiheadAttention(E, H, add_bias_kv=True, add_zero_attn=True), seq-first layout; eval mode unless
    `dropout_mult` is given: the (B*H, Lq, S+2) multipliers (0 or 1/(1-p)) F.dropout would apply to the softmax
    probabilities in train() mode (functional.py:6640-6645, dropout_p = 0.1 from modeling.py:879) — passed explicitly so
    the gradient oracle and the device kernels use the SAME mask.

    Follows torch/nn/functional.py multi_head_attention_forward (SURVEY.md Appendix A):
      in-projection (functional.py:5798-5868), bias_k/bias_v appended AFTER projection (:6531-6537), head split,
      one zero key/value per head appended (:6585-6602), q scaled by 1/sqrt(hd) (:6632), softmax, PV, out_proj
      (:6647-6653).  Call sites: modeling.py:986-987, 1007-1008, 1025-1026, 1078.
    query (Lq, B, E), key/value (S, B, E) -> (Lq, B, E).
    """
    Lq, B, E = query.shape
    S = key.shape[0]
    hd = E // num_heads
    W, bias = w("in_proj_weight"), w("in_proj_bias")
    q = F.linear(query, W[:E], bias[:E])
    k = F.linear(key, W[E:2 * E], bias[E:2 * E])
    v = F.linear(value, W[2 * E:], bias[2 * E:])
    k = torch.cat([k, w("bias_k").expand(1, B, E)], dim=0)
    v = torch.cat([v, w("bias_v").expand(1, B, E)], dim=0)
    q = q.reshape(Lq, B * num_heads, hd).transpose(0, 1)
    k = k.reshape(S + 1, B * num_heads, hd).transpose(0, 1)
    v = v.reshape(S + 1, B * num_heads, hd).transpose(0, 1)
    zeros = torch.zeros(B * num_heads, 1, hd, dtype=k.dtype, device=k.device)
    k = torch.cat([k, zeros], dim=1)
    v = torch.cat([v, zeros], dim=1)
    q = q * (1.0 / math.sqrt(hd))
    p = torch.softmax(torch.bmm(q, k.transpose(1, 2)), dim=-1)
    if dropout_mult is not None:
        p = p * dropout_mult.to(p.dtype)
    ctx = torch.bmm(p, v).transpose(0, 1).reshape(Lq, B, E)
    return F.linear(ctx, w("out_proj.weight"), w("out_proj.bias"))


def align_block(feats: Tensor, table: Tensor, conv: _SD, lin: _SD, mha: _SD, stride: int, num_heads: int,
                dropout_mult: Optional[Tensor] = None) -> Tensor:
    """One modality of modeling.py:982-987 / 999-1008 / 1022-1026: Conv1d over tokens -> Linear C->E -> MHA(Q=feats,
    K=V=the whole embedding table).  The reference repeats the table per batch element (modeling.py:974-975); K/V
    are batch-invariant, so this restatement projects them once and broadcasts — numerically the same function.
    feats (B, N, C), table (V, E) -> (B, Lq, E)."""
    y = F.conv1d(feats.transpose(1, 2), conv("weight"), conv("bias"), stride=stride).transpose(1, 2)
    z = F.linear(y, lin("weight"), lin("bias"))
    B = z.shape[0]
    kv = table.unsqueeze(1).expand(-1, B, -1)
    return mha_forward(z.transpose(0, 1), kv, kv, mha, num_heads, dropout_mult).transpose(0, 1)


# ------------------------------------------------------------------------------------------------ CLIP vision tower
def clip_tokens(images: Tensor, w: _SD, hp: dict) -> Tensor:
    """`visual_projection(vision_model(images)[0])[:, 1:, :]` (modeling.py:1092): the UN-pooled last hidden state (no
    post_layernorm), projected per token, CLS dropped.  Restates transformers modeling_clip.py CLIPVisionEmbeddings
    (:138-219), CLIPAttention / CLIPMLP / CLIPEncoderLayer (:261-386), CLIPVisionTransformer.forward (:667-691)."""
    c = hp["clip"]
    vm = w.sub("vision_model.")
    B = images.shape[0]
    x = F.conv2d(images, vm("embeddings.patch_embedding.weight"), stride=c["patch"]).flatten(2).transpose(1, 2)
    cls = vm("embeddings.class_embedding").expand(B, 1, -1)
    x = torch.cat([cls, x], dim=1) + vm("embeddings.position_embedding.weight")[None]
    D, H = c["hidden"], c["heads"]
    hd = D // H
    x = F.layer_norm(x, (D,), vm("pre_layrnorm.weight"), vm("pre_layrnorm.bias"), c["eps"])
    act = _act(c["act"])
    for i in range(c["layers"]):
        l = vm.sub(f"encoder.layers.{i}.")
        h = F.layer_norm(x, (D,), l("layer_norm1.weight"), l("layer_norm1.bias"), c["eps"])
        q = F.linear(h, l("self_attn.q_proj.weight"), l("self_attn.q_proj.bias")).view(B, -1, H, hd).transpose(1, 2)
        k = F.linear(h, l("self_attn.k_proj.weight"), l("self_attn.k_proj.bias")).view(B, -1, H, hd).transpose(1, 2)
        v = F.linear(h, l("self_attn.v_proj.weight"), l("self_attn.v_proj.bias")).view(B, -1, H, hd).transpose(1, 2)
        p = torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1)
        a = (p @ v).transpose(1, 2).reshape(B, -1, D)
        x = x + F.linear(a, l("self_attn.out_proj.weight"), l("self_attn.out_proj.bias"))
        h = F.layer_norm(x, (D,), l("layer_norm2.weight"), l("layer_norm2.bias"), c["eps"])
        h = F.linear(act(F.linear(h, l("mlp.fc1.weight"), l("mlp.fc1.bias"))), l("mlp.fc2.weight"), l("mlp.fc2.bias"))
        x = x + h
    return F.linear(x, w("visual_projection.weight"))[:, 1:, :]


# ------------------------------------------------------------------------------------------------ Whisper encoder
def whisper_encode(mel: Tensor, w: _SD, hp: dict) -> Tensor:
    """`audio_encoder.encoder(mel)[0]` (modeling.py:1081-1083).  Restates transformers modeling_whisper.py
    WhisperEncoder.forward (:593-647), WhisperAttention (:241-357; q scaled, k_proj bias-free), WhisperEncoderLayer
    (:360-415).  mel (B, 80, 3000) -> (B, 1500, d_model)."""
    c = hp["whisper"]
    D, H = c["d_model"], c["heads"]
    hd = D // H
    act = _act(c["act"])
    x = F.gelu(F.conv1d(mel, w("conv1.weight"), w("conv1.bias"), padding=1))
    x = F.gelu(F.conv1d(x, w("conv2.weight"), w("conv2.bias"), stride=2, padding=1))
    x = x.permute(0, 2, 1) + w("embed_positions.weight")[None]
    B = x.shape[0]
    for i in range(c["layers"]):
        l = w.sub(f"layers.{i}.")
        h = F.layer_norm(x, (D,), l("self_attn_layer_norm.weight"), l("self_attn_layer_norm.bias"), 1e-5)
        q = (F.linear(h, l("self_attn.q_proj.weight"), l("self_attn.q_proj.bias")) * hd ** -0.5)
        q = q.view(B, -1, H, hd).transpose(1, 2)
        k = F.linear(h, l("self_attn.k_proj.weight")).view(B, -1, H, hd).transpose(1, 2)
        v = F.linear(h, l("self_attn.v_proj.weight"), l("self_attn.v_proj.bias")).view(B, -1, H, hd).transpose(1, 2)
        p = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
        a = (p @ v).transpose(1, 2).reshape(B, -1, D)
        x = x + F.linear(a, l("self_attn.out_proj.weight"), l("self_attn.out_proj.bias"))
        h = F.layer_norm(x, (D,), l("final_layer_norm.weight"), l("final_layer_norm.bias"), 1e-5)
        x = x + F.linear(act(F.linear(h, l("fc1.weight"), l("fc1.bias"))), l("fc2.weight"), l("fc2.bias"))
    return F.layer_norm(x, (D,), w("layer_norm.weight"), w("layer_norm.bias"), 1e-5)


# ------------------------------------------------------------------------------------------------ video-long
def video_positional_encoding(L: int, h: int, dtype=torch.float32) -> Tensor:
    """create_positional_encoding (modeling.py:1095-1106), vectorised.  The reference computes, in fp32,
    div = exp(-(ln(10000)/h) * (2*i)) for even i (note 2*i with i already even — a non-standard frequency ladder),
    pe[pos, i] = sin(pos * div), pe[pos, i+1] = cos(pos * div).  Computed in fp32 exactly as written, then cast."""
    # the exponent is a python double rounded to fp32 by torch.tensor(.), then exp() runs in fp32 (modeling.py:1102)
    arg = torch.tensor([-(math.log(10000.0) / h * (2 * i)) for i in range(0, h, 2)], dtype=torch.float32)
    div = torch.exp(arg)
    pos = torch.arange(L, dtype=torch.float32)[:, None]
    pe = torch.zeros(L, h, dtype=torch.float32)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe.to(dtype)


def encode_video_long(videos: Tensor, sd: _SD, hp: dict, dropout_mult: Optional[Tensor] = None) -> Tensor:
    """modeling.py:1070-1079: CLIP per frame -> (B, F*256, D) -> + sinusoid PE -> video_long_self_attention(x, x, x)."""
    F_ = hp["n_frames"]
    frames = videos.reshape(-1, *videos.shape[-3:])
    tok = clip_tokens(frames, sd.sub("video_encoder."), hp)
    B = frames.shape[0] // F_
    x = tok.reshape(B, F_ * tok.shape[1], -1)
    x = x + video_positional_encoding(x.shape[1], x.shape[2], x.dtype)[None]
    xs = x.transpose(0, 1)
    return mha_forward(xs, xs, xs, sd.sub("video_long_self_attention."), hp["attention_heads"], dropout_mult).transpose(0, 1)


# ------------------------------------------------------------------------------------------------ LLaMA
def llama_forward(embeds: Tensor, attention_mask: Optional[Tensor], sd: _SD, hp: dict) -> Tensor:
    """Vendored LlamaModel + lm_head (modeling.py:397-522, 597): position_ids = arange(T) regardless of padding
    (:434-439); additive causal + padding mask clamped at finfo.min (:373-394, 210-211); rotate-half RoPE base 1e4
    (:76-123); fp32 softmax (:214); RMSNorm with fp32 variance (:311-319); SwiGLU MLP (:139-140).
    embeds (B, T, E), attention_mask (B, T) of {0,1} or None -> logits (B, T, V)."""
    c = hp["llama"]
    E, H = c["hidden"], c["heads"]
    hd = E // H
    B, T, _ = embeds.shape
    dt = embeds.dtype
    fmin = torch.finfo(dt).min
    causal = torch.full((T, T), fmin, dtype=dt)
    causal = torch.triu(causal, diagonal=1)
    mask = causal[None, None].expand(B, 1, T, T)
    if attention_mask is not None:
        inv = 1.0 - attention_mask[:, None, None, :].to(dt).expand(B, 1, T, T)
        mask = inv.masked_fill(inv.bool(), fmin) + mask
    inv_freq = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
    freqs = torch.arange(T).float()[:, None] * inv_freq[None]
    emb = torch.cat([freqs, freqs], dim=-1)
    cos, sin = emb.cos().to(dt)[None, None], emb.sin().to(dt)[None, None]

    def rms(x, wt):
        var = x.float().pow(2).mean(-1, keepdim=True)
        return wt * (x * torch.rsqrt(var + c["eps"])).to(dt)

    def rot(x):
        return torch.cat([-x[..., hd // 2:], x[..., : hd // 2]], dim=-1)

    x = embeds
    m = sd.sub("llm.model.")
    for i in range(c["layers"]):
        l = m.sub(f"layers.{i}.")
        h = rms(x, l("input_layernorm.weight"))
        q = F.linear(h, l("self_attn.q_proj.weight")).view(B, T, H, hd).transpose(1, 2)
        k = F.linear(h, l("self_attn.k_proj.weight")).view(B, T, H, hd).transpose(1, 2)
        v = F.linear(h, l("self_attn.v_proj.weight")).view(B, T, H, hd).transpose(1, 2)
        q, k = q * cos + rot(q) * sin, k * cos + rot(k) * sin
        s = q @ k.transpose(2, 3) / math.sqrt(hd) + mask
        s = torch.max(s, torch.tensor(fmin, dtype=dt))
        p = torch.softmax(s, dim=-1, dtype=torch.float32).to(dt)
        a = (p @ v).transpose(1, 2).reshape(B, T, E)
        x = x + F.linear(a, l("self_attn.o_proj.weight"))
        h = rms(x, l("post_attention_layernorm.weight"))
        h = F.linear(F.silu(F.linear(h, l("mlp.gate_proj.weight"))) * F.linear(h, l("mlp.up_proj.weight")),
                     l("mlp.down_proj.weight"))
        x = x + h
    x = rms(x, m("norm.weight"))
    return F.linear(x, sd("llm.lm_head.weight"))


def shifted_ce(logits: Tensor, labels: Tensor) -> Tensor:
    """modeling.py:600-610: logits[:, :-1] vs labels[:, 1:], mean over labels != -100."""
    V = logits.shape[-1]
    return F.cross_entropy(logits[:, :-1].reshape(-1, V).float(), labels[:, 1:].reshape(-1), ignore_index=-100)


# ------------------------------------------------------------------------------------------------ whole forward
def prepare_inputs(inputs: dict, sd_raw: Dict[str, Tensor], hp: dict, dtype=torch.float32, keep_graph: bool = False,
                   dropout: Optional[Dict[str, Tensor]] = None):
    """MM_LLMs.prepare_inputs_for_generation (modeling.py:965-1048) -> (embeds, attention_mask | None, labels | None).
    dropout: train()-mode attention-dropout multipliers per MHA, keys "image" / "audio" / "video" / "video_long"."""
    dropout = dropout or {}
    sd = _SD(sd_raw, dtype, keep_graph=keep_graph)
    table = sd("llm.model.embed_tokens.weight")
    H2 = hp["attention_heads"] * 2
    cast = lambda t: None if t is None else t.to("cpu").to(dtype)
    image_feats = clip_tokens(cast(inputs["images"]), sd.sub("image_encoder."), hp) if inputs.get("images") is not None else None
    audio_feats = whisper_encode(cast(inputs["audios"]), sd.sub("audio_encoder.encoder."), hp) if inputs.get("audios") is not None else None
    video_feats = (encode_video_long(cast(inputs["videos"]), sd, hp, dropout.get("video_long"))
                   if inputs.get("videos") is not None else None)
    ids = inputs["input_ids"].to("cpu").long()
    text = table[ids]
    n_ignore = 0
    # order matters: video, then audio, then image — each block is spliced right after BOS (modeling.py:978-1034)
    for name, feats in (("video", video_feats), ("audio", audio_feats), ("image", image_feats)):
        if feats is None:
            continue
        starts = table[inputs[f"{name}_starts"].to("cpu").long()].unsqueeze(1)
        ends = table[inputs[f"{name}_ends"].to("cpu").long()].unsqueeze(1)
        out = align_block(feats, table, sd.sub(f"project_{name}."), sd.sub(f"transform_{name}_to_hidden."),
                          sd.sub(f"{name}_align_attention."), hp[f"{name}_conv"][1], H2, dropout.get(name))
        block = torch.cat([starts, out, ends], dim=1)
        text = torch.cat([text[:, :1], block, text[:, 1:]], dim=1)
        n_ignore += block.shape[1]
    B = text.shape[0]
    mask = labels = None
    if "attention_mask" in inputs:
        mask = torch.cat([torch.ones(B, n_ignore, dtype=torch.int64), inputs["attention_mask"].to("cpu").long()], dim=1)
    if inputs.get("labels") is not None:
        labels = torch.cat([torch.full((B, n_ignore), -100, dtype=torch.int64), inputs["labels"].to("cpu").long()], dim=1)
    return text, mask, labels


def forward(inputs: dict, sd_raw: Dict[str, Tensor], hp: dict, dtype=torch.float32):
    """MM_LLMs.forward (modeling.py:941-963) without the generate branch -> dict(loss | None, logits, embeds, mask, labels)."""
    with torch.no_grad():
        embeds, mask, labels = prepare_inputs(inputs, sd_raw, hp, dtype)
        logits = llama_forward(embeds, mask, _SD(sd_raw, dtype), hp)
        loss = shifted_ce(logits, labels) if labels is not None else None
    return dict(loss=loss, logits=logits, embeds=embeds, attention_mask=mask, labels=labels)


def generate_greedy(inputs: dict, sd_raw: Dict[str, Tensor], hp: dict, max_new_tokens: int = 128, eos_token_id: int = 2,
                    pad_token_id: int = 32006, dtype=torch.float32, forced_tokens: Optional[Tensor] = None):
    """The generate branch (modeling.py:954-960 -> HF greedy search on inputs_embeds, no attention mask, only new tokens
    returned), restated WITHOUT a KV cache: the whole sequence is re-run every step.  With `forced_tokens` (B, n) the
    given tokens are fed instead of the argmax (teacher forcing) and the per-step logits are returned as well."""
    with torch.no_grad():
        embeds, _, _ = prepare_inputs({k: v for k, v in inputs.items() if k not in ("labels", "attention_mask")}, sd_raw, hp, dtype)
        sd = _SD(sd_raw, dtype)
        table = sd("llm.model.embed_tokens.weight")
        B = embeds.shape[0]
        finished = torch.zeros(B, dtype=torch.bool)
        out, step_logits = [], []
        for step in range(max_new_tokens):
            logits = llama_forward(embeds, None, sd, hp)[:, -1, :]
            step_logits.append(logits)
            tok = logits.argmax(-1)
            if forced_tokens is not None:
                tok = forced_tokens[:, step].to(tok.dtype)
            tok = torch.where(finished, torch.full_like(tok, pad_token_id), tok)
            out.append(tok)
            finished |= tok == eos_token_id
            if bool(finished.all()) or (forced_tokens is not None and step + 1 == forced_tokens.shape[1]):
                break
            embeds = torch.cat([embeds, table[tok.clamp(max=table.shape[0] - 1)].unsqueeze(1)], dim=1)
    return torch.stack(out, dim=1), torch.stack(step_logits, dim=1)


# ------------------------------------------------------------------------------------------------ gradient oracle
def llama_loss_and_grads(inputs: dict, sd_raw: Dict[str, Tensor], hp: dict, dtype=torch.float32):
    """Loss of MM_LLMs.forward (modeling.py:941-963, 597-610) and its autograd gradients w.r.t. every `llm.*` parameter,
    as the HF Trainer obtains them (llm_trainer.py:184-188: `loss = model(**inputs)[0]`; `loss.backward()`), with the
    ALIGNED rows of the multimodal prefix held constant (they are computed without a graph): the gradient then reaches
    the embedding table through the gathered rows only (BOS / text tokens, start / end tokens), which is the
    differentiable set of this repo's training step (macaw-llm_b200/training.py).  For text-only inputs this IS the
    reference's full gradient.  -> (loss, {name: grad}, d loss / d inputs_embeds)."""
    with torch.no_grad():
        embeds_c, mask, labels = prepare_inputs(inputs, sd_raw, hp, dtype)
    leaves = {k: v.detach().to("cpu").to(dtype).clone().requires_grad_(True) for k, v in sd_raw.items()
              if k.startswith("llm.") and v.is_floating_point() and not k.endswith("inv_freq")}
    table = leaves["llm.model.embed_tokens.weight"]
    ids = inputs["input_ids"].to("cpu").long()
    B, L = ids.shape
    n_prefix = embeds_c.shape[1] - L
    rows = [table[ids[:, :1]]]
    off = 1
    # final layout [BOS, <image> .. </image>, <audio> .. </audio>, <video> .. </video>, text[1:]]
    for name, key in (("image", "images"), ("audio", "audios"), ("video", "videos")):
        if inputs.get(key) is None:
            continue
        Lq = None
        # block length: scan for the end token position is ambiguous; recompute from the conv geometry
        kk, ss = hp[f"{name}_conv"]
        n_tok = {"image": (hp["clip"]["image_size"] // hp["clip"]["patch"]) ** 2, "audio": hp["whisper"]["max_pos"],
                 "video": hp["n_frames"] * (hp["clip"]["image_size"] // hp["clip"]["patch"]) ** 2}[name]
        Lq = (n_tok - kk) // ss + 1
        rows.append(table[inputs[f"{name}_starts"].to("cpu").long()].unsqueeze(1))
        rows.append(embeds_c[:, off + 1: off + 1 + Lq])
        rows.append(table[inputs[f"{name}_ends"].to("cpu").long()].unsqueeze(1))
        off += Lq + 2
    assert off == 1 + n_prefix, (off, n_prefix)
    rows.append(table[ids[:, 1:]])
    embeds = torch.cat(rows, dim=1)
    embeds.retain_grad()
    logits = llama_forward(embeds, mask, _SD(leaves, dtype, keep_graph=True), hp)
    loss = shifted_ce(logits, labels)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaves.items()}, embeds.grad


ALIGN_PREFIXES = tuple(f"project_{n}." for n in ("image", "audio", "video")) + \
    tuple(f"transform_{n}_to_hidden." for n in ("image", "audio", "video")) + \
    tuple(f"{n}_align_attention." for n in ("image", "audio", "video")) + ("video_long_self_attention.",)


def full_loss_and_grads(inputs: dict, sd_raw: Dict[str, Tensor], hp: dict, dtype=torch.float32,
                        dropout: Optional[Dict[str, Tensor]] = None):
    """Loss of MM_LLMs.forward and its autograd gradients w.r.t. every `llm.*` parameter AND the alignment modules
    (project_*, transform_*_to_hidden, *_align_attention) — the gradient the HF Trainer obtains from the reference in eval-
    mode arithmetic (dropout off), with the encoders frozen (run_clm_llms.py:390-393).  The embedding table is
    differentiated through the gathered rows AND as the keys / values of the alignment attention (modeling.py:974-975).
    `video_long_self_attention` is differentiated too (its input, frozen CLIP features + PE, is a constant).
    `dropout`: explicit train()-mode attention-dropout multipliers per MHA (see mha_forward); None = dropout off.
    -> (loss, {name: grad})."""
    merged, leaves = {}, {}
    for k, v in sd_raw.items():
        if not v.is_floating_point():
            merged[k] = v
            continue
        t = v.detach().to("cpu").to(dtype)
        if (k.startswith("llm.") and not k.endswith("inv_freq")) or k.startswith(ALIGN_PREFIXES):
            t = t.clone().requires_grad_(True)
            leaves[k] = t
        merged[k] = t
    embeds, mask, labels = prepare_inputs(inputs, merged, hp, dtype, keep_graph=True, dropout=dropout)
    logits = llama_forward(embeds, mask, _SD(merged, dtype, keep_graph=True), hp)
    loss = shifted_ce(logits, labels)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaves.items()}
