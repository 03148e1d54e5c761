"""KV-cached restatement of `oracle.macaw_oracle.llama_forward` with the generate branch's semantics, for the decode tests.

generate() hands the decoder no attention mask and positions are indices in the sequence (reference modeling.py:954-960,
434-439).  This module runs that computation the way a cached decoder does — prefill over the prompt, then one token
per step against the growing key / value cache — in float64 on any device, following the oracle's rules so that it
equals a full recompute by the oracle (tests/test_decode_cpu.py):
  * RMSNorm with the variance in fp32 (modeling.py:311-319), gain applied after;
  * rotate-half RoPE, base 1e4, angles and cos / sin computed in fp32 on the CPU exactly as the oracle does, then widened;
  * scores clamped at the format's minimum, softmax in fp32 (modeling.py:214);
  * SwiGLU MLP and lm_head.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F


def rope_tables(T: int, hd: int):
    """cos / sin (T, hd / 2) fp32 on the CPU: the oracle's angles (fp32 inv_freq, fp32 products) and fp32 cos / sin."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
    freqs = torch.arange(T).float()[:, None] * inv_freq[None]
    return freqs.cos(), freqs.sin()


class CachedDecoder:
    """The decoder of a state dict (keys `llm.model.*`, `llm.lm_head.weight`) with a per-layer K / V cache.

    hp: the oracle's hyper-parameters (`oracle.macaw_oracle.hp_from_config`; only hp["llama"] is read)."""

    def __init__(self, sd: Dict[str, torch.Tensor], hp: dict, device="cpu", dtype=torch.float64):
        c = hp["llama"]
        self.E, self.H, self.L, self.eps = c["hidden"], c["heads"], c["layers"], c["eps"]
        self.hd = self.E // self.H
        self.dev, self.dt = torch.device(device), dtype
        self.sd = sd
        self.k = [None] * self.L  # (B, H, T, hd) per layer
        self.v = [None] * self.L
        self._rope = None

    def w(self, name: str) -> torch.Tensor:
        return self.sd[name].detach().to(device=self.dev, dtype=self.dt)

    def _tables(self, T: int):
        if self._rope is None or self._rope[0].shape[0] < T:
            cos, sin = rope_tables(max(T, 256), self.hd)
            emb = lambda t: torch.cat([t, t], -1).to(device=self.dev, dtype=self.dt)  # noqa: E731
            self._rope = (emb(cos), emb(sin))
        return self._rope

    def _rms(self, x, wt):
        var = x.float().pow(2).mean(-1, keepdim=True)
        return wt * (x * torch.rsqrt(var + self.eps)).to(self.dt)

    def _rot(self, x):
        hd = self.hd
        return torch.cat([-x[..., hd // 2:], x[..., : hd // 2]], dim=-1)

    def _run(self, x: torch.Tensor, pos0: int) -> torch.Tensor:
        """x (B, T, E) at positions pos0 .. pos0 + T - 1 -> final hidden states (B, T, E); the cache grows by T."""
        B, T, E = x.shape
        H, hd = self.H, self.hd
        cos_t, sin_t = self._tables(pos0 + T)
        cos, sin = cos_t[pos0:pos0 + T][None, None], sin_t[pos0:pos0 + T][None, None]
        fmin = torch.finfo(self.dt).min
        Tk = pos0 + T
        # query i (position pos0 + i) sees keys 0 .. pos0 + i
        mask = torch.triu(torch.full((T, Tk), fmin, dtype=self.dt, device=self.dev), diagonal=pos0 + 1)[None, None]
        for i in range(self.L):
            p = f"llm.model.layers.{i}."
            h = self._rms(x, self.w(p + "input_layernorm.weight"))
            q = F.linear(h, self.w(p + "self_attn.q_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            k = F.linear(h, self.w(p + "self_attn.k_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            v = F.linear(h, self.w(p + "self_attn.v_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            q, k = q * cos + self._rot(q) * sin, k * cos + self._rot(k) * sin
            if pos0 > 0:
                k = torch.cat([self.k[i], k], dim=2)
                v = torch.cat([self.v[i], v], dim=2)
            self.k[i], self.v[i] = k, v
            s = q @ k.transpose(2, 3) / math.sqrt(hd) + mask
            s = torch.max(s, torch.tensor(fmin, dtype=self.dt, device=self.dev))
            a = (torch.softmax(s, dim=-1, dtype=torch.float32).to(self.dt) @ v).transpose(1, 2).reshape(B, T, E)
            x = x + F.linear(a, self.w(p + "self_attn.o_proj.weight"))
            h = self._rms(x, self.w(p + "post_attention_layernorm.weight"))
            x = x + F.linear(F.silu(F.linear(h, self.w(p + "mlp.gate_proj.weight"))) * F.linear(h, self.w(p + "mlp.up_proj.weight")),
                             self.w(p + "mlp.down_proj.weight"))
        return x

    def _logits(self, x):
        return F.linear(self._rms(x, self.w("llm.model.norm.weight")), self.w("llm.lm_head.weight"))

    def prefill(self, embeds: torch.Tensor) -> torch.Tensor:
        """embeds (B, T, E) at positions 0 .. T - 1 -> logits (B, T, V) of every prompt position; fills the cache."""
        x = self._run(embeds.to(device=self.dev, dtype=self.dt), 0)
        self.pos = embeds.shape[1]
        return self._logits(x)

    def step(self, embed: torch.Tensor) -> torch.Tensor:
        """embed (B, E) of the next token -> logits (B, V) at its position; appends it to the cache."""
        x = self._run(embed.to(device=self.dev, dtype=self.dt)[:, None], self.pos)
        self.pos += 1
        return self._logits(x)[:, 0]


def decode_logits(sd: Dict[str, torch.Tensor], hp: dict, embeds: torch.Tensor, tokens: torch.Tensor,
                  device="cpu", dtype=torch.float64):
    """Teacher-forced cached decode: prefill over embeds (B, T0, E), then feed tokens[:, s] (rows of the embedding table,
    ids clamped to it as generate does for finished rows) one per step.  -> (prefill logits (B, T0, V), step logits
    (B, n + 1, V)): entry 0 is the prefill's last position, entry s the logits after feeding tokens[:, s - 1]."""
    dec = CachedDecoder(sd, hp, device, dtype)
    table = sd["llm.model.embed_tokens.weight"]
    with torch.no_grad():
        pre = dec.prefill(embeds)
        steps = [pre[:, -1]]
        for s in range(tokens.shape[1]):
            steps.append(dec.step(table[tokens[:, s].to(table.device).clamp(0, table.shape[0] - 1)]))
    return pre, torch.stack(steps, dim=1)
