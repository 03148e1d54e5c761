"""The int8 KV-cache rule and a KV-cached decoder that stores its keys and values by it, for the int8 KV-cache tests.

Rule, per cached key vector and per cached value vector of one token and one head (128 elements), for v as the 16-bit
cache would store it:  s = fp32(max |v|) / 127 (IEEE division),  q = clamp(rint(v / s), -127, 127) with IEEE division and
ties to even,  q = 0 and s = 0 for an all-zero vector.  The dequantized value is the fp32 product q * s.

An fp32 quotient is the fp64 quotient of the same operands rounded once to fp32 (fp64 carries more than 2 * 24 + 2 bits),
so the restatement divides in fp64 and rounds; numpy keeps subnormals, so heads whose scale is subnormal follow IEEE too.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import decode_reference as R


def quantize(v: np.ndarray):
    """v (..., 128) fp32 values -> (q int8 (..., 128), s fp32 (...))."""
    v = np.asarray(v, dtype=np.float32)
    mx = np.abs(v).max(axis=-1)
    s = (mx.astype(np.float64) / 127.0).astype(np.float32)
    safe = np.where(s == 0, np.float32(1), s)
    r = np.rint((v.astype(np.float64) / safe.astype(np.float64)[..., None]).astype(np.float32))
    q = np.where((s == 0)[..., None], 0, np.clip(r, -127, 127)).astype(np.int8)
    return q, s


def quantize_torch(v: torch.Tensor):
    """`quantize` on a torch tensor (any device, 16-bit or fp32 values) -> (q int8, s fp32) on the same device."""
    q, s = quantize(v.float().cpu().numpy())
    return torch.from_numpy(q).to(v.device), torch.from_numpy(s).to(v.device)


def quantize_cache(cache: torch.Tensor, H: int):
    """A 16-bit cache (B, Tmax, 2, E) -> (int8 (B, Tmax, 2, E), scales fp32 (B, 2, H, Tmax)): the int8 cache's layout."""
    B, Tmax, _, E = cache.shape
    q, s = quantize_torch(cache.view(B, Tmax, 2, H, E // H))
    return q.view(B, Tmax, 2, E), s.permute(0, 2, 3, 1).contiguous()


def dequantize_cache(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """(int8 (B, Tmax, 2, E), fp32 (B, 2, H, Tmax)) -> fp64 (B, Tmax, 2, H, 128) values q * s (the fp32 product, widened)."""
    B, Tmax, _, E = q.shape
    H = s.shape[2]
    return (q.view(B, Tmax, 2, H, E // H).float() * s.permute(0, 3, 1, 2)[..., None]).double()


class QuantCachedDecoder(R.CachedDecoder):
    """`decode_reference.CachedDecoder` whose cache holds keys and values by the int8 rule: every key / value vector is
    rounded to `fmt` (the 16-bit format the cache would store), then quantized and kept as its fp64 dequantized value.
    The prefill's attention reads the exact k / v, as the engine's does; decode steps read the cache.  With quant=False
    this is CachedDecoder, bit for bit."""

    def __init__(self, sd, hp, device="cpu", dtype=torch.float64, fmt=torch.bfloat16, quant=True):
        super().__init__(sd, hp, device, dtype)
        self.fmt, self.quant = fmt, quant

    def _store(self, t: torch.Tensor) -> torch.Tensor:
        """(B, H, T, hd) -> its values after the cache's round trip."""
        if not self.quant:
            return t
        q, s = quantize_torch(t.to(self.fmt))
        return (q.float() * s[..., None]).to(self.dt)

    def _run(self, x: torch.Tensor, pos0: int) -> torch.Tensor:
        F = torch.nn.functional
        B, T, E = x.shape
        H, hd = self.H, self.hd
        cos_t, sin_t = self._tables(pos0 + T)
        cos, sin = cos_t[pos0:pos0 + T][None, None], sin_t[pos0:pos0 + T][None, None]
        fmin = torch.finfo(self.dt).min
        Tk = pos0 + T
        mask = torch.triu(torch.full((T, Tk), fmin, dtype=self.dt, device=self.dev), diagonal=pos0 + 1)[None, None]
        for i in range(self.L):
            p = f"llm.model.layers.{i}."
            h = self._rms(x, self.w(p + "input_layernorm.weight"))
            q = F.linear(h, self.w(p + "self_attn.q_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            k = F.linear(h, self.w(p + "self_attn.k_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            v = F.linear(h, self.w(p + "self_attn.v_proj.weight")).view(B, T, H, hd).transpose(1, 2)
            q, k = q * cos + self._rot(q) * sin, k * cos + self._rot(k) * sin
            kc, vc = self._store(k), self._store(v)
            if pos0 > 0:  # a decode step attends over the cache, its own new row included
                k = torch.cat([self.k[i], kc], dim=2)
                v = torch.cat([self.v[i], vc], dim=2)
                self.k[i], self.v[i] = k, v
            else:  # the prefill attends over its exact rows and leaves the cache's values behind
                self.k[i], self.v[i] = kc, vc
            s = q @ k.transpose(2, 3) / math.sqrt(hd) + mask
            s = torch.max(s, torch.tensor(fmin, dtype=self.dt, device=self.dev))
            a = (torch.softmax(s, dim=-1, dtype=torch.float32).to(self.dt) @ v).transpose(1, 2).reshape(B, T, E)
            x = x + F.linear(a, self.w(p + "self_attn.o_proj.weight"))
            h = self._rms(x, self.w(p + "post_attention_layernorm.weight"))
            x = x + F.linear(F.silu(F.linear(h, self.w(p + "mlp.gate_proj.weight"))) * F.linear(h, self.w(p + "mlp.up_proj.weight")),
                             self.w(p + "mlp.down_proj.weight"))
        return x


def decode_logits(sd, hp, embeds, tokens, device="cpu", fmt=torch.bfloat16, quant=True):
    """`decode_reference.decode_logits` through QuantCachedDecoder."""
    dec = QuantCachedDecoder(sd, hp, device, fmt=fmt, quant=quant)
    table = sd["llm.model.embed_tokens.weight"]
    with torch.no_grad():
        pre = dec.prefill(embeds)
        steps = [pre[:, -1]]
        for s in range(tokens.shape[1]):
            steps.append(dec.step(table[tokens[:, s].to(table.device).clamp(0, table.shape[0] - 1)]))
    return pre, torch.stack(steps, dim=1)
