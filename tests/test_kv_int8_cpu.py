"""CPU tier of the int8 KV cache: the rule's restatement (tests/kv_int8_reference.py) on crafted head vectors, the
quantizing cached decoder against decode_reference.CachedDecoder, and the new entry points' argument checks."""
import ctypes

import numpy as np
import torch

from tests import decode_reference as R
from tests import kv_int8_reference as Q
from tests.test_decode_cpu import _random_decoder


def _head(*vals, fill=0.0):
    v = np.full(128, fill, dtype=np.float32)
    v[: len(vals)] = vals
    return v


def test_rule_on_crafted_heads():
    """max 127 makes s = 1, so q = rint(v): ties at .5 go to even; the element at the max is 127; -max is -127."""
    v = _head(127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.5, 126.5, -127.0, 0.49999997)
    q, s = Q.quantize(v)
    assert s == np.float32(1.0)
    assert q[:11].tolist() == [127, 0, 2, 2, 0, -2, -2, 4, 126, -127, 0]
    # s = fl(max / 127) and q = fl(v / s) in fp32: a scale that rounds down still maps the max to 127
    for mx in (1.0, 3.0, 100.0, 1e-3, 65504.0, 3.3895e38):
        q, s = Q.quantize(_head(np.float32(mx), -np.float32(mx) / 2, fill=np.float32(mx) / 3))
        assert s == np.float32(np.float32(mx) / np.float32(127))
        assert q[0] == 127 and abs(int(q[1])) in (63, 64) and q[1] < 0


def test_rule_all_zero_and_signed_zero_heads():
    for v in (np.zeros(128, np.float32), -np.zeros(128, np.float32)):
        q, s = Q.quantize(v)
        assert s == 0 and not q.any()


def test_rule_subnormal_scales_clamp():
    """A head whose max is near the bottom of fp32 gets a subnormal scale with few significant bits: v / s reaches past
    127.5 and is clamped to +-127.  The restatement's fp64 quotient rounded to fp32 equals numpy's fp32 division."""
    tiny = np.float32(2.0 ** -140)  # bf16 holds it; max / 127 is subnormal in fp32
    v = _head(tiny, -tiny, tiny * 0.75, fill=tiny / 2)
    q, s = Q.quantize(v)
    assert 0 < s < np.finfo(np.float32).tiny
    raw = np.rint(v / s)  # numpy's own fp32 division
    assert raw[0] > 127 and q[0] == 127 and q[1] == -127
    assert q.tolist() == np.clip(raw, -127, 127).astype(np.int8).tolist()
    # the smallest subnormal max: s rounds to 0, so q = 0 (the all-zero rule)
    q, s = Q.quantize(_head(np.float32(2.0 ** -149)))
    assert s == 0 and not q.any()


def test_rule_matches_fp32_division_on_random_heads():
    g = np.random.default_rng(3)
    v = (g.standard_normal((4096, 128)) * np.exp(g.uniform(-40, 40, (4096, 1)))).astype(np.float32)
    v = torch.from_numpy(v).to(torch.bfloat16).float().numpy()  # values the bf16 cache holds
    q, s = Q.quantize(v)
    s32 = np.abs(v).max(1) / np.float32(127)
    assert np.array_equal(s, s32)
    assert np.array_equal(q, np.clip(np.rint(v / s32[:, None]), -127, 127).astype(np.int8))
    err = np.abs(q.astype(np.float64) * s[:, None] - v).max(1)
    assert (err <= s.astype(np.float64) / 2 + np.spacing(np.abs(v).max(1))).all()  # half a step, and v / s's rounding


def test_quantize_cache_layout():
    """quantize_cache gives the (B, Tmax, 2, E) values and (B, 2, H, Tmax) scales of each (token, k / v, head) vector."""
    g = torch.Generator().manual_seed(1)
    B, Tmax, H = 2, 5, 3
    cache = torch.randn(B, Tmax, 2, H * 128, generator=g).to(torch.bfloat16)
    q, s = Q.quantize_cache(cache, H)
    assert q.shape == cache.shape and q.dtype == torch.int8 and tuple(s.shape) == (B, 2, H, Tmax)
    for b, t, w, h in ((0, 0, 0, 0), (1, 4, 1, 2), (0, 3, 1, 1)):
        qq, ss = Q.quantize(cache[b, t, w, h * 128:(h + 1) * 128].float().numpy())
        assert np.array_equal(q[b, t, w, h * 128:(h + 1) * 128].numpy(), qq) and s[b, w, h, t].item() == ss
    deq = Q.dequantize_cache(q, s)
    assert float((deq.view(B, Tmax, 2, H * 128) - cache.double()).abs().max()) <= float(s.max()) / 2 * 1.001


def test_quant_decoder_off_equals_cached_decoder_bitwise():
    E, H, L, I, V = 256, 2, 2, 512, 512
    sd, hp = _random_decoder(E, H, L, I, V, seed=11)
    g = torch.Generator().manual_seed(12)
    prompt, toks = torch.randint(0, V, (2, 9), generator=g), torch.randint(0, V, (2, 12), generator=g)
    table = sd["llm.model.embed_tokens.weight"]
    pre, steps = R.decode_logits(sd, hp, table[prompt], toks)
    pre_q, steps_q = Q.decode_logits(sd, hp, table[prompt], toks, quant=False)
    assert torch.equal(pre, pre_q) and torch.equal(steps, steps_q)


def test_quant_decoder_prefill_is_exact_and_steps_are_close():
    """With quantization on, the prefill's logits are the exact decoder's (its attention reads exact k / v) and the steps
    differ by the cache's quantization only: small against the logits, but not zero."""
    E, H, L, I, V = 256, 2, 2, 512, 512
    sd, hp = _random_decoder(E, H, L, I, V, seed=13)
    g = torch.Generator().manual_seed(14)
    prompt, toks = torch.randint(0, V, (2, 9), generator=g), torch.randint(0, V, (2, 12), generator=g)
    table = sd["llm.model.embed_tokens.weight"]
    pre, steps = R.decode_logits(sd, hp, table[prompt], toks)
    pre_q, steps_q = Q.decode_logits(sd, hp, table[prompt], toks)
    assert torch.equal(pre, pre_q) and torch.equal(steps[:, 0], steps_q[:, 0])
    rel = float((steps_q[:, 1:] - steps[:, 1:]).norm() / steps[:, 1:].norm())
    print(f"\n[int8 KV restatement] step logits vs the exact cache: {rel:.2e}")
    assert 0 < rel < 2e-2


def test_entry_points_refuse_bad_arguments():
    """Argument checks run before any CUDA call: null pointers, a count above the capacity, a missing workspace, and the
    int8 tail without the QKV mode or without its scale buffer."""
    from macaw_llm_b200 import _lib

    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)
    assert lib.mm_kv_append_i8(p, 3 * 4096, 1, 1, 4096, p, None, 64, 0, None, None) != 0
    assert b"mm_kv_append_i8" in lib.mm_last_error()
    assert lib.mm_kv_append_i8(p, 3 * 4096, 1, 2, 4096, p, p, 64, 63, None, None) != 0
    ws = int(lib.mm_attn_decode_i8_workspace_bytes(8, 32, 2112))
    assert ws > 0 and ws % ((128 + 2) * 4 * 8 * 32) == 0
    assert lib.mm_attn_decode_i8(p, 3 * 4096, p, p, p, 4096, 8, 32, 2112, 2113, None, 0.088, p, ws, None) != 0
    assert b"bad shape" in lib.mm_last_error()
    assert lib.mm_attn_decode_i8(p, 3 * 4096, p, p, p, 4096, 8, 32, 2112, 2112, None, 0.088, p, ws - 4, None) != 0
    assert b"workspace" in lib.mm_last_error()
    a = _lib.ThinArgs()
    a.part, a.out, a.splits, a.N, a.M, a.ldp, a.mode = 1 << 20, 1 << 20, 1, 3 * 4096, 1, 4, 0
    a.rope_cos = a.rope_sin = a.cache = 1 << 20
    a.E, a.Tmax = 4096, 64
    assert lib.mm_thin_fused_kv_i8(ctypes.byref(a), p, None) != 0 and b"MM_THIN_QKV" in lib.mm_last_error()
    a.mode = 2
    assert lib.mm_thin_fused_kv_i8(ctypes.byref(a), None, None) != 0 and b"cache_scale" in lib.mm_last_error()
