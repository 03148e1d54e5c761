"""The int8 KV cache on the H100: the decode tail's int8 mode, mm_kv_append_i8 and mm_attn_decode_i8 at the kernel tier
(bf16 and fp16), and generate() with the int8 cache at 7B width and on the tiny model, with 16-bit, int8 and FP8 weights.

The writers are held bitwise to the rule (tests/kv_int8_reference.py) applied to what the 16-bit writers store; the
attention to fp64 over the dequantized cache at the 16-bit decode tests' bar (5e-3); the engine's step logits to 1.5x
the larger of two errors against the unquantized fp64 decoder: the 16-bit-cache engine's own and that of the fp64 decoder
whose cache holds the quantized values (the format's yardstick).  Measured values are printed (-s)."""
import pytest
import torch

from tests import decode_reference as R
from tests import helpers as H
from tests import kv_int8_reference as Q
from tests.test_decode_gpu import (DEV, _attn64, _hp, _model_7b, _prompt, _ref_state, _weights_7b, act, bits, rel64,
                                   rnd)

pytestmark = pytest.mark.gpu

__all__ = ["act"]  # the fixture, imported for this module's tests


def _ops():
    from macaw_llm_b200 import ops

    return ops


# ------------------------------------------------------------------------------------------------ decode tail
@pytest.mark.parametrize("M", [1, 8, 64])
def test_tail_int8_mode_writes_the_rule_of_the_16bit_slot(act, M):
    """At the 7B QKV shape (12288 x 4096), on the same split-K partials: the int8-mode tail writes rule(slot the 16-bit
    tail writes), values and scales bitwise, nothing outside its slot, and the same q rows."""
    from macaw_llm_b200.engine import Engine

    ops = _ops()
    E, Hh, Tmax = 4096, 32, 8
    w = _weights_7b(act)
    x = rnd(M, E, dt=act, seed=400 + M)
    rs = torch.rand(M, device=DEV) + 0.5
    cos, sin = Engine(None).rope_tables(2048, 128, torch.device(DEV))
    sent16 = torch.full((M, Tmax, 2, E), 777.0, device=DEV, dtype=act)
    sent_q = torch.full((M, Tmax, 2, E), 99, device=DEV, dtype=torch.int8)
    sent_s = torch.full((M, 2, Hh, Tmax), -5.0, device=DEV)
    for pos, slot in ((0, 0), (64, 5), (2047, 7)):
        kw = dict(row_scale=rs, rope=(cos, sin, torch.tensor([pos], device=DEV, dtype=torch.int32)),
                  t0_dev=torch.tensor([slot], device=DEV, dtype=torch.int32))
        c16 = sent16.clone()
        out16 = ops.linear_thin_fused(x, w["qkv"], ops.THIN_QKV, cache=c16, **kw)
        cq, cs = sent_q.clone(), sent_s.clone()
        out8 = ops.linear_thin_fused(x, w["qkv"], ops.THIN_QKV, cache=cq, cache_scale=cs, **kw)
        assert torch.equal(bits(out8[:, :E]), bits(out16[:, :E])), pos
        q_ref, s_ref = Q.quantize_cache(c16[:, slot:slot + 1], Hh)
        assert torch.equal(cq[:, slot], q_ref[:, 0]), pos
        assert torch.equal(cs[..., slot].view(torch.int32), s_ref[..., 0].view(torch.int32)), pos
        # the host slot form writes the same
        cq2, cs2 = sent_q.clone(), sent_s.clone()
        ops.linear_thin_fused(x, w["qkv"], ops.THIN_QKV, row_scale=rs, rope=(cos[pos:], sin[pos:], None), cache=cq2,
                              cache_scale=cs2, t0=slot)
        assert torch.equal(cq2, cq) and torch.equal(cs2.view(torch.int32), cs.view(torch.int32)), pos
        cq[:, slot], cs[..., slot] = sent_q[:, slot], sent_s[..., slot]
        assert torch.equal(cq, sent_q) and torch.equal(cs.view(torch.int32), sent_s.view(torch.int32)), pos


# ------------------------------------------------------------------------------------------------ append
@pytest.mark.parametrize("B,T_new", [(1, 1), (1, 37), (65, 1), (65, 37)])
def test_kv_append_i8_is_the_rule_of_kv_append(act, B, T_new):
    ops = _ops()
    E, Hh, Tmax = 4096, 32, 64
    buf = rnd(B * T_new, 3 * E + 64, dt=act, seed=B + T_new, scale=3.0)
    buf[0, E:E + 128] = 0  # an all-zero key head
    qkv = buf[:, :3 * E]  # row stride 3E + 64
    sent_q = torch.full((B, Tmax, 2, E), -99, device=DEV, dtype=torch.int8)
    sent_s = torch.full((B, 2, Hh, Tmax), float("nan"), device=DEV)
    for t0, dev_t0 in ((3, None), (Tmax - T_new, None), (17, 17)):
        c16 = torch.zeros((B, Tmax, 2, E), device=DEV, dtype=act)
        ops.kv_append(qkv, B, T_new, c16, t0)
        q_ref, s_ref = Q.quantize_cache(c16[:, t0:t0 + T_new], Hh)
        cq, cs = sent_q.clone(), sent_s.clone()
        if dev_t0 is None:
            ops.kv_append_i8(qkv, B, T_new, cq, cs, t0)
        else:  # the host offset is ignored when the device one is given
            ops.kv_append_i8(qkv, B, T_new, cq, cs, 0, torch.tensor([dev_t0], device=DEV, dtype=torch.int32))
        assert torch.equal(cq[:, t0:t0 + T_new], q_ref), t0
        assert torch.equal(cs[..., t0:t0 + T_new].view(torch.int32), s_ref.view(torch.int32)), t0
        cq[:, t0:t0 + T_new], cs[..., t0:t0 + T_new] = sent_q[:, t0:t0 + T_new], sent_s[..., t0:t0 + T_new]
        assert torch.equal(cq, sent_q) and torch.equal(cs.view(torch.int32), sent_s.view(torch.int32)), t0


# ------------------------------------------------------------------------------------------------ attention
def _i8_operands(B, Hh, Tmax, dt, seed):
    """q as the q-third of a fused activation and an int8 cache + scales quantized from a random 16-bit cache."""
    qkv = rnd(B, 1, 3, Hh, 128, dt=dt, seed=seed)
    cache = rnd(B, Tmax, 2, Hh * 128, dt=dt, seed=seed + 1)
    kq, ks = Q.quantize_cache(cache, Hh)
    return qkv[:, :, 0], kq, ks


def _garbage(kq, ks, tk):
    """Rows and scales past tk overwritten: random int8 values, scales NaN / +inf / -inf / 1e30."""
    kq, ks = kq.clone(), ks.clone()
    n = kq.shape[1] - tk
    if n > 0:
        kq[:, tk:] = torch.randint(-128, 128, kq[:, tk:].shape, device=DEV, dtype=torch.int8)
        vals = torch.tensor([float("nan"), float("inf"), -float("inf"), 1e30], device=DEV)
        ks[..., tk:] = vals[torch.arange(n, device=DEV) % 4]
    return kq, ks


@pytest.mark.parametrize("B", [1, 7, 65, 96])
def test_attention_decode_i8_over_the_cache(act, B):
    """1 to 256 keys of a 256-row cache, H = 32, against fp64 over the dequantized cache; rows and scales past the count
    (garbage, NaN / inf scales), a host count and a device count above the capacity change no bit; two launches agree."""
    ops = _ops()
    Hh, Tmax, scale = 32, 256, 128 ** -0.5
    q, kq, ks = _i8_operands(B, Hh, Tmax, act, seed=20 * B)
    deq = Q.dequantize_cache(kq, ks)
    errs = []
    for tk in (1, 31, 63, 64, 65, 129, 200, 256):
        tk_dev = torch.tensor([tk], device=DEV, dtype=torch.int32)
        out = ops.attention_decode_i8(q, kq, ks, scale=scale, tk_dev=tk_dev)
        ref = _attn64(q[:, 0], deq[:, :tk, 0], deq[:, :tk, 1], scale)
        e = rel64(out[:, 0], ref)
        errs.append(e)
        assert e < 5e-3, (tk, e)
        gq, gs = _garbage(kq, ks, tk)
        runs = dict(garbage=ops.attention_decode_i8(q, gq, gs, scale=scale, tk_dev=tk_dev),
                    host=ops.attention_decode_i8(q, gq, gs, scale=scale, Tk=tk),
                    again=ops.attention_decode_i8(q, kq, ks, scale=scale, tk_dev=tk_dev))
        if tk == Tmax:
            runs["clamp"] = ops.attention_decode_i8(q, kq, ks, scale=scale,
                                                    tk_dev=torch.tensor([Tmax + 37], device=DEV, dtype=torch.int32))
        for name, o in runs.items():
            assert torch.equal(bits(o), bits(out)), (tk, name)
    print(f"\n[attention decode int8 {act} B={B}] max err vs fp64 of the dequantized cache {max(errs):.2e} (bar 5e-3)")


def test_attention_decode_i8_long_rising_scores(act):
    """2048 keys of a 2112-row cache whose scores rise along the sequence: the running max moves in every split."""
    ops = _ops()
    B, Hh, Tmax, tk, scale = 2, 32, 2112, 2048, 128 ** -0.5
    qkv = rnd(B, 1, 3, Hh, 128, dt=act, seed=91)
    q = qkv[:, :, 0]
    cache = rnd(B, Tmax, 2, Hh * 128, dt=act, seed=92)
    ramp = torch.linspace(0.0, 2.0, Tmax, device=DEV)[None, :, None, None]
    k = 0.5 * cache[:, :, 0].float().view(B, Tmax, Hh, 128) + ramp * q[:, 0].float()[:, None]
    cache[:, :, 0] = k.reshape(B, Tmax, Hh * 128).to(act)
    kq, ks = Q.quantize_cache(cache, Hh)
    deq = Q.dequantize_cache(kq, ks)
    gq, gs = _garbage(kq, ks, tk)
    out = ops.attention_decode_i8(q, gq, gs, scale=scale, tk_dev=torch.tensor([tk], device=DEV, dtype=torch.int32))
    ref = _attn64(q[:, 0], deq[:, :tk, 0], deq[:, :tk, 1], scale)
    s = torch.einsum("bhd,bthd->bht", q[:, 0].double(), deq[:, :tk, 0]) * scale
    tile_max = s.view(B, Hh, tk // 64, 64).amax(-1)
    assert float((tile_max[..., 1:] > tile_max[..., :-1].cummax(-1).values).float().mean()) > 0.5
    e = rel64(out[:, 0], ref)
    print(f"\n[attention decode int8 {act} Tk=2048 rising scores] err vs fp64 {e:.2e} (bar 5e-3)")
    assert e < 5e-3


def test_attention_decode_i8_in_a_graph_with_advancing_count(act):
    """Captured once, replayed while the device count advances: each replay equals the eager launch at that count."""
    ops = _ops()
    B, Hh, Tmax, scale = 8, 32, 320, 128 ** -0.5
    q, kq, ks = _i8_operands(B, Hh, Tmax, act, seed=55)
    tk_dev = torch.tensor([1], device=DEV, dtype=torch.int32)
    ops.attention_decode_i8(q, kq, ks, scale=scale, tk_dev=tk_dev)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.attention_decode_i8(q, kq, ks, scale=scale, tk_dev=tk_dev)
    for tk in (1, 2, 63, 64, 65, 200, 319, 320):
        tk_dev.fill_(tk)
        g.replay()
        eager = ops.attention_decode_i8(q, kq, ks, scale=scale, Tk=tk)
        assert torch.equal(bits(out), bits(eager)), tk


def test_attention_decode_i8_refuses_a_key_mask():
    ops = _ops()
    q, kq, ks = _i8_operands(1, 32, 64, torch.bfloat16, seed=3)
    with pytest.raises(NotImplementedError):
        ops.attention_decode_i8(q, kq, ks, scale=0.088, key_mask=torch.ones((1, 64), device=DEV, dtype=torch.int32))


# ------------------------------------------------------------------------------------------------ engine, 7B width
def _drive(model, ids, n_new, int8, forced=None):
    """Prefill + n_new - 1 decode steps through the engine's own calls with a 16-bit or int8 cache (device positions, as
    the captured graph reads them), feeding back the GPU's argmax, or step s the token forced[:, s - 1].
    -> (tokens (B, n_new), step logits (B, n_new, V), prefill's last-position logits, cache object after the prefill)."""
    from macaw_llm_b200.engine import KVCache, KVCacheInt8

    ops = _ops()
    eng = model.engine
    B, T0 = ids.shape
    with torch.no_grad():
        eng.set_format()
        table = eng.w(model.llm.model.embed_tokens.weight, "llm.embed")
        E = table.shape[1]
        t_max = (T0 + n_new + 63) // 64 * 64
        embeds = ops.embed_gather(table, ids).view(B, T0, E)
        cache = (KVCacheInt8 if int8 else KVCache).allocate(B, t_max, len(model.llm.model.layers), E, torch.device(DEV))
        x = eng._llama_layers(embeds.reshape(B * T0, E).clone(), B, T0, None, 0, cache, t_max)
        lg = eng._lm_head(x, rows=x.view(B, T0, E)[:, -1, :])
        snap = [c.clone() for c in cache.layers], [s.clone() for s in getattr(cache, "ks", [])]
        toks, logits = [ops.argmax_rows(lg)], [lg]
        pos_dev = torch.zeros((2,), device=DEV, dtype=torch.int32)
        for s in range(1, n_new):
            pos0 = T0 + s - 1
            pos_dev.copy_(torch.tensor([pos0, pos0 + 1], dtype=torch.int32))
            feed = toks[-1] if forced is None else forced[:, s - 1]
            x1 = eng._llama_layers(ops.embed_gather(table, feed), B, 1, None, 1, cache, t_max, pos_dev)
            lg = eng._lm_head(x1)
            logits.append(lg)
            toks.append(ops.argmax_rows(lg))
    return torch.stack(toks, 1), torch.stack(logits, 1), snap


T0, N_NEW = 60, 80


@pytest.mark.parametrize("dt,B", [(torch.bfloat16, 1), (torch.bfloat16, 8), (torch.bfloat16, 64), (torch.bfloat16, 65),
                                  (torch.float16, 8)], ids=["bf16-B1", "bf16-B8", "bf16-B64", "bf16-B65", "fp16-B8"])
def test_7b_width_int8_cache_steps_vs_fp64(dt, B):
    """2 layers at 7B width, 80 steps after a 60-token prompt.  After the prefill every layer's int8 cache is the rule of
    the 16-bit cache bitwise, and the prefill logits / first token are the 16-bit cache's.  Teacher-forced on the int8
    run's tokens, the step logits are within 1.5x max(16-bit-cache engine error, quantized fp64 decoder error) of the
    unquantized fp64 decoder."""
    model = _model_7b(dt)
    ids = _prompt(B, T0, seed=B)
    Hh = model.llm.config.num_attention_heads
    toks8, lg8, (kq, ks) = _drive(model, ids, N_NEW, int8=True)
    _, lg16, (c16, _) = _drive(model, ids, N_NEW, int8=False, forced=toks8)
    assert torch.equal(bits(lg8[:, 0]), bits(lg16[:, 0]))
    for i, c in enumerate(c16):
        q_ref, s_ref = Q.quantize_cache(c[:, :T0], Hh)
        assert torch.equal(kq[i][:, :T0], q_ref) and torch.equal(ks[i][..., :T0].view(torch.int32), s_ref.view(torch.int32)), i
    sd, hp = _ref_state(model), _hp(model)
    table = sd["llm.model.embed_tokens.weight"]
    _, ref = R.decode_logits(sd, hp, table[ids], toks8[:, :-1], device=DEV)
    _, ref_q = Q.decode_logits(sd, hp, table[ids], toks8[:, :-1], device=DEV, fmt=dt)
    e8, e16, eq = (rel64(t[:, 1:], ref[:, 1:]) for t in (lg8, lg16, ref_q))
    bar = 1.5 * max(e16, eq)
    print(f"\n[7B width int8 KV {dt} B={B}] step logits vs fp64: int8-cache engine {e8:.3e}, 16-bit-cache engine "
          f"{e16:.3e}, quantized fp64 decoder {eq:.3e} (bar {bar:.3e})")
    assert e16 < 3e-2 and e8 <= bar


@pytest.mark.parametrize("B", [8, 65])
def test_7b_width_int8_generate_matches_driven_loop_reuses_caches_and_turns_off(B):
    """generate() with the int8 cache emits the driven loop's tokens; a second call on the reused caches emits a fresh
    engine's; with the flag off again, the 16-bit cache's tokens of a fresh engine."""
    from macaw_llm_b200.engine import Engine

    model = _model_7b(torch.bfloat16)
    ids = _prompt(B, T0, seed=B)
    toks, _, _ = _drive(model, ids, N_NEW, int8=True)
    seen = set(toks.flatten().tolist())
    eos = next(i for i in range(3, 32000) if i not in seen)
    eng = model.engine
    eng.enable_int8_kv_cache()
    try:
        got = eng.generate(dict(input_ids=ids), max_new_tokens=N_NEW, eos_token_id=eos)
        assert got.shape == (B, N_NEW) and torch.equal(got, toks)
        ids2 = _prompt(B, 40, seed=100 + B)
        second = eng.generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos)
        fresh = Engine(model)
        fresh.enable_int8_kv_cache(True)
        assert torch.equal(second, fresh.generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos))
    finally:
        eng.enable_int8_kv_cache(False)
    assert not eng._decode
    off = eng.generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos)
    assert torch.equal(off, Engine(model).generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos))


# ------------------------------------------------------------------------------------------------ tiny model, combinations
@pytest.mark.parametrize("weights", ["16bit", "int8", "fp8"])
@pytest.mark.parametrize("do_sample", [False, True], ids=["greedy", "sampled"])
def test_tiny_int8_cache_with_each_weight_format(weights, do_sample):
    """The all3 case at B = 2 generates past 128 keys with the int8 cache under 16-bit, int8 and FP8 decoder weights; the
    first token is the 16-bit cache's (same prefill, same draw), and with 16-bit weights greedy it is oracle.generate_greedy's
    top-1 (or a near-tie)."""
    from oracle import macaw_oracle as O

    model, spec, hp, wts = H.build_tiny_model(DEV, torch.bfloat16)
    if weights != "16bit":
        getattr(model, f"quantize_llm_{weights}")()
    inp = H.case_inputs(spec, H.load_case("all3"))
    inp = {k: v for k, v in inp.items() if k not in ("labels", "attention_mask")}
    dev_in = {k: (v.to(DEV).to(torch.bfloat16) if isinstance(v, torch.Tensor) and v.is_floating_point()
                  else v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    kw = dict(max_new_tokens=100, do_sample=do_sample, top_k=20, seed=1234, eos_token_id=40000)
    model.enable_int8_kv_cache(True)
    t8 = model.engine.generate(dev_in, **kw)
    model.enable_int8_kv_cache(False)
    t16 = model.engine.generate(dev_in, **kw)
    T = model.prepare_inputs_for_generation(dev_in)[0].shape[1]
    assert t8.shape == (2, 100) and T + 99 > 128
    assert torch.equal(t8[:, 0], t16[:, 0])
    if weights == "16bit" and not do_sample:
        sub = {k: (v.float() if v.is_floating_point() else v) if isinstance(v, torch.Tensor) else v for k, v in inp.items()}
        _, o_logits = O.generate_greedy(sub, H.bf16_round(wts), hp, max_new_tokens=1, forced_tokens=t8[:, :1].cpu())
        for b in range(2):
            row = o_logits[b, 0]
            assert float(row.max() - row[int(t8[b, 0])]) <= 0.05 * float(row.std()) + 1e-3, b
