"""The decode step on the H100 past one key tile and at LLaMA-7B width, against fp64.

Kernel tier (bf16 and fp16 activation formats): `ops.attention` in the decode step's form (Tq = 1 over strided cache
views, key count on the device), `ops.kv_append`, `ops.argmax_rows`, `ops.embed_gather` with out-of-range ids, and
`ops.linear_thin_fused` at the 7B fused shapes.  Step tier: a 2-layer decoder at 7B width driven through the engine's
own prefill / decode calls, device positions against host positions bitwise and logits against the KV-cached fp64
reference (tests/decode_reference.py); `generate()` against that driven loop, and a second `generate()` on reused
caches.  Tiny model: a long greedy generation teacher-forced against `oracle.generate_greedy`.

Bars: norm-wise relative errors, the suite's existing ones (attention 5e-3, GEMM tails 4e-3 / SwiGLU 5e-3, logits 3e-2);
the measured values are printed (-s)."""
import numpy as np
import pytest
import torch

from tests import decode_reference as R
from tests import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from macaw_llm_b200 import ops

    return ops


@pytest.fixture(params=[torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def act(request):
    """Run the test in one activation format and restore bf16 afterwards."""
    ops = _ops()
    ops.set_act_format(request.param)
    try:
        yield request.param
    finally:
        ops.set_act_format(torch.bfloat16)


def rnd(*shape, dt, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dt)


def rel64(a, b) -> float:
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-300))


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ attention, decode form
def _attn64(q, k, v, scale, keep=None):
    """q (B, H, hd), k / v (B, Tk, H, hd), keep (B, Tk) bool | None -> (B, H, hd) fp64; a row with no key gives zeros."""
    s = torch.einsum("bhd,bthd->bht", q.double(), k.double()) * scale
    if keep is not None:
        s = s.masked_fill(~keep[:, None, :], float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    return torch.einsum("bht,bthd->bhd", p, v.double())


def _decode_operands(B, H, hd, Tmax, dt, seed):
    """q as the q-third of a fused (B, 1, 3, H, hd) activation, and a (B, Tmax, 2, H * hd) cache, as the engine holds them."""
    qkv = rnd(B, 1, 3, H, hd, dt=dt, seed=seed)
    cache = rnd(B, Tmax, 2, H * hd, dt=dt, seed=seed + 1)
    return qkv[:, :, 0], cache


def _stale(cache, tk, dt):
    """The cache with every row past tk replaced by large finite values (K ~ +-1e4, V ~ 1e30 or fp16's 6e4)."""
    st = cache.clone()
    n = st.shape[1] - tk
    if n > 0:
        sign = torch.where(torch.rand(st[:, tk:, 0].shape, device=DEV) < 0.5, -1.0, 1.0)
        st[:, tk:, 0] = (1e4 * sign).to(dt)
        st[:, tk:, 1] = 1e30 if dt == torch.bfloat16 else 6e4
    return st


@pytest.mark.parametrize("B,H,hd", [(1, 32, 128), (7, 32, 128), (64, 32, 128), (65, 32, 128), (7, 32, 64)])
def test_attention_decode_over_the_cache(act, B, H, hd):
    """Tq = 1 over a (B, 256, 2, H, hd) cache with the key count on the device: one key, a partial first tile, whole
    tiles, a partial tile after whole ones, the full capacity.  Against fp64; the rows past the count — stale values,
    zeros, or absent (host length) — do not change a bit; a count above the capacity clamps to it."""
    ops = _ops()
    Tmax, scale = 256, hd ** -0.5
    q, cache = _decode_operands(B, H, hd, Tmax, act, seed=10 * B + hd)
    qr = q[:, 0]
    errs = []
    for tk in (1, 63, 64, 65, 129, 200, 256):
        tk_dev = torch.tensor([tk], device=DEV, dtype=torch.int32)
        runs = {}
        for name, c in (("stale", _stale(cache, tk, act)), ("zero", cache.clone())):
            if name == "zero":
                c[:, tk:] = 0
            kv = c.unflatten(-1, (H, hd))
            runs[name] = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, tk_dev=tk_dev)
        kv = cache[:, :tk].unflatten(-1, (H, hd))
        runs["host"] = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale)
        if tk == Tmax:
            kv = cache.unflatten(-1, (H, hd))
            runs["clamp"] = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale,
                                          tk_dev=torch.tensor([Tmax + 37], device=DEV, dtype=torch.int32))
        ref = _attn64(qr, kv[:, :tk, 0], kv[:, :tk, 1], scale)
        e = rel64(runs["stale"][:, 0], ref)
        errs.append(e)
        assert e < 5e-3, (tk, e)
        for name, out in runs.items():
            assert torch.equal(bits(out), bits(runs["stale"])), (tk, name)
    print(f"\n[attention decode {act} B={B} hd={hd}] max err vs fp64 {max(errs):.2e} (bar 5e-3)")


def test_attention_decode_key_mask_and_zero_keys(act):
    """tk_dev together with a (B, Tmax) key mask that masks keys below the count, and a count of zero (every key masked:
    zeros, DESIGN.md "unspecified rows")."""
    ops = _ops()
    B, H, hd, Tmax, scale = 5, 32, 128, 256, 128 ** -0.5
    q, cache = _decode_operands(B, H, hd, Tmax, act, seed=77)
    g = torch.Generator(device=DEV).manual_seed(78)
    km = (torch.rand(B, Tmax, generator=g, device=DEV) > 0.3).to(torch.int32)
    km[:, 0] = 1
    kv = cache.unflatten(-1, (H, hd))
    for tk in (1, 65, 129, 200):
        out = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, key_mask=km,
                            tk_dev=torch.tensor([tk], device=DEV, dtype=torch.int32))
        ref = _attn64(q[:, 0], kv[:, :tk, 0], kv[:, :tk, 1], scale, keep=km[:, :tk].bool())
        assert rel64(out[:, 0], ref) < 5e-3, tk
    out = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, tk_dev=torch.zeros(1, device=DEV, dtype=torch.int32))
    assert float(out.abs().max()) == 0.0


def test_attention_decode_long_rising_scores(act):
    """Tk = 2048 keys at Tq = 1 whose scores keep growing along the sequence: the running max is rescaled at every one of
    the 32 key tiles."""
    ops = _ops()
    B, H, hd, Tmax, tk = 2, 32, 128, 2112, 2048
    scale = hd ** -0.5
    q, cache = _decode_operands(B, H, hd, Tmax, act, seed=90)
    qf = q[:, 0].float()  # (B, H, hd)
    ramp = torch.linspace(0.0, 2.0, Tmax, device=DEV)[None, :, None, None]
    k = 0.5 * cache[:, :, 0].float().view(B, Tmax, H, hd) + ramp * qf[:, None]
    cache[:, :, 0] = k.reshape(B, Tmax, H * hd).to(act)
    kv = _stale(cache, tk, act).unflatten(-1, (H, hd))
    out = ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, tk_dev=torch.tensor([tk], device=DEV, dtype=torch.int32))
    ref = _attn64(q[:, 0], kv[:, :tk, 0], kv[:, :tk, 1], scale)
    s = torch.einsum("bhd,bthd->bht", q[:, 0].double(), kv[:, :tk, 0].double()) * scale
    tile_max = s.view(B, H, tk // 64, 64).amax(-1)
    assert float((tile_max[..., 1:] > tile_max[..., :-1].cummax(-1).values).float().mean()) > 0.5  # the max keeps moving
    e = rel64(out[:, 0], ref)
    print(f"\n[attention decode {act} Tk=2048 rising scores] err vs fp64 {e:.2e} (bar 5e-3)")
    assert e < 5e-3


# ------------------------------------------------------------------------------------------------ kv_append
@pytest.mark.parametrize("B,T_new", [(1, 1), (1, 37), (65, 1), (65, 37)])
def test_kv_append_writes_only_its_slots(act, B, T_new):
    ops = _ops()
    E, Tmax = 4096, 64
    buf = rnd(B * T_new, 3 * E + 64, dt=act, seed=B + T_new)
    qkv = buf[:, :3 * E]  # row stride 3E + 64
    sentinel = torch.full((B, Tmax, 2, E), -1234.5, device=DEV, dtype=act)
    new_k = qkv[:, E:2 * E].reshape(B, T_new, E)
    new_v = qkv[:, 2 * E:].reshape(B, T_new, E)
    for t0, dev_t0 in ((3, None), (Tmax - T_new, None), (17, 17)):
        cache = sentinel.clone()
        if dev_t0 is None:
            ops.kv_append(qkv, B, T_new, cache, t0)
        else:  # the host offset is ignored when the device one is given
            ops.kv_append(qkv, B, T_new, cache, 0, torch.tensor([dev_t0], device=DEV, dtype=torch.int32))
        assert torch.equal(bits(cache[:, t0:t0 + T_new, 0]), bits(new_k)), t0
        assert torch.equal(bits(cache[:, t0:t0 + T_new, 1]), bits(new_v)), t0
        cache[:, t0:t0 + T_new] = sentinel[:, t0:t0 + T_new]
        assert torch.equal(bits(cache), bits(sentinel)), t0


# ------------------------------------------------------------------------------------------------ argmax_rows
def _crafted_rows(V):
    """Rows where the lowest-index rule matters: ties across threads, warps and loop iterations of the 512-thread CTA."""
    rows = []

    def base(seed):
        return torch.randn(V, generator=torch.Generator().manual_seed(seed))

    for c, others in ((5, (6, 37, 517, 8197)), (40, (72,)), (300, (812,)), (511, (8703,)), (0, (V - 1,)), (1, (31999,))):
        r = base(c)
        for i in (c,) + others:
            if i < V:
                r[i] = 40.0
        rows.append(r)
    rows.append(torch.full((V,), 3.0))                      # all equal -> 0
    rows.append(torch.full((V,), float("-inf")))            # all -inf -> 0
    r = base(99)
    r[V // 3] = float("inf")
    r[V - 1] = float("inf")
    rows.append(r)                                           # +inf, twice
    r = base(98)
    r[V - 1] = float("inf")
    rows.append(r)                                           # +inf at the end
    return rows


@pytest.mark.parametrize("V", [1, 512, 32000, 32007])
@pytest.mark.parametrize("rows", [1, 64, 65])
def test_argmax_rows_first_occurrence(act, V, rows):
    """mm_argmax_rows against torch.argmax (first occurrence), bitwise, on row-strided views (ld > V)."""
    ops = _ops()
    crafted = _crafted_rows(V)
    for start in range(0, len(crafted), rows):
        g = torch.Generator().manual_seed(start + V)
        x = torch.randn(rows, V + 13, generator=g)
        for i, r in enumerate(crafted[start:start + rows]):
            x[i, :V] = r
        xd = x.to(act).to(DEV)[:, :V]  # ties also arise from rounding to 16 bits
        got = ops.argmax_rows(xd)
        ref = xd.float().cpu().argmax(dim=1)
        assert torch.equal(got.cpu(), ref), (start, torch.nonzero(got.cpu() != ref).flatten().tolist())
    if V > 1:  # the all-equal and all -inf rows
        assert int(ops.argmax_rows(torch.full((2, V), 3.0, device=DEV, dtype=act)).max()) == 0
        assert int(ops.argmax_rows(torch.full((2, V), float("-inf"), device=DEV, dtype=act)).max()) == 0


# ------------------------------------------------------------------------------------------------ embed_gather
def test_embed_gather_clamps_out_of_range_ids(act):
    """Ids outside the table read its nearest row: the pad id 32006 of a finished row and anything larger read row V - 1,
    negative ids row 0 (the clamp `oracle.generate_greedy` applies), bit for bit, for int64 and int32 ids."""
    ops = _ops()
    V, E = 32000, 512
    table = rnd(V, E, dt=act, seed=5)
    ids = torch.tensor([0, 7, V - 1, V, 32006, 40000, 2 ** 31 - 1, 2 ** 40, -1, -32006, -2 ** 40, 1234], device=DEV)
    ref = table[ids.clamp(0, V - 1)]
    assert torch.equal(bits(ops.embed_gather(table, ids)), bits(ref))
    ids32 = ids.clamp(-2 ** 31, 2 ** 31 - 1).to(torch.int32)
    assert torch.equal(bits(ops.embed_gather(table, ids32)), bits(table[ids32.long().clamp(0, V - 1)]))
    out = torch.zeros((ids.numel(), E + 64), device=DEV, dtype=act)
    ops.embed_gather(table, ids, out=out[:, :E])
    assert torch.equal(bits(out[:, :E]), bits(ref)) and float(out[:, E:].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ rope tables
def test_engine_rope_tables_match_the_oracles():
    """Engine.rope_tables computes cos / sin on the device; they are within a few fp32 ulps of the oracle's CPU tables up
    to position 2047, so the fp64 references below (which widen the CPU tables) use the engine's own angles."""
    from macaw_llm_b200.engine import Engine

    cos_d, sin_d = Engine(None).rope_tables(2048, 128, torch.device(DEV))
    cos_h, sin_h = R.rope_tables(2048, 128)
    n_ulp = []
    for d, h in ((cos_d, cos_h), (sin_d, sin_h)):
        ulp = torch.from_numpy(np.spacing(h.abs().numpy()))
        n_ulp.append(float(((d.cpu() - h).abs() / ulp).max()))
    print(f"\n[rope tables] max distance from the oracle's tables: cos {n_ulp[0]:.0f} ulp, sin {n_ulp[1]:.0f} ulp (bar 4)")
    assert max(n_ulp) <= 4, n_ulp


# ------------------------------------------------------------------------------------------------ thin GEMM tails, 7B
_W7 = {}


def _weights_7b(dt):
    if dt not in _W7:
        _W7.clear()
        E, I = 4096, 11008
        _W7[dt] = dict(qkv=rnd(3 * E, E, dt=dt, scale=E ** -0.5, seed=1), gu=rnd(2 * I, E, dt=dt, scale=E ** -0.5, seed=2),
                       o=rnd(E, E, dt=dt, scale=E ** -0.5, seed=3), d=rnd(E, I, dt=dt, scale=I ** -0.5, seed=4))
    return _W7[dt]


@pytest.mark.parametrize("M", [1, 8, 13, 64])
def test_thin_fused_tails_at_the_7b_shapes(act, M):
    """mm_thin_fused after the split-K thin GEMM at the 7B fused shapes: QKV (12288 x 4096) with RoPE from the engine's
    tables at positions up to 2047 (device position / slot, and the host offset form bitwise), SwiGLU (22016 x 4096) with
    the row scale from RMS statistics, residual o_proj (4096 x 4096) and down_proj (4096 x 11008) with the statistics out."""
    from macaw_llm_b200.engine import Engine

    ops = _ops()
    E, I, eps, Tmax = 4096, 11008, 1e-6, 8
    w = _weights_7b(act)
    x = rnd(M, E, dt=act, seed=100 + M)
    errs = {}
    # QKV + RoPE + cache slot
    cos, sin = Engine(None).rope_tables(2048, 128, torch.device(DEV))
    c64, s64 = [t.double().to(DEV) for t in R.rope_tables(2048, 128)]
    rs = torch.rand(M, device=DEV) + 0.5
    y = ((x.double() * rs.double()[:, None]) @ w["qkv"].double().t()).view(M, 3, E // 128, 2, 64)
    sentinel = torch.full((M, Tmax, 2, E), 777.0, device=DEV, dtype=act)
    for pos, slot in ((0, 0), (63, 5), (64, 1), (1000, 7), (2047, 3)):
        c, s = c64[pos][None, None], s64[pos][None, None]
        rot = lambda t: torch.stack([t[:, :, 0] * c - t[:, :, 1] * s, t[:, :, 1] * c + t[:, :, 0] * s], 2).reshape(M, E)  # noqa: E731
        cache = sentinel.clone()
        out = ops.linear_thin_fused(x, w["qkv"], ops.THIN_QKV, row_scale=rs, cache=cache,
                                    rope=(cos, sin, torch.tensor([pos], device=DEV, dtype=torch.int32)),
                                    t0_dev=torch.tensor([slot], device=DEV, dtype=torch.int32))
        errs[f"q@{pos}"] = rel64(out[:, :E], rot(y[:, 0]))
        errs[f"k@{pos}"] = rel64(cache[:, slot, 0], rot(y[:, 1]))
        errs[f"v@{pos}"] = rel64(cache[:, slot, 1], y[:, 2].reshape(M, E))
        others = cache.clone()
        others[:, slot] = sentinel[:, slot]
        assert torch.equal(bits(others), bits(sentinel)), pos  # only slot `slot` was written
        cache2 = sentinel.clone()
        out2 = ops.linear_thin_fused(x, w["qkv"], ops.THIN_QKV, row_scale=rs, rope=(cos[pos:], sin[pos:], None),
                                     cache=cache2, t0=slot)
        assert torch.equal(bits(out2[:, :E]), bits(out[:, :E])) and torch.equal(bits(cache2), bits(cache)), pos
    # RES (o_proj, down_proj) in place on the residual stream, statistics of the stored values out
    stream0 = rnd(M, E, dt=act, seed=200 + M)
    for name, K in (("o", E), ("d", I)):
        a = rnd(M, K, dt=act, seed=300 + K + M)
        stream, ss = stream0.clone(), torch.empty((M, E // 32), device=DEV, dtype=torch.float32)
        ops.linear_thin_fused(a, w[name], ops.THIN_RES, residual=stream, out=stream, sumsq_out=ss)
        errs[f"res_{name}"] = rel64(stream, a.double() @ w[name].double().t() + stream0.double())
        errs[f"sumsq_{name}"] = rel64(ss, stream.double().view(M, E // 32, 32).pow(2).sum(-1))
        assert errs[f"sumsq_{name}"] < 1e-5
    # SWIGLU with the RMSNorm row scale from the statistics of the stream
    ss = stream.float().view(M, E // 32, 32).pow(2).sum(-1).contiguous()
    gsw = ops.linear_thin_fused(stream, w["gu"], ops.THIN_SWIGLU, rms_from=(ss, eps))
    rstd = torch.rsqrt(stream.double().pow(2).mean(1, keepdim=True) + eps)
    yy = ((stream.double() * rstd) @ w["gu"].double().t()).view(M, I // 32, 2, 32)
    errs["swiglu"] = rel64(gsw, (torch.nn.functional.silu(yy[:, :, 0]) * yy[:, :, 1]).reshape(M, I))
    print(f"\n[thin tails 7B {act} M={M}] " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < (5e-3 if k == "swiglu" else 4e-3), (k, v)


# ------------------------------------------------------------------------------------------------ step tier: 7B width
_MODELS = {}


def _model_7b(dt):
    """bench.real_configs() with 2 decoder layers (encoders cut to 1 layer: text-only prompts never run them)."""
    if dt not in _MODELS:
        import bench
        from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

        _MODELS.clear()
        torch.cuda.empty_cache()
        (clip, whisper, llama), hyper = bench.real_configs()
        clip.vision_config.num_hidden_layers = 1
        whisper.encoder_layers = 1
        llama.num_hidden_layers = 2
        cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
        _MODELS[dt] = MM_LLMs.build_random(cfg, device=DEV, dtype=dt, seed=3)
    return _MODELS[dt]


def _prompt(B, T, seed):
    ids = torch.randint(3, 32000 - 6, (B, T), generator=torch.Generator().manual_seed(seed))
    ids[:, 0] = 1
    return ids.to(DEV)


def _drive(model, ids, n_new, host_too=False):
    """Prefill + n_new - 1 decode steps through the engine's own calls, as Engine.generate makes them (the decode step
    eagerly, with the device-side position the captured graph reads), feeding back the GPU's argmax.  With host_too the
    same steps also run with host positions on a copy of the prefilled cache.  -> (tokens (B, n_new), step logits list,
    host-position step logits list, engine prefill logits (B, T0, V))."""
    ops = _ops()
    eng = model.engine
    B, T0 = ids.shape
    with torch.no_grad():
        eng.set_format()
        table = eng.w(model.llm.model.embed_tokens.weight, "llm.embed")
        E = table.shape[1]
        t_max = (T0 + n_new + 63) // 64 * 64
        embeds = ops.embed_gather(table, ids).view(B, T0, E)
        pre_logits = eng.llama_forward(embeds.clone(), None)
        cache = [torch.zeros((B, t_max, 2, E), device=DEV, dtype=table.dtype) for _ in model.llm.model.layers]
        x = eng._llama_layers(embeds.reshape(B * T0, E).clone(), B, T0, None, 0, cache, t_max)
        lg = eng._lm_head(x, rows=x.view(B, T0, E)[:, -1, :])
        cache_h = [c.clone() for c in cache] if host_too else None
        toks, dev_logits, host_logits = [ops.argmax_rows(lg)], [lg], [lg]
        pos_dev = torch.zeros((2,), device=DEV, dtype=torch.int32)
        for s in range(1, n_new):
            pos0 = T0 + s - 1
            pos_dev.copy_(torch.tensor([pos0, pos0 + 1], dtype=torch.int32))
            x1 = eng._llama_layers(ops.embed_gather(table, toks[-1]), B, 1, None, 1, cache, t_max, pos_dev)
            lg = eng._lm_head(x1)
            dev_logits.append(lg)
            if host_too:
                x1 = eng._llama_layers(ops.embed_gather(table, toks[-1]), B, 1, None, pos0, cache_h, t_max)
                host_logits.append(eng._lm_head(x1))
            toks.append(ops.argmax_rows(lg))
    return torch.stack(toks, 1), dev_logits, host_logits, pre_logits


def _ref_state(model):
    return {k: v.detach().to(torch.float64) for k, v in model.state_dict().items()
            if k.startswith("llm.") and v.is_floating_point() and not k.endswith("inv_freq")}


def _hp(model):
    c = model.llm.config
    return dict(llama=dict(hidden=c.hidden_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                           eps=c.rms_norm_eps, vocab=c.vocab_size))


def _check_tokens(toks, ref_steps, logits):
    """Every emitted token is the reference's top-1 or within 0.05 std of it (test_generate_greedy_vs_oracle's rule), or
    within 6x the RMS error of that step's logits: at 7B width the bf16 logits carry ~0.012 RMS error each, so among
    thousands of tokens a near-tie a little wider than 0.05 std (0.065 here) flips now and then; two logits whose errors
    differ by 6x the RMS error is a 4-sigma event."""
    top = ref_steps.max(-1).values
    got = ref_steps.gather(-1, toks[..., None].to(ref_steps.device))[..., 0]
    gap = top - got
    rms = (logits.double() - ref_steps).pow(2).mean(-1).sqrt()
    bar = torch.maximum(0.05 * ref_steps.std(-1) + 1e-3, 6 * rms)
    bad = torch.nonzero(gap > bar)
    assert bad.numel() == 0, [(int(b), int(s), float(gap[b, s]), float(bar[b, s])) for b, s in bad[:5].tolist()]


T0, N_NEW = 60, 80  # t_max 192: the key count crosses 64 and 128


@pytest.mark.parametrize("dt,B", [(torch.bfloat16, 1), (torch.bfloat16, 8), (torch.bfloat16, 64), (torch.bfloat16, 65),
                                  (torch.float16, 8)], ids=["bf16-B1", "bf16-B8", "bf16-B64", "bf16-B65", "fp16-B8"])
def test_7b_width_decode_steps_vs_fp64(dt, B):
    """Real width, 2 layers, 80 greedy steps after a 60-token prompt.  Each step's logits with device positions equal
    those with host positions bitwise; at the first step, at 64 / 65 / 128 / 129 keys and at the last step they are as
    close to the fp64 reference as the engine's own prefill logits are (1.5x, and 3e-2); every token is the reference's
    top-1, or a near-tie within the greedy test's margin or the step's own logit error (_check_tokens)."""
    model = _model_7b(dt)
    ids = _prompt(B, T0, seed=B)
    toks, dev_logits, host_logits, pre_logits = _drive(model, ids, N_NEW, host_too=True)
    for s, (a, b) in enumerate(zip(dev_logits, host_logits)):
        assert torch.equal(bits(a), bits(b)), s
    sd = _ref_state(model)
    table = sd["llm.model.embed_tokens.weight"]
    ref_pre, ref_steps = R.decode_logits(sd, _hp(model), table[ids], toks[:, :-1], device=DEV)
    e_pre = rel64(pre_logits, ref_pre)
    bar = min(1.5 * e_pre, 3e-2)
    errs = {}
    for tk in (T0 + 1, 64, 65, 128, 129, T0 + N_NEW - 1):
        s = tk - T0  # step s attends over T0 + s keys
        errs[tk] = rel64(dev_logits[s], ref_steps[:, s])
    print(f"\n[7B width {dt} B={B}] prefill logits err {e_pre:.3e}; decode step err by key count "
          + " ".join(f"{k}:{v:.3e}" for k, v in errs.items()) + f" (bar {bar:.3e})")
    for tk, e in errs.items():
        assert e <= bar, (tk, e, bar)
    _check_tokens(toks, ref_steps, torch.stack(dev_logits, 1))


@pytest.mark.parametrize("B", [8, 65])
def test_7b_width_generate_matches_driven_loop_and_reuses_caches(B):
    """generate() (eager first step, then graph replays) emits the driven loop's tokens bitwise; a second call on the same
    (batch, capacity) caches — shorter prompt, more new tokens, stale rows left from the first call — emits the tokens of
    a fresh engine."""
    from macaw_llm_b200.engine import Engine

    model = _model_7b(torch.bfloat16)
    ids = _prompt(B, T0, seed=B)
    toks, _, _, _ = _drive(model, ids, N_NEW)
    seen = set(toks.flatten().tolist())
    eos = next(i for i in range(3, 32000) if i not in seen)  # never emitted: all 80 steps run
    eng = model.engine
    got =eng.generate(dict(input_ids=ids), max_new_tokens=N_NEW, eos_token_id=eos)
    assert got.shape == (B, N_NEW) and torch.equal(got, toks)
    ids2 = _prompt(B, 40, seed=100 + B)
    assert (40 + 100 + 63) // 64 * 64 == (T0 + N_NEW + 63) // 64 * 64
    second = eng.generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos)
    fresh = Engine(model).generate(dict(input_ids=ids2), max_new_tokens=100, eos_token_id=eos)
    assert second.shape == fresh.shape and torch.equal(second, fresh)


# ------------------------------------------------------------------------------------------------ tiny model, long run
@pytest.mark.parametrize("B", [2, 66])
def test_tiny_long_generation_vs_oracle(B):
    """The all3 case (T = 50) with 90 new tokens, so the key count passes 128; at B = 66 (the samples replicated) the
    16-bit B > 64 decode path meets an independent reference.  Teacher-forced against oracle.generate_greedy."""
    from oracle import macaw_oracle as O

    model, spec, hp, weights = H.build_tiny_model(DEV, torch.bfloat16)
    inp = H.case_inputs(spec, H.load_case("all3"))
    inp = {k: v for k, v in inp.items() if k not in ("labels", "attention_mask")}
    B0 = inp["input_ids"].shape[0]
    idx = torch.arange(B) % B0
    big = {k: (v[idx] if isinstance(v, torch.Tensor) and v.shape[0] == B0 else v) for k, v in inp.items()}
    big = {k: (v.to(torch.bfloat16) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in big.items()}
    n_new = 90
    toks = model(dict({k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in big.items()}, inference=True,
                      max_new_tokens=n_new)).cpu()
    T = model.prepare_inputs_for_generation({k: (v.to(DEV) if isinstance(v, torch.Tensor) else v)
                                             for k, v in big.items()})[0].shape[1]
    alive = (toks != 32006).sum(1)  # tokens each row emitted before and including its EOS
    assert T + int(alive.max()) - 1 > 128, (T, toks.shape)
    # rows that share a sample and a token sequence share the oracle run
    uniq = {}
    for b in range(B):
        uniq.setdefault((b % B0, tuple(toks[b].tolist())), b)
    rows = list(uniq.values())
    sub = {k: (v[rows].float() if v.is_floating_point() else v[rows]) if isinstance(v, torch.Tensor) else v
           for k, v in big.items()}
    _, o_logits = O.generate_greedy(sub, H.bf16_round(weights), hp, max_new_tokens=toks.shape[1], forced_tokens=toks[rows])
    n_cmp = 0
    for j, b in enumerate(rows):
        for s_ in range(o_logits.shape[1]):
            t = int(toks[b, s_])
            if t == 32006:
                continue
            row = o_logits[j, s_]
            gap = float(row.max() - row[t])
            assert gap <= 0.05 * float(row.std()) + 1e-3, (b, s_, t, int(row.argmax()), gap)
            n_cmp += 1
    print(f"\n[tiny long generate B={B}] T={T}, {toks.shape[1]} steps, {len(rows)} distinct rows, {n_cmp} tokens checked")
