"""GPU tier of the int8 decoder weights (quant.py, csrc/quant.cu): the quantization kernel bit-exact against the CPU rule,
the dequantization bit-exact in both fused layouts, the int8 decode GEMM with each tail against fp64, the tiny model's
forward bitwise against the engine on the dequantized weights, generation against the oracle, a 7B decode step against a
fresh prefill, and the lifecycle (memory, stale graphs, state dicts, refusals).  Every model here is built by this file."""
import copy
import re

import pytest
import torch

from tests import helpers as H
from tests.test_quant_cpu import crafted_rows, quantize_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops(dt=torch.bfloat16):
    from macaw_llm_b200 import ops

    ops.set_act_format(dt)
    return ops


def rnd(*shape, scale=1.0, seed=0, dt=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dt)


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(4096, 4096), (11008, 4096), (4096, 11008)])
def test_quantize_kernel_is_bit_exact(shape, dt):
    ops = _ops(dt)
    N, K = shape
    w = rnd(N, K, scale=0.02, seed=N + K, dt=dt)
    c = crafted_rows(K).to(DEV).to(dt)
    w[: c.shape[0]] = c
    w[7, 100] = 3.0  # an outlier row
    q, s = ops.quantize_rows_int8(w)
    qr, sr = quantize_ref(w.cpu())
    assert torch.equal(s.cpu(), sr) and torch.equal(q.cpu(), qr)
    # a strided view quantizes the same rows
    wide = torch.zeros((N, K + 64), device=DEV, dtype=dt)
    wide[:, :K] = w
    q2, s2 = ops.quantize_rows_int8(wide[:, :K])
    assert torch.equal(q2, q) and torch.equal(s2, s)


def _sources(rows, K, seed, dt=torch.bfloat16):
    from macaw_llm_b200 import ops

    qs, ss = [], []
    for j, r in enumerate(rows):
        q, s = ops.quantize_rows_int8(rnd(r, K, scale=0.02, seed=seed + j, dt=dt))
        qs.append(q)
        ss.append(s)
    return qs, ss


def _deq(q, s):
    return q.float() * s[:, None]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_dequant_rows_bit_exact_in_both_layouts(dt):
    ops = _ops(dt)
    E, I = 512, 1024
    g1 = (1.0 + rnd(E, scale=0.1, seed=1, dt=dt).float()).to(dt)
    qs, ss = _sources((E, E, E), E, 10, dt)
    got = ops.dequant_rows(ops.W8Matrix(qs, ss, gain=g1))
    ref = (torch.cat([_deq(q, s) for q, s in zip(qs, ss)], 0) * g1.float()[None, :]).to(dt)
    assert torch.equal(got, ref)
    qs, ss = _sources((I, I), E, 20, dt)
    got = ops.dequant_rows(ops.W8Matrix(qs, ss, interleave=True, gain=g1))
    ref = torch.stack([(_deq(qs[0], ss[0]) * g1.float()[None]).to(dt).view(I // 32, 32, E),
                       (_deq(qs[1], ss[1]) * g1.float()[None]).to(dt).view(I // 32, 32, E)], 1).reshape(2 * I, E)
    assert torch.equal(got, ref)
    qs, ss = _sources((E,), I, 30, dt)
    assert torch.equal(ops.dequant_rows(ops.W8Matrix(qs, ss)), _deq(qs[0], ss[0]).to(dt))


SHAPES = {"real": (4096, 11008), "tiny": (256, 512)}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M", [1, 8, 13, 64])
@pytest.mark.parametrize("size", ["real", "tiny"])
def test_w8_decode_gemm_with_each_tail(size, M, dt):
    """s_n * sum q x~ (x~ = round16(x g)) through the three mm_thin_fused tails against fp64: RES with statistics (o_proj
    and down_proj shapes), SWIGLU with rms_from, QKV with RoPE and the cache write at host and device positions."""
    ops = _ops(dt)
    E, I = SHAPES[size]
    Tmax, t0, eps = 24, 5, 1e-6
    d = lambda t: t.double().cpu()  # noqa: E731
    g1 = (1.0 + rnd(E, scale=0.1, seed=2, dt=dt).float()).to(dt)
    g2 = (1.0 + rnd(E, scale=0.1, seed=3, dt=dt).float()).to(dt)
    xt = lambda x, g: (x.float() * g.float()[None]).to(dt) if g is not None else x  # noqa: E731  x~ = round16(x g)

    # RES (o_proj: E x E), in place on the residual stream, statistics out
    x, res = rnd(M, E, seed=300, dt=dt), rnd(M, E, seed=302, dt=dt)
    qo, so = _sources((E,), E, 40, dt)
    ss = torch.empty((M, E // 32), device=DEV, dtype=torch.float32)
    stream = res.clone()
    ops.linear_w8_thin_fused(x, ops.W8Matrix(qo, so), ops.THIN_RES, residual=stream, out=stream, sumsq_out=ss)
    ref = d(x) @ d(_deq(qo[0], so[0])).t() + d(res)
    assert H.rel_err(stream, ref) < 4e-3
    assert H.rel_err(ss.sum(1), stream.float().pow(2).sum(1)) < 1e-5
    # RES (down_proj: E x I)
    h = rnd(M, I, seed=305, dt=dt)
    qd, sd = _sources((E,), I, 50, dt)
    out = ops.linear_w8_thin_fused(h, ops.W8Matrix(qd, sd), ops.THIN_RES, residual=res)
    assert H.rel_err(out, d(h) @ d(_deq(qd[0], sd[0])).t() + d(res)) < 4e-3
    # SWIGLU with the row scale from those statistics, gain g2 on the activation rows
    qg, sg = _sources((I, I), E, 60, dt)
    g = ops.linear_w8_thin_fused(stream, ops.W8Matrix(qg, sg, interleave=True, gain=g2), ops.THIN_SWIGLU, rms_from=(ss, eps))
    rstd = torch.rsqrt(d(stream).pow(2).mean(1, keepdim=True) + eps)
    xs = d(xt(stream, g2))
    gate, up = rstd * (xs @ d(_deq(qg[0], sg[0])).t()), rstd * (xs @ d(_deq(qg[1], sg[1])).t())
    assert H.rel_err(g, torch.nn.functional.silu(gate) * up) < 5e-3
    # QKV: gain g1, RoPE at the device-side position, q -> out, k / v -> the cache slot
    qq, sq = _sources((E, E, E), E, 70, dt)
    W = ops.W8Matrix(qq, sq, gain=g1)
    rs = torch.rand(M, device=DEV) + 0.5
    cos, sin = torch.rand(Tmax, 64, device=DEV), torch.rand(Tmax, 64, device=DEV)
    cache = torch.zeros((M, Tmax, 2, E), device=DEV, dtype=dt)
    pos = torch.tensor([t0], device=DEV, dtype=torch.int32)
    out = ops.linear_w8_thin_fused(x, W, ops.THIN_QKV, row_scale=rs, rope=(cos, sin, pos), cache=cache, t0_dev=pos)
    y = (d(rs)[:, None] * (d(xt(x, g1)) @ torch.cat([d(_deq(q, s)) for q, s in zip(qq, sq)]).t())).view(M, 3, E // 128, 128)
    c = torch.cat([cos[t0], cos[t0]]).double().cpu()[None, None, :]
    s_ = torch.cat([sin[t0], sin[t0]]).double().cpu()[None, None, :]
    rot = lambda t: t * c + torch.cat([-t[..., 64:], t[..., :64]], -1) * s_  # noqa: E731
    assert H.rel_err(out[:, :E], rot(y[:, 0]).reshape(M, E)) < 4e-3
    assert H.rel_err(cache[:, t0, 0], rot(y[:, 1]).reshape(M, E)) < 4e-3
    assert H.rel_err(cache[:, t0, 1], y[:, 2].reshape(M, E)) < 4e-3
    assert float(cache[:, :t0].abs().sum()) == 0 and float(cache[:, t0 + 1:].abs().sum()) == 0
    cache2 = torch.zeros_like(cache)
    out2 = ops.linear_w8_thin_fused(x, W, ops.THIN_QKV, row_scale=rs, rope=(cos[t0:], sin[t0:], None), cache=cache2, t0=t0)
    assert torch.equal(out2[:, :E], out[:, :E]) and torch.equal(cache2, cache)


@pytest.mark.parametrize("M", [1, 8, 64])
def test_w8_decode_gemm_at_the_7b_fused_shapes(M):
    """The fused [q; k; v] (12288 x 4096) and [gate | up] (22016 x 4096) launches at LLaMA-7B width, bf16 and fp16."""
    for dt in (torch.bfloat16, torch.float16):
        ops = _ops(dt)
        E, I = 4096, 11008
        x = rnd(M, E, seed=M, dt=dt)
        for rows, inter in (((E, E, E), False), ((I, I), True)):
            qs, ss = _sources(rows, E, 80, dt)
            W = ops.W8Matrix(qs, ss, interleave=inter)
            out = ops.linear_w8_thin_fused(x, W, ops.THIN_RES, residual=torch.zeros((M, W.N), device=DEV, dtype=dt))
            ref = (x.double().cpu() @ ops.dequant_rows(W).double().cpu().t())
            assert H.rel_err(out, ref) < 4e-3, (dt, rows)


# ---------------------------------------------------------------------------------------------------- tiny model
def _inputs(spec, name, dt, drop=("labels",)):
    inp = H.case_inputs(spec, H.load_case(name))
    return {k: (v.to(dt).cuda() if isinstance(v, torch.Tensor) and v.is_floating_point() else
                (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items() if k not in drop}


def _twin_on_dequantized(model16, qmodel):
    """A copy of the 16-bit model whose decoder projections hold the fp32 values q * s of the quantized model."""
    from macaw_llm_b200 import quant

    twin = copy.deepcopy(model16)
    for lt, lq in zip(twin.llm.model.layers, qmodel.llm.model.layers):
        for parent, name in quant.PROJECTIONS:
            getattr(getattr(lt, parent), name).weight = torch.nn.Parameter(
                getattr(getattr(lq, parent), name).dequantized(), requires_grad=False)
    return twin


def _oracle_sd(weights, qmodel, dt):
    sd = {k: (v.to(dt).float() if v.is_floating_point() else v) for k, v in weights.items()}
    for k, v in qmodel.state_dict().items():
        if k.endswith(".weight") and v.dtype == torch.int8:
            sd[k] = v.float().cpu() * qmodel.state_dict()[k + "_scale"].cpu()[:, None]
    return sd


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_tiny_model_forward_and_generate(dt):
    from oracle import macaw_oracle as O

    model16, spec, hp, weights = H.build_tiny_model("cuda", dt)
    qm = copy.deepcopy(model16)
    qm.quantize_llm_int8()
    twin = _twin_on_dequantized(model16, qm)
    for name in ("all3", "text"):
        inp = _inputs(spec, name, dt, drop=())
        a, b = qm(inp), twin(inp)
        assert torch.equal(a.logits, b.logits), name  # prefill on dequantized weights == the engine on q * s in fp32
        if a.loss is not None:  # mm_ce_loss sums rows with atomicAdd: the order, hence the last bit, may vary per call
            assert abs(float(a.loss) - float(b.loss)) <= 1e-6 * abs(float(b.loss))
    # eval forward against the oracle on q * s
    case = H.load_case("all3")
    inp = _inputs(spec, "all3", dt, drop=())
    out = qm(inp)
    host = {k: (v.float().cpu() if isinstance(v, torch.Tensor) and v.is_floating_point() else
                (v.cpu() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()}
    o = O.forward(host, _oracle_sd(weights, qm, dt), hp, dtype=torch.float32)
    valid = torch.from_numpy(case["attention_mask"]).bool()
    e_log = H.rel_err(out.logits.cpu()[valid], o["logits"][valid])
    print(f"\n[int8 {dt}] logits vs oracle on q*s: {e_log:.3e}")
    assert e_log < (2e-3 if dt == torch.float16 else 3e-2)
    # greedy generate, teacher-forced against the oracle (criterion of test_generate_greedy_vs_oracle)
    n_new = 6
    inp = _inputs(spec, "all3", dt)
    toks = qm(dict(inp, inference=True, max_new_tokens=n_new))
    assert toks.dtype == torch.int64 and toks.shape[0] == 2 and 1 <= toks.shape[1] <= n_new
    host = {k: (v.float().cpu() if isinstance(v, torch.Tensor) and v.is_floating_point() else
                (v.cpu() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()}
    _, o_logits = O.generate_greedy(host, _oracle_sd(weights, qm, dt), hp, max_new_tokens=toks.shape[1],
                                    forced_tokens=toks.cpu())
    for b in range(toks.shape[0]):
        for s_ in range(toks.shape[1]):
            t = int(toks[b, s_])
            if t == 32006:
                continue
            row = o_logits[b, s_]
            gap = float(row.max() - row[t])
            assert gap <= 0.05 * float(row.std()) + 1e-3, (b, s_, t, int(row.argmax()), gap)


def _proj_elems(model):
    from macaw_llm_b200 import quant

    return sum(getattr(getattr(l, p), n).weight.numel() for l in model.llm.model.layers for p, n in quant.PROJECTIONS)


def test_lifecycle():
    from macaw_llm_b200 import quant
    from macaw_llm_b200.lora import LoraConfig

    model, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    inp = _inputs(spec, "image", torch.bfloat16)
    gen = dict(inp, inference=True, max_new_tokens=5)
    n_w = _proj_elems(model)
    model(gen)  # 16-bit: derived fused weights, KV caches and the decode graph exist now
    torch.cuda.synchronize()
    mem16 = torch.cuda.memory_allocated()
    model.quantize_llm_int8()
    toks_after = model(gen)
    torch.cuda.synchronize()
    mem8 = torch.cuda.memory_allocated()
    assert mem16 - mem8 >= n_w, (mem16, mem8, n_w)
    for l in model.llm.model.layers:
        for p, n in quant.PROJECTIONS:
            lin = getattr(getattr(l, p), n)
            assert isinstance(lin, quant.Int8Linear) and lin.weight.dtype == torch.int8
            assert {t.dtype for t in lin.parameters()} == {torch.int8, torch.float32}
    derived = [k for k in model.engine._cache if re.match(r"(lora:|shadow:)?llm\.l\d", k)]
    assert not derived, derived
    # a freshly quantized twin gives the same tokens: nothing stale from the 16-bit model is replayed
    twin, _, _, _ = H.build_tiny_model("cuda", torch.bfloat16)
    twin.quantize_llm_int8()
    assert torch.equal(twin(gen), toks_after)
    # sampled decoding with a fixed seed is reproducible
    eng = model.engine
    s1 = eng.generate(inp, max_new_tokens=5, do_sample=True, top_k=20, temperature=1.3, seed=77)
    s2 = eng.generate(inp, max_new_tokens=5, do_sample=True, top_k=20, temperature=1.3, seed=77)
    assert torch.equal(s1, s2)
    # load_state_dict between quantized models: the weights, derived state and graphs follow
    other, _, _, _ = H.build_tiny_model("cuda", torch.bfloat16)
    with torch.no_grad():
        for p in other.llm.model.layers.parameters():
            p.mul_(-1.0)
    other.quantize_llm_int8()
    other(gen)
    other.load_state_dict(model.state_dict())
    assert torch.equal(other(gen), toks_after)
    # refusals
    with pytest.raises(RuntimeError, match="int8"):
        model.add_lora(LoraConfig(r=8))
    model.train()
    with pytest.raises(RuntimeError, match="cannot be trained"):
        model(_inputs(spec, "image", torch.bfloat16, drop=()))
    model.eval()
    with pytest.raises(RuntimeError, match="already quantized"):
        model.quantize_llm_int8()


def test_cuda_graph_forward_on_a_quantized_model():
    model, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    model.quantize_llm_int8()
    inp = _inputs(spec, "all3", torch.bfloat16, drop=())
    ref = model(inp).logits.clone()
    model.engine.enable_cuda_graphs(True)
    try:
        a = model(inp).logits.clone()
        b = model(inp).logits.clone()
    finally:
        model.engine.enable_cuda_graphs(False)
    assert torch.equal(a, ref) and torch.equal(b, ref)


# ---------------------------------------------------------------------------------------------------- 7B, full depth
def test_7b_decode_step_matches_full_recompute():
    """Real width and depth (LLaMA-7B, random fp16 weights, quantized): the logits of a cached decode step (int8 GEMMs)
    against a fresh prefill over the extended sequence (dequantized 16-bit GEMMs) on the same model."""
    import bench
    from macaw_llm_b200 import ops
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    (clip, whisper, llama), hyper = bench.real_configs()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device="cuda", dtype=torch.float16, seed=0)
    model.quantize_llm_int8()
    eng = model.engine
    B, T = 2, 40
    with torch.no_grad():
        eng.set_format()
        table = eng.w(model.llm.model.embed_tokens.weight, "llm.embed")
        ids = torch.randint(3, 32000, (B, T + 1), generator=torch.Generator().manual_seed(5)).cuda()
        embeds = table[ids[:, :T]]
        E = embeds.shape[-1]
        full = eng.llama_forward(table[ids].clone(), None)[:, -1, :]
        cache = [torch.empty((B, T + 4, 2, E), device="cuda", dtype=torch.float16) for _ in model.llm.model.layers]
        x = embeds.reshape(B * T, E).clone()
        eng._llama_layers(x, B, T, None, 0, cache, T + 4)
        x1 = ops.embed_gather(table, ids[:, T])
        x1 = eng._llama_layers(x1, B, 1, None, T, cache, T + 4)
        step = eng._lm_head(x1)
    torch.cuda.synchronize()
    err = H.rel_err(step, full)
    print(f"\n[int8 7B] decode step vs full recompute: {err:.3e}")
    assert err < 1e-2


def test_generate_beyond_the_thin_decode_batch():
    """B > 64 has no thin decode path: every step runs the dequantized 16-bit GEMMs, so the tokens equal those of the
    engine on the fp32 values q * s bit for bit."""
    model16, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    qm = copy.deepcopy(model16)
    qm.quantize_llm_int8()
    twin = _twin_on_dequantized(model16, qm)
    inp = _inputs(spec, "image", torch.bfloat16)
    B0 = inp["input_ids"].shape[0]
    reps = -(-66 // B0)
    big = {k: (v.repeat(reps, *([1] * (v.dim() - 1)))[:66] if isinstance(v, torch.Tensor) and v.shape[0] == B0 else v)
           for k, v in inp.items()}
    gen = dict(big, inference=True, max_new_tokens=4)
    a, b = qm(gen), twin(gen)
    assert a.shape[0] == 66 and torch.equal(a, b)
