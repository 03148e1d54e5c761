"""GPU tier of the FP8 decoder: the e4m3 quantization kernel bit-exact against the restated rule, the e4m3 GEMM element by
element against fp64 of its quantized operands with each epilogue the decoder uses, determinism under a CUDA graph, the
e4m3 decode kernel against fp64, the tiny model end to end, and the lifecycle (freed weights, no fused copy, refusals).
Measured error ratios are printed (pytest -s)."""
import math

import pytest
import torch

from tests import decode_reference as R
from tests import helpers as H
from tests.fp8_reference import E4M3, gemm_ref, half_ulp, quantize_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
E, I = 4096, 11008
# The bound of an e4m3 GEMM output before the epilogue: kappa 2^-P sqrt(K) (|q_x| s_x)(|q_w| s_w)^T, kappa = 1.  P comes from a
# measurement (H100, fp32 outputs, this file's cases): the promoted kernel's worst error is 4.4 2^-24 sqrt(K) |.||.| (M = 1,
# K = 4096; 1.8 at M = 264, K = 11008), the unpromoted comparison instance's 88 2^-24 sqrt(K) |.||.|.  P = 21 (kappa 8 at
# p = 24) leaves the promoted kernel about 2x headroom and puts the unpromoted one about 11x above the bar, so a kernel that
# lost its promotion fails.  Each case prints its worst ratio; DESIGN records them.
P = 21

# epi 0 std | 1 SwiGLU | 2 RoPE; rows: the weight's sources (the B operand is read through the chunk map)
GEMM_CASES = [
    dict(epi=0, M=1, N=E, K=E, rows=[E], tail="plain"),
    dict(epi=0, M=13, N=E, K=I, rows=[E], tail="residual"),
    dict(epi=0, M=264, N=E, K=E, rows=[E], tail="residual"),
    dict(epi=0, M=2112, N=E, K=I, rows=[E], tail="residual"),
    dict(epi=2, M=13, N=3 * E, K=E, rows=[E] * 3, tail="rope"),
    dict(epi=2, M=264, N=3 * E, K=E, rows=[E] * 3, tail="rope"),
    dict(epi=1, M=13, N=2 * I, K=E, rows=[I] * 2, tail="swiglu"),
    dict(epi=1, M=2112, N=2 * I, K=E, rows=[I] * 2, tail="swiglu"),
    dict(epi=0, M=264, N=E, K=I, rows=[E], tail="plain", unpromoted=True),
]


def _ops(dt=torch.bfloat16):
    from macaw_llm_b200 import ops

    ops.set_act_format(dt)
    return ops


def rnd(*shape, scale=1.0, seed=0, dt=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dt)


# ---------------------------------------------------------------------------------------------------- quantization
@pytest.mark.parametrize("gain", [False, True])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("shape", [(4096, 4096), (11008, 4096), (4096, 11008)])
def test_quantize_kernel_is_bit_exact(shape, dt, gain):
    from tests.test_fp8_cpu import crafted_rows

    ops = _ops(torch.float16 if dt == torch.float16 else torch.bfloat16)
    R, K = shape
    x = rnd(R, K, scale=0.7, seed=R + K, dt=dt)
    c = crafted_rows(K).to(DEV).to(dt)
    x[: c.shape[0]] = c
    x[7, 100] = 30.0
    g = (1.0 + rnd(K, scale=0.2, seed=5, dt=ops.ACT()).float()).to(ops.ACT()) if gain else None
    q, s = ops.quantize_rows_e4m3(x, g)
    qr, sr = quantize_ref(x.cpu(), None if g is None else g.cpu())
    assert torch.equal(s.cpu(), sr)
    assert torch.equal(q.view(torch.uint8).cpu(), qr.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------- e4m3 GEMM
def _weight(rows, K, seed, interleave):
    from macaw_llm_b200 import ops

    qs, ss = [], []
    for j, r in enumerate(rows):
        q, s = ops.quantize_rows_e4m3(rnd(r, K, scale=0.02, seed=seed + j))
        qs.append(q)
        ss.append(s)
    W = ops.W8Matrix(qs, ss, interleave=interleave)
    chunks = ops.w8_chunk_map(rows, interleave)
    qf = torch.cat([qs[int(j)][int(r):int(r) + 32] for j, r in chunks])       # the fused weight the GEMM stands for
    sf = torch.cat([ss[int(j)][int(r):int(r) + 32] for j, r in chunks])
    return W, qf, sf


def _case(c, dt, unpromoted=None):
    """Run one case; -> worst |err| / bar with kappa = 1 at P."""
    ops = _ops(dt)
    M, N, K, epi = c["M"], c["N"], c["K"], c["epi"]
    W, qf, sf = _weight(c["rows"], K, seed=N + K, interleave=epi == 1)
    x = rnd(M, K, seed=M + K, dt=dt)
    g = (1.0 + rnd(K, scale=0.2, seed=9, dt=dt).float()).to(dt)
    qx, sx = ops.quantize_rows_e4m3(x, g)
    ref, mag = gemm_ref(qx, sx, qf, sf)  # fp64 on the device
    acc_bar = 2.0 ** -P * math.sqrt(K) * mag
    fp32 = 2.0 ** -22 * mag  # a few fp32 roundings of the scaling and the epilogue
    unp = c.get("unpromoted", False) if unpromoted is None else unpromoted
    d = lambda t: t.double()  # noqa: E731
    if c["tail"] == "plain":
        out = ops.linear_e4m3(qx, sx, W, unpromoted=unp, out_dtype=torch.float32)
        err, bar = (d(out) - ref).abs(), acc_bar + fp32
    elif c["tail"] == "residual":
        res = rnd(M, N, seed=3, dt=dt)
        out = res.clone()
        ss = torch.empty((M, N // 32), device=DEV, dtype=torch.float32)
        ops.linear_e4m3(qx, sx, W, residual=out, out=out, sumsq_out=ss)
        y = ref + d(res)
        err, bar = (d(out) - y).abs(), half_ulp(y, dt) + acc_bar + fp32
        assert H.rel_err(ss, out.float().pow(2).view(M, N // 32, 32).sum(2)) < 1e-5
    elif c["tail"] == "rope":
        parts = torch.rand(M, E // 32, device=DEV) + 0.5
        eps = 1e-6
        rs = 1.0 / torch.sqrt(d(parts).sum(1, keepdim=True) / K + eps)
        T = 64
        cos, sin = torch.rand(T, 64, device=DEV), torch.rand(T, 64, device=DEV)
        out = ops.linear_e4m3(qx, sx, W, epi=ops.EPI_ROPE, rope=(cos, sin, T, 2 * E), rms_from=(parts, eps))
        pos = torch.arange(M, device=DEV) % T
        cc = torch.cat([d(cos)[pos], d(cos)[pos]], 1).repeat(1, N // 128)
        sn = torch.cat([d(sin)[pos], d(sin)[pos]], 1).repeat(1, N // 128)
        cols = torch.arange(N, device=DEV)
        partner = cols + torch.where(cols % 128 < 64, 64, -64)
        sign = torch.where(cols % 128 < 64, -1.0, 1.0).double()
        rot = cols < 2 * E  # q and k heads rotate, v does not
        a = rs * ref
        y = torch.where(rot, a * cc + sign * a[:, partner] * sn, a)
        ab = rs * (acc_bar + fp32)
        bar = half_ulp(y, dt) + torch.where(rot, ab * cc.abs() + ab[:, partner] * sn.abs(), ab) + 2.0 ** -22 * rs * mag * 2
        err = (d(out) - y).abs()
    else:  # swiglu: fused rows [32 gate | 32 up]
        parts = torch.rand(M, E // 32, device=DEV) + 0.5
        eps = 1e-6
        rs = 1.0 / torch.sqrt(d(parts).sum(1, keepdim=True) / K + eps)
        out = ops.linear_e4m3(qx, sx, W, epi=ops.EPI_SWIGLU, rms_from=(parts, eps))
        gi = torch.arange(N, device=DEV).view(N // 64, 2, 32)
        gate, up = rs * ref[:, gi[:, 0].reshape(-1)], rs * ref[:, gi[:, 1].reshape(-1)]
        bg = rs * (acc_bar + fp32)[:, gi[:, 0].reshape(-1)]
        bu = rs * (acc_bar + fp32)[:, gi[:, 1].reshape(-1)]
        sig = torch.sigmoid(gate)
        y = gate * sig * up
        dsilu = sig * (1 + gate * (1 - sig))
        bar = half_ulp(y, dt) + (dsilu * up).abs() * bg + (gate * sig).abs() * bu + 2.0 ** -20 * y.abs()
        err = (d(out) - y).abs()
    assert torch.isfinite(d(out)).all()
    return float((err / bar).max())


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ci", range(len(GEMM_CASES)))
def test_e4m3_gemm_against_fp64(ci, dt):
    c = GEMM_CASES[ci]
    ratio = _case(c, dt)
    print(f"\n[fp8 gemm] {c} {dt}: worst err / bar (kappa 1, P {P}) = {ratio:.3f}")
    if c.get("unpromoted"):
        promoted = _case(c, dt, unpromoted=False)
        print(f"[fp8 gemm] same case promoted: {promoted:.3f}")
        # the promoted kernel meets the bound; accumulating all of K inside the MMA does not: the promotion is what the
        # bound rests on
        assert promoted <= 1.0 and ratio > 2.0, (promoted, ratio)
    else:
        assert ratio <= 1.0


def test_e4m3_gemm_plan_matches_the_launch():
    ops = _ops()
    from macaw_llm_b200 import ops as o

    W, _, _ = _weight([E] * 3, E, 1, False)
    qx, sx = ops.quantize_rows_e4m3(rnd(264, E))
    o.PLANS = []
    try:
        ops.linear_e4m3(qx, sx, W)
        assert o.PLANS == [ops.linear_e4m3(qx, sx, W, plan_only=True)]
    finally:
        o.PLANS = None


def test_determinism_and_graph_replay():
    ops = _ops()
    W, _, _ = _weight([I] * 2, E, 7, True)
    x = rnd(2112, E, seed=4)
    g = (1.0 + rnd(E, scale=0.2, seed=9).float()).to(torch.bfloat16)
    parts = torch.rand(2112, E // 32, device=DEV) + 0.5

    def run():
        qx, sx = ops.quantize_rows_e4m3(x, g)
        return ops.linear_e4m3(qx, sx, W, epi=ops.EPI_SWIGLU, rms_from=(parts, 1e-6))

    a, b = run(), run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(graph):
        c = run()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c)


# ---------------------------------------------------------------------------------------------------- e4m3 decode GEMM
@pytest.mark.parametrize("M", [1, 8, 64])
def test_e4m3_decode_gemm_at_the_7b_fused_shapes(M):
    """s_n sum_k e4m3(q) round16(x g) at the fused [q; k; v] and [gate | up] shapes through each mm_thin_fused tail (RES,
    SWIGLU, QKV with RoPE and the KV-cache write at a device-side position), element by element against fp64 with the
    GEMM tests' bound (half an output ulp + 2^-22 sqrt(K) |x~| |q s|^T, carried through RoPE / SwiGLU); bf16 and fp16."""
    Tmax, t0 = 24, 5
    for dt in (torch.bfloat16, torch.float16):
        ops = _ops(dt)
        x = rnd(M, E, seed=M, dt=dt)
        g = (1.0 + rnd(E, scale=0.2, seed=9, dt=dt).float()).to(dt)
        xt = (x.float() * g.float()[None]).to(dt).double()
        ratio = lambda out, y, bar: float(((out.double() - y).abs() / bar).max())  # noqa: E731
        # RES on the fused [q; k; v] rows
        W, qf, sf = _weight([E] * 3, E, 80, False)
        W = ops.W8Matrix(W._keep[0], W._keep[1], gain=g)
        wd = qf.double() * sf.double()[:, None]
        ref, mag = xt @ wd.t(), xt.abs() @ wd.abs().t()
        acc = 2.0 ** -22 * math.sqrt(E) * mag
        out = ops.linear_w8_thin_fused(x, W, ops.THIN_RES, residual=torch.zeros((M, W.N), device=DEV, dtype=dt))
        assert ratio(out, ref, half_ulp(ref, dt) + acc) <= 1.0, (dt, "res")
        # QKV: row scale, RoPE at the device-side position t0, q -> out, k / v -> the cache slot t0
        rs = (torch.rand(M, device=DEV) + 0.5)
        cos, sin = torch.rand(Tmax, 64, device=DEV), torch.rand(Tmax, 64, device=DEV)
        cache = torch.zeros((M, Tmax, 2, E), device=DEV, dtype=dt)
        pos = torch.tensor([t0], device=DEV, dtype=torch.int32)
        out = ops.linear_w8_thin_fused(x, W, ops.THIN_QKV, row_scale=rs, rope=(cos, sin, pos), cache=cache, t0_dev=pos)
        r = rs.double()[:, None]
        a, ab = r * ref, r * (acc + 2.0 ** -22 * mag)
        cols = torch.arange(3 * E, device=DEV)
        partner = cols + torch.where(cols % 128 < 64, 64, -64)
        sign = torch.where(cols % 128 < 64, -1.0, 1.0).double()
        cc = torch.cat([cos[t0], cos[t0]]).double().repeat(3 * E // 128)[None]
        sn = torch.cat([sin[t0], sin[t0]]).double().repeat(3 * E // 128)[None]
        rot = cols < 2 * E
        y = torch.where(rot, a * cc + sign * a[:, partner] * sn, a)
        bar = half_ulp(y, dt) + torch.where(rot, ab * cc.abs() + ab[:, partner] * sn.abs(), ab)
        got = torch.cat([out[:, :E], cache[:, t0, 0], cache[:, t0, 1]], 1)
        assert ratio(got, y, bar) <= 1.0, (dt, "qkv")
        assert float(cache[:, :t0].abs().sum()) == 0 and float(cache[:, t0 + 1:].abs().sum()) == 0
        # SWIGLU on the interleaved [gate | up] rows (unit row scale)
        Wg, qg, sg = _weight([I] * 2, E, 90, True)
        Wg = ops.W8Matrix(Wg._keep[0], Wg._keep[1], interleave=True, gain=g)
        out = ops.linear_w8_thin_fused(x, Wg, ops.THIN_SWIGLU, row_scale=torch.ones(M, device=DEV))
        wg = qg.double() * sg.double()[:, None]
        r, mg = xt @ wg.t(), xt.abs() @ wg.abs().t()
        gi = torch.arange(2 * I, device=DEV).view(I // 32, 2, 32)
        gcol, ucol = gi[:, 0].reshape(-1), gi[:, 1].reshape(-1)
        gate, up = r[:, gcol], r[:, ucol]
        bg = 2.0 ** -22 * (math.sqrt(E) + 1) * mg[:, gcol]
        bu = 2.0 ** -22 * (math.sqrt(E) + 1) * mg[:, ucol]
        sig = torch.sigmoid(gate)
        y = gate * sig * up
        bar = half_ulp(y, dt) + (sig * (1 + gate * (1 - sig)) * up).abs() * bg + (gate * sig).abs() * bu + 2.0 ** -20 * y.abs()
        assert ratio(out, y, bar) <= 1.0, (dt, "swiglu")


# ---------------------------------------------------------------------------------------------------- tiny model
def _inputs(spec, name, dt, drop=("labels",)):
    inp = H.case_inputs(spec, H.load_case(name))
    return {k: (v.to(dt).cuda() if isinstance(v, torch.Tensor) and v.is_floating_point() else
                v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items() if k not in drop}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_tiny_model_forward_and_generate(dt):
    model16, spec, _, _ = H.build_tiny_model(DEV, dt)
    qm, _, _, _ = H.build_tiny_model(DEV, dt)
    qm.quantize_llm_fp8()
    with torch.no_grad():
        for name in ("text", "all3"):
            a = qm(_inputs(spec, name, dt)).logits
            b = model16(_inputs(spec, name, dt)).logits
            err = H.rel_err(a, b)
            print(f"\n[fp8 tiny] {dt} {name}: logits rel err vs 16-bit {err:.3e}")
            assert torch.isfinite(a.float()).all() and err < 0.2
        inp = _inputs(spec, "all3", dt, drop=("labels", "attention_mask"))
        t1 = qm.engine.generate(inp, max_new_tokens=12)
        t2 = qm.engine.generate(inp, max_new_tokens=12)
        assert torch.equal(t1, t2) and t1.shape[1] >= 1
        s1 = qm.engine.generate(inp, max_new_tokens=12, do_sample=True, top_k=20, seed=7)
        s2 = qm.engine.generate(inp, max_new_tokens=12, do_sample=True, top_k=20, seed=7)
        assert torch.equal(s1, s2)
        # the graphed forward replays the eager FP8 forward bitwise
        eager = qm(_inputs(spec, "text", dt)).logits.clone()
        qm._engine.enable_cuda_graphs(True)
        try:
            g1 = qm(_inputs(spec, "text", dt)).logits.clone()
        finally:
            qm._engine.enable_cuda_graphs(False)
        assert torch.equal(eager, g1)


def test_generate_beyond_the_thin_decode_batch():
    """B > 64 runs quantize -> e4m3 GEMM in every decode step (with device positions under the captured graph)."""
    qm, spec, _, _ = H.build_tiny_model(DEV, torch.bfloat16)
    qm.quantize_llm_fp8()
    inp = _inputs(spec, "text", torch.bfloat16, drop=("labels", "attention_mask"))
    inp = {k: (v.repeat(33, *([1] * (v.dim() - 1))) if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    with torch.no_grad():
        t = qm.engine.generate(inp, max_new_tokens=6)
    assert t.shape[0] == inp["input_ids"].shape[0] and t.shape[0] > 64


# ---------------------------------------------------------------------------------------------------- 7B width, end to end
class _QuantDecoder:
    """An fp64 restatement of the FP8 decoder with the engine's quantization points: weights q s; in the prefill (and in
    decode steps above 64 samples) each GEMM input row -- x g1, the attention output, x g2, the SwiGLU output -- quantized
    by the e4m3 rule, the RMSNorm statistic applied after the GEMM; decode steps of up to 64 samples quantize no
    activation.  `store` (a 16-bit dtype) rounds what the engine stores in 16 bits -- the residual stream, q / k / v, the
    attention probabilities and output, the decode steps' x~ = x g, the SwiGLU output and the logits -- before it is used:
    that twin is the yardstick."""

    def __init__(self, sd, hp, store=None, quant_steps=False):
        c = hp["llama"]
        self.sd, self.E, self.H, self.L, self.eps = sd, c["hidden"], c["heads"], c["layers"], c["eps"]
        self.hd = self.E // self.H
        self.store, self.quant_steps = store, quant_steps
        self.k, self.v = [None] * self.L, [None] * self.L
        cos, sin = R.rope_tables(512, self.hd)
        self.cos, self.sin = (torch.cat([t, t], -1).to(DEV, torch.float64) for t in (cos, sin))

    def st(self, t):
        return t if self.store is None else t.to(self.store).double()

    @staticmethod
    def quant(v):
        s = v.abs().amax(-1, keepdim=True) / 448.0
        z = s == 0
        q = torch.where(z, 0.0, v / torch.where(z, 1.0, s)).clamp(-448.0, 448.0).float().to(E4M3).double()
        return q * s

    def _rot(self, x):
        return torch.cat([-x[..., self.hd // 2:], x[..., : self.hd // 2]], -1)

    def run(self, x, pos0):
        B, T, E = x.shape
        H, hd, w, st = self.H, self.hd, self.sd, self.st
        aq = pos0 == 0 or self.quant_steps
        inp = (lambda v: self.quant(v)) if aq else st  # a GEMM input: e4m3 rows, or x~ stored in 16 bits
        cos, sin = self.cos[pos0:pos0 + T][None, None], self.sin[pos0:pos0 + T][None, None]
        mask = torch.triu(torch.full((T, pos0 + T), float("-inf"), device=DEV, dtype=torch.float64), pos0 + 1)
        x = st(x)
        for i in range(self.L):
            p = f"llm.model.layers.{i}."
            rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps)
            h = inp(x * w[p + "input_layernorm.weight"])
            q, k, v = ((rstd * (h @ w[p + f"self_attn.{n}_proj.weight"].t())).view(B, T, H, hd).transpose(1, 2)
                       for n in "qkv")
            q, k, v = st(q * cos + self._rot(q) * sin), st(k * cos + self._rot(k) * sin), st(v)
            if pos0 > 0:
                k, v = torch.cat([self.k[i], k], 2), torch.cat([self.v[i], v], 2)
            self.k[i], self.v[i] = k, v
            prob = st(torch.softmax(q @ k.transpose(2, 3) / math.sqrt(hd) + mask, -1))
            a = st((prob @ v).transpose(1, 2).reshape(B, T, E))
            x = st(x + inp(a) @ w[p + "self_attn.o_proj.weight"].t())
            rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps)
            h = inp(x * w[p + "post_attention_layernorm.weight"])
            gate, up = (rstd * (h @ w[p + f"mlp.{n}_proj.weight"].t()) for n in ("gate", "up"))
            g = st(torch.nn.functional.silu(gate) * up)
            x = st(x + inp(g) @ w[p + "mlp.down_proj.weight"].t())
        rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps)
        return st(rstd * ((x * w["llm.model.norm.weight"]) @ w["llm.lm_head.weight"].t()))


def _fp8_model_7b(dt):
    """bench.real_configs() with 2 decoder layers, RMSNorm gains drawn around 1 (so that where the gain is applied
    matters), quantized with quantize_llm_fp8()."""
    import bench
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    (clip, whisper, llama), hyper = bench.real_configs()
    clip.vision_config.num_hidden_layers = 1
    whisper.encoder_layers = 1
    llama.num_hidden_layers = 2
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=DEV, dtype=dt, seed=3)
    gen = torch.Generator(device=DEV).manual_seed(4)
    with torch.no_grad():
        for name, p in model.llm.named_parameters():
            if name.endswith("norm.weight"):
                p.copy_(1.0 + 0.25 * torch.randn(p.shape, generator=gen, device=DEV))
    model.quantize_llm_fp8()
    return model


def _fp8_ref_state(model):
    sd = model.state_dict()
    out = {}
    for k, v in sd.items():
        if not k.startswith("llm.") or k.endswith(("weight_scale", "inv_freq")) or not v.is_floating_point():
            continue
        out[k] = v.double() * sd[k + "_scale"].double()[:, None] if v.dtype == E4M3 else v.double()
    return out


@pytest.mark.parametrize("dt,B", [(torch.bfloat16, 8), (torch.bfloat16, 65), (torch.float16, 8)],
                         ids=["bf16-B8", "bf16-B65", "fp16-B8"])
def test_7b_width_fp8_decoder_vs_fp64_restatement(dt, B):
    """A 2-layer FP8 decoder at LLaMA-7B width: prefill of a 60-token prompt and 80 greedy decode steps (B = 8: the e4m3
    thin kernel with each tail; B = 65: quantize -> e4m3 GEMM in every step), through the engine's own calls as
    generate() makes them.  The logits of the prefill and of the steps at 61, 64, 65, 128, 129 and 139 keys are held to
    1.5x a yardstick measured here: the fp64 restatement with the engine's quantization points against the same
    restatement with its activations stored in 16 bits before quantization (e4m3 rounding flips that 16-bit storage alone
    causes)."""
    from tests.test_decode_gpu import _drive, _hp, _prompt, rel64

    model = _fp8_model_7b(dt)
    T0, n_new = 60, 80
    ids = _prompt(B, T0, seed=B)
    toks, dev_logits, _, pre_logits = _drive(model, ids, n_new)
    sd = _fp8_ref_state(model)
    table = sd["llm.model.embed_tokens.weight"]
    refs = {}
    with torch.no_grad():
        for name, store in (("fp64", None), ("16-bit", dt)):
            dec = _QuantDecoder(sd, _hp(model), store=store, quant_steps=B > 64)
            pre = dec.run(table[ids], 0)
            steps = [pre[:, -1]]
            for s in range(1, n_new):
                steps.append(dec.run(table[toks[:, s - 1]][:, None], T0 + s - 1)[:, 0])
            refs[name] = (pre, steps)
    checks = [("prefill", pre_logits, refs["fp64"][0], refs["16-bit"][0])]
    for tk in (T0 + 1, 64, 65, 128, 129, T0 + n_new - 1):
        s = tk - T0
        checks.append((f"{tk} keys", dev_logits[s], refs["fp64"][1][s], refs["16-bit"][1][s]))
    del model
    torch.cuda.empty_cache()
    lines = []
    for name, got, ref, yard in checks:
        e, y = rel64(got, ref), rel64(yard, ref)
        lines.append((name, e, y))
    print(f"\n[fp8 7B width {dt} B={B}] logits error vs fp64 restatement / 16-bit-storage yardstick: "
          + "; ".join(f"{n} {e:.3e} / {y:.3e}" for n, e, y in lines))
    for n, e, y in lines:
        assert e <= 1.5 * y, (n, e, y)


# ---------------------------------------------------------------------------------------------------- lifecycle
def test_lifecycle_and_refusals():
    from macaw_llm_b200.lora import LoraConfig

    model, spec, _, _ = H.build_tiny_model(DEV, torch.bfloat16)
    eng = model._engine
    with torch.no_grad():
        model(_inputs(spec, "text", torch.bfloat16))
    assert any("wqkv" in k for k in eng._cache)
    model._engine.enable_cuda_graphs(True)
    with torch.no_grad():
        model(_inputs(spec, "text", torch.bfloat16))
    assert eng._graphs
    model.quantize_llm_fp8()
    assert not eng._graphs and not eng._cache  # forward graphs and derived 16-bit copies dropped
    lin = model.llm.model.layers[0].self_attn.q_proj
    assert lin.weight.dtype == E4M3 and lin.weight_scale.dtype == torch.float32
    with torch.no_grad():
        model(_inputs(spec, "text", torch.bfloat16))
    model._engine.enable_cuda_graphs(False)
    # no fused or 16-bit copy of a decoder projection is derived on the FP8 path
    assert not [k for k in eng._cache if any(s in k for s in ("wqkv", "wgu", ".wo", ".wd"))], list(eng._cache)
    with pytest.raises(RuntimeError, match="already quantized"):
        model.quantize_llm_fp8()
    with pytest.raises(RuntimeError, match="already quantized"):
        model.quantize_llm_int8()
    with pytest.raises(RuntimeError, match="FP8-quantized"):
        model.add_lora(LoraConfig(r=8))
    model.train()
    with pytest.raises(RuntimeError, match="cannot be trained"):
        model(_inputs(spec, "text", torch.bfloat16, drop=()))
    m2, _, _, _ = H.build_tiny_model(DEV, torch.bfloat16)
    m2.add_lora(LoraConfig(r=8, target_modules=["q_proj"]))
    with pytest.raises(RuntimeError, match="merge_lora"):
        m2.quantize_llm_fp8()


def test_7b_width_memory_holds_no_fused_copy():
    """A 2-layer decoder at LLaMA-7B width: after quantize_llm_fp8 the projections take one byte per weight, and a
    prefill allocates no fused FP8 or 16-bit copy of them (peak stays below one layer's 16-bit weights above the start)."""
    from macaw_llm_b200 import quant
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    spec, _, _ = H.load_shapes()
    from tests.golden import gen

    clip, whisper, llama = gen.build_configs(spec)
    llama.hidden_size, llama.intermediate_size, llama.num_attention_heads, llama.num_hidden_layers = E, I, 32, 2
    llama.vocab_size = 512
    cfg = MM_LLMs_Config(n_frames=spec["n_frames"], attention_heads=spec["attention_heads"], clip_config=clip,
                         whisper_config=whisper, llm_config=llama)
    torch.manual_seed(0)
    model = MM_LLMs(cfg).to(DEV, torch.bfloat16).eval()
    with torch.no_grad():
        for p in model.llm.parameters():
            p.normal_(0, 0.02)
    model.quantize_llm_fp8()
    proj = sum(getattr(getattr(l, a), b).weight.numel() for l in model.llm.model.layers for a, b in quant.PROJECTIONS)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    emb = torch.randn(1, 256, E, device=DEV, dtype=torch.bfloat16) * 0.1
    with torch.no_grad():
        logits = model._engine.llama_forward(emb, None)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    print(f"\n[fp8 7b-width] projections {proj / 2**20:.1f} MiB in e4m3; prefill peak above start {extra / 2**20:.1f} MiB")
    assert torch.isfinite(logits.float()).all()
    assert extra < proj  # one layer's projections in 16 bits: proj / 2 weights of 2 bytes
