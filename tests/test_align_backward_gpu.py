"""The alignment block's training backward (training.AlignTrainer) on the H100 in both model formats.

Part A: the row / column kernels the backward is built from, each against an fp64 restatement of the formula in its
comment in csrc/train_kernels.cu — mm_align_softmax_bwd (with four wrong variants of the formula, to show the bars
discriminate), mm_align_dropout_fwd, mm_head_weighted_colsum, mm_window_gather_add (col2im) and mm_cast_f16_bf16.

Part B: the whole backward of the three alignment blocks (and video_long_self_attention) at REAL width (V = 32000,
E = 4096, 16 heads of 256) through the public `model(inputs).loss.backward()` path, against fp64 autograd of the oracle's
restatement on the GPU.  The bar of every gradient tensor is set by a yardstick measured in the same test: the same
restatement run by torch autograd in the model's own 16-bit format, which is how the reference trains."""
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
E32 = 2.0 ** -24  # unit roundoff of fp32
SENT16 = 0x5A5A   # sentinel bit pattern of untouched 16-bit output columns


def _ops():
    from macaw_llm_b200 import ops

    return ops


@pytest.fixture(params=[BF16, F16], ids=["bf16", "fp16"])
def act(request):
    """Runs the test in each activation format (the format of the backward's 16-bit outputs)."""
    ops = _ops()
    ops.set_act_format(request.param)
    try:
        yield request.param
    finally:
        ops.set_act_format(BF16)


def _u(dt) -> float:
    """Unit roundoff of a 16-bit format: one round-to-nearest moves a normal value by at most u |x|."""
    return torch.finfo(dt).eps / 2


def _half_sub(dt) -> float:
    """Half the spacing of the format's subnormals: the rounding error bound where a value is subnormal."""
    fi = torch.finfo(dt)
    return fi.smallest_normal * fi.eps / 2


def _ratio(got, ref, tol) -> float:
    """max |got - ref| / tol: <= 1 passes an element-wise bar."""
    return float(((got.double() - ref.double()).abs() / tol).max())


# ---------------------------------------------------------------------------------------------------- part A
def _softmax_inputs(R: int, V: int, regime: str, seed: int):
    """Probabilities of the (V + 2)-key alignment softmax as the fused forward keeps them: fp16 P' = exp(s - rho) over
    the V real keys, 1 / l with l = sum of the rounded P' + the two synthetic keys' terms, and the un-dropped p_extra.
    flat: P ~ 1/V (fp16-subnormal at V = 32000); sharp: scores spanning > 20 nats; extra: p_extra ~ 1."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    if regime == "flat":
        s = torch.randn(R, V, generator=g, dtype=F64) * 0.02
        ext = torch.randn(R, generator=g, dtype=F64) * 0.02
    elif regime == "sharp":
        s = torch.randn(R, V, generator=g, dtype=F64) * 6.0
        ext = torch.randn(R, generator=g, dtype=F64) * 6.0
    else:
        s = torch.randn(R, V, generator=g, dtype=F64)
        ext = torch.full((R,), math.log(V + 2) + 6.0, dtype=F64)
    rho = torch.maximum(torch.maximum(s.amax(1), ext), torch.zeros_like(ext))
    Pp = torch.exp(s - rho[:, None]).to(F16)
    l = Pp.double().sum(1) + torch.exp(ext - rho) + torch.exp(-rho)
    inv_l = (1.0 / l).float()
    pe = (torch.exp(ext - rho) / l).float()
    span = float((s.amax(1) - s.amin(1)).min())
    return Pp, inv_l, pe, span


def _softmax_bwd_ref(Pp, inv_l, G, dpsr, pe, dpe, m, gscale, V, variant=None):
    """fp64 restatement of align_softmax_bwd_kernel's comment (m: (R, V + 1) dropout multipliers, column V = bias_k key):
        dP_v = m_v (G_v + dpsr),  D = sum_v P_v dP_v + p_extra m_V dpe,  dS_v = P_v (dP_v - D),
        Pd = m P,  dstats[0] = gscale sum_v dS_v,  dstats[1] = gscale p_extra (m_V dpe - D).
    `variant` makes one deliberate mistake: "no_dpsr", "no_extra" (extra-key term left out of D), "dropped_pe" (the
    dropped p_extra used in place of the raw one) or "no_gscale"."""
    P = Pp.double() * inv_l.double()[:, None]
    mr, mV = m[:, :V], m[:, V]
    a = 0.0 if variant == "no_dpsr" else dpsr.double()[:, None]
    dP = mr * (G.double() + a)
    pex = pe.double() * mV if variant == "dropped_pe" else pe.double()
    dpe = dpe.double()
    D = (P * dP).sum(1) + (0.0 if variant == "no_extra" else pex * mV * dpe)
    dS = P * (dP - D[:, None])
    gs = 1.0 if variant == "no_gscale" else gscale
    dstats = torch.stack([gs * dS.sum(1), gs * pex * (mV * dpe - D)])
    scale_r = (P * dP).abs().sum(1) + (pe.double() * mV * dpe).abs() + 1e-30  # magnitude of the terms D sums
    return mr * P, dS, dstats, dict(P=P, dP=dP, D=D, scale_r=scale_r)


SOFTMAX_CASES = [(32000, 97), (519, 37), (1, 5), (4097, 37)]


@pytest.mark.parametrize("regime", ["flat", "sharp", "extra"])
@pytest.mark.parametrize("dropout", [False, True], ids=["nodrop", "drop"])
@pytest.mark.parametrize("V,R", SOFTMAX_CASES, ids=[f"V{v}-R{r}" for v, r in SOFTMAX_CASES])
def test_align_softmax_bwd(act, V, R, dropout, regime):
    """mm_align_softmax_bwd through the C entry with sentinel-filled outputs, ldg > V, ldp > V, ldo > ldp and NaN in the
    input columns >= V (which must not be read): Pd and dS within one rounding to the format (or half a subnormal
    spacing), dstats within 1e-5 of the magnitude of the row's terms; columns >= V of Pd / dS untouched.  Four wrong
    variants of the formula must miss by >= 10x the bar in the p_extra ~ 1 regime with dropout on (V > 1)."""
    from macaw_llm_b200 import _lib

    ops = _ops()
    fmt = act
    seed_i = 1000 * V + 10 * R + {"flat": 0, "sharp": 1, "extra": 2}[regime] + 5 * int(dropout)
    Pp, inv_l, pe, span = _softmax_inputs(R, V, regime, seed_i)
    if regime == "sharp" and V >= 519:
        assert span > 20.0
    g = torch.Generator(device="cpu").manual_seed(seed_i + 1)
    G = torch.randn(R, V, generator=g)
    dpsr, dpe = torch.randn(R, generator=g) * 0.5, torch.randn(R, generator=g) * 0.5
    gscale = 0.125 if dropout else 1.0
    ldg, ldp = V + 5, (V + 7) // 8 * 8 + 8
    ldo = ldp + 16
    Gb = torch.full((R, ldg), float("nan"), device=DEV)
    Gb[:, :V] = G.to(DEV)
    Pb = torch.full((R, ldp), float("nan"), device=DEV, dtype=F16)
    Pb[:, :V] = Pp.to(DEV)
    inv_l_d, pe_d, dpsr_d, dpe_d = (t.to(DEV).contiguous() for t in (inv_l, pe, dpsr, dpe))
    Pd = torch.empty((R, ldo), device=DEV, dtype=fmt)
    dS = torch.empty((R, ldo), device=DEV, dtype=fmt)
    Pd.view(torch.int16).fill_(SENT16)
    dS.view(torch.int16).fill_(SENT16)
    dst = torch.full((2 * R + 8,), 1234.5, device=DEV)
    seed = torch.tensor([(7 << 32) | (seed_i & 0xFFFFFFF)], dtype=torch.int64, device=DEV)
    p, sid = (0.1, 5) if dropout else (0.0, 0)
    rc = _lib.load().mm_align_softmax_bwd(Gb.data_ptr(), ldg, Pb.data_ptr(), ldp, inv_l_d.data_ptr(), dpsr_d.data_ptr(),
                                          pe_d.data_ptr(), dpe_d.data_ptr(), gscale, Pd.data_ptr(), dS.data_ptr(), ldo,
                                          dst.data_ptr(), R, V, p, seed.data_ptr() if dropout else None, sid,
                                          ops._stream())
    ops._check(rc, "mm_align_softmax_bwd")
    m = (ops.dropout_mask(R, V + 1, (p, seed, sid), DEV).double() if dropout
         else torch.ones(R, V + 1, device=DEV, dtype=F64))
    if dropout and R * V >= 1000:
        assert abs(float((m != 0).double().mean()) - 0.9) < 0.02
    G64, Pp64 = G.to(DEV), Pp.to(DEV)
    Pd_ref, dS_ref, st_ref, aux = _softmax_bwd_ref(Pp64, inv_l_d, G64, dpsr_d, pe_d, dpe_d, m, gscale, V)
    torch.cuda.synchronize()
    assert bool((Pd.view(torch.int16)[:, V:] == SENT16).all()) and bool((dS.view(torch.int16)[:, V:] == SENT16).all())
    assert bool((dst[2 * R:] == 1234.5).all())
    # bars: one rounding to the format (or half a subnormal spacing) + the fp32 arithmetic before it; the fp32 row
    # reduction of D (<= V/512 sequential adds per thread + 10 shuffle / shared-memory levels) is bounded by dD
    u, hs = _u(fmt), _half_sub(fmt)
    P, dP, D, scale_r = aux["P"], aux["dP"], aux["D"], aux["scale_r"]
    dD = (V / 512 + 16) * E32 * scale_r
    tol_P = torch.clamp(u * Pd_ref.abs(), min=hs) + 4 * E32 * Pd_ref.abs()
    tol_dS = (torch.clamp(u * dS_ref.abs(), min=hs) + P * (4 * E32 * (dP.abs() + D.abs()[:, None]) + dD[:, None])
              + 2 * E32 * dS_ref.abs())
    tol_st = (1e-5 * abs(gscale) * scale_r).expand(2, R)
    got_st = dst[:2 * R].view(2, R)
    r_P, r_dS, r_st = _ratio(Pd[:, :V], Pd_ref, tol_P), _ratio(dS[:, :V], dS_ref, tol_dS), _ratio(got_st, st_ref, tol_st)
    sub = float((dS_ref.abs() < torch.finfo(F16).smallest_normal).double().mean())
    # discrimination: each wrong variant against the correct result, in units of the same bars
    disc = {}
    for var, affects in (("no_dpsr", ("dS", "dstats")), ("no_extra", ("dS", "dstats")),
                         ("dropped_pe", ("dS", "dstats")), ("no_gscale", ("dstats",))):
        _, dS_w, st_w, _ = _softmax_bwd_ref(Pp64, inv_l_d, G64, dpsr_d, pe_d, dpe_d, m, gscale, V, variant=var)
        r = {"dS": _ratio(dS_w, dS_ref, tol_dS), "dstats": _ratio(st_w, st_ref, tol_st)}
        disc[var] = max(r[k] for k in affects)
    print(f"\n[align_softmax_bwd {str(fmt)[6:]} V={V} R={R} {regime} drop={int(dropout)}] error/bar: Pd {r_P:.3f} "
          f"dS {r_dS:.3f} dstats {r_st:.3f} (dS fp16-subnormal share {sub:.2f}); wrong variants / bar: "
          + " ".join(f"{k} {v:.3g}" for k, v in disc.items()))
    assert r_P <= 1.0 and r_dS <= 1.0 and r_st <= 1.0, (r_P, r_dS, r_st)
    if regime == "extra" and dropout and V > 1:
        # asserted on these inputs only, where every term of the formula matters (p_extra ~ 1, a live mask on the bias_k
        # key, gscale != 1); with p_extra ~ 1/V (flat / sharp rows) the extra-key and raw-p_extra mistakes move the outputs
        # by ~p_extra relative and cannot show, so there the ratios are printed only
        for var, r in disc.items():
            assert r >= 10.0, (var, r)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("V,R", SOFTMAX_CASES, ids=[f"V{v}-R{r}" for v, r in SOFTMAX_CASES])
def test_align_dropout_fwd(act, V, R, p):
    """mm_align_dropout_fwd: Pm = P' where kept and +0 where dropped, bit for bit; rs = fp32(1/l) * fp32(1/(1-p)) exactly
    (within one fp32 ulp of the exact quotient); p_extra_d = p_extra * m_V exactly; p_sum_real_d against fp64."""
    ops = _ops()
    Pp, inv_l, pe, _ = _softmax_inputs(R, V, "sharp", 31 * V + R)
    ldp = (V + 7) // 8 * 8 + 8
    Pb = torch.full((R, ldp), float("nan"), device=DEV, dtype=F16)
    Pb[:, :V] = Pp.to(DEV)
    inv_l_d, pe_d = inv_l.to(DEV), pe.to(DEV)
    seed = torch.tensor([(3 << 32) | (V + R)], dtype=torch.int64, device=DEV)
    drop = (p, seed, 2)
    Pm, rs, psum_d, pext_d = ops.align_dropout_fwd(Pb, inv_l_d, pe_d, V, drop)
    m = ops.dropout_mask(R, V + 1, drop, DEV) if p > 0 else torch.ones(R, V + 1, device=DEV)
    want = torch.where(m[:, :V] != 0, Pb[:, :V], torch.zeros_like(Pb[:, :V]))
    torch.cuda.synchronize()
    assert torch.equal(Pm[:, :V].view(torch.int16), want.view(torch.int16))
    scale = (torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32))) if p > 0 else torch.tensor(1.0)
    assert torch.equal(rs, inv_l_d * scale.to(DEV))
    exact = inv_l_d.double() / (1.0 - float(np.float32(p)))
    assert bool(((rs.double() - exact).abs() <= 2.0 ** -23 * (1 + 2.0 ** -20) * exact.abs()).all())  # two fp32 roundings
    assert torch.equal(pext_d, pe_d * m[:, V])
    ref = exact * (Pb[:, :V].double() * (m[:, :V] != 0)).sum(1)
    e = float(((psum_d.double() - ref).abs() / ref.abs().clamp_min(1e-300)).max())
    print(f"\n[align_dropout_fwd V={V} R={R} p={p}] p_sum_real_d max rel err {e:.2e}")
    assert e < 1e-5


HWC_CASES = [(4096, 256, 816), (4096, 256, 12), (768, 96, 816), (768, 96, 1)]


@pytest.mark.parametrize("xdt", [BF16, F16], ids=["x_bf16", "x_fp16"])
@pytest.mark.parametrize("E,hd,Nq", HWC_CASES, ids=[f"E{e}-hd{h}-Nq{n}" for e, h, n in HWC_CASES])
def test_head_weighted_colsum(act, E, hd, Nq, xdt):
    """mm_head_weighted_colsum on a strided x view, accumulating into a non-zero out, against fp64: element-wise within the
    worst-case bound of Nq sequential fp32 adds plus the final add into out."""
    ops = _ops()
    H = E // hd
    g = torch.Generator(device=DEV).manual_seed(E + hd + Nq)
    base = torch.randn(Nq, E + 72, generator=g, device=DEV).to(xdt)
    x = base[:, 40:40 + E]
    assert x.stride(0) == E + 72
    w = torch.randn(H * Nq, generator=g, device=DEV)
    out0 = torch.randn(E, generator=g, device=DEV)
    out = ops.head_weighted_colsum(x, w, hd, out0.clone())
    xv, wv = x.double().reshape(Nq, H, hd), w.double().view(H, Nq)
    ref = out0.double() + torch.einsum("hn,nhd->hd", wv, xv).reshape(E)
    mag = torch.einsum("hn,nhd->hd", wv.abs(), xv.abs()).reshape(E) + out0.double().abs()
    r = _ratio(out, ref, (Nq + 2) * E32 * mag + 1e-30)
    print(f"\n[head_weighted_colsum E={E} hd={hd} Nq={Nq} {str(xdt)[6:]}] error / worst-case bound {r:.3f}")
    assert r <= 1.0


def _col2im(dwin, B, N, C, Lq, kk, ss, dtype):
    """dfeats[b, t, c] = sum over the windows l covering token t, in ascending l, of dwin[b*Lq + l, (t - l*ss)*C + c],
    accumulated in `dtype` (fp32 restates the kernel's order exactly)."""
    d = dwin.to(dtype).view(B, Lq, kk, C)
    t = torch.arange(N, device=dwin.device)
    l_lo = torch.where(t - kk + 1 <= 0, torch.zeros_like(t), torch.div(t - kk + ss, ss, rounding_mode="floor"))
    l_hi = torch.clamp(torch.div(t, ss, rounding_mode="floor"), max=Lq - 1)
    acc = torch.zeros((B, N, C), device=dwin.device, dtype=dtype)
    cover = torch.zeros((N,), device=dwin.device, dtype=torch.int64)
    for j in range(-(-kk // ss) + 1):
        l = l_lo + j
        k = t - l * ss
        ok = (l <= l_hi) & (k >= 0) & (k < kk)
        v = d[:, l.clamp(0, Lq - 1), k.clamp(0, kk - 1), :]
        acc = torch.where(ok[None, :, None], acc + v, acc)
        cover += ok.long()
    return acc, cover


GEOMS = [("image", 2, 256, 768, 48, 36), ("audio", 2, 1500, 512, 240, 220), ("video", 2, 1536, 768, 36, 30),
         ("gaps", 2, 100, 64, 5, 8), ("lq1", 1, 50, 768, 48, 36)]


@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_window_gather_add(act, geom):
    """mm_window_gather_add (Conv1d data gradient, col2im over overlapping windows): bit-exact against the fp32 restatement
    rounded once; against fp64 autograd of F.conv1d's input gradient within the rounding of dwin and of the output;
    tokens no window covers (gaps when s > k, the trailing tokens) exactly +0."""
    ops = _ops()
    fmt = act
    name, B, N, C, kk, ss = geom
    Lq = (N - kk) // ss + 1
    g = torch.Generator(device=DEV).manual_seed(N + kk)
    dy = torch.randn(B, Lq, C, generator=g, device=DEV, dtype=F64)
    W = torch.randn(C, C, kk, generator=g, device=DEV, dtype=F64) * (C * kk) ** -0.5
    dwin64 = dy.reshape(B * Lq, C) @ W.permute(0, 2, 1).reshape(C, kk * C)
    dwin = dwin64.to(fmt).contiguous()
    got = ops.window_gather_add(dwin, B, N, C, Lq, kk, ss)
    want, cover = _col2im(dwin, B, N, C, Lq, kk, ss, torch.float32)
    x = torch.zeros(B, N, C, device=DEV, dtype=F64, requires_grad=True)
    F.conv1d(x.transpose(1, 2), W, stride=ss).backward(dy.transpose(1, 2))
    mag, _ = _col2im(dwin64.abs(), B, N, C, Lq, kk, ss, F64)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.to(fmt).view(torch.int16))
    u, hs = _u(fmt), _half_sub(fmt)
    ref = x.grad
    r = _ratio(got, ref, torch.clamp(u * ref.abs(), min=hs) + u * mag + hs)
    n_free = int((cover == 0).sum())
    assert bool((got.view(torch.int16)[:, cover == 0] == 0).all())
    print(f"\n[window_gather_add {name} k={kk} s={ss} N={N} Lq={Lq}] vs fp64 conv1d grad: error / bar {r:.3f}; "
          f"{n_free} tokens in no window")
    assert r <= 1.0
    assert n_free == {"image": 28, "audio": 160, "video": 0, "lq1": 2}.get(name, n_free)
    if name == "gaps":
        assert n_free == (Lq - 1) * (ss - kk) + (N - (Lq - 1) * ss - kk)


def test_cast_bf16_all_fp16_patterns(act):
    """mm_cast_f16_bf16 (ops.cast_bf16) against torch's fp16 -> bf16 conversion over all 65536 fp16 bit patterns, bit for
    bit (NaNs as NaN), in three row shapes."""
    ops = _ops()
    x = torch.from_numpy(np.arange(65536, dtype=np.uint16).view(np.int16)).view(F16).to(DEV)
    want = x.to(BF16)
    nan = torch.isnan(want)
    assert int(nan.sum()) == 2046
    for shape in ((65536,), (256, 256), (2048, 32)):
        got = ops.cast_bf16(x.view(shape)).view(-1)
        assert torch.equal(torch.isnan(got), nan)
        assert torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan])


# ---------------------------------------------------------------------------------------------------- part B
ALIGN = ("image", "audio", "video")
TABLE = "llm.model.embed_tokens.weight"


@pytest.fixture(scope="module", params=[BF16, F16], ids=["bf16", "fp16"])
def real_width(request):
    """The bench's real configs with the depths cut (CLIP 2, Whisper 1, LLaMA 1 layers; default 6 frames) in one model
    format, every alignment bias (bias_k / bias_v included) re-drawn non-zero, and a B = 2 image + audio + video batch."""
    import bench
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from oracle import macaw_oracle as O

    fmt = request.param
    (clip, whisper, llama), hyper = bench.real_configs()
    clip.vision_config.num_hidden_layers = 2
    whisper.encoder_layers = 1
    llama.num_hidden_layers = 1
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=DEV, dtype=fmt, seed=3)
    g = torch.Generator(device=DEV).manual_seed(17)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.startswith(O.ALIGN_PREFIXES) and name.endswith(("bias", "bias_k", "bias_v")):
                p.copy_(torch.randn(p.shape, generator=g, device=DEV) * 0.02)
    gc = torch.Generator().manual_seed(23)
    B, L, V = 2, 12, llama.vocab_size
    inp = dict(images=torch.randn(B, 3, 224, 224, generator=gc), audios=torch.randn(B, 80, 3000, generator=gc),
               videos=torch.randn(B, cfg.n_frames, 3, 224, 224, generator=gc),
               input_ids=torch.randint(3, V - 6, (B, L), generator=gc), attention_mask=torch.ones(B, L, dtype=torch.int64))
    inp["input_ids"][:, 0] = 1
    inp["labels"] = inp["input_ids"].clone()
    inp["labels"][:, :2] = -100
    for i, name in enumerate(ALIGN):
        inp[f"{name}_starts"] = torch.full((B,), V - 6 + 2 * i, dtype=torch.int32)
        inp[f"{name}_ends"] = torch.full((B,), V - 5 + 2 * i, dtype=torch.int32)
    inp = {k: (v.to(DEV).to(fmt) if v.is_floating_point() else v.to(DEV)) for k, v in inp.items()}
    yield fmt, model, inp
    del model
    torch.cuda.empty_cache()


def _score_span(model, name, feats) -> float:
    """Median over query rows and heads of (max - min) of the real keys' scores s q_h . (W_k[h] table_v + b_k[h]), fp64."""
    conv, lin = getattr(model, f"project_{name}"), getattr(model, f"transform_{name}_to_hidden")
    mha = getattr(model, f"{name}_align_attention")
    table = model.llm.model.embed_tokens.weight.detach().double()
    y = F.conv1d(feats.double().transpose(1, 2), conv.weight.detach().double(), conv.bias.detach().double(),
                 stride=conv.stride[0]).transpose(1, 2)
    z = F.linear(y, lin.weight.detach().double(), lin.bias.detach().double())
    E, H = z.shape[-1], mha.num_heads
    hd = E // H
    W, b = mha.in_proj_weight.detach().double(), mha.in_proj_bias.detach().double()
    q = F.linear(z, W[:E], b[:E]).reshape(-1, H, hd)
    k = F.linear(table, W[E:2 * E], b[E:2 * E]).view(-1, H, hd)
    s = torch.einsum("nhd,vhd->nhv", q, k) * hd ** -0.5
    return float((s.amax(-1) - s.amin(-1)).median())


def _sharpen(model, inp, fmt, target=40.0):
    """Scale W_q and W_k of each alignment attention by one factor c (scores scale by ~c^2) so that a row's scores span
    ~`target` nats.  -> the original in-projection weights, for restoring."""
    ops = _ops()
    prev = ops.ACT()
    ops.set_act_format(fmt)  # the eval-mode encoders run in the thread's format
    try:
        with torch.no_grad():
            feats = dict(image=model.encode_image(inp["images"]), audio=model.encode_audio(inp["audios"]),
                         video=model.encode_video_long(inp["videos"]))
    finally:
        ops.set_act_format(prev)
    with torch.no_grad():
        saved, spans = {}, {}
        for n in ALIGN:
            mha = getattr(model, f"{n}_align_attention")
            E = mha.embed_dim
            saved[n] = mha.in_proj_weight.detach().clone()
            s0 = _score_span(model, n, feats[n])
            c = math.sqrt(target / s0)
            mha.in_proj_weight[:2 * E].mul_(c)
            spans[n] = (s0, c, _score_span(model, n, feats[n]))
    print("\n[sharp regime] median score span (nats) default weights -> W_q, W_k scaled by c: "
          + ", ".join(f"{n} {s0:.2f} -> c {c:.2f} -> {s:.1f}" for n, (s0, c, s) in spans.items()))
    spans = {n: v[2] for n, v in spans.items()}
    assert min(spans.values()) > 20.0
    return saved


def _train_backward(model, inp, fmt, dropout, monkeypatch):
    """One `model.train(); model(inp).loss.backward()` (fp16: DynamicLossScaler at its default 2^16), recording what each
    AlignTrainer.backward receives and the d(feats) its video block hands to video_long_backward.
    -> (records, loss scale S, dropout seed)."""
    from macaw_llm_b200 import training

    rec = {}
    orig, orig_vl = training.AlignTrainer.backward, training.AlignTrainer.video_long_backward

    def spy(self, name, sv, d_embeds, video_long=None):
        rec[name] = dict(d=d_embeds.clone(), feats=sv["feats"].clone(), off=int(sv["row_off"]) + 1, Lq=int(sv["Lq"]),
                         xp=None if video_long is None else video_long["xp"].clone())
        return orig(self, name, sv, d_embeds, video_long)

    def spy_vl(self, sv, d_feats):
        rec["video_d_feats"] = d_feats.clone()
        return orig_vl(self, sv, d_feats)

    monkeypatch.setattr(training.AlignTrainer, "backward", spy)
    monkeypatch.setattr(training.AlignTrainer, "video_long_backward", spy_vl)
    model.train()
    model.train_step.attention_dropout = bool(dropout)
    try:
        for p in model.parameters():
            p.grad = None
        out = model(inp)
        if fmt == F16:
            scaler = training.DynamicLossScaler()
            scaler.scale(out.loss).backward()
            S = scaler.loss_scale
        else:
            out.loss.backward()
            S = 1.0
        torch.cuda.synchronize()
    finally:
        model.train_step.attention_dropout = True
        model.eval()
        monkeypatch.undo()
    assert sorted(rec) == sorted(ALIGN + ("video_d_feats",)) and rec["video"]["xp"] is not None
    return rec, S, model.train_step.last_seed if dropout else None


def _masks(model, seed, B):
    """The attention-dropout multipliers of the latest training forward in the oracle's (B*H, Lq, S+2) layout."""
    ops = _ops()
    if seed is None:
        return {}
    eng = model.engine
    V = model.llm.model.embed_tokens.weight.shape[0]
    masks = {}
    for n in ALIGN:
        mha = getattr(model, f"{n}_align_attention")
        Hh, Lq = mha.num_heads, eng.last_lens[n]
        m = ops.dropout_mask(Hh * B * Lq, V + 2, (mha.dropout, seed, eng.DROPOUT_SID[n]), DEV)
        masks[n] = m.view(Hh, B, Lq, V + 2).permute(1, 0, 2, 3).reshape(B * Hh, Lq, V + 2)
    mha = model.video_long_self_attention
    N = eng._video_long_len
    masks["video_long"] = ops.dropout_mask(B * mha.num_heads * N, N + 2, (mha.dropout, seed, eng.DROPOUT_SID["video_long"]),
                                           DEV).view(B * mha.num_heads, N, N + 2)
    return masks


def _restated_grads(model, rec, masks, dtype, S):
    """Autograd of the oracle's alignment blocks (+ video_long_self_attention on the recorded xp) on the GPU in `dtype`:
    leaves are copies of the model's weights and table, the recorded feats are constants (video: the value is the recorded
    one, the gradient flows into video_long_self_attention), the upstream gradient is the recorded d_embeds rows.
    -> ({parameter: gradient / S}, table gradient / S, gradient / S of the video feats), fp32-stored."""
    from oracle import macaw_oracle as O

    named = dict(model.named_parameters())
    table = named[TABLE].detach().to(dtype).clone().requires_grad_(True)
    grads = {}
    for n in ALIGN:
        pre = (f"project_{n}.", f"transform_{n}_to_hidden.", f"{n}_align_attention.") + \
            (("video_long_self_attention.",) if n == "video" else ())
        leaves = {k: p.detach().to(dtype).clone().requires_grad_(True) for k, p in named.items() if k.startswith(pre)}
        sd = O._SD(leaves, dtype, keep_graph=True)
        r = rec[n]
        feats = r["feats"].to(dtype)
        if n == "video":
            feats = f_leaf = feats.clone().requires_grad_(True)
            mv = model.video_long_self_attention
            B, N, P = feats.shape
            xs = r["xp"].to(dtype).view(B, N, P).transpose(0, 1)
            vl = O.mha_forward(xs, xs, xs, sd.sub("video_long_self_attention."), mv.num_heads,
                               masks.get("video_long")).transpose(0, 1)
            feats = feats + (vl - vl.detach())
        mha = getattr(model, f"{n}_align_attention")
        out = O.align_block(feats, table, sd.sub(f"project_{n}."), sd.sub(f"transform_{n}_to_hidden."),
                            sd.sub(f"{n}_align_attention."), getattr(model, f"project_{n}").stride[0], mha.num_heads,
                            masks.get(n))
        out.backward(r["d"][:, r["off"]:r["off"] + r["Lq"]].to(dtype))
        for k, t in leaves.items():
            grads[k] = (t.grad.double() / S).float()  # fp32 storage: 6e-8 relative, far below the errors compared
        del leaves, sd, out, feats
    tg = (table.grad.double() / S).float()
    dfe = (f_leaf.grad.double() / S).float()
    del table, f_leaf
    torch.cuda.empty_cache()
    return grads, tg, dfe


def _gathered_rows(model, inp, rec, S):
    """fp64 gradient the table receives through the gathered rows (BOS, text, start / end tokens) from the recorded
    d_embeds, and the ids those rows use."""
    d = rec["image"]["d"].double() / S
    B, T, E = d.shape
    ids_in = inp["input_ids"]
    L = ids_in.shape[1]
    ids = torch.full((B, T), -1, dtype=torch.int64, device=DEV)
    ids[:, 0] = ids_in[:, 0]
    ids[:, T - L + 1:] = ids_in[:, 1:]
    for n in ALIGN:
        r = rec[n]
        ids[:, r["off"] - 1] = inp[f"{n}_starts"].long()
        ids[:, r["off"] + r["Lq"]] = inp[f"{n}_ends"].long()
    sel = ids >= 0
    V = model.llm.model.embed_tokens.weight.shape[0]
    g = torch.zeros((V, E), device=DEV, dtype=F64).index_add_(0, ids[sel], d[sel])
    return g.float(), ids[sel].unique()


def _rel(a, b) -> float:
    b = b.double()
    return float((a.double() - b).norm() / b.norm().clamp_min(1e-300))


ABS_BAR = 6e-3  # the per-op bar of the training kernels' bf16 / fp16 tests (one 16-bit rounding + 16-bit inputs)


@pytest.mark.parametrize("dropout", [False, True], ids=["nodrop", "drop"])
@pytest.mark.parametrize("regime", ["flat", "sharp"])
def test_real_width_align_backward(real_width, regime, dropout, monkeypatch):
    """Every alignment parameter's gradient (in-projections split into their q / k / v parts) and the table gradient
    (rows no input id touches: the alignment contribution alone; all rows: plus the gathered-row term) from the public
    training path, against fp64 autograd of the oracle; each must satisfy err < max(ABS_BAR, 2 x the torch-16-bit
    yardstick's err)."""
    fmt, model, inp = real_width
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    saved = _sharpen(model, inp, fmt) if regime == "sharp" else None
    try:
        rec, S, seed = _train_backward(model, inp, fmt, dropout, monkeypatch)
        named = dict(model.named_parameters())
        from oracle import macaw_oracle as O

        ours = {k: (p.grad.detach().double() / S).float() for k, p in named.items()
                if p.grad is not None and k.startswith(O.ALIGN_PREFIXES)}
        ours_t = (named[TABLE].grad.detach().double() / S).float()
        for p in model.parameters():
            p.grad = None
        B = inp["input_ids"].shape[0]
        masks = _masks(model, seed, B)
        ref, ref_t, ref_df = _restated_grads(model, rec, masks, F64, S)
        yard, yard_t, yard_df = _restated_grads(model, rec, masks, fmt, S)
        ours_df = (rec["video_d_feats"].double() / S).float().view_as(ref_df)
        gath, touched = _gathered_rows(model, inp, rec, S)
    finally:
        if saved is not None:
            with torch.no_grad():
                for n, w in saved.items():
                    getattr(model, f"{n}_align_attention").in_proj_weight.copy_(w)
    assert sorted(ours) == sorted(ref), sorted(set(ours) ^ set(ref))
    # the video block's d(feats), where the alignment backward hands over to video_long_self_attention's backward
    rows = [("video: d(feats) into video_long_self_attention", _rel(ours_df, ref_df), _rel(yard_df, ref_df))]
    for k in sorted(ref):
        if k.endswith(("in_proj_weight", "in_proj_bias")):
            n3 = ref[k].shape[0] // 3
            parts = [(f"{k}[{s}]", slice(i * n3, (i + 1) * n3)) for i, s in enumerate("qkv")]
        else:
            parts = [(k, slice(None))]
        for lbl, sl in parts:
            rows.append((lbl, _rel(ours[k][sl], ref[k][sl]), _rel(yard[k][sl], ref[k][sl])))
    free = torch.ones(ref_t.shape[0], dtype=torch.bool, device=DEV)
    free[touched] = False
    rows.append(("table, rows no input id touches", _rel(ours_t[free], ref_t[free]), _rel(yard_t[free], ref_t[free])))
    rows.append(("table, all rows", _rel(ours_t, ref_t + gath), _rel(yard_t + gath, ref_t + gath)))
    # free the device tensors before any assertion: a failing test's traceback would keep them alive for the next test
    del ours, ours_t, ref, ref_t, yard, yard_t, gath, free, rec, masks, ours_df, ref_df, yard_df
    torch.cuda.empty_cache()
    tag = f"{str(fmt)[6:]} {regime} dropout={'on' if dropout else 'off'}"
    bad = []
    # a mistake that changes a gradient by a relative d gives an error >= d - err, so the bar catches every d > bar + err
    print(f"\n[align backward, real width, {tag}] err (ours vs fp64) | yardstick (torch {str(fmt)[6:]} vs fp64) | bar | "
          f"smallest relative change caught")
    for lbl, e, y in rows:
        bar = max(ABS_BAR, 2.0 * y)
        print(f"  {lbl:58s} {e:.3e} | {y:.3e} | {bar:.3e} | {bar + e:.3e}{'   FAIL' if not e < bar else ''}")
        if not e < bar:
            bad.append((lbl, e, bar))
    print(f"[align backward, real width, {tag}] wall {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    assert not bad, bad
