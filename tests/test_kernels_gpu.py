"""Per-kernel numerics on the H100: every C-ABI kernel against a plain torch fp32 restatement of the same op
(bf16-rounded inputs, fp32 math).  Tolerances are norm-wise relative errors; bf16 output rounding alone is ~2e-3
element-wise / ~1.5e-3 norm-wise, so GEMM-class outputs are held to 4e-3 and fp32 outputs to 1e-4."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from macaw_llm_b200 import ops

    return ops


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-20))


def test_attention_lazy_rescale_large_scores():
    """Scores with a large dynamic range (row max grows by >> 2^8 between key tiles) exercise the running-max rescale."""
    ops = _ops()
    B, H, T, hd = 1, 2, 512, 128
    q = rnd(B, T, H, hd, scale=2.0, seed=60)
    k = rnd(B, T, H, hd, scale=2.0, seed=61)
    v = rnd(B, T, H, hd, seed=62)
    # make later keys systematically larger so the running max keeps jumping
    k = (k.float() * torch.linspace(0.2, 3.0, T, device=DEV)[None, :, None, None]).to(torch.bfloat16)
    out = ops.attention(q, k, v, scale=hd ** -0.5)
    ref = _attn_ref(q, k, v, hd ** -0.5, False, None)
    assert rel_err(out, ref) < 1e-2


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize(
    "M,N,K",
    [
        (128, 256, 64),      # one tile, one k-block
        (128, 256, 256),     # one tile, pipeline wraps
        (256, 512, 4096),    # several tiles
        (264, 4096, 4096),   # LLaMA B=1 shape (M tail)
        (6, 4096, 768),      # alignment Linear C->E (tiny M)
        (300, 1000, 1096),   # ragged everything (N % 32 != 0, K % 64 != 0)
        (2112, 11008, 4096), # LLaMA MLP up, many tiles -> multi-wave persistent loop
        (1500, 512, 2048),   # Whisper fc2
    ],
)
def test_gemm_plain(M, N, K):
    ops = _ops()
    x, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    out = ops.linear(x, w)
    ref = x.float() @ w.float().t()
    assert rel_err(out, ref) < 4e-3
    out32 = ops.linear(x, w, out_fp32=True)
    assert rel_err(out32, ref) < 1e-4


@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_gemm_bias_act_residual(act):
    ops = _ops()
    M, N, K = 514, 1024, 1024
    x, w, b = rnd(M, K, seed=3), rnd(N, K, scale=K ** -0.5, seed=4), rnd(N, seed=5)
    res = rnd(M, N, seed=6)
    out = ops.linear(x, w, b, act=act, residual=res)
    y = x.float() @ w.float().t() + b.float()
    if act == 1:
        y = torch.nn.functional.gelu(y)
    elif act == 2:
        y = y * torch.sigmoid(1.702 * y)
    elif act == 3:
        y = torch.nn.functional.silu(y)
    ref = y + res.float()
    assert rel_err(out, ref) < 4e-3


def test_gemm_residual_row_mod_and_inplace():
    ops = _ops()
    M, N, K = 771, 1024, 640  # 3 x 257 rows, CLIP-like
    x, w = rnd(M, K, seed=7), rnd(N, K, scale=K ** -0.5, seed=8)
    pos = rnd(257, N, seed=9)
    out = ops.linear(x, w, residual=pos, res_row_mod=257)
    ref = x.float() @ w.float().t() + pos.float().repeat(3, 1)
    assert rel_err(out, ref) < 4e-3
    # in-place residual add (out aliases residual) as used for the transformer residual stream
    h = rnd(M, N, seed=10)
    ref2 = x.float() @ w.float().t() + h.float()
    ops.linear(x, w, residual=h, out=h)
    assert rel_err(h, ref2) < 4e-3


def test_gemm_row_scale_alpha():
    ops = _ops()
    M, N, K = 200, 512, 512
    x, w = rnd(M, K, seed=11), rnd(N, K, scale=K ** -0.5, seed=12)
    rs = torch.rand(M, device=DEV) + 0.5
    out = ops.linear(x, w, row_scale=rs, alpha=0.25, out_fp32=True)
    ref = (x.float() @ w.float().t()) * rs[:, None] * 0.25
    assert rel_err(out, ref) < 1e-4


def test_gemm_swiglu():
    ops = _ops()
    M, K, I = 300, 1024, 2752
    x = rnd(M, K, seed=13)
    wg, wu = rnd(I, K, scale=K ** -0.5, seed=14), rnd(I, K, scale=K ** -0.5, seed=15)
    # interleave rows in blocks of 32: [g0..g31, u0..u31, g32.., ...]
    wgu = torch.stack([wg.view(I // 32, 32, K), wu.view(I // 32, 32, K)], dim=1).reshape(2 * I, K).contiguous()
    out = ops.linear(x, wgu, epi=ops.EPI_SWIGLU)
    ref = torch.nn.functional.silu(x.float() @ wg.float().t()) * (x.float() @ wu.float().t())
    assert out.shape == (M, I)
    assert rel_err(out, ref) < 4e-3


def test_gemm_rope():
    ops = _ops()
    B, T, E, H = 2, 100, 512, 4  # head_dim 128
    x = rnd(B * T, E, seed=16)
    w = rnd(3 * E, E, scale=E ** -0.5, seed=17)
    inv = 1.0 / (10000 ** (torch.arange(0, 128, 2, device=DEV).float() / 128))
    ang = torch.arange(T, device=DEV).float()[:, None] * inv[None, :]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    out = ops.linear(x, w, epi=ops.EPI_ROPE, rope=(cos, sin, T, 2 * E))
    y = (x.float() @ w.float().t()).view(B, T, 3, H, 128)
    c = torch.cat([cos, cos], -1)[None, :, None, None, :]
    s = torch.cat([sin, sin], -1)[None, :, None, None, :]
    rot = torch.cat([-y[..., 64:], y[..., :64]], -1)
    yr = y * c + rot * s
    ref = torch.cat([yr[:, :, :2], y[:, :, 2:]], dim=2).reshape(B * T, 3 * E)
    assert rel_err(out, ref) < 4e-3


def test_gemm_batched_strided_and_mn_major():
    ops = _ops()
    # per-head absorbed query: q (Nq, 16*256) x W_k[h] (256, E) -> (H, Nq, E); B operand is MN-major (N contiguous)
    Nq, H, hd, E = 24, 4, 256, 1024
    q = rnd(Nq, H * hd, seed=18)
    wk = rnd(H * hd, E, scale=hd ** -0.5, seed=19)
    out = torch.empty(H, Nq, E, device=DEV, dtype=torch.bfloat16)
    ops.gemm_raw(M=Nq, N=E, K=hd, batch=H, A=q.data_ptr(), lda=q.stride(0), a_bs=hd, B=wk.data_ptr(), ldb=E,
                 b_bs=hd * E, b_mn_major=True, Cout=out.data_ptr(), ldc=E, c_bs=Nq * E, alpha=0.5)
    ref = 0.5 * torch.einsum("nhd,hde->hne", q.float().view(Nq, H, hd), wk.float().view(H, hd, E))
    assert rel_err(out, ref) < 4e-3


def test_gemm_mn_major_long_k():
    ops = _ops()
    # P (R, V) x table (V, E): K = V is the table's row index -> MN-major B, ragged K
    R, V, E = 200, 3001, 512
    P = rnd(R, 3008, seed=20).abs()
    P[:, V:] = 0
    tab = rnd(V, E, seed=21)
    out = torch.empty(R, E, device=DEV, dtype=torch.float32)
    ops.gemm_raw(M=R, N=E, K=V, A=P.data_ptr(), lda=P.stride(0), B=tab.data_ptr(), ldb=E, b_mn_major=True,
                 Cout=out.data_ptr(), ldc=E, c_fp32=True)
    ref = P[:, :V].float() @ tab.float()
    assert rel_err(out, ref) < 1e-4


def test_gemm_overlapping_rows_conv_view_and_splitk():
    ops = _ops()
    # Conv1d(C, C, k, stride s) over the token axis as a GEMM on overlapping row views, split over K
    B, Ntok, Cc, k, s = 3, 256, 64, 48, 36
    Lq = (Ntok - k) // s + 1
    x = rnd(B, Ntok, Cc, seed=22)
    w = rnd(Cc, Cc, k, scale=(Cc * k) ** -0.5, seed=23)       # torch Conv1d weight (out, in, k)
    bias = rnd(Cc, seed=24)
    wp = w.permute(0, 2, 1).reshape(Cc, k * Cc).contiguous()    # (out, k*in): matches the contiguous token window
    S = 4
    Kc = k * Cc // S
    part = torch.empty(S, B * Lq, Cc, device=DEV, dtype=torch.float32)
    # inner batch = K split, outer batch (batch2) = sample; one launch
    ops.gemm_raw(M=Lq, N=Cc, K=Kc, batch=S, batch2=B, A=x.data_ptr(), lda=s * Cc, a_bs=Kc, a_bs2=Ntok * Cc,
                 B=wp.data_ptr(), ldb=k * Cc, b_bs=Kc, b_bs2=0, Cout=part.data_ptr(), ldc=Cc, c_bs=B * Lq * Cc,
                 c_bs2=Lq * Cc, c_fp32=True)
    out = torch.empty(B * Lq, Cc, device=DEV, dtype=torch.bfloat16)
    ops.splitk_reduce(part, bias, out)
    ref = torch.nn.functional.conv1d(x.float().transpose(1, 2), w.float(), bias.float(), stride=s).transpose(1, 2)
    assert rel_err(out, ref.reshape(B * Lq, Cc)) < 4e-3


# ------------------------------------------------------------------------------------------------ attention
def _attn_ref(q, k, v, scale, causal, key_mask):
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))  # B H T d
    s = (qf @ kf.transpose(-1, -2)) * scale
    Tq, Tk = s.shape[-2:]
    if causal:
        i = torch.arange(Tq, device=s.device)[:, None]
        j = torch.arange(Tk, device=s.device)[None, :]
        s = s.masked_fill(j > i + (Tk - Tq), float("-inf"))
    if key_mask is not None:
        s = s.masked_fill(key_mask[:, None, None, :] == 0, float("-inf"))
    p = torch.softmax(s, dim=-1)
    p = torch.nan_to_num(p, nan=0.0)
    return (p @ vf).permute(0, 2, 1, 3)


@pytest.mark.parametrize(
    "B,H,Tq,Tk,hd,causal,masked",
    [
        (2, 4, 257, 257, 64, False, False),    # CLIP
        (1, 8, 1500, 1500, 64, False, False),  # Whisper
        (1, 8, 200, 202, 96, False, False),    # video-long (two synthetic keys appended)
        (2, 4, 264, 264, 128, True, False),    # LLaMA causal
        (2, 4, 130, 130, 128, True, True),     # LLaMA causal + right padding
        (1, 2, 64, 64, 128, True, False),
        (1, 2, 1, 70, 64, False, False),
        (2, 32, 528, 528, 128, True, True),    # cfg4 LLaMA shape: 5 query tiles (ragged first tile), padding
        (1, 3, 300, 300, 64, True, False),
    ],
)
def test_attention(B, H, Tq, Tk, hd, causal, masked):
    ops = _ops()
    # q/k/v as strided views of one fused (B, T, 3, H, hd) projection output, as the engine uses them
    qkv_q = rnd(B, Tq, 3, H, hd, seed=30)
    qkv_k = qkv_q if Tq == Tk else rnd(B, Tk, 3, H, hd, seed=31)
    q, k, v = qkv_q[:, :, 0], qkv_k[:, :, 1], qkv_k[:, :, 2]
    km = None
    if masked:
        km = torch.ones(B, Tk, dtype=torch.int32, device=DEV)
        km[0, Tk - 17:] = 0
    scale = hd ** -0.5
    out = ops.attention(q, k, v, scale=scale, causal=causal, key_mask=km)
    ref = _attn_ref(q, k, v, scale, causal, km)
    if masked:  # rows whose own key is padding are unspecified (DESIGN.md); compare valid query rows only
        valid = km.bool()[:, -Tq:]
        out, ref = out[valid], ref[valid]
    assert rel_err(out, ref) < 5e-3


# ------------------------------------------------------------------------------------------------ norms & misc
def test_rmsnorm_layernorm():
    ops = _ops()
    x, w, b = rnd(300, 4096, seed=40), rnd(4096, seed=41), rnd(4096, seed=42)
    y = ops.rmsnorm(x, w, 1e-6)
    xf = x.float()
    ref = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * w.float()
    assert rel_err(y, ref) < 3e-3
    for cols in (128, 512, 1024, 2048):  # warp-per-row kernels (<= 1024) and the CTA-per-row kernel
        x2 = rnd(517, cols, seed=43)
        y2 = ops.layernorm(x2, w[:cols].contiguous(), b[:cols].contiguous(), 1e-5)
        ref2 = torch.nn.functional.layer_norm(x2.float(), (cols,), w[:cols].float(), b[:cols].float(), 1e-5)
        assert rel_err(y2, ref2) < 3e-3, cols


def test_embed_gather_and_splice_bit_exact():
    ops = _ops()
    V, E, B, L, P = 1000, 256, 3, 17, 8
    table = rnd(V, E, seed=44)
    ids = torch.randint(0, V, (B, L), device=DEV)
    text = ops.embed_gather(table, ids).view(B, L, E)
    assert torch.equal(text, table[ids])
    prefix = rnd(B, P, E, seed=45)
    mask = torch.randint(0, 2, (B, L), device=DEV)
    labels = torch.randint(-100, V, (B, L), device=DEV)
    emb, m, l = ops.splice_prefix(text, prefix, mask, labels)
    ref = torch.cat([text[:, :1], prefix, text[:, 1:]], dim=1)
    assert torch.equal(emb, ref)
    assert torch.equal(m, torch.cat([torch.ones(B, P, dtype=torch.int64, device=DEV), mask], 1))
    assert torch.equal(l, torch.cat([torch.full((B, P), -100, dtype=torch.int64, device=DEV), labels], 1))
    emb2, m2, l2 = ops.splice_prefix(text, None, None, None)
    assert torch.equal(emb2, text) and m2 is None and l2 is None


def test_patchify_transpose_addrows():
    ops = _ops()
    img = rnd(2, 3, 28, 42, seed=46)
    out = ops.patchify(img, 14, 640)
    ref = torch.nn.functional.unfold(img.float(), kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588)
    assert torch.equal(out[:, :588].float(), ref) and float(out[:, 588:].abs().max()) == 0.0
    x = rnd(2, 80, 300, seed=47)
    t = ops.transpose_pad(x, 1)
    assert torch.equal(t[:, 1:-1], x.transpose(1, 2)) and float(t[:, 0].abs().max()) == 0 and float(t[:, -1].abs().max()) == 0
    a, add = rnd(514, 1024, seed=48), rnd(257, 1024, seed=49)
    y = torch.empty_like(a)
    ops.add_rows(a, add, y)
    assert rel_err(y, a.float() + add.float().repeat(2, 1)) < 3e-3


def test_ce_loss():
    ops = _ops()
    B, T, V = 3, 21, 5000
    logits = rnd(B, T, V, scale=3.0, seed=50)
    labels = torch.randint(0, V, (B, T), device=DEV)
    labels[:, :5] = -100
    loss = ops.ce_loss(logits, labels)
    ref = torch.nn.functional.cross_entropy(logits[:, :-1].float().reshape(-1, V), labels[:, 1:].reshape(-1))
    assert abs(float(loss) - float(ref)) < 1e-3 * abs(float(ref))


def test_rms_rstd_and_fused_norm_linear():
    """RMSNorm folded into the next GEMM: rstd * (x (W diag g)^T) == RMSNorm(x) W^T."""
    ops = _ops()
    M, K, N = 300, 4096, 512
    x, g, w = rnd(M, K, seed=70), (1.0 + 0.1 * torch.randn(K)).to(DEV).to(torch.bfloat16), rnd(N, K, scale=K ** -0.5, seed=71)
    rstd = ops.rms_rstd(x, 1e-6)
    ref_rstd = torch.rsqrt(x.float().pow(2).mean(-1) + 1e-6)
    assert rel_err(rstd, ref_rstd) < 1e-5
    wg = (w.float() * g.float()[None, :]).to(torch.bfloat16)
    out = ops.linear(x, wg, row_scale=rstd)
    ref = (x.float() * ref_rstd[:, None] * g.float()) @ w.float().t()
    assert rel_err(out, ref) < 5e-3


@pytest.mark.parametrize(
    "M,N,K,kind",
    [
        (4224, 4096, 512, "std"),      # 33 M tiles
        (4096, 2560, 1024, "bias_res"),
        (4096, 4096, 1024, "rope"),
        (4096, 5504, 1024, "swiglu"),
        (3072, 4096, 3001, "mn"),      # P x table shape, MN-major B, ragged K
        (16896, 4096, 4096, "std"),    # cfg4 o_proj
        (2176, 12288, 4096, "rope"),   # 17 M tiles: a partial last wave
        (2112, 4096, 11008, "bias_res"),
    ],
)
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_gemm_wide_shapes(M, N, K, kind, dtype):
    """The wide, multi-wave GEMMs of the LLaMA stack and the alignment chain, with bf16 and with fp16 operands /
    activations."""
    ops = _ops()
    dt = torch.float16 if dtype == "fp16" else torch.bfloat16
    ops.set_act_format(dt)
    _wide_case(M, N, K, kind, dt)
    torch.cuda.synchronize()


def _wide_case(M, N, K, kind, dt):
    ops = _ops()
    x = rnd(M, K, seed=80).to(dt)
    if kind == "mn":
        P = rnd(M, 3008, seed=81).abs().to(dt)
        P[:, K:] = 0
        tab = rnd(K, N, seed=82).to(dt)
        out = torch.empty(M, N, device=DEV, dtype=dt)
        ops.gemm_raw(M=M, N=N, K=K, A=P.data_ptr(), lda=P.stride(0), B=tab.data_ptr(), ldb=N, b_mn_major=True,
                     Cout=out.data_ptr(), ldc=N)
        assert rel_err(out, P[:, :K].float() @ tab.float()) < 4e-3
        return
    if kind == "swiglu":
        I = N // 2
        wg, wu = rnd(I, K, scale=K ** -0.5, seed=83).to(dt), rnd(I, K, scale=K ** -0.5, seed=84).to(dt)
        wgu = torch.stack([wg.view(I // 32, 32, K), wu.view(I // 32, 32, K)], dim=1).reshape(2 * I, K).contiguous()
        out = ops.linear(x, wgu, epi=ops.EPI_SWIGLU)
        ref = torch.nn.functional.silu(x.float() @ wg.float().t()) * (x.float() @ wu.float().t())
        assert rel_err(out, ref) < 4e-3
        return
    w = rnd(N, K, scale=K ** -0.5, seed=85).to(dt)
    if kind == "rope":
        T = 128
        inv = 1.0 / (10000 ** (torch.arange(0, 128, 2, device=DEV).float() / 128))
        ang = torch.arange(T, device=DEV).float()[:, None] * inv[None, :]
        cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
        out = ops.linear(x, w, epi=ops.EPI_ROPE, rope=(cos, sin, T, N))
        y = (x.float() @ w.float().t()).view(M // T, T, N // 128, 128)
        c = torch.cat([cos, cos], -1)[None, :, None, :]
        s_ = torch.cat([sin, sin], -1)[None, :, None, :]
        ref = (y * c + torch.cat([-y[..., 64:], y[..., :64]], -1) * s_).reshape(M, N)
        assert rel_err(out, ref) < 4e-3
        return
    if kind == "bias_res":
        b, res = rnd(N, seed=86).to(dt), rnd(M, N, seed=87).to(dt)
        out = ops.linear(x, w, b, residual=res)
        assert rel_err(out, x.float() @ w.float().t() + b.float() + res.float()) < 4e-3
        return
    out = ops.linear(x, w)
    assert rel_err(out, x.float() @ w.float().t()) < 4e-3


@pytest.mark.parametrize("M,N,K,kind", [
    (2112, 4096, 4096, "res_stats"),   # o_proj at 4 samples/GPU: 17 x 64 = 1088 tiles of 128 x 64 -> 8 waves + 32
    (2112, 4096, 11008, "res_stats"),  # down_proj, K = 172 k-blocks
    (2112, 12288, 4096, "rope"),       # QKV + RoPE: 17 x 96 = 1632 tiles -> 12 waves + 48
    (264, 12288, 4096, "rope"),        # cfg2 QKV + RoPE (B=1, T=264): 3 x 96 = 288 tiles -> 2 waves + 24; each RoPE
                                       # warp owns columns (i, i + 64) of a head: its partials must come from that warp
    (1200, 4096 * 2, 1024, "swiglu"),  # 10 x 64 = 640 tiles -> 4 waves + 112: shares of ~14 of a tile's 16 k-blocks
    (19072, 256, 4096, "plain"),       # 149 x 4 = 596 tiles of 128 x 64 -> 4 waves + 68: a narrow N, long K
    (17024, 64, 4096, "plain"),        # 133 tiles -> 1 wave + 1: ONE tile split over all CTAs (64 k-blocks on 132 CTAs)
    (640, 7680, 512, "plain"),         # 5 x 120 = 600 tiles, num_k = 8: shares shorter than one k-block for most CTAs
])
def test_gemm_streamk_tail(M, N, K, kind):
    """Stream-K tail (mm_gemm_args.sk_workspace): the partial last wave's k-blocks are split evenly over all CTAs, partial
    accumulators handed over through the workspace.  Against the fp32 reference at the usual bar, against the plain
    data-parallel launch (same math, different fp32 summation order: a handful of 1-ulp flips), bit-identical across
    repeated launches (fixed summation order; the flags re-arm themselves)."""
    ops = _ops()
    x, w = rnd(M, K, seed=190), rnd(N, K, scale=K ** -0.5, seed=191)
    ws = ops.streamk_workspace(x.device)

    def run():
        if kind == "res_stats":
            res = rnd(M, N, seed=192)
            ss = torch.empty((M, N // 32), device=DEV, dtype=torch.float32)
            out = ops.linear(x, w, residual=res, sumsq_out=ss)
            return out, ss
        if kind == "rope":
            return ops.linear(x, w, epi=ops.EPI_ROPE, rope=(cos_g, sin_g, 528, N * 2 // 3)), None
        if kind == "swiglu":
            return ops.linear(x, w, epi=ops.EPI_SWIGLU), None
        return ops.linear(x, w), None

    cos_g, sin_g = torch.rand(528, 64, device=DEV), torch.rand(528, 64, device=DEV)
    from macaw_llm_b200 import _lib

    base, base_ss = run()
    ops.STREAMK = ws
    prev = _lib.load().mm_gemm_streamk_mode(2)  # force: the default policy skips shapes where it does not pay (o_proj)
    try:
        outs = [run() for _ in range(3)]
    finally:
        ops.STREAMK = None
        _lib.load().mm_gemm_streamk_mode(prev)
    torch.cuda.synchronize()
    assert int(ws[:2048].abs().sum()) == 0  # every flag re-armed
    got, got_ss = outs[0]
    for o, o_ss in outs[1:]:
        assert torch.equal(o, got)
        assert o_ss is None or torch.equal(o_ss, got_ss)
    assert rel_err(got, base) < 1e-3
    frac = float((got != base).float().mean())
    assert frac < 0.02, frac
    assert float(ws[2048:].view(torch.float32).abs().sum()) > 0  # partial accumulators did pass through the workspace
    if kind == "plain":
        assert rel_err(got, x.float() @ w.float().t()) < 4e-3
    if kind == "res_stats":
        ref = x.float() @ w.float().t() + rnd(M, N, seed=192).float()
        assert rel_err(got, ref) < 4e-3
        assert rel_err(got_ss.sum(1), got.float().pow(2).sum(1)) < 1e-5


@pytest.mark.parametrize("M", [1, 8, 32, 50])
def test_linear_thin_swapped_operands(M, thin_streamk):
    """Decode-step GEMMs: operands swapped (weights on the 128-row side), transposed epilogue."""
    ops = _ops()
    K, N = 1024, 1536
    x, w, b = rnd(M, K, seed=90), rnd(N, K, scale=K ** -0.5, seed=91), rnd(N, seed=92)
    res = rnd(M, N, seed=93)
    rs = torch.rand(M, device=DEV) + 0.5
    out = ops.linear_thin(x, w, b, act=ops.ACT_GELU, residual=res, row_scale=rs)
    ref = torch.nn.functional.gelu((x.float() @ w.float().t()) * rs[:, None] + b.float()) + res.float()
    assert rel_err(out, ref) < 4e-3
    h = res.clone()
    ops.linear_thin(x, w, residual=h, out=h)  # in-place residual stream update
    assert rel_err(h, x.float() @ w.float().t() + res.float()) < 4e-3


@pytest.fixture(params=[False, True], ids=["splitk4", "streamk"])
def thin_streamk(request):
    """Thin (decode) GEMMs either with the fixed split-K factor or with the stream-K workspace (fewer tiles than SMs:
    the whole GEMM is divided evenly along K over all SMs)."""
    ops = _ops()
    ops.STREAMK = ops.streamk_workspace(torch.device(DEV, 0)) if request.param else None
    yield request.param
    ws, ops.STREAMK = ops.STREAMK, None
    if ws is not None:
        torch.cuda.synchronize()
        assert int(ws[:2048].abs().sum()) == 0  # every hand-over flag re-armed


@pytest.mark.parametrize("M", [1, 8, 13])
def test_linear_thin_fused_decode_tails(M, thin_streamk):
    """mm_thin_fused: the three fused tails of the decode step's thin GEMMs against fp32 references — residual +
    next-RMSNorm statistic, SwiGLU on the interleaved product with the row scale taken from such statistics, and
    QKV + RoPE with k / v landing in the KV cache slot."""
    ops = _ops()
    E, I, Tmax, t0, eps = 512, 1280, 24, 5, 1e-6
    x = rnd(M, E, seed=300)
    # RES: o_proj-like, in place on the residual stream, statistics out
    wo, res = rnd(E, E, scale=E ** -0.5, seed=301), rnd(M, E, seed=302)
    ss = torch.empty((M, E // 32), device=DEV, dtype=torch.float32)
    stream = res.clone()
    ops.linear_thin_fused(x, wo, ops.THIN_RES, residual=stream, out=stream, sumsq_out=ss)
    ref = x.float() @ wo.float().t() + res.float()
    assert rel_err(stream, ref) < 4e-3
    assert rel_err(ss.sum(1), stream.float().pow(2).sum(1)) < 1e-5
    # SWIGLU with the row scale derived from those statistics (RMSNorm of `stream`)
    wgu = rnd(2 * I, E, scale=E ** -0.5, seed=303)
    g = ops.linear_thin_fused(stream, wgu, ops.THIN_SWIGLU, rms_from=(ss, eps))
    rstd = torch.rsqrt(stream.float().pow(2).mean(1, keepdim=True) + eps)
    y = ((stream.float() * rstd) @ wgu.float().t()).view(M, I // 32, 2, 32)
    ref_g = (torch.nn.functional.silu(y[:, :, 0]) * y[:, :, 1]).reshape(M, I)
    assert rel_err(g, ref_g) < 5e-3
    # QKV: RoPE at device-side position, q -> out[:, :E], k / v -> cache slot
    wqkv = rnd(3 * E, E, scale=E ** -0.5, seed=304)
    rs = torch.rand(M, device=DEV) + 0.5
    cos, sin = torch.rand(Tmax, 64, device=DEV), torch.rand(Tmax, 64, device=DEV)
    cache = torch.zeros((M, Tmax, 2, E), device=DEV, dtype=torch.bfloat16)
    pos = torch.tensor([t0], device=DEV, dtype=torch.int32)
    out = ops.linear_thin_fused(x, wqkv, ops.THIN_QKV, row_scale=rs, rope=(cos, sin, pos), cache=cache, t0_dev=pos)
    y = ((x.float() * rs[:, None]) @ wqkv.float().t()).view(M, 3, E // 128, 128)
    c = torch.cat([cos[t0], cos[t0]])[None, None, :]
    s_ = torch.cat([sin[t0], sin[t0]])[None, None, :]
    rot = lambda t: t * c + torch.cat([-t[..., 64:], t[..., :64]], -1) * s_  # noqa: E731
    assert rel_err(out[:, :E], rot(y[:, 0]).reshape(M, E)) < 4e-3
    assert rel_err(cache[:, t0, 0], rot(y[:, 1]).reshape(M, E)) < 4e-3
    assert rel_err(cache[:, t0, 1], y[:, 2].reshape(M, E)) < 4e-3
    assert float(cache[:, :t0].abs().sum()) == 0 and float(cache[:, t0 + 1:].abs().sum()) == 0
    # host-side slot / table offset instead of the device scalars (eager decode path)
    cache2 = torch.zeros_like(cache)
    out2 = ops.linear_thin_fused(x, wqkv, ops.THIN_QKV, row_scale=rs, rope=(cos[t0:], sin[t0:], None), cache=cache2, t0=t0)
    assert torch.equal(out2[:, :E], out[:, :E]) and torch.equal(cache2, cache)


def test_rms_statistics_carried_by_gemm_epilogues_match_rms_rstd():
    """The GEMM that writes the residual stream leaves per-(row, 32-column) sums of squares of the STORED values; the
    consuming GEMM derives the RMSNorm row scale from them (no separate pass).  Must equal the rms_rstd kernel's result.
    The two row scales agree to a few fp32 ulps, not bit for bit (different summation orders), so the outputs are
    compared in fp32, where such a difference is visible and a wrong statistic is far outside 1e-5; a 16-bit output
    may sit at a rounding tie and move by one ulp, which is all the 16-bit comparison allows."""
    ops = _ops()
    M, E, N2 = 300, 512, 384
    h, wo, res = rnd(M, 256, seed=70), rnd(E, 256, scale=1 / 16, seed=71), rnd(M, E, seed=72)
    ss = torch.empty(M, E // 32, device=DEV, dtype=torch.float32)
    x = ops.linear(h, wo, residual=res, sumsq_out=ss)                       # new residual stream + its statistics
    assert rel_err(ss.sum(-1), x.float().pow(2).sum(-1)) < 1e-6             # of the values as stored (bf16-rounded)
    w2 = rnd(N2, E, scale=E ** -0.5, seed=73)
    y_fused = ops.linear(x, w2, rms_from=(ss, 1e-6))
    y_two = ops.linear(x, w2, row_scale=ops.rms_rstd(x, 1e-6))
    assert rel_err(y_fused, y_two) < 1e-5
    ref = (x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-6)) @ w2.float().t()
    assert rel_err(y_fused, ref) < 4e-3
    # SwiGLU and RoPE epilogues take the same statistics
    wg = rnd(2 * 256, E, scale=E ** -0.5, seed=74)
    rstd = ops.rms_rstd(x, 1e-6)
    f32 = torch.float32
    assert rel_err(ops.linear(x, wg, epi=ops.EPI_SWIGLU, rms_from=(ss, 1e-6), out_dtype=f32),
                   ops.linear(x, wg, epi=ops.EPI_SWIGLU, row_scale=rstd, out_dtype=f32)) < 1e-5
    a = ops.linear(x, wg, epi=ops.EPI_SWIGLU, rms_from=(ss, 1e-6)).float()
    b = ops.linear(x, wg, epi=ops.EPI_SWIGLU, row_scale=rstd).float()
    ulp = torch.ldexp(torch.ones_like(a), torch.frexp(torch.maximum(a.abs(), b.abs()))[1] - 8)  # bf16 ulp
    assert bool(((a - b).abs() <= ulp).all())


def test_rope_rows():
    ops = _ops()
    B, E = 8, 512
    x = rnd(B, 3 * E, seed=94)
    T = 40
    inv = 1.0 / (10000 ** (torch.arange(0, 128, 2, device=DEV).float() / 128))
    ang = torch.arange(T, device=DEV).float()[:, None] * inv[None, :]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    pos = torch.tensor([17], device=DEV, dtype=torch.int32)
    y = x.clone()
    ops.rope_rows(y, 2 * E, cos, sin, 1, pos)
    xf = x.float().view(B, 3, E // 128, 128)
    c = torch.cat([cos[17], cos[17]])[None, None, None, :]
    s_ = torch.cat([sin[17], sin[17]])[None, None, None, :]
    rot = torch.cat([-xf[..., 64:], xf[..., :64]], -1)
    ref = xf.clone()
    ref[:, :2] = (xf * c + rot * s_)[:, :2]
    assert rel_err(y, ref.view(B, 3 * E)) < 3e-3


# ------------------------------------------------------------------------------------------------ fp16 activation chain
def test_gemm_fp16_operands():
    """wgmma .f16 with fp16 A and B operands and fp16 output: the alignment chain's format.  One fp16 rounding is
    ~1.4e-4 norm-wise (bf16: ~1.1e-3).  Mixed f16 x bf16 is rejected up front: wgmma takes one input type for both
    operands."""
    ops = _ops()
    M, N, K = 200, 768, 1096
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(M, K, generator=g)).to(DEV).to(torch.float16)
    w = rnd(N, K, scale=K ** -0.5, seed=6).to(torch.float16)
    b = rnd(N, seed=7)
    y = ops.linear(x, w, b, out_dtype=torch.float16)
    ref = x.float() @ w.float().t() + b.float()
    assert y.dtype == torch.float16 and rel_err(y, ref) < 4e-4
    y32 = ops.linear(x, w, b, out_fp32=True)
    assert rel_err(y32, ref) < 2e-5
    with pytest.raises(RuntimeError, match="share one 16-bit format"):
        ops.linear(x, w.to(torch.bfloat16), b)
    src = rnd(33, 64, seed=8)
    c = ops.cast_f16(src)
    assert c.dtype == torch.float16 and torch.equal(c, src.to(torch.float16))
    big = src.float().abs() >= 2.0 ** -14  # fp16's normal range: the conversion is exact there
    assert torch.equal(c.float()[big], src.float()[big])


def test_gemm_row_scaled_bias_terms():
    """out = A B^T + rs1[m] * bias[n] + rs2[m] * bias2[n] per batch (value-side bias terms of the absorbed alignment)."""
    ops = _ops()
    Hh, nq, hd, E = 4, 37, 64, 256
    g = torch.Generator().manual_seed(8)
    a = torch.randn(Hh, nq, E, generator=g).to(DEV).to(torch.float16)
    w = rnd(Hh * hd, E, scale=E ** -0.5, seed=9).to(torch.float16)
    b1, b2 = rnd(Hh * hd, seed=10), rnd(Hh * hd, seed=11)
    r1 = torch.rand(Hh * nq, generator=g).to(DEV)
    r2 = torch.rand(Hh * nq, generator=g).to(DEV)
    out = torch.empty(nq, Hh * hd, device=DEV, dtype=torch.float16)
    ops.gemm_raw(M=nq, N=hd, K=E, batch=Hh, A=a.data_ptr(), lda=E, a_bs=nq * E, B=w.data_ptr(), ldb=E, b_bs=hd * E,
                 Cout=out.data_ptr(), ldc=Hh * hd, c_bs=hd, a_fp16=True, b_fp16=True, c_fp16=True, bias=b1.data_ptr(),
                 bias_bs=hd,
                 bias_rs=r1.data_ptr(), bias2=b2.data_ptr(), bias2_rs=r2.data_ptr())
    ref = torch.empty(nq, Hh * hd, device=DEV)
    for h in range(Hh):
        sl = slice(h * hd, (h + 1) * hd)
        ref[:, sl] = (a[h].float() @ w[sl].float().t() + r1[h * nq:(h + 1) * nq, None] * b1[sl].float()
                      + r2[h * nq:(h + 1) * nq, None] * b2[sl].float())
    assert rel_err(out, ref) < 4e-4


def _align_ref(qt, table, stats):
    V = table.shape[0]
    s = qt.double() @ table.double().t() + stats[:, :1].double()
    full = torch.cat([s, stats[:, 1:2].double(), torch.zeros_like(stats[:, :1]).double()], dim=1)
    p = torch.softmax(full, dim=-1)
    return (p[:, :V] @ table.double()).float(), p[:, :V].sum(-1).float(), p[:, V].float()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize(
    "R,V,E,qs,kind",
    [
        (37, 32000, 4096, 1.0, "real width, ragged rows"),
        (300, 519, 256, 1.0, "odd vocab (resized table), several row blocks"),
        (384, 1000, 512, 1.0, "vocab not a multiple of the 256-key tile"),
        (130, 2048, 256, 40.0, "scores far above the synthetic keys: overflow flag -> exact-max second attempt"),
        (64, 2048, 256, -1.0, "real keys far BELOW the zero key (all mass on the synthetic keys)"),
    ],
)
def test_align_fused(R, V, E, qs, kind, mode):
    """mm_align_fwd (one persistent kernel: scores + fp16 probabilities, then P . table) vs an fp64 softmax over the
    V + 2 keys.  fp16 P' and fp16 output: ~2e-4 norm-wise each."""
    ops = _ops()
    g = torch.Generator().manual_seed(R + V)
    table = (torch.randn(V, E, generator=g) * 0.5).to(DEV).to(torch.bfloat16).to(torch.float16)
    qt = (torch.randn(R, E, generator=g) * (abs(qs) * 2.0 / math.sqrt(E))).to(DEV).to(torch.float16)
    stats = torch.randn(R, 2, generator=g).to(DEV)
    if qs < 0:  # push every real score ~60 nats below zero
        stats[:, 0] = -60.0
    out, psum, pext = ops.align_fused(table, qt, stats.contiguous(), mode=mode)
    torch.cuda.synchronize()
    ref, rsum, rext = _align_ref(qt, table, stats)
    e = (rel_err(out, ref) if qs > 0 else float((out.float() - ref).abs().max()), rel_err(psum, rsum) if qs > 0 else float((psum - rsum).abs().max()),
         rel_err(pext, rext))
    print(f"\n[align_fused mode {mode}] {kind}: ctx~ {e[0]:.2e}  p_sum_real {e[1]:.2e}  p_extra {e[2]:.2e}")
    assert e[0] < 6e-4 and e[1] < 2e-4 and e[2] < 2e-4
