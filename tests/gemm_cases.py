"""The table of fp64 GEMM cases (tests/test_gemm_fp64_gpu.py) and the kernel instance each one must launch.

Every case is one mm_gemm_fwd launch: shape, layout, format, modes (mm_gemm_overlap_mode 0 / 1 / 2,
mm_gemm_streamk_mode 0 / 2) and epilogue options.  raw_args() turns a case into the exact gemm_raw() arguments its
wrapper issues, from base addresses that are real on the GPU and fake (with the same alignment) on the CPU, and
instance() names the kernel template that the dispatcher's plan for those arguments launches:
  ("tile", BN, EPI, B_MN, A_MN, F16, EWG)  gemm_bf16_kernel<BN, EPI, B_MN, A_MN, F16, EWG>
  ("wide", EPI, F16)                       gemm_wide_kernel<EPI, F16>
Shapes were chosen so that the table reaches every instance with 132 SMs (an H100 SXM) and with 114 (an H100 PCIe).
"""
from __future__ import annotations

from dataclasses import dataclass

from macaw_llm_b200 import ops

E, I = 4096, 11008
F16, BF16 = "fp16", "bf16"


@dataclass(frozen=True)
class Case:
    name: str
    kind: str                 # linear | thin | dx | dw | batched | align
    M: int                    # rows of x (linear / thin), of dy (dx / dw); per batch entry for batched / align
    N: int                    # output features (linear / thin), columns of dy (dx / dw)
    K: int                    # input features (linear / thin), columns of w (dx) / x (dw)
    fmt: str = BF16
    overlap: int = 0
    streamk: int = 0          # 0 off, 2: stream-K tail whenever the schedule allows (a workspace is passed)
    out: str = "act"          # act (the operand format) | fp32
    epi: int = ops.EPI_STD
    act: int = ops.ACT_NONE
    bias: bool = False
    residual: bool = False
    res_row_mod: int = 0
    alpha: float = 1.0
    row_scale: bool = False
    rms: bool = False         # rs_sumsq: the RMSNorm row scale from partial sums of squares
    sumsq: bool = False       # sumsq_out
    ldc_pad: int = 0          # output view of a (M, n_out + ldc_pad + c_off) buffer
    c_off: int = 0            # element offsets of C / bias / residual from a 16-byte aligned base
    bias_off: int = 0
    res_off: int = 0
    rope_cols: int = 0
    rope_T: int = 0
    rope_pos: int = 0         # device-side position offset (0: none)
    gate_std: float = 1.0     # standard deviation of the pre-activations (SiLU / SwiGLU gates)
    tiny: bool = False        # outputs in fp16's subnormal range
    cancel: bool = False      # residual of the product's scale and opposite sign
    batch: int = 1
    batch2: int = 1

    @property
    def n_out(self):
        return self.N // 2 if self.epi == ops.EPI_SWIGLU else self.N

    @property
    def ldc(self):
        return self.n_out + self.ldc_pad + self.c_off


def _cases():
    c = []
    for fmt in (BF16, F16):
        # ---- K-major operands, standard epilogue: BN 32 / 64 / 128 in modes 0 and 1, tile pairs in mode 2
        for ov in (0, 1):
            c.append(Case(f"ragged_bias_gelu_{fmt}_m{ov}", "linear", 300, 1000, 2120, fmt, ov, bias=True,
                          act=ops.ACT_GELU))                                    # BN 32, partial last chunk (vector)
            c.append(Case(f"bias_silu_res_{fmt}_m{ov}", "linear", 300, 2048, 2112, fmt, ov, bias=True,
                          act=ops.ACT_SILU, residual=True, gate_std=4.0))       # BN 64, gates to about +-12
            c.append(Case(f"lm_head_{fmt}_m{ov}", "linear", 384, 32007, E, fmt, ov, out="fp32"))  # BN 128, scalar
            c.append(Case(f"dx_{fmt}_m{ov}", "dx", 300, 2112, 2048, fmt, ov))   # MN-major B, BN 64
            c.append(Case(f"dx_acc_{fmt}_m{ov}", "dx", 300, 2112, 4096, fmt, ov, residual=True))  # BN 128
            c.append(Case(f"dw_{fmt}_m{ov}", "dw", 2112, 304, 2048, fmt, ov))   # MN-major A and B, BN 64
            c.append(Case(f"dw_acc_{fmt}_m{ov}", "dw", 2112, 304, 4096, fmt, ov, residual=True))  # BN 128
        for ov in (0, 1, 2):
            c.append(Case(f"qkv_rope_{fmt}_m{ov}", "linear", 300, 3 * E, E, fmt, ov, epi=ops.EPI_ROPE,
                          rope_cols=2 * E, rope_T=100, rope_pos=37, rms=True))  # decoder width
            c.append(Case(f"gate_up_swiglu_{fmt}_m{ov}", "linear", 300, 2 * I, E, fmt, ov, epi=ops.EPI_SWIGLU,
                          rms=True, gate_std=4.0))                              # decoder width
        c.append(Case(f"o_proj_res_sumsq_{fmt}_m2", "linear", 2560, E, E, fmt, 2, residual=True, sumsq=True,
                      cancel=True))                                             # tile pairs, standard epilogue
        # ---- stream-K tails (consumer epilogue) with each epilogue and with MN-major operands
        c.append(Case(f"sk_fp32_{fmt}", "linear", 2112, E, 1024, fmt, 2, streamk=2, out="fp32", row_scale=True,
                      alpha=0.37))
        c.append(Case(f"sk_rope_{fmt}", "linear", 300, 3 * E, E, fmt, 1, streamk=2, epi=ops.EPI_ROPE,
                      rope_cols=2 * E, rope_T=300))
        c.append(Case(f"sk_swiglu_{fmt}", "linear", 300, 2 * I, E, fmt, 1, streamk=2, epi=ops.EPI_SWIGLU, rms=True,
                      gate_std=4.0))
        c.append(Case(f"sk_dx_{fmt}", "dx", 2112, 1024, E, fmt, 1, streamk=2))
        # ---- the scalar (non-vectorised) epilogue: odd ldc, C / bias / residual one element off 16 bytes
        c.append(Case(f"odd_ldc_bias_qgelu_res_{fmt}", "linear", 300, 1000, 2120, fmt, 1, bias=True,
                      act=ops.ACT_QUICK_GELU, residual=True, ldc_pad=1, gate_std=4.0))
        c.append(Case(f"c_off_bias_off_{fmt}", "linear", 300, 1000, 1000, fmt, 0, bias=True, c_off=1, ldc_pad=1,
                      bias_off=1))
        c.append(Case(f"res_off_mod_{fmt}", "linear", 300, 2048, 2112, fmt, 0, residual=True, res_off=1,
                      res_row_mod=77, cancel=True))
        c.append(Case(f"sk_scalar_bias_res_{fmt}", "linear", 2112, E, 1024, fmt, 0, streamk=2, bias=True,
                      residual=True, bias_off=1, res_off=1))
        # ---- decode (c_trans) at M = 1, 8, 64
        for m in (1, 8, 64):
            c.append(Case(f"thin_m{m}_{fmt}", "thin", m, E, E, fmt, 1 if m != 8 else 0, bias=True, act=ops.ACT_SILU,
                          residual=True, row_scale=True, gate_std=4.0))
        # ---- 4-D batching: shared B, per-batch bias, residual strides
        c.append(Case(f"batched_{fmt}", "batched", 136, 200, 520, fmt, 0, bias=True, residual=True, batch=3, batch2=2))
    # fp16 outputs in the subnormal range, bf16 residual cancellation at short K, row scale + alpha
    c.append(Case("tiny_fp16", "linear", 300, 1000, 2120, F16, 1, alpha=2.0 ** -16, tiny=True))
    c.append(Case("row_scale_alpha_bf16", "linear", 300, 2048, 2112, BF16, 1, row_scale=True, alpha=0.37))
    # the alignment's value projection: per-head batches, interleaved head columns, row-scaled bias pair (fp16)
    c.append(Case("align_bias_pair_fp16", "align", 250, 256, E, F16, 0, batch=16))
    # accumulation at the table's largest K, fp32 out (calibrates KAPPA)
    for fmt in (BF16, F16):
        c.append(Case(f"down_fp32_{fmt}", "linear", 300, E, I, fmt, 0, out="fp32"))
    return c


CASES = _cases()


def raw_args(c: Case, p: dict) -> dict:
    """The gemm_raw() keyword arguments of case `c`'s launch, as its wrapper (ops.linear, linear_thin, gemm_dx,
    gemm_dw) or the engine's raw call issues them.  `p` holds the base addresses: x, w, out, bias, res, rs, ss, ssq,
    cos, sin, pos, ws, bias2, brs, b2rs (offsets of the case are added here)."""
    f16 = c.fmt == F16
    osz = 4 if c.out == "fp32" else 2
    kw = dict(a_fp16=f16, b_fp16=f16, c_fp32=c.out == "fp32", c_fp16=f16 and c.out != "fp32")
    if c.streamk:
        kw.update(streamk=(p["ws"], p["ws_bytes"]))
    if c.kind == "linear":
        kw.update(M=c.M, N=c.N, K=c.K, A=p["x"], lda=c.K, B=p["w"], ldb=c.K, Cout=p["out"] + c.c_off * osz, ldc=c.ldc,
                  epi=c.epi, act=c.act, alpha=c.alpha)
        if c.bias:
            kw.update(bias=p["bias"] + 2 * c.bias_off)
        if c.row_scale:
            kw.update(row_scale=p["rs"])
        if c.residual:
            kw.update(residual=p["res"] + 2 * c.res_off, ldr=c.n_out + 2 * c.res_off, res_row_mod=c.res_row_mod)
        if c.rms:
            kw.update(rs_sumsq=p["ssq"], rs_parts=32, rs_eps=1e-6)
        if c.sumsq:
            kw.update(sumsq_out=p["ss"])
        if c.epi == ops.EPI_ROPE:
            kw.update(rope_cos=p["cos"], rope_sin=p["sin"], rope_T=c.rope_T, rope_cols=c.rope_cols,
                      rope_pos=p["pos"] if c.rope_pos else None)
    elif c.kind == "thin":
        kw.update(M=c.N, N=c.M, K=c.K, A=p["w"], lda=c.K, B=p["x"], ldb=c.K, Cout=p["out"], ldc=c.N, act=c.act,
                  bias=p["bias"], row_scale=p["rs"], residual=p["res"], ldr=c.N, c_trans=True)
    elif c.kind == "dx":  # dx (M, K) = dy (M, N) @ w (N, K)
        kw.update(M=c.M, N=c.K, K=c.N, A=p["x"], lda=c.N, B=p["w"], ldb=c.K, b_mn_major=True, Cout=p["out"], ldc=c.K)
        if c.residual:
            kw.update(residual=p["out"], ldr=c.K)
    elif c.kind == "dw":  # dw (N, K) (+)= dy (M, N)^T @ x (M, K)
        kw.update(M=c.N, N=c.K, K=c.M, A=p["x"], lda=c.N, a_mn_major=True, B=p["w"], ldb=c.K, b_mn_major=True,
                  Cout=p["out"], ldc=c.K)
        if c.residual:
            kw.update(residual=p["out"], ldr=c.K)
    elif c.kind == "batched":  # A (b2, b, M, K), shared B (N, K), C (b2, b, M, N), bias (b, N), residual (b2, b, M, N)
        bl = c.batch
        kw.update(M=c.M, N=c.N, K=c.K, batch=bl, batch2=c.batch2, A=p["x"], lda=c.K, a_bs=c.M * c.K,
                  a_bs2=bl * c.M * c.K, B=p["w"], ldb=c.K, b_bs=0, b_bs2=0, Cout=p["out"], ldc=c.N, c_bs=c.M * c.N,
                  c_bs2=bl * c.M * c.N, bias=p["bias"], bias_bs=c.N, residual=p["res"], ldr=c.N, r_bs=c.M * c.N,
                  r_bs2=bl * c.M * c.N)
    elif c.kind == "align":  # Engine.align's value projection: heads as batch, head columns interleaved in ctx rows
        H, hd = c.batch, c.N
        kw.update(M=c.M, N=hd, K=c.K, batch=H, A=p["x"], lda=c.K, a_bs=c.M * c.K, B=p["w"], ldb=c.K, b_bs=hd * c.K,
                  Cout=p["out"], ldc=H * hd, c_bs=hd, bias=p["bias"], bias_bs=hd, bias_rs=p["brs"], bias2=p["bias2"],
                  bias2_rs=p["b2rs"])
    else:
        raise ValueError(c.kind)
    return kw


def fake_ptrs() -> dict:
    """16-byte aligned, distinct fake addresses: mm_gemm_plan checks pointers for null and alignment only."""
    keys = ("x", "w", "out", "bias", "res", "rs", "ss", "ssq", "cos", "sin", "pos", "ws", "bias2", "brs", "b2rs")
    d = {k: (1 << 24) * (i + 1) for i, k in enumerate(keys)}
    d["ws_bytes"] = 1 << 30
    return d


def plan(c: Case, p: dict) -> dict:
    """The dispatcher's plan for case `c` under its modes (restored afterwards)."""
    from macaw_llm_b200 import _lib

    lib = _lib.load()
    prev_o, prev_s = lib.mm_gemm_overlap_mode(c.overlap), lib.mm_gemm_streamk_mode(c.streamk)
    try:
        return ops.gemm_raw(plan_only=True, **raw_args(c, p))
    finally:
        lib.mm_gemm_overlap_mode(prev_o)
        lib.mm_gemm_streamk_mode(prev_s)


def instance(c: Case, pl: dict) -> tuple:
    """The kernel template of plan `pl` for case `c`."""
    f16 = c.fmt == F16
    if pl["kernel"] == ops.GEMM_TILE_PAIRS:
        return ("wide", c.epi, f16)
    a_mn = c.kind == "dw"
    b_mn = c.kind in ("dx", "dw")
    return ("tile", pl["block_n"], c.epi, b_mn, a_mn, f16, pl["kernel"] == ops.GEMM_EPILOGUE_WARPGROUP)


def all_instances() -> set:
    """The 42 kernel instances mm_gemm_fwd can launch (the dispatch in gemm_wgmma.cu)."""
    out = set()
    for f16 in (False, True):
        for ewg in (False, True):
            for bn in (32, 64, 128):
                out.add(("tile", bn, ops.EPI_STD, False, False, f16, ewg))
            for bn in (64, 128):
                out.add(("tile", bn, ops.EPI_STD, True, False, f16, ewg))
                out.add(("tile", bn, ops.EPI_STD, True, True, f16, ewg))
            out.add(("tile", 128, ops.EPI_SWIGLU, False, False, f16, ewg))
            out.add(("tile", 128, ops.EPI_ROPE, False, False, f16, ewg))
        for epi in (ops.EPI_STD, ops.EPI_SWIGLU, ops.EPI_ROPE):
            out.add(("wide", epi, f16))
    return out
