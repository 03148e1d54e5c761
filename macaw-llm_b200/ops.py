"""torch-tensor front end of the C ABI (include/macaw_b200.h).

torch is used only for device memory and streams; every function here launches kernels from libmacaw_b200.so on
torch's current CUDA stream and raises if an operand is not a CUDA tensor (there is no CPU or eager fallback).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import AlignArgs, AttnArgs, GemmArgs

ACT_NONE, ACT_GELU, ACT_QUICK_GELU, ACT_SILU = 0, 1, 2, 3
EPI_STD, EPI_SWIGLU, EPI_ROPE = 0, 1, 2
GEMM_CONSUMER_EPILOGUE, GEMM_EPILOGUE_WARPGROUP, GEMM_TILE_PAIRS = 0, 1, 2  # gemm_plan()["kernel"]: MM_GEMM_KERNEL_*

_BF16 = torch.bfloat16
_F16 = torch.float16
_ACT_DTYPE = torch.bfloat16


def ACT():
    """16-bit storage dtype of activations / parameters of the model being run (see set_act_format)."""
    return _ACT_DTYPE


def set_act_format(dtype) -> None:
    """Select the activation format (torch.bfloat16 | torch.float16) for this thread: the Python-side dtype checks and
    the kernel library's thread-local format (mm_set_act_format) move together."""
    global _ACT_DTYPE
    if dtype not in _16BIT:
        raise TypeError(f"macaw_b200: activation format must be bf16 or fp16, got {dtype}")
    if dtype != _ACT_DTYPE or int(_lib.load().mm_get_act_format()) != int(dtype == _F16):
        _lib.load().mm_set_act_format(int(dtype == _F16))
        _ACT_DTYPE = dtype
_16BIT = (torch.bfloat16, torch.float16)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {_lib.last_error()}")


def _cuda(t: torch.Tensor, dtype=None, name: str = "tensor") -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"macaw_b200: {name} must be a CUDA tensor (no CPU fallback exists)")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"macaw_b200: {name} must be {dtype}, got {t.dtype}")
    if t.device.index != torch.cuda.current_device():
        # kernels are launched on the CURRENT device's stream: a tensor of another GPU would be used with the wrong stream
        raise RuntimeError(f"macaw_b200: {name} lives on {t.device} but the current CUDA device is "
                           f"cuda:{torch.cuda.current_device()}; wrap the call in torch.cuda.device(...)")
    return t


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# Optional per-launch CUDA-event profiling of the GEMM kernel (bench.py's live roofline): when PROFILE is a list, every
# mm_gemm_fwd launch appends (TAG, flops, start_event, end_event) recorded on the launching stream.
PROFILE = None
TAG = "gemm"


def launch_count() -> int:
    return int(_lib.load().mm_launch_count())


def launch_count_reset() -> None:
    _lib.load().mm_launch_count_reset()


# ---------------------------------------------------------------------------------------------------- GEMM
def gemm_raw(*, M, N, K, A, lda, B, ldb, Cout, ldc, batch=1, a_bs=0, b_bs=0, c_bs=0, batch2=1, a_bs2=0, b_bs2=0,
             c_bs2=0, b_mn_major=False, c_fp32=False, epi=EPI_STD, act=ACT_NONE, alpha=1.0, bias=None, bias_bs=0,
             row_scale=None, residual=None, ldr=0, r_bs=0, r_bs2=0, res_row_mod=0, rope_cos=None, rope_sin=None,
             rope_T=0, rope_cols=0, rope_pos=None, c_trans=False, a_fp16=None, b_fp16=None, c_fp16=None,
             bias_rs=None, bias2=None, bias2_rs=None, a_mn_major=False, sumsq_out=None, rs_sumsq=None, rs_parts=0,
             rs_eps=0.0, streamk=None, plan_only: bool = False, e4m3: Optional[_lib.GemmE4m3Args] = None):
    """Direct binding of mm_gemm_fwd; pointers are ints (data_ptr() + byte offsets).  Operand / output formats default to
    the current activation format (ACT()): fp16 for an fp16 model, bf16 otherwise.  `streamk` is a workspace tensor, or
    (address, bytes).  plan_only=True launches nothing and returns the gemm_plan() dict of exactly these arguments
    (mm_gemm_plan: no memory is touched, so the pointers may be fake); while PLANS is a list, every launch appends its own.
    With `e4m3` (mm_gemm_e4m3_args) the call goes to mm_gemm_e4m3_fwd / mm_gemm_e4m3_plan instead: A is the e4m3
    activation, B is ignored (the weight is e4m3.w)."""
    f16 = ACT() == _F16
    a_fp16 = f16 if a_fp16 is None else a_fp16
    b_fp16 = f16 if b_fp16 is None else b_fp16
    c_fp16 = (f16 and not c_fp32) if c_fp16 is None else c_fp16
    if isinstance(streamk, torch.Tensor):
        streamk = (streamk.data_ptr(), streamk.numel() * streamk.element_size())
    a = GemmArgs(M, N, K, batch, batch2, A, lda, a_bs, a_bs2, B, ldb, b_bs, b_bs2, int(b_mn_major), Cout, ldc, c_bs,
                 c_bs2, int(c_fp32), epi, act, float(alpha), bias, bias_bs, row_scale, residual, ldr, r_bs, r_bs2,
                 res_row_mod, rope_cos, rope_sin, rope_T, rope_cols, rope_pos, int(c_trans), int(a_fp16), int(b_fp16), int(c_fp16),
                 bias_rs, bias2, bias2_rs, int(a_mn_major), sumsq_out, rs_sumsq, int(rs_parts), float(rs_eps),
                 None if streamk is None else streamk[0], 0 if streamk is None else streamk[1])
    if plan_only or PLANS is not None:
        plan = _plan_of(a, e4m3)
        if plan_only:
            return plan
        PLANS.append(plan)
    if e4m3 is None:
        fwd, args, what = _lib.load().mm_gemm_fwd, (C.byref(a),), "mm_gemm_fwd"
    else:
        fwd, args, what = _lib.load().mm_gemm_e4m3_fwd, (C.byref(a), C.byref(e4m3)), "mm_gemm_e4m3_fwd"
    if PROFILE is None:
        _check(fwd(*args, _stream()), what)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _check(fwd(*args, _stream()), what)
    e1.record()
    PROFILE.append((TAG, 2.0 * M * N * K * batch * max(1, batch2), e0, e1))


def gemm_plan(*, M: int, N: int, K: int, batch: int = 1, batch2: int = 1, epi: int = EPI_STD, b_mn_major: bool = False,
              a_mn_major: bool = False, c_fp32: bool = False, c_trans: bool = False, fp16: bool = False,
              streamk: bool = False) -> dict:
    """The schedule mm_gemm_fwd would pick for a dense, 16-byte-aligned GEMM of this shape (mm_gemm_plan: the host-side
    dispatch run without touching memory or launching — works without a GPU, where the library assumes the 132 SMs of an H100 SXM).
    `streamk=True` hands the dispatcher a stream-K workspace, as the LLaMA stack does."""
    lib = _lib.load()
    fake = 1 << 20  # operand addresses are only checked for null / alignment
    lda = M if a_mn_major else K
    ldb = N if b_mn_major else K
    n_out = N // 2 if epi == EPI_SWIGLU else N
    ldc = M if c_trans else n_out
    ws = int(lib.mm_gemm_streamk_workspace_bytes()) if streamk else 0
    rope = dict(rope_cos=fake, rope_sin=fake, rope_T=max(1, M), rope_cols=(N // 128) * 128) if epi == EPI_ROPE else {}
    kw = dict(M=M, N=N, K=K, batch=batch, batch2=batch2, A=fake, lda=lda, a_bs=M * K, a_bs2=M * K * batch, B=fake, ldb=ldb,
              b_bs=N * K, b_bs2=N * K * batch, b_mn_major=int(b_mn_major), C=fake, ldc=ldc, c_bs=M * n_out,
              c_bs2=M * n_out * batch, c_fp32=int(c_fp32), epi=epi, act=ACT_NONE, alpha=1.0, c_trans=int(c_trans),
              a_fp16=int(fp16), b_fp16=int(fp16), c_fp16=int(fp16 and not c_fp32), a_mn_major=int(a_mn_major),
              sk_workspace=fake if streamk else None, sk_workspace_bytes=ws, **rope)
    return _plan_of(GemmArgs(**kw))


# While a list, gemm_raw appends the gemm_plan() dict of every launch's own arguments (what the dispatcher decided).
PLANS = None


def _plan_of(a: GemmArgs, e4m3=None) -> dict:
    plan = _lib.GemmPlan()
    if e4m3 is None:
        _check(_lib.load().mm_gemm_plan(C.byref(a), C.byref(plan)), "mm_gemm_plan")
    else:
        _check(_lib.load().mm_gemm_e4m3_plan(C.byref(a), C.byref(e4m3), C.byref(plan)), "mm_gemm_e4m3_plan")
    d = {name: int(getattr(plan, name)) for name, _ in _lib.GemmPlan._fields_}
    d["fill"] = d["units"] / float(d["waves"] * d["workers"])  # share of the scheduled tile slots that carry work
    return d


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: int = ACT_NONE,
           residual: Optional[torch.Tensor] = None, res_row_mod: int = 0, out: Optional[torch.Tensor] = None,
           out_fp32: bool = False, alpha: float = 1.0, row_scale: Optional[torch.Tensor] = None, epi: int = EPI_STD,
           rope=None, out_dtype=None, sumsq_out: Optional[torch.Tensor] = None, rms_from=None) -> torch.Tensor:
    """out = epilogue(alpha * x @ w.T): x (M, K) bf16 or fp16 with unit inner stride, w (N, K) bf16 or fp16 (an nn.Linear
    weight); out bf16 (default), fp16 or fp32 (`out_dtype` / the dtype of `out`)."""
    _cuda(x, None, "x"); _cuda(w, None, "w")
    assert x.dtype in _16BIT and w.dtype in _16BIT, (x.dtype, w.dtype)
    assert x.dim() == 2 and w.dim() == 2 and x.shape[1] == w.shape[1], (x.shape, w.shape)
    assert x.stride(1) == 1 and w.stride(1) == 1
    M, K = x.shape
    N = w.shape[0]
    n_out = N // 2 if epi == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), device=x.device,
                          dtype=out_dtype if out_dtype is not None else (torch.float32 if out_fp32 else ACT()))
    assert out.shape[0] == M and out.shape[1] == n_out and out.stride(1) == 1
    kw = {}
    if residual is not None:
        _cuda(residual, ACT(), "residual")
        assert residual.stride(-1) == 1
        kw.update(residual=residual.data_ptr(), ldr=residual.stride(0), res_row_mod=res_row_mod)
    if rope is not None:
        cos, sin, T, cols = rope[:4]
        kw.update(rope_cos=cos.data_ptr(), rope_sin=sin.data_ptr(), rope_T=T, rope_cols=cols)
        if len(rope) > 4 and rope[4] is not None:  # device-side position offset (int32 tensor)
            kw.update(rope_pos=rope[4].data_ptr())
    if sumsq_out is not None:  # (M, N/32) fp32: per-chunk sums of squares of the stored outputs (next RMSNorm's statistic)
        assert sumsq_out.dtype == torch.float32 and sumsq_out.is_contiguous() and sumsq_out.shape == (M, (N + 31) // 32)
        kw.update(sumsq_out=sumsq_out.data_ptr())
    if rms_from is not None:   # (partials (M, parts) fp32, eps): RMSNorm row scale derived in this GEMM's epilogue
        parts, eps = rms_from
        assert parts.dtype == torch.float32 and parts.is_contiguous() and parts.shape[0] == M and row_scale is None
        kw.update(rs_sumsq=parts.data_ptr(), rs_parts=parts.shape[1], rs_eps=eps)
    if STREAMK is not None and STREAMK.device == x.device:
        kw.update(streamk=STREAMK)
    gemm_raw(M=M, N=N, K=K, A=x.data_ptr(), lda=x.stride(0), B=w.data_ptr(), ldb=w.stride(0), Cout=out.data_ptr(),
             ldc=out.stride(0), c_fp32=out.dtype == torch.float32, c_fp16=out.dtype == _F16, a_fp16=x.dtype == _F16,
             b_fp16=w.dtype == _F16, epi=epi, act=act, alpha=alpha, bias=_ptr(bias), row_scale=_ptr(row_scale), **kw)
    return out


# Stream-K workspace handed to every `linear()` launch while set (see mm_gemm_args.sk_workspace).  The OWNER sets it
# around a section whose GEMMs run one after another on a single stream (the LLaMA stack) and clears it afterwards: two
# GEMMs sharing one workspace must never run concurrently.
STREAMK: Optional[torch.Tensor] = None


def streamk_workspace(device) -> torch.Tensor:
    """A zero-initialised stream-K workspace (flags + one fp32 accumulator slot per SM) on `device`."""
    _lib.load()
    with torch.cuda.device(device):
        n = int(_lib.load().mm_gemm_streamk_workspace_bytes())
    return torch.zeros((n + 15) // 16 * 4, device=device, dtype=torch.int32)


def linear_thin(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: int = ACT_NONE,
                residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                row_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(x @ w.T) for a THIN x (a few rows, e.g. one decode step): operands are swapped so the weight rows
    fill the 128-row MMA tile (weight-streaming regime) and the epilogue stores transposed.  Same semantics as `linear`
    with the standard epilogue: row_scale scales rows of x, bias is per output feature, residual/out are (M, N)."""
    _cuda(x, ACT(), "x"); _cuda(w, ACT(), "w")
    M, K = x.shape
    N = w.shape[0]
    assert x.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] == K
    if out is None:
        out = torch.empty((M, N), device=x.device, dtype=ACT())
    assert out.shape == (M, N) and out.stride(1) == 1
    kw = {}
    if residual is not None:
        assert residual.stride(1) == 1
        kw.update(residual=residual.data_ptr(), ldr=residual.stride(0))
    # swapped problem: M' = N (weight rows), N' = M (activation rows)
    if STREAMK is not None and STREAMK.device == x.device:
        kw.update(streamk=STREAMK)
    gemm_raw(M=N, N=M, K=K, A=w.data_ptr(), lda=w.stride(0), B=x.data_ptr(), ldb=x.stride(0), Cout=out.data_ptr(),
             ldc=out.stride(0), c_fp32=out.dtype == torch.float32, act=act, bias=_ptr(bias), row_scale=_ptr(row_scale),
             c_trans=True, **kw)
    return out


THIN_SPLITS = 4  # K slices of a thin (decode) GEMM: 32..172-tile grids become 128..688 units on 132 SMs


THIN_RES, THIN_SWIGLU, THIN_QKV = 0, 1, 2


def linear_thin_fused(x: torch.Tensor, w: torch.Tensor, mode: int, *, row_scale: Optional[torch.Tensor] = None,
                      rms_from=None, residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                      sumsq_out: Optional[torch.Tensor] = None, rope=None, cache: Optional[torch.Tensor] = None, t0: int = 0,
                      t0_dev: Optional[torch.Tensor] = None, splits: Optional[int] = None,
                      cache_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decode-step GEMM x (M <= 64, K) @ w (N, K)^T with K split over `splits` CTAs per weight tile (fp32 partials) and ONE
    fused tail kernel (mm_thin_fused):
      THIN_RES     out = rs * xW^T + residual (in place allowed); sumsq_out (M, N/32) fp32 receives the next RMSNorm's statistic
      THIN_SWIGLU  out (M, N/2) = silu(gate) * up of the [32 gate | 32 up]-interleaved fused weight
      THIN_QKV     N = 3E: RoPE on q / k (rope = (cos, sin, pos_dev | None)), q -> out (M, 3E) columns [0, E), k / v -> `cache`
                   (B, Tmax, 2, E) at slot t0 / *t0_dev; an int8 `cache` with `cache_scale` (B, 2, H, Tmax) fp32 receives
                   k / v by the int8 KV-cache rule (kv_append_i8)
    rs: `row_scale` (M,) fp32, or rms_from = (partials (M, parts) fp32, eps): rsqrt(mean(x^2) + eps) from a THIN_RES pass."""
    _cuda(x, ACT(), "x"); _cuda(w, ACT(), "w")
    M, K = x.shape
    N = w.shape[0]
    assert x.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] == K and M <= 64
    sk = None  # stream-K needs a full wave of tiles to hide its hand-over behind: a decode GEMM has 32..172 tiles
    S = THIN_SPLITS if splits is None else int(splits)
    if S < 1 or K % (S * 64) != 0:
        S = 1
    Kc = K // S
    Mp = (M + 3) // 4 * 4
    dev = x.device
    part = torch.empty((S, N, Mp), device=dev, dtype=torch.float32)
    # fixed split-K factor; the tail kernel adds the partial sums up
    gemm_raw(M=N, N=M, K=Kc, batch=S, A=w.data_ptr(), lda=w.stride(0), a_bs=Kc, B=x.data_ptr(), ldb=x.stride(0), b_bs=Kc,
             Cout=part.data_ptr(), ldc=Mp, c_bs=N * Mp, c_fp32=True, streamk=sk)
    return _thin_tail(part, M, K, mode, row_scale=row_scale, rms_from=rms_from, residual=residual, out=out,
                      sumsq_out=sumsq_out, rope=rope, cache=cache, t0=t0, t0_dev=t0_dev, cache_scale=cache_scale)


def _thin_tail(part: torch.Tensor, M: int, K: int, mode: int, *, row_scale=None, rms_from=None, residual=None, out=None,
               sumsq_out=None, rope=None, cache=None, t0: int = 0, t0_dev=None, cache_scale=None) -> torch.Tensor:
    """mm_thin_fused over the split-K partial sums part (S, N, Mp) of a thin GEMM with M rows and K columns."""
    S, N, Mp = part.shape
    dev = part.device
    n_out = N // 2 if mode == THIN_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), device=dev, dtype=ACT())
    assert out.shape == (M, n_out) and out.stride(1) == 1
    a = _lib.ThinArgs()
    a.part, a.splits, a.N, a.M, a.ldp, a.mode = part.data_ptr(), S, N, M, Mp, int(mode)
    a.row_scale = _ptr(row_scale)
    if rms_from is not None:
        parts, eps = rms_from
        assert row_scale is None and parts.dtype == torch.float32 and parts.is_contiguous() and parts.shape[0] == M
        a.rs_sumsq, a.rs_parts, a.rs_K, a.rs_eps = parts.data_ptr(), parts.shape[1], K, float(eps)
    if residual is not None:
        _cuda(residual, ACT(), "residual")
        assert mode == THIN_RES and residual.stride(1) == 1
        a.residual, a.ldr = residual.data_ptr(), residual.stride(0)
    a.out, a.ldo = out.data_ptr(), out.stride(0)
    if sumsq_out is not None:
        assert mode == THIN_RES and sumsq_out.dtype == torch.float32 and sumsq_out.is_contiguous() and sumsq_out.shape == (M, N // 32)
        a.sumsq_out = sumsq_out.data_ptr()
    if mode == THIN_QKV:
        cos, sin, pos_dev = rope
        E = N // 3
        if cache_scale is None:
            _cuda(cache, ACT(), "cache")
        else:
            _check_kv_i8(cache, cache_scale, M)
        assert cache.is_contiguous() and cache.dim() == 4 and cache.shape[0] == M and cache.shape[2] == 2 and cache.shape[3] == E
        a.rope_cos, a.rope_sin, a.pos_dev, a.E = cos.data_ptr(), sin.data_ptr(), _ptr(pos_dev), E
        a.cache, a.Tmax, a.t0, a.t0_dev = cache.data_ptr(), cache.shape[1], int(t0), _ptr(t0_dev)
    if cache_scale is None:
        _check(_lib.load().mm_thin_fused(C.byref(a), _stream()), "mm_thin_fused")
    else:
        _check(_lib.load().mm_thin_fused_kv_i8(C.byref(a), cache_scale.data_ptr(), _stream()), "mm_thin_fused_kv_i8")
    return out


# ---------------------------------------------------------------------------------------------------- int8 weights
_W8_FORMAT = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 2}  # mm_quantize_rows_int8's w_format


def quantize_rows_int8(w: torch.Tensor):
    """Per-row int8 quantization of a (rows, K) bf16 / fp16 / fp32 weight (mm_quantize_rows_int8) -> (q int8 (rows, K),
    scale fp32 (rows,)):  s = fp32(max |w|) / 127,  q = clamp(rint(w / s), -127, 127),  q = 0 where s = 0."""
    if not isinstance(w, torch.Tensor) or w.dim() != 2 or w.dtype not in _W8_FORMAT or w.stride(1) != 1:
        raise TypeError("macaw_b200: quantize_rows_int8 takes a 2-D bf16 / fp16 / fp32 tensor with unit column stride")
    _cuda(w, None, "w")
    rows, K = w.shape
    q = torch.empty((rows, K), device=w.device, dtype=torch.int8)
    s = torch.empty((rows,), device=w.device, dtype=torch.float32)
    _check(_lib.load().mm_quantize_rows_int8(w.data_ptr(), w.stride(0), _W8_FORMAT[w.dtype], rows, K, q.data_ptr(),
                                             s.data_ptr(), _stream()), "mm_quantize_rows_int8")
    return q, s


def w8_chunk_map(rows, interleave: bool = False) -> torch.Tensor:
    """The (source, first source row) of every 32-row chunk of a fused weight matrix, int32 (N / 32, 2) on the CPU.
    interleave=False: the sources' rows one after another (torch.cat, the [q; k; v] weight); True: two sources of equal
    height in alternating 32-row groups (fused row 64j + r is row 32j + r of source 0, row 64j + 32 + r of source 1: the
    [gate | up] weight)."""
    rows = [int(r) for r in rows]
    if any(r <= 0 or r % 32 for r in rows):
        raise ValueError(f"macaw_b200: fused sources need a positive multiple of 32 rows, got {rows}")
    if interleave:
        if len(rows) != 2 or rows[0] != rows[1]:
            raise ValueError(f"macaw_b200: an interleaved fused matrix has two sources of equal height, got {rows}")
        c = torch.arange(2 * rows[0] // 32)
        return torch.stack([c % 2, 32 * (c // 2)], 1).to(torch.int32)
    return torch.cat([torch.stack([torch.full((r // 32,), j), 32 * torch.arange(r // 32)], 1)
                      for j, r in enumerate(rows)]).to(torch.int32)


_W8_CHUNKS = {}  # device copies of the chunk maps, by (rows, interleave, device)


class W8Matrix:
    """A fused int8 (or e4m3: `fp8`) weight (N, K) over up to three per-row-quantized sources (mm_w8_matrix), the
    sources' rows arranged as `w8_chunk_map(rows, interleave)` says; `gain` (K,) 16-bit: the RMSNorm gain folded into the
    product, or None."""

    def __init__(self, qs, scales, interleave: bool = False, gain: Optional[torch.Tensor] = None):
        qs, scales = list(qs), list(scales)
        if not 1 <= len(qs) <= _lib.W8_MAX_SRC or len(scales) != len(qs):
            raise ValueError(f"macaw_b200: a fused int8 weight has 1..{_lib.W8_MAX_SRC} sources, each with its scales")
        K = qs[0].shape[1]
        self.fp8 = qs[0].dtype == _E4M3
        for q, s in zip(qs, scales):
            if self.fp8 and (q.dtype != _E4M3 or q.dim() != 2 or not q.is_contiguous() or q.shape[1] != K):
                raise TypeError("macaw_b200: e4m3 sources must be contiguous (rows, K) float8_e4m3fn tensors with one K")
            if not self.fp8 and (q.dtype != torch.int8 or q.dim() != 2 or not q.is_contiguous() or q.shape[1] != K):
                raise TypeError("macaw_b200: int8 sources must be contiguous (rows, K) int8 tensors with one K")
            if s.dtype != torch.float32 or tuple(s.shape) != (q.shape[0],) or not s.is_contiguous():
                raise TypeError("macaw_b200: each source needs a contiguous fp32 scale per row")
        chunks = w8_chunk_map([q.shape[0] for q in qs], interleave)
        N = 32 * chunks.shape[0]
        if N % 64 or K % 16:
            raise ValueError(f"macaw_b200: int8 weights need N % 64 == 0 and K % 16 == 0, got N={N}, K={K}")
        if gain is not None and (gain.dtype != ACT() or tuple(gain.shape) != (K,) or not gain.is_contiguous()):
            raise TypeError(f"macaw_b200: the gain must be a contiguous ({K},) {ACT()} tensor")
        for i, t in enumerate(qs + scales + ([gain] if gain is not None else [])):
            _cuda(t, None, f"int8 weight operand {i}")
        dev = qs[0].device
        key = (tuple(q.shape[0] for q in qs), bool(interleave), str(dev))
        dchunks = _W8_CHUNKS.get(key)
        if dchunks is None:
            dchunks = _W8_CHUNKS[key] = chunks.to(dev)
        self.N, self.K, self.gain = N, K, gain
        self._keep = (qs, scales, dchunks, gain)
        self.args = _lib.W8Matrix()
        for j, (q, s) in enumerate(zip(qs, scales)):
            self.args.q[j], self.args.scale[j], self.args.rows[j] = q.data_ptr(), s.data_ptr(), q.shape[0]
        self.args.chunks, self.args.N, self.args.K, self.args.gain = dchunks.data_ptr(), N, K, _ptr(gain)


def dequant_rows(w: W8Matrix, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The fused 16-bit weight (N, K) in the activation format: round16(fp32(fp32(q s) g)) (mm_dequant_rows)."""
    dev = w._keep[0][0].device
    if out is None:
        out = torch.empty((w.N, w.K), device=dev, dtype=ACT())
    _cuda(out, ACT(), "out")
    assert out.shape == (w.N, w.K) and out.stride(1) == 1
    _check(_lib.load().mm_dequant_rows(C.byref(w.args), out.data_ptr(), out.stride(0), _stream()), "mm_dequant_rows")
    return out


def w8_thin_splits(N: int, K: int, n_sms: int) -> int:
    """K slices of an int8 decode GEMM: at least two, and enough CTAs (64 weight rows each) for two per SM; at most one
    slice per 128-column stage.  With two slices the x~ of up to 8 activation rows of a 4096-column slice half fits the
    kernel's staging buffer, so one-token decode steps at small batch need no extra launch."""
    return min((K + 127) // 128, max(2, -(-2 * n_sms // (N // 64))))


def linear_w8_thin_fused(x: torch.Tensor, w: W8Matrix, mode: int, *, splits: Optional[int] = None, **tail) -> torch.Tensor:
    """`linear_thin_fused` on an int8 fused weight: mm_gemm_w8_thin writes the split-K partial sums
    s_n * sum_k q[n, k] round16(x[m, k] g[k]) and the same mm_thin_fused tail finishes them (keywords as there).  An e4m3
    weight (w.fp8) runs mm_gemm_e4m3_thin, the same kernel with e4m3(q[n, k])."""
    _cuda(x, ACT(), "x")
    M, K = x.shape
    assert x.stride(1) == 1 and K == w.K and 1 <= M <= 64
    dev = x.device
    S = w8_thin_splits(w.N, K, torch.cuda.get_device_properties(dev).multi_processor_count) if splits is None else int(splits)
    Mp = (M + 3) // 4 * 4
    part = torch.empty((S, w.N, Mp), device=dev, dtype=torch.float32)
    xs_work = torch.empty((M, (K + 127) // 128 * 128), device=dev, dtype=ACT())  # x~ when it is streamed
    fn, what = (_lib.load().mm_gemm_e4m3_thin, "mm_gemm_e4m3_thin") if w.fp8 else (_lib.load().mm_gemm_w8_thin, "mm_gemm_w8_thin")
    _check(fn(C.byref(w.args), x.data_ptr(), x.stride(0), M, part.data_ptr(), S, Mp, xs_work.data_ptr(), _stream()), what)
    return _thin_tail(part, M, K, mode, **tail)


# ---------------------------------------------------------------------------------------------------- e4m3 (FP8)
_E4M3 = torch.float8_e4m3fn


def quantize_rows_e4m3(x: torch.Tensor, gain: Optional[torch.Tensor] = None):
    """Per-row e4m3 quantization of a (rows, K) bf16 / fp16 / fp32 matrix (mm_quantize_rows_e4m3) -> (q float8_e4m3fn
    (rows, K), scale fp32 (rows,)):  v = x g (fp32),  s = max |v| / 448,  q = e4m3(v / s) (nearest even, saturated),
    q = 0 where s = 0.  `gain` (K,) in the activation format, or None."""
    if not isinstance(x, torch.Tensor) or x.dim() != 2 or x.dtype not in _W8_FORMAT or x.stride(1) != 1:
        raise TypeError("macaw_b200: quantize_rows_e4m3 takes a 2-D bf16 / fp16 / fp32 tensor with unit column stride")
    _cuda(x, None, "x")
    rows, K = x.shape
    if gain is not None:
        _cuda(gain, ACT(), "gain")
        assert tuple(gain.shape) == (K,) and gain.is_contiguous()
    q = torch.empty((rows, K), device=x.device, dtype=_E4M3)
    s = torch.empty((rows,), device=x.device, dtype=torch.float32)
    args = (x.data_ptr(), x.stride(0), _W8_FORMAT[x.dtype], rows, K, _ptr(gain), q.data_ptr(), K, s.data_ptr(), _stream())
    if PROFILE is None:
        _check(_lib.load().mm_quantize_rows_e4m3(*args), "mm_quantize_rows_e4m3")
        return q, s
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _check(_lib.load().mm_quantize_rows_e4m3(*args), "mm_quantize_rows_e4m3")
    e1.record()
    PROFILE.append((TAG + ".quantize", 0.0, e0, e1))  # no GEMM FLOPs: its time, next to the GEMMs'
    return q, s


def _e4m3_args(a_scale: int, w: W8Matrix, unpromoted: bool) -> _lib.GemmE4m3Args:
    if not w.fp8:
        raise TypeError("macaw_b200: the e4m3 GEMM needs an e4m3 weight")
    e = _lib.GemmE4m3Args()
    e.a_scale, e.unpromoted = a_scale, int(unpromoted)
    C.memmove(C.byref(e.w), C.byref(w.args), C.sizeof(_lib.W8Matrix))
    e.w.gain = None  # the gain was applied to the activation rows before they were quantized
    return e


def linear_e4m3(xq: torch.Tensor, xs: torch.Tensor, w: W8Matrix, *, epi: int = EPI_STD, residual=None,
                out: Optional[torch.Tensor] = None, out_dtype=None, row_scale: Optional[torch.Tensor] = None, rope=None,
                sumsq_out: Optional[torch.Tensor] = None, rms_from=None, unpromoted: bool = False,
                plan_only: bool = False):
    """`linear` on per-row e4m3 operands: out = epilogue((acc * xs[m]) * s_w[n]), acc = sum_k xq[m, k] q_w[n, k]
    (mm_gemm_e4m3_fwd).  xq (M, K) float8_e4m3fn with unit column stride and xs (M,) fp32 from quantize_rows_e4m3; w an
    e4m3 W8Matrix (its gain is not used).  Epilogue keywords as in `linear`; unpromoted=True runs the comparison instance
    whose MMAs accumulate all of K in place; plan_only=True returns the plan of this launch."""
    _cuda(xq, _E4M3, "xq"); _cuda(xs, torch.float32, "xs")
    M, K = xq.shape
    assert xq.stride(1) == 1 and xs.shape == (M,) and xs.is_contiguous() and K == w.K
    N = w.N
    n_out = N // 2 if epi == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), device=xq.device, dtype=out_dtype if out_dtype is not None else ACT())
    assert out.shape == (M, n_out) and out.stride(1) == 1
    kw = {}
    if residual is not None:
        _cuda(residual, ACT(), "residual")
        assert residual.stride(-1) == 1
        kw.update(residual=residual.data_ptr(), ldr=residual.stride(0))
    if rope is not None:
        cos, sin, T, cols = rope[:4]
        kw.update(rope_cos=cos.data_ptr(), rope_sin=sin.data_ptr(), rope_T=T, rope_cols=cols)
        if len(rope) > 4 and rope[4] is not None:
            kw.update(rope_pos=rope[4].data_ptr())
    if sumsq_out is not None:
        assert sumsq_out.dtype == torch.float32 and sumsq_out.is_contiguous() and sumsq_out.shape == (M, (N + 31) // 32)
        kw.update(sumsq_out=sumsq_out.data_ptr())
    if rms_from is not None:
        parts, eps = rms_from
        assert parts.dtype == torch.float32 and parts.is_contiguous() and parts.shape[0] == M and row_scale is None
        kw.update(rs_sumsq=parts.data_ptr(), rs_parts=parts.shape[1], rs_eps=eps)
    e = _e4m3_args(xs.data_ptr(), w, unpromoted)
    plan = gemm_raw(M=M, N=N, K=K, A=xq.data_ptr(), lda=xq.stride(0), B=0, ldb=K, Cout=out.data_ptr(), ldc=out.stride(0),
                    c_fp32=out.dtype == torch.float32, c_fp16=out.dtype == _F16, epi=epi, row_scale=_ptr(row_scale),
                    plan_only=plan_only, e4m3=e, **kw)
    return plan if plan_only else out


def gemm_e4m3_plan(*, M: int, N: int, K: int, epi: int = EPI_STD, rows=None, lda: Optional[int] = None,
                   a_scale: bool = True, w_scale: bool = True) -> dict:
    """The launch mm_gemm_e4m3_fwd would make for M activation rows against an e4m3 weight (N, K) whose sources have
    `rows` (default one source of N rows), 16-byte-aligned fake operands (mm_gemm_e4m3_plan: nothing is touched, no GPU
    needed).  a_scale / w_scale=False pass null scales (argument checks)."""
    lib = _lib.load()
    fake = 1 << 20
    rows = [N] if rows is None else list(rows)
    n_out = N // 2 if epi == EPI_SWIGLU else N
    rope = dict(rope_cos=fake, rope_sin=fake, rope_T=max(1, M), rope_cols=(N // 128) * 128) if epi == EPI_ROPE else {}
    a = GemmArgs(M=M, N=N, K=K, batch=1, batch2=1, A=fake, lda=K if lda is None else lda, B=fake, ldb=K, C=fake,
                 ldc=n_out, epi=epi, alpha=1.0, c_fp16=int(ACT() == _F16), **rope)
    e = _lib.GemmE4m3Args()
    e.a_scale = fake if a_scale else None
    for j, r in enumerate(rows):
        e.w.q[j], e.w.scale[j], e.w.rows[j] = fake, fake if w_scale else None, r
    e.w.chunks, e.w.N, e.w.K = fake, N, K
    return _plan_of(a, e)


def splitk_reduce(partial: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor) -> torch.Tensor:
    _cuda(partial, torch.float32, "partial"); _cuda(out, None, "out")
    assert out.dtype in _16BIT
    S, M, N = partial.shape
    _check(_lib.load().mm_splitk_reduce(partial.data_ptr(), S, M, N, _ptr(bias), out.data_ptr(), out.stride(0),
                                        int(out.dtype == _F16), _stream()), "mm_splitk_reduce")
    return out


# ---------------------------------------------------------------------------------------------------- attention
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, scale: float, causal: bool = False,
              key_mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
              tk_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q (B, Tq, H, hd), k/v (B, Tk, H, hd) bf16 views (hd contiguous, arbitrary other strides) -> (B, Tq, H, hd)."""
    for n, t in (("q", q), ("k", k), ("v", v)):
        _cuda(t, ACT(), n)
        assert t.dim() == 4 and t.stride(3) == 1
    B, Tq, H, hd = q.shape
    Tk = k.shape[1]
    if out is None:
        out = torch.empty((B, Tq, H, hd), device=q.device, dtype=ACT())
    if key_mask is not None:
        _cuda(key_mask, torch.int32, "key_mask")
        assert key_mask.shape == (B, Tk) and key_mask.is_contiguous()
    a = AttnArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Tq, Tk, hd,
                 q.stride(0), q.stride(1), q.stride(2), k.stride(0), k.stride(1), k.stride(2),
                 v.stride(0), v.stride(1), v.stride(2), out.stride(0), out.stride(1), out.stride(2),
                 _ptr(key_mask), int(causal), float(scale), _ptr(tk_dev))
    _check(_lib.load().mm_attn_fwd(C.byref(a), _stream()), "mm_attn_fwd")
    return out


# ---------------------------------------------------------------------------------------------------- norms
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, ACT(), "x"); _cuda(w, ACT(), "w")
    assert x.is_contiguous()
    cols = x.shape[-1]
    rows = x.numel() // cols
    if out is None:
        out = torch.empty_like(x)
    _check(_lib.load().mm_rmsnorm_fwd(x.data_ptr(), w.data_ptr(), out.data_ptr(), rows, cols, float(eps), _stream()),
           "mm_rmsnorm_fwd")
    return out


def rms_rstd(x: torch.Tensor, eps: float) -> torch.Tensor:
    """fp32 rsqrt(mean(x^2) + eps) per row of a contiguous bf16 (rows, cols) tensor."""
    _cuda(x, ACT(), "x")
    assert x.is_contiguous()
    cols = x.shape[-1]
    rows = x.numel() // cols
    out = torch.empty((rows,), device=x.device, dtype=torch.float32)
    _check(_lib.load().mm_rms_rstd(x.data_ptr(), out.data_ptr(), rows, cols, float(eps), _stream()), "mm_rms_rstd")
    return out


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x (rows, cols) bf16 with unit inner stride (row stride free)."""
    _cuda(x, ACT(), "x"); _cuda(w, ACT(), "w"); _cuda(b, ACT(), "b")
    assert x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), device=x.device, dtype=ACT())
    _check(_lib.load().mm_layernorm_fwd(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                        out.stride(0), rows, cols, float(eps), _stream()), "mm_layernorm_fwd")
    return out


# ---------------------------------------------------------------------------------------------------- gathers / layout
def embed_gather(table: torch.Tensor, ids: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[i] = table[ids[i]]; ids any integer dtype (converted to int64 on device), out (n, dim) row stride free."""
    _cuda(table, ACT(), "table"); _cuda(ids, None, "ids")
    ids64 = ids.reshape(-1).to(torch.int64).contiguous()  # (a strided 1-D view survives reshape(-1))
    n, dim = ids64.numel(), table.shape[1]
    if out is None:
        out = torch.empty((n, dim), device=table.device, dtype=ACT())
    assert out.stride(-1) == 1
    _check(_lib.load().mm_embed_gather(table.data_ptr(), table.shape[0], dim, ids64.data_ptr(), n, out.data_ptr(),
                                       out.stride(0), _stream()), "mm_embed_gather")
    return out


def splice_prefix(text: torch.Tensor, prefix: Optional[torch.Tensor], mask_in: Optional[torch.Tensor],
                  labels_in: Optional[torch.Tensor]):
    """text (B, L, E), prefix (B, P, E) -> embeds (B, P + L, E), mask (B, P + L) | None, labels (B, P + L) | None."""
    _cuda(text, ACT(), "text")
    B, L, E = text.shape
    P = 0 if prefix is None else prefix.shape[1]
    assert text.is_contiguous() and (prefix is None or prefix.is_contiguous())
    dst = torch.empty((B, P + L, E), device=text.device, dtype=ACT())
    mask_out = labels_out = None
    if mask_in is not None:
        mask_in = _cuda(mask_in, None, "attention_mask").to(torch.int64).contiguous()
        mask_out = torch.empty((B, P + L), device=text.device, dtype=torch.int64)
    if labels_in is not None:
        labels_in = _cuda(labels_in, None, "labels").to(torch.int64).contiguous()
        labels_out = torch.empty((B, P + L), device=text.device, dtype=torch.int64)
    _check(_lib.load().mm_splice_prefix(text.data_ptr(), _ptr(prefix), dst.data_ptr(), B, L, P, E, _ptr(mask_in),
                                        _ptr(mask_out), _ptr(labels_in), _ptr(labels_out), _stream()),
           "mm_splice_prefix")
    return dst, mask_out, labels_out


def patchify(images: torch.Tensor, patch: int, ldo: int) -> torch.Tensor:
    _cuda(images, ACT(), "images")
    assert images.is_contiguous()
    B, Cc, H, W = images.shape
    out = torch.empty((B * (H // patch) * (W // patch), ldo), device=images.device, dtype=ACT())
    _check(_lib.load().mm_patchify(images.data_ptr(), B, Cc, H, W, patch, out.data_ptr(), ldo, _stream()),
           "mm_patchify")
    return out


def transpose_pad(x: torch.Tensor, pad: int) -> torch.Tensor:
    """(B, C, T) -> (B, T + 2 pad, C) with zero pad rows."""
    _cuda(x, ACT(), "x")
    assert x.is_contiguous()
    B, Cc, T = x.shape
    out = torch.empty((B, T + 2 * pad, Cc), device=x.device, dtype=ACT())
    _check(_lib.load().mm_transpose_pad(x.data_ptr(), B, Cc, T, pad, out.data_ptr(), _stream()), "mm_transpose_pad")
    return out


def cast_f16(x: torch.Tensor) -> torch.Tensor:
    """bf16 (..., cols) contiguous -> fp16 copy (mm_cast_bf16_f16)."""
    _cuda(x, torch.bfloat16, "x")
    assert x.is_contiguous()
    cols = x.shape[-1]
    rows = x.numel() // cols
    y = torch.empty(x.shape, device=x.device, dtype=_F16)
    _check(_lib.load().mm_cast_bf16_f16(x.data_ptr(), cols, y.data_ptr(), cols, rows, cols, _stream()), "mm_cast_bf16_f16")
    return y


def add_rows(x: torch.Tensor, add: Optional[torch.Tensor], out: torch.Tensor) -> torch.Tensor:
    """out[r] = x[r] + add[r % add.shape[0]] over 2-D bf16 views with unit inner stride."""
    _cuda(x, ACT(), "x"); _cuda(out, ACT(), "out")
    rows, cols = x.shape
    assert x.stride(1) == 1 and out.stride(1) == 1 and out.shape == x.shape
    if add is None:
        _check(_lib.load().mm_copy_rows(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), rows, cols,
                                        _stream()), "mm_copy_rows")
    else:
        _cuda(add, ACT(), "add")
        assert add.stride(1) == 1 and add.shape[1] == cols
        _check(_lib.load().mm_add_rows(x.data_ptr(), x.stride(0), add.data_ptr(), add.stride(0), add.shape[0],
                                       out.data_ptr(), out.stride(0), rows, cols, _stream()), "mm_add_rows")
    return out


# ---------------------------------------------------------------------------------------------------- alignment
ALIGN_MODE = 0  # 0: one cooperative launch with grid-wide barriers between the phases; 1: three stream-ordered launches


def align_fused(table: torch.Tensor, qt: torch.Tensor, stats: torch.Tensor, out: Optional[torch.Tensor] = None,
                mode: Optional[int] = None, keep: Optional[dict] = None):
    """Fused absorbed-form alignment attention (mm_align_fwd).  table (V, E) fp16; qt (R, E) fp16 absorbed queries;
    stats (R, 2) fp32 = [row_bias, extra score] -> (ctx~ (R, E) fp16, p_sum_real (R,), p_extra (R,))."""
    _cuda(table, _F16, "table"); _cuda(qt, _F16, "qt"); _cuda(stats, torch.float32, "stats")
    R, E = qt.shape
    V = table.shape[0]
    assert table.shape[1] == E and table.stride(1) == 1 and qt.stride(1) == 1 and stats.shape == (R, 2) and stats.is_contiguous()
    dev = qt.device
    if out is None:
        out = torch.empty((R, E), device=dev, dtype=_F16)
    assert out.shape == (R, E) and out.stride(1) == 1 and out.dtype == _F16
    Vp = (V + 7) // 8 * 8
    P = torch.empty((R, Vp), device=dev, dtype=_F16)
    lib = _lib.load()
    ws = torch.empty((int(lib.mm_align_workspace_bytes(R, V)) + 15) // 16 * 4, device=dev, dtype=torch.int32)
    psum = torch.empty((R,), device=dev, dtype=torch.float32)
    pext = torch.empty((R,), device=dev, dtype=torch.float32)
    inv_l = torch.empty((R,), device=dev, dtype=torch.float32) if keep is not None else None
    a = AlignArgs(table.data_ptr(), V, E, table.stride(0), qt.data_ptr(), R, qt.stride(0), stats.data_ptr(),
                  stats.data_ptr() + 4, 2, out.data_ptr(), out.stride(0), psum.data_ptr(), pext.data_ptr(), P.data_ptr(), Vp,
                  ws.data_ptr(), ALIGN_MODE if mode is None else int(mode), _ptr(inv_l))
    if keep is not None:  # the training step keeps the un-normalised probabilities and 1 / l for the backward pass
        keep.update(P=P, inv_l=inv_l)
    if PROFILE is None:
        _check(lib.mm_align_fwd(C.byref(a), _stream()), "mm_align_fwd")
    else:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _check(lib.mm_align_fwd(C.byref(a), _stream()), "mm_align_fwd")
        e1.record()
        PROFILE.append(("align.fused", 4.0 * R * V * E, e0, e1))
    return out, psum, pext


# ---------------------------------------------------------------------------------------------------- decode helpers
def kv_append(qkv: torch.Tensor, B: int, T_new: int, cache: torch.Tensor, t0: int,
              t0_dev: Optional[torch.Tensor] = None) -> None:
    """qkv (B*T_new, 3E) fused activation -> cache (B, Tmax, 2, E) at positions t0 .. t0+T_new-1 (K and V thirds)."""
    _cuda(qkv, ACT(), "qkv"); _cuda(cache, ACT(), "cache")
    E = cache.shape[-1]
    assert qkv.shape == (B * T_new, 3 * E) and qkv.stride(1) == 1 and cache.is_contiguous() and cache.shape[2] == 2
    _check(_lib.load().mm_kv_append(qkv.data_ptr(), qkv.stride(0), B, T_new, E, cache.data_ptr(), cache.shape[1], t0,
                                    _ptr(t0_dev), _stream()), "mm_kv_append")


# ---------------------------------------------------------------------------------------------------- int8 KV cache
def _check_kv_i8(cache: torch.Tensor, cache_scale: torch.Tensor, B: int) -> None:
    """cache int8 (B, Tmax, 2, E) and cache_scale fp32 (B, 2, E / 128, Tmax), both contiguous (mm_kv_append_i8's layout)."""
    _cuda(cache, torch.int8, "cache"); _cuda(cache_scale, torch.float32, "cache_scale")
    assert cache.dim() == 4 and cache.is_contiguous() and cache.shape[0] == B and cache.shape[2] == 2, cache.shape
    _, Tmax, _, E = cache.shape
    assert tuple(cache_scale.shape) == (B, 2, E // 128, Tmax) and cache_scale.is_contiguous(), cache_scale.shape


def kv_append_i8(qkv: torch.Tensor, B: int, T_new: int, cache: torch.Tensor, cache_scale: torch.Tensor, t0: int,
                 t0_dev: Optional[torch.Tensor] = None) -> None:
    """`kv_append` into an int8 cache: each k / v head vector of the rows (16-bit, as the 16-bit cache stores it) is
    quantized by the int8 KV-cache rule (mm_kv_append_i8): s = fp32(max |v|) / 127, q = clamp(rint(v / s), -127, 127),
    q = 0 where s = 0; q -> cache (B, Tmax, 2, E), s -> cache_scale (B, 2, H, Tmax)."""
    _cuda(qkv, ACT(), "qkv")
    _check_kv_i8(cache, cache_scale, B)
    E = cache.shape[-1]
    assert qkv.shape == (B * T_new, 3 * E) and qkv.stride(1) == 1
    _check(_lib.load().mm_kv_append_i8(qkv.data_ptr(), qkv.stride(0), B, T_new, E, cache.data_ptr(), cache_scale.data_ptr(),
                                       cache.shape[1], t0, _ptr(t0_dev), _stream()), "mm_kv_append_i8")


def attention_decode_i8(q: torch.Tensor, cache: torch.Tensor, cache_scale: torch.Tensor, *, scale: float,
                        Tk: Optional[int] = None, tk_dev: Optional[torch.Tensor] = None,
                        key_mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Attention of one query row per (sample, head) over an int8 cache (mm_attn_decode_i8): q (B, 1, H, 128) 16-bit view
    (head_dim contiguous, heads 128 apart), cache / cache_scale as kv_append_i8 fills them -> (B, 1, H, 128).  The key count
    is Tk (default: the capacity), or min(*tk_dev, Tk) read on the device.  There is no key mask: generate never passes one."""
    if key_mask is not None:
        raise NotImplementedError("macaw_b200: the int8 KV cache's decode attention takes no key mask")
    _cuda(q, ACT(), "q")
    B, Tq, H, hd = q.shape
    assert Tq == 1 and hd == 128 and q.stride(3) == 1 and q.stride(2) == 128, (q.shape, q.stride())
    _check_kv_i8(cache, cache_scale, B)
    Tmax = cache.shape[1]
    assert cache.shape[3] == H * hd
    Tk = Tmax if Tk is None else int(Tk)
    if tk_dev is not None:
        _cuda(tk_dev, torch.int32, "tk_dev")
    if out is None:
        out = torch.empty((B, 1, H, hd), device=q.device, dtype=ACT())
    assert out.shape == (B, 1, H, hd) and out.stride(3) == 1 and out.stride(2) == 128
    lib = _lib.load()
    nbytes = int(lib.mm_attn_decode_i8_workspace_bytes(B, H, Tmax))
    ws = torch.empty(((nbytes + 15) // 16 * 4,), device=q.device, dtype=torch.float32)
    _check(lib.mm_attn_decode_i8(q.data_ptr(), q.stride(0), cache.data_ptr(), cache_scale.data_ptr(), out.data_ptr(),
                                 out.stride(0), B, H, Tmax, Tk, _ptr(tk_dev), float(scale), ws.data_ptr(), ws.numel() * 4,
                                 _stream()), "mm_attn_decode_i8")
    return out


def rope_rows(x: torch.Tensor, rot_cols: int, cos: torch.Tensor, sin: torch.Tensor, rope_T: int,
              pos_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """In-place rotate-half RoPE (head_dim 128) on the first rot_cols columns of 16-bit rows (x, cos and sin tables (T, 64))."""
    _cuda(x, ACT(), "x")
    assert x.dim() == 2 and x.stride(1) == 1
    _check(_lib.load().mm_rope_rows(x.data_ptr(), x.stride(0), x.shape[0], rot_cols, cos.data_ptr(), sin.data_ptr(), rope_T,
                                    _ptr(pos_dev), _stream()), "mm_rope_rows")
    return x


def argmax_rows(logits: torch.Tensor) -> torch.Tensor:
    """Greedy token per row of bf16 logits (rows, V) with unit inner stride -> int64 (rows,)."""
    _cuda(logits, ACT(), "logits")
    assert logits.dim() == 2 and logits.stride(1) == 1
    out = torch.empty((logits.shape[0],), device=logits.device, dtype=torch.int64)
    _check(_lib.load().mm_argmax_rows(logits.data_ptr(), logits.stride(0), logits.shape[0], logits.shape[1],
                                      out.data_ptr(), _stream()), "mm_argmax_rows")
    return out


def sample_rows(logits: torch.Tensor, seen: torch.Tensor, *, do_sample: bool, repetition_penalty: float = 1.0,
                temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, seed_dev: Optional[torch.Tensor] = None,
                step_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Next token per row of 16-bit logits (rows, V) under HF's repetition penalty / temperature / top-k / top-p chain
    (mm_sample_rows) -> int64 (rows,).  seen: int32 (rows, ceil(V/32)) bitmap of the tokens generated so far, updated
    in place with the emitted token.  seed_dev (int64 (1,)) and step_dev (int32 (1,)) are read on the device, so a
    captured CUDA graph draws fresh numbers when they change; greedy (do_sample=False) does not read them."""
    _cuda(logits, ACT(), "logits"); _cuda(seen, torch.int32, "seen")
    assert logits.dim() == 2 and logits.stride(1) == 1
    rows, V = logits.shape
    assert seen.is_contiguous() and tuple(seen.shape) == (rows, (V + 31) // 32)
    if do_sample:
        _cuda(seed_dev, torch.int64, "seed_dev"); _cuda(step_dev, torch.int32, "step_dev")
    out = torch.empty((rows,), device=logits.device, dtype=torch.int64)
    _check(_lib.load().mm_sample_rows(logits.data_ptr(), logits.stride(0), rows, V, seen.data_ptr(),
                                      float(repetition_penalty), float(temperature), int(top_k), float(top_p),
                                      int(bool(do_sample)), _ptr(seed_dev), _ptr(step_dev), out.data_ptr(), _stream()),
           "mm_sample_rows")
    return out


# ---------------------------------------------------------------------------------------------------- loss
def ce_loss(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """Shifted CE (mean over labels != -100) of bf16 logits (B, T, V) against int64 labels (B, T); returns fp32 scalar."""
    return ce_loss_with_count(logits, labels)[0]


# ---------------------------------------------------------------------------------------------------- training step
def gemm_dx(dy: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """Input gradient of y = x @ w.T:  dx (M, K) = dy (M, N) @ w (N, K) — w is read as an MN-major B operand in place."""
    _cuda(dy, ACT(), "dy"); _cuda(w, ACT(), "w")
    M, N = dy.shape
    K = w.shape[1]
    assert w.shape[0] == N and dy.stride(1) == 1 and w.stride(1) == 1
    if out is None:
        assert not accumulate
        out = torch.empty((M, K), device=dy.device, dtype=ACT())
    kw = dict(residual=out.data_ptr(), ldr=out.stride(0)) if accumulate else {}
    gemm_raw(M=M, N=K, K=N, A=dy.data_ptr(), lda=dy.stride(0), B=w.data_ptr(), ldb=w.stride(0), b_mn_major=True,
             Cout=out.data_ptr(), ldc=out.stride(0), **kw)
    return out


def gemm_dw(dy: torch.Tensor, x: torch.Tensor, out: torch.Tensor, accumulate: bool) -> torch.Tensor:
    """Weight gradient of y = x @ w.T:  dw (N, K) (+)= dy (M, N).T @ x (M, K) — both activations are read as stored
    (MN-major A and B operands), no transposes."""
    _cuda(dy, ACT(), "dy"); _cuda(x, ACT(), "x"); _cuda(out, ACT(), "dw")
    M, N = dy.shape
    K = x.shape[1]
    assert x.shape[0] == M and out.shape == (N, K) and dy.stride(1) == 1 and x.stride(1) == 1 and out.stride(1) == 1
    kw = dict(residual=out.data_ptr(), ldr=out.stride(0)) if accumulate else {}
    gemm_raw(M=N, N=K, K=M, A=dy.data_ptr(), lda=dy.stride(0), a_mn_major=True, B=x.data_ptr(), ldb=x.stride(0),
             b_mn_major=True, Cout=out.data_ptr(), ldc=out.stride(0), **kw)
    return out


def rmsnorm_bwd(dy: torch.Tensor, x: torch.Tensor, rstd: torch.Tensor, g: torch.Tensor, dres: Optional[torch.Tensor],
                dg: Optional[torch.Tensor]) -> torch.Tensor:
    """dx of y = x * rstd * g (+ dres); dg (fp32, cols) is accumulated in place."""
    _cuda(dy, ACT(), "dy"); _cuda(x, ACT(), "x"); _cuda(rstd, torch.float32, "rstd"); _cuda(g, ACT(), "g")
    assert dy.is_contiguous() and x.is_contiguous() and (dres is None or dres.is_contiguous())
    rows, cols = x.shape
    dx = torch.empty_like(x)
    lib = _lib.load()
    parts = None
    if dg is not None:  # per-CTA partial column sums, reduced in a fixed order (no atomics)
        with torch.cuda.device(x.device):
            parts = torch.empty((int(lib.mm_rmsnorm_bwd_parts(rows)), cols), device=x.device, dtype=torch.float32)
    _check(lib.mm_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr(), g.data_ptr(), _ptr(dres), dx.data_ptr(),
                              _ptr(dg), _ptr(parts), rows, cols, _stream()), "mm_rmsnorm_bwd")
    return dx


def swiglu_fwd(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    _cuda(gate, ACT(), "gate"); _cuda(up, ACT(), "up")
    assert gate.is_contiguous() and up.is_contiguous() and gate.shape == up.shape
    h = torch.empty_like(gate)
    _check(_lib.load().mm_swiglu_fwd(gate.data_ptr(), up.data_ptr(), h.data_ptr(), gate.numel(), _stream()), "mm_swiglu_fwd")
    return h


def swiglu_bwd(dh: torch.Tensor, gate: torch.Tensor, up: torch.Tensor):
    _cuda(dh, ACT(), "dh")
    assert dh.is_contiguous() and gate.is_contiguous() and up.is_contiguous()
    dg, du = torch.empty_like(gate), torch.empty_like(up)
    _check(_lib.load().mm_swiglu_bwd(dh.data_ptr(), gate.data_ptr(), up.data_ptr(), dg.data_ptr(), du.data_ptr(), dh.numel(),
                                     _stream()), "mm_swiglu_bwd")
    return dg, du


def _drop_args(dropout):
    """dropout = None | (p, seed_dev int64 1-element CUDA tensor, stream id) -> (p, seed pointer, sid) for the C ABI."""
    if dropout is None:
        return 0.0, None, 0
    p, seed, sid = dropout
    if float(p) <= 0.0:
        return 0.0, None, 0
    assert seed.is_cuda and seed.dtype == torch.int64 and seed.numel() == 1
    return float(p), seed.data_ptr(), int(sid)


def dropout_mask(rows: int, cols: int, dropout, device) -> torch.Tensor:
    """fp32 (rows, cols) multipliers (0 or 1/(1-p)) the dropout kernels apply for this (seed, stream id): tests only."""
    p, seed, sid = _drop_args(dropout)
    out = torch.empty((rows, cols), device=device, dtype=torch.float32)
    _check(_lib.load().mm_dropout_mask(out.data_ptr(), cols, rows, cols, p, seed, sid, _stream()), "mm_dropout_mask")
    return out


def attention_train_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, scale: float, causal: bool = False,
                        key_mask: Optional[torch.Tensor] = None, dropout=None) -> torch.Tensor:
    """Training-mode forward of a DROPOUT attention (the flash kernel has no dropout): S = q k^T (fp32, batched wgmma
    GEMM), Pd = dropout(softmax(scale S)) (one row-wise kernel, Philox mask), O = Pd v.  Same operand conventions as
    attention_bwd; returns O (B, Tq, H, hd) contiguous."""
    for n, t in (("q", q), ("k", k), ("v", v)):
        _cuda(t, ACT(), n)
        assert t.dim() == 4 and t.stride(3) == 1
    B, Tq, H, hd = q.shape
    Tk = k.shape[1]
    dev = q.device
    Tp = (Tk + 7) // 8 * 8
    S = torch.empty((B, H, Tq, Tp), device=dev, dtype=torch.float32)
    gemm_raw(M=Tq, N=Tk, K=hd, batch=H, batch2=B, A=q.data_ptr(), lda=q.stride(1), a_bs=q.stride(2), a_bs2=q.stride(0),
             B=k.data_ptr(), ldb=k.stride(1), b_bs=k.stride(2), b_bs2=k.stride(0), Cout=S.data_ptr(), ldc=Tp, c_bs=Tq * Tp,
             c_bs2=H * Tq * Tp, c_fp32=True)
    P = torch.empty((B, H, Tq, Tp), device=dev, dtype=ACT())
    if key_mask is not None:
        _cuda(key_mask, torch.int32, "key_mask")
    pd, seed, sid = _drop_args(dropout)
    _check(_lib.load().mm_attn_softmax_fwd(S.data_ptr(), P.data_ptr(), B, H, Tq, Tk, Tp, float(scale), int(causal),
                                           _ptr(key_mask), pd, seed, sid, _stream()), "mm_attn_softmax_fwd")
    del S
    o = torch.empty((B, Tq, H, hd), device=dev, dtype=ACT())
    gemm_raw(M=Tq, N=hd, K=Tk, batch=H, batch2=B, A=P.data_ptr(), lda=Tp, a_bs=Tq * Tp, a_bs2=H * Tq * Tp,
             B=v.data_ptr(), ldb=v.stride(1), b_bs=v.stride(2), b_bs2=v.stride(0), b_mn_major=True, Cout=o.data_ptr(),
             ldc=o.stride(1), c_bs=o.stride(2), c_bs2=o.stride(0))
    return o


def attention_bwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, do: torch.Tensor, *, scale: float, causal: bool,
                  key_mask: Optional[torch.Tensor] = None, dropout=None):
    """Backward of mm_attn_fwd composed from wgmma GEMMs: S = q k^T and dP = dO v^T (fp32, batched over (b, h)), one
    row-wise softmax-backward kernel (P, dS in bf16), then dV = P^T dO, dK = dS^T q (MN-major A), dQ = dS k.
    q / do (B, Tq, H, hd), k / v (B, Tk, H, hd): bf16 views with unit head-dim stride.  Returns contiguous dq, dk, dv.
    dropout = (p, seed_dev, sid): backward of attention_train_fwd with the same mask (regenerated, not stored).

    fp16: dS is stored UNSCALED, as torch's autograd keeps it (the scale goes into the fp32 score GEMM's alpha and into the
    dK / dQ GEMMs' alpha).  With the scale folded in, scale * P (dP - D) of a flat softmax row (P ~ 1 / Tk) under a small
    upstream gradient lands in fp16's subnormal range: a 1 / sqrt(96) scale there cost video_long_self_attention's key-side
    gradients 5-7x the error of torch's fp16 autograd.  bf16 keeps the folded scale (no subnormals at these magnitudes)."""
    for n, t in (("q", q), ("k", k), ("v", v), ("do", do)):
        _cuda(t, ACT(), n)
        assert t.dim() == 4 and t.stride(3) == 1
    B, Tq, H, hd = q.shape
    Tk = k.shape[1]
    dev = q.device
    Tp = (Tk + 7) // 8 * 8
    S = torch.empty((B, H, Tq, Tp), device=dev, dtype=torch.float32)
    dP = torch.empty((B, H, Tq, Tp), device=dev, dtype=torch.float32)

    def bat(t):  # (lda, head stride, sample stride) of a (B, T, H, hd) view
        return dict(ld=t.stride(1), bs=t.stride(2), bs2=t.stride(0))

    # (alpha of the score GEMM, scale passed to the softmax kernel, alpha of the dK / dQ GEMMs)
    s_alpha, k_scale, g_alpha = (float(scale), 1.0, float(scale)) if ACT() == _F16 else (1.0, float(scale), 1.0)

    def scores(a, b, out, alpha=1.0):
        sa, sb = bat(a), bat(b)
        gemm_raw(M=Tq, N=Tk, K=hd, batch=H, batch2=B, A=a.data_ptr(), lda=sa["ld"], a_bs=sa["bs"], a_bs2=sa["bs2"],
                 B=b.data_ptr(), ldb=sb["ld"], b_bs=sb["bs"], b_bs2=sb["bs2"], Cout=out.data_ptr(), ldc=Tp, c_bs=Tq * Tp,
                 c_bs2=H * Tq * Tp, c_fp32=True, alpha=alpha)

    scores(q, k, S, s_alpha)
    scores(do, v, dP)
    P = torch.empty((B, H, Tq, Tp), device=dev, dtype=ACT())
    dS = torch.empty((B, H, Tq, Tp), device=dev, dtype=ACT())
    if key_mask is not None:
        _cuda(key_mask, torch.int32, "key_mask")
    pd, seed, sid = _drop_args(dropout)
    _check(_lib.load().mm_attn_softmax_bwd(S.data_ptr(), dP.data_ptr(), P.data_ptr(), dS.data_ptr(), B, H, Tq, Tk, Tp,
                                           k_scale, int(causal), _ptr(key_mask), pd, seed, sid, _stream()),
           "mm_attn_softmax_bwd")
    del S, dP
    dq = torch.empty((B, Tq, H, hd), device=dev, dtype=ACT())
    dk = torch.empty((B, Tk, H, hd), device=dev, dtype=ACT())
    dv = torch.empty((B, Tk, H, hd), device=dev, dtype=ACT())

    def pt_x(p_, x_, out, alpha=1.0):  # out_bh (Tk, hd) = alpha * p_bh^T (Tk x Tq) @ x_bh (Tq, hd)
        sx, so = bat(x_), bat(out)
        gemm_raw(M=Tk, N=hd, K=Tq, batch=H, batch2=B, A=p_.data_ptr(), lda=Tp, a_bs=Tq * Tp, a_bs2=H * Tq * Tp,
                 a_mn_major=True, B=x_.data_ptr(), ldb=sx["ld"], b_bs=sx["bs"], b_bs2=sx["bs2"], b_mn_major=True,
                 Cout=out.data_ptr(), ldc=so["ld"], c_bs=so["bs"], c_bs2=so["bs2"], alpha=alpha)

    pt_x(P, do, dv)
    pt_x(dS, q, dk, g_alpha)
    sk, so = bat(k), bat(dq)
    gemm_raw(M=Tq, N=hd, K=Tk, batch=H, batch2=B, A=dS.data_ptr(), lda=Tp, a_bs=Tq * Tp, a_bs2=H * Tq * Tp,
             B=k.data_ptr(), ldb=sk["ld"], b_bs=sk["bs"], b_bs2=sk["bs2"], b_mn_major=True, Cout=dq.data_ptr(),
             ldc=so["ld"], c_bs=so["bs"], c_bs2=so["bs2"], alpha=g_alpha)
    return dq, dk, dv


def ce_loss_with_count(logits: torch.Tensor, labels: torch.Tensor):
    """mm_ce_loss -> (loss fp32 scalar tensor, n_valid int32 1-element tensor)."""
    _cuda(logits, ACT(), "logits"); _cuda(labels, torch.int64, "labels")
    assert logits.is_contiguous() and labels.is_contiguous()
    B, T, V = logits.shape
    acc = torch.zeros((2,), device=logits.device, dtype=torch.float32)
    cnt = acc[1:].view(torch.int32)
    _check(_lib.load().mm_ce_loss(logits.data_ptr(), labels.data_ptr(), B, T, V, acc.data_ptr(), cnt.data_ptr(),
                                  _stream()), "mm_ce_loss")
    return acc[0] / cnt[0].to(torch.float32), cnt


def ce_bwd(logits: torch.Tensor, labels: torch.Tensor, n_valid: torch.Tensor, grad_scale=1.0) -> torch.Tensor:
    """d loss / d logits, written IN PLACE over the bf16 logits.  grad_scale: python float or a device fp32 scalar tensor
    (the upstream gradient of the loss, read by the kernel — no host sync, CUDA-graph capturable)."""
    B, T, V = logits.shape
    gs_dev = None
    if isinstance(grad_scale, torch.Tensor):
        gs_dev = _cuda(grad_scale.reshape(1).to(torch.float32), torch.float32, "grad_scale")
        grad_scale = 1.0
    _check(_lib.load().mm_ce_bwd(logits.data_ptr(), labels.data_ptr(), logits.data_ptr(), B, T, V, n_valid.data_ptr(),
                                 float(grad_scale), _ptr(gs_dev), _stream()), "mm_ce_bwd")
    return logits


def embed_scatter_add(dx: torch.Tensor, ids: torch.Tensor, dtable: torch.Tensor) -> None:
    """dtable[ids[i]] += dx[i] for bf16 rows dx (n, dim) with unit inner stride."""
    _cuda(dx, ACT(), "dx"); _cuda(dtable, ACT(), "dtable")
    ids64 = ids.reshape(-1).to(torch.int64).contiguous()  # (a strided 1-D view survives reshape(-1))
    assert dx.dim() == 2 and dx.stride(1) == 1 and dx.shape[0] == ids64.numel() and dtable.is_contiguous()
    _check(_lib.load().mm_embed_scatter_add(dx.data_ptr(), dx.stride(0), ids64.data_ptr(), ids64.numel(), dx.shape[1],
                                            dtable.shape[0], dtable.data_ptr(), _stream()), "mm_embed_scatter_add")


def colsum(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _cuda(x, ACT(), "x"); _cuda(out, torch.float32, "out")
    assert x.dim() == 2 and x.stride(1) == 1 and out.numel() == x.shape[1]
    _check(_lib.load().mm_colsum(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], out.data_ptr(), _stream()), "mm_colsum")
    return out


def adamw(p: torch.Tensor, g: torch.Tensor, master: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *, lr: float,
          beta1: float, beta2: float, eps: float, weight_decay: float, step: int, grad_scale: float = 1.0,
          step_dev: Optional[torch.Tensor] = None, grad_mult_dev: Optional[torch.Tensor] = None,
          skip_dev: Optional[torch.Tensor] = None, lr_dev: Optional[torch.Tensor] = None) -> None:
    """Fused AdamW on one tensor (p, g in the activation format).  grad_mult_dev: device fp32 scalar replacing grad_scale;
    skip_dev: device int32 scalar, non-zero = write nothing; lr_dev: device fp32 scalar replacing lr (the output of
    `lr_schedule`) (see mm_adamw)."""
    _cuda(p, ACT(), "p"); _cuda(g, ACT(), "g")
    assert p.is_contiguous() and g.is_contiguous() and master.numel() == p.numel()
    _check(_lib.load().mm_adamw(p.data_ptr(), g.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
                                _ptr(step_dev), float(grad_scale), _ptr(grad_mult_dev), _ptr(skip_dev), _ptr(lr_dev),
                                _stream()),
           "mm_adamw")


LR_SCHEDULE_KINDS = {"linear": 0, "cosine": 1, "constant_with_warmup": 2}  # mm_lr_schedule's `kind`


def lr_schedule(step_dev: torch.Tensor, lr_out: torch.Tensor, *, base_lr: float, kind: str, warmup_steps: int,
                training_steps: int) -> None:
    """lr_out (device fp32 scalar) = fp32(base_lr * lambda(t - 1)), t = *step_dev the AdamW step counter after it has
    advanced, lambda HF's multiplier of schedule `kind` (LR_SCHEDULE_KINDS); one single-thread launch (mm_lr_schedule)."""
    _cuda(step_dev, torch.int32, "step_dev"); _cuda(lr_out, torch.float32, "lr_out")
    assert step_dev.numel() == 1 and lr_out.numel() == 1
    if kind not in LR_SCHEDULE_KINDS:
        raise ValueError(f"lr_schedule: unknown kind {kind!r}; supported: {', '.join(LR_SCHEDULE_KINDS)}")
    _check(_lib.load().mm_lr_schedule(step_dev.data_ptr(), float(base_lr), LR_SCHEDULE_KINDS[kind], int(warmup_steps),
                                      int(training_steps), lr_out.data_ptr(), _stream()), "mm_lr_schedule")


class HostBlock:
    """`nbytes` of page-locked host memory mapped into the device's address space (mm_host_alloc): AdamW state that does not
    fit in HBM, updated in place by `adamw_host` over PCIe.  `view(offset, numel)` is a CPU float32 tensor over part of the
    block.  The block lives until `free()` (idempotent); views must not be used after it."""

    def __init__(self, nbytes: int):
        if nbytes <= 0:
            raise ValueError("HostBlock: nbytes must be > 0")
        h, d = C.c_void_p(), C.c_void_p()
        _check(_lib.load().mm_host_alloc(int(nbytes), C.byref(h), C.byref(d)), "mm_host_alloc")
        self.nbytes, self.host, self.dev = int(nbytes), int(h.value), int(d.value)
        self._flat = torch.frombuffer((C.c_char * self.nbytes).from_address(self.host), dtype=torch.uint8)

    def view(self, offset: int, numel: int) -> torch.Tensor:
        """float32 CPU tensor of `numel` elements at byte `offset` (16-byte aligned)."""
        if offset % 16 or offset < 0 or offset + 4 * numel > self.nbytes:
            raise ValueError(f"HostBlock.view: [{offset}, {offset + 4 * numel}) is not a 16-byte aligned range of the block")
        return self._flat[offset:offset + 4 * numel].view(torch.float32)

    def dev_ptr(self, t: torch.Tensor) -> int:
        """Device alias of the data of `t`, a contiguous float32 view of this block."""
        off = t.data_ptr() - self.host
        if t.device.type != "cpu" or t.dtype != torch.float32 or not t.is_contiguous() or off < 0 or \
                off + 4 * t.numel() > self.nbytes:
            raise ValueError("HostBlock.dev_ptr: not a contiguous float32 view of this block")
        return self.dev + off

    def free(self) -> None:
        if self.host:
            self._flat = None
            _check(_lib.load().mm_host_free(self.host), "mm_host_free")
            self.host = self.dev = 0


def host_alloc(nbytes: int) -> HostBlock:
    """Exactly `nbytes` of mapped, page-locked host memory (mm_host_alloc; not torch's pinned allocator, which rounds every
    block up to a power of two)."""
    return HostBlock(nbytes)


def adamw_host(p: torch.Tensor, g: torch.Tensor, master: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *,
               block: HostBlock, lr: float, beta1: float, beta2: float, eps: float, weight_decay: float, step: int,
               grad_scale: float = 1.0, step_dev: Optional[torch.Tensor] = None,
               grad_mult_dev: Optional[torch.Tensor] = None, skip_dev: Optional[torch.Tensor] = None,
               lr_dev: Optional[torch.Tensor] = None) -> None:
    """`adamw` with master / m / v CPU float32 views of `block` (host memory, reached by the kernel over PCIe); p, g on the
    device.  Bit-identical to `adamw` on device copies of the same state (mm_adamw_host)."""
    _cuda(p, ACT(), "p"); _cuda(g, ACT(), "g")
    assert p.is_contiguous() and g.is_contiguous() and master.numel() == m.numel() == v.numel() == p.numel()
    _check(_lib.load().mm_adamw_host(p.data_ptr(), g.data_ptr(), block.dev_ptr(master), block.dev_ptr(m), block.dev_ptr(v),
                                     p.numel(), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
                                     int(step), _ptr(step_dev), float(grad_scale), _ptr(grad_mult_dev), _ptr(skip_dev),
                                     _ptr(lr_dev), _stream()),
           "mm_adamw_host")


def grad_sumsq_parts(n: int) -> int:
    """Size of the fp32 partials workspace mm_grad_sumsq uses for n elements (on the current device)."""
    return int(_lib.load().mm_grad_sumsq_parts(int(n)))


def grad_sumsq(g: torch.Tensor, out: torch.Tensor, partials: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (device fp32 scalar) += sum(g.float() ** 2) over a contiguous bf16 / fp16 tensor, deterministically; a NaN / Inf
    element makes the result non-finite (mm_grad_sumsq)."""
    _cuda(g, None, "g"); _cuda(out, torch.float32, "out")
    assert g.dtype in _16BIT and g.is_contiguous() and out.numel() == 1
    n = g.numel()
    if partials is None:
        partials = torch.empty((grad_sumsq_parts(n),), device=g.device, dtype=torch.float32)
    assert partials.dtype == torch.float32 and partials.numel() >= grad_sumsq_parts(n)
    _check(_lib.load().mm_grad_sumsq(g.data_ptr(), n, int(g.dtype == _F16), out.data_ptr(), partials.data_ptr(), _stream()),
           "mm_grad_sumsq")
    return out


LOSS_SCALE_STATE_WORDS = 12  # sizeof(mm_loss_scale_state) / 4


def loss_scale_update(state: torch.Tensor, sumsq: torch.Tensor, *, max_norm: Optional[float], dynamic: bool,
                      window: int, hysteresis: int, min_scale: float) -> None:
    """One step of the device loss scaler / clipper over `state` (int32 (12,) tensor laid out as mm_loss_scale_state);
    consumes and zeroes `sumsq` (mm_loss_scale_update)."""
    _cuda(state, torch.int32, "state"); _cuda(sumsq, torch.float32, "sumsq")
    assert state.numel() == LOSS_SCALE_STATE_WORDS and state.is_contiguous() and sumsq.numel() == 1
    _check(_lib.load().mm_loss_scale_update(state.data_ptr(), sumsq.data_ptr(), float(max_norm or 0.0), int(dynamic),
                                            int(window), int(hysteresis), float(min_scale), _stream()),
           "mm_loss_scale_update")


def cast_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp16 contiguous tensor -> bf16 copy (mm_cast_f16_bf16): the alignment backward of a bf16 model runs in bf16."""
    _cuda(x, _F16, "x")
    assert x.is_contiguous()
    cols = x.shape[-1]
    rows = x.numel() // cols
    y = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    _check(_lib.load().mm_cast_f16_bf16(x.data_ptr(), cols, y.data_ptr(), cols, rows, cols, _stream()), "mm_cast_f16_bf16")
    return y


def align_dropout_fwd(P_unnorm: torch.Tensor, inv_l: torch.Tensor, pe: torch.Tensor, V: int, dropout):
    """Training-mode dropout of the alignment probabilities -> (Pm fp16 (R, ldp) kept entries, rs (R,) = (1/l)/(1-p),
    p_sum_real_d (R,), p_extra_d (R,)); see mm_align_dropout_fwd."""
    _cuda(P_unnorm, _F16, "P")
    R, ldp = P_unnorm.shape
    dev = P_unnorm.device
    Pm = torch.empty_like(P_unnorm)
    rs, psum_d, pext_d = (torch.empty((R,), device=dev, dtype=torch.float32) for _ in range(3))
    pd, seed, sid = _drop_args(dropout)
    _check(_lib.load().mm_align_dropout_fwd(P_unnorm.data_ptr(), Pm.data_ptr(), ldp, inv_l.data_ptr(), pe.data_ptr(),
                                            rs.data_ptr(), psum_d.data_ptr(), pext_d.data_ptr(), R, V, pd, seed, sid,
                                            _stream()), "mm_align_dropout_fwd")
    return Pm, rs, psum_d, pext_d


def align_softmax_bwd(G: torch.Tensor, P_unnorm: torch.Tensor, inv_l: torch.Tensor, dpsr: torch.Tensor, pe: torch.Tensor,
                      dpe: torch.Tensor, gscale: float, V: int, dropout=None):
    """-> (Pd (R, ldp), dS (R, ldp) in the activation format, dstats fp32 (2, R)); see mm_align_softmax_bwd."""
    _cuda(G, torch.float32, "G"); _cuda(P_unnorm, _F16, "P")
    R, ldp = P_unnorm.shape
    assert G.shape[0] == R and G.stride(1) == 1 and P_unnorm.stride(1) == 1
    for t in (inv_l, dpsr, pe, dpe):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == R
    P = torch.empty((R, ldp), device=G.device, dtype=ACT())
    dS = torch.empty((R, ldp), device=G.device, dtype=ACT())
    dstats = torch.empty((2, R), device=G.device, dtype=torch.float32)
    pd, seed, sid = _drop_args(dropout)
    _check(_lib.load().mm_align_softmax_bwd(G.data_ptr(), G.stride(0), P_unnorm.data_ptr(), ldp, inv_l.data_ptr(), dpsr.data_ptr(),
                                            pe.data_ptr(), dpe.data_ptr(), float(gscale), P.data_ptr(), dS.data_ptr(), ldp,
                                            dstats.data_ptr(), R, V, pd, seed, sid, _stream()), "mm_align_softmax_bwd")
    return P, dS, dstats


def head_weighted_colsum(x: torch.Tensor, w: torch.Tensor, head_dim: int, out: torch.Tensor) -> torch.Tensor:
    """out[h*hd + d] += sum_n w[h, n] * x[n, h*hd + d]; x (Nq, E) bf16 / fp16, w (H*Nq,) fp32 contiguous, out fp32 (E,)."""
    _cuda(x, None, "x"); _cuda(w, torch.float32, "w"); _cuda(out, torch.float32, "out")
    assert x.dtype in _16BIT and x.stride(1) == 1 and w.is_contiguous()
    Nq, E = x.shape
    assert w.numel() == (E // head_dim) * Nq and out.numel() == E
    _check(_lib.load().mm_head_weighted_colsum(x.data_ptr(), x.stride(0), int(x.dtype == _F16), w.data_ptr(), 1, Nq, E,
                                               head_dim, out.data_ptr(), _stream()), "mm_head_weighted_colsum")
    return out


def window_gather_add(dwin: torch.Tensor, B: int, N: int, C: int, Lq: int, kk: int, ss: int) -> torch.Tensor:
    """Conv1d data gradient: dwin (B*Lq, kk*C) -> dfeats (B, N, C), both in the activation format (mm_window_gather_add)."""
    _cuda(dwin, ACT(), "dwin")
    assert dwin.is_contiguous() and dwin.shape == (B * Lq, kk * C)
    out = torch.empty((B, N, C), device=dwin.device, dtype=ACT())
    _check(_lib.load().mm_window_gather_add(dwin.data_ptr(), B, N, C, Lq, kk, ss, out.data_ptr(), _stream()),
           "mm_window_gather_add")
    return out


# ---------------------------------------------------------------------------------------------------- LoRA adapters
def _lora_args(M: int, K: int, N: int, r: int, n: int, scaling: float = 1.0, dropout=None) -> "_lib.LoraArgs":
    """mm_lora_args for n adapters; dropout = None | (p, seed_dev int64 (1,), [stream id per adapter])."""
    assert 1 <= n <= _lib.LORA_MAX
    a = _lib.LoraArgs()
    a.n, a.M, a.K, a.N, a.r, a.scaling = n, M, K, N, r, float(scaling)
    if dropout is not None and float(dropout[0]) > 0.0:
        p, seed, sids = dropout
        _cuda(seed, torch.int64, "seed")
        assert seed.numel() == 1 and len(sids) == n
        a.p_drop, a.seed_dev = float(p), seed.data_ptr()
        for j, s in enumerate(sids):
            a.sid[j] = int(s)
    return a


def _lora_weights(As, Bs):
    for A in As:
        _cuda(A, ACT(), "lora_A")
        assert A.is_contiguous()
    for Bw in Bs:
        _cuda(Bw, ACT(), "lora_B")
        assert Bw.is_contiguous()


def lora_down(x: torch.Tensor, As, dropout=None):
    """u_j (M, r) fp32 = drop_j(x) A_j^T for adapters sharing the input x (M, K) (mm_lora_down); As: lora_A weights (r, K)."""
    _cuda(x, ACT(), "x")
    _lora_weights(As, ())
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    r = As[0].shape[0]
    assert all(A.shape == (r, K) for A in As)
    a = _lora_args(M, K, 1, r, len(As), dropout=dropout)
    a.x, a.ldx = x.data_ptr(), x.stride(0)
    us = [torch.empty((M, r), device=x.device, dtype=torch.float32) for _ in As]
    for j, (A, u) in enumerate(zip(As, us)):
        a.A[j], a.u[j] = A.data_ptr(), u.data_ptr()
    _check(_lib.load().mm_lora_down(C.byref(a), _stream()), "mm_lora_down")
    return us


def lora_up(ys, us, Bs, scaling: float, rope=None) -> None:
    """In place: y_j <- round(rope(y_j + scaling u_j B_j^T)) (mm_lora_up); ys (M, N) 16-bit views with unit inner stride and
    one row stride, us (M, r) fp32, Bs lora_B weights (N, r); rope = (cos, sin, T) applies RoPE over 128-wide heads."""
    _lora_weights((), Bs)
    M, N = ys[0].shape
    r = Bs[0].shape[1]
    for y, u, Bw in zip(ys, us, Bs):
        _cuda(y, ACT(), "y"); _cuda(u, torch.float32, "u")
        assert y.shape == (M, N) and y.stride(1) == 1 and y.stride(0) == ys[0].stride(0)
        assert u.shape == (M, r) and u.is_contiguous() and Bw.shape == (N, r)
    a = _lora_args(M, 8, N, r, len(ys), scaling)
    a.ldy = ys[0].stride(0)
    for j, (y, u, Bw) in enumerate(zip(ys, us, Bs)):
        a.y[j], a.u[j], a.B[j] = y.data_ptr(), u.data_ptr(), Bw.data_ptr()
    if rope is not None:
        cos, sin, T = rope
        a.rope_cos, a.rope_sin, a.rope_T = cos.data_ptr(), sin.data_ptr(), int(T)
    _check(_lib.load().mm_lora_up(C.byref(a), _stream()), "mm_lora_up")


def lora_bwd_dy(dys, us, Bs, dBs, scaling: float, accumulate):
    """g_j (M, r) fp32 = scaling dy_j B_j and dB_j (+)= scaling dy_j^T u_j (mm_lora_bwd_dy) -> [g_j]; dBs: gradient views
    (N, r) in the activation format, accumulate[j]: add into dB_j instead of overwriting it."""
    _lora_weights((), Bs)
    M, N = dys[0].shape
    r = Bs[0].shape[1]
    for dy, u, Bw, dB in zip(dys, us, Bs, dBs):
        _cuda(dy, ACT(), "dy"); _cuda(u, torch.float32, "u"); _cuda(dB, ACT(), "dB")
        assert dy.shape == (M, N) and dy.stride(1) == 1 and dy.stride(0) == dys[0].stride(0)
        assert u.shape == (M, r) and u.is_contiguous() and Bw.shape == (N, r) and dB.shape == (N, r) and dB.is_contiguous()
    a = _lora_args(M, 8, N, r, len(dys), scaling)
    a.ldy = dys[0].stride(0)
    gs = [torch.empty((M, r), device=dys[0].device, dtype=torch.float32) for _ in dys]
    for j, (dy, u, Bw, dB, g) in enumerate(zip(dys, us, Bs, dBs, gs)):
        a.y[j], a.u[j], a.B[j], a.dB[j], a.g[j] = dy.data_ptr(), u.data_ptr(), Bw.data_ptr(), dB.data_ptr(), g.data_ptr()
        a.accumulate[j] = int(bool(accumulate[j]))
    lib = _lib.load()
    ws = torch.empty(((int(lib.mm_lora_workspace_bytes(C.byref(a), 2)) + 15) // 16 * 4,), device=dys[0].device,
                     dtype=torch.float32)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel() * 4
    _check(lib.mm_lora_bwd_dy(C.byref(a), _stream()), "mm_lora_bwd_dy")
    return gs


def lora_bwd_x(x: torch.Tensor, gs, As, dAs, dx: torch.Tensor, accumulate, dropout=None) -> None:
    """dA_j (+)= g_j^T drop_j(x) and, in place, dx <- round(dx + sum_j drop_j(g_j A_j)) for adapters sharing the input x
    (mm_lora_bwd_x); dropout as in lora_down (the same masks)."""
    _cuda(x, ACT(), "x"); _cuda(dx, ACT(), "dx")
    _lora_weights(As, ())
    M, K = x.shape
    r = As[0].shape[0]
    assert x.stride(1) == 1 and dx.shape == (M, K) and dx.stride(1) == 1
    for g, A, dA in zip(gs, As, dAs):
        _cuda(g, torch.float32, "g"); _cuda(dA, ACT(), "dA")
        assert g.shape == (M, r) and g.is_contiguous() and A.shape == (r, K) and dA.shape == (r, K) and dA.is_contiguous()
    a = _lora_args(M, K, 1, r, len(As), dropout=dropout)
    a.x, a.ldx, a.dx, a.lddx = x.data_ptr(), x.stride(0), dx.data_ptr(), dx.stride(0)
    for j, (g, A, dA) in enumerate(zip(gs, As, dAs)):
        a.g[j], a.A[j], a.dA[j] = g.data_ptr(), A.data_ptr(), dA.data_ptr()
        a.accumulate[j] = int(bool(accumulate[j]))
    lib = _lib.load()
    ws = torch.empty(((int(lib.mm_lora_workspace_bytes(C.byref(a), 3)) + 15) // 16 * 4,), device=x.device,
                     dtype=torch.float32)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel() * 4
    _check(lib.mm_lora_bwd_x(C.byref(a), _stream()), "mm_lora_bwd_x")


# ---------------------------------------------------------------------------------------------------- JPEG decode
def jpeg_decode(data: torch.Tensor, desc: torch.Tensor, layout: dict):
    """mm_jpeg_decode over a packed batch (jpeg.pack): `data` the scan bytes and `desc` the descriptor bytes, both uint8
    device tensors.  Allocates the coefficient, plane and output buffers; returns (out uint8, status int32 per image)
    without synchronising."""
    _cuda(data, torch.uint8, "data"); _cuda(desc, torch.uint8, "desc")
    dev = data.device
    coef = torch.empty(layout["coef"], dtype=torch.int16, device=dev)
    planes = torch.empty(layout["planes"], dtype=torch.uint8, device=dev)
    out = torch.empty(layout["out"], dtype=torch.uint8, device=dev)
    status = torch.empty(layout["n_images"], dtype=torch.int32, device=dev)
    base, off = desc.data_ptr(), layout["off"]
    a = _lib.JpegArgs(layout["n_images"], layout["n_segments"], layout["n_huff"], layout["n_quant"], data.data_ptr(),
                      layout["data_bytes"], base + off["images"], base + off["segments"], base + off["huff"],
                      base + off["quant"], coef.data_ptr(), coef.numel(), planes.data_ptr(), planes.numel(),
                      out.data_ptr(), out.numel(), status.data_ptr(), layout["max_blocks"], layout["max_pixels"])
    _check(_lib.load().mm_jpeg_decode(C.byref(a), _stream()), "mm_jpeg_decode")
    return out, status
