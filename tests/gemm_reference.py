"""fp64 restatement of mm_gemm_fwd (ops.gemm_raw) and a per-element error bar for it.

gemm_ref() computes, in float64 from the exact 16-bit operands, what the GEMM is defined to return: the product, the
row scale (row_scale / the RMSNorm statistic from rs_sumsq), alpha, bias or the alignment's row-scaled bias pair,
the exact activation (erf-GELU, x sigma(1.702 x), x sigma(x)), the residual, SwiGLU on the [32 gate | 32 up]
interleaved columns, RoPE from the fp32 cos / sin tables the kernel is handed, and the transposed store of a c_trans
launch.  Next to the value it returns the bound on |kernel - value| that an honest fp32 implementation meets:

  bar = half an ulp of the output format at |ref|                                     (output rounding, 0 for fp32)
      + KAPPA 2^-24 sqrt(K) (|A| |B|^T), carried through the epilogue by |d out / d acc| (tensor-core accumulation)
      + EPI_ULPS fp32 ulps of every epilogue operation, carried the same way            (epilogue evaluation)

with sigma's own allowance of (5 + 1.2 |z|) ulps (CUDA's documented __expf bound, a rounded add and an approximate
reciprocal) and erfc's of a few ulps plus the rounding of its exponent's argument (about 1.5 x^2 ulps).  A kernel
passes when max |got - ref| / bar <= 1.  All of it runs on whatever device the operands are on.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

ACT_NONE, ACT_GELU, ACT_QUICK_GELU, ACT_SILU = 0, 1, 2, 3
EPI_STD, EPI_SWIGLU, EPI_ROPE = 0, 1, 2

U = 2.0 ** -24  # unit roundoff of fp32
# Accumulation constant.  Mode-0 launches with fp32 output at K = 11008, the largest K of the table (down_fp32_*), on an
# H100 80GB HBM3 (700 W limit): the worst element reached 0.17 (bf16) and 0.19 (fp16) of 2^-24 sqrt(K) (|A| |B|^T).
KAPPA = 1.0
EPI_ULPS = 4.0  # fp32 ulps allowed per epilogue operation (one rounding is 0.5)


def half_ulp(x: torch.Tensor, fmt) -> torch.Tensor:
    """Half an ulp of `fmt` (torch.bfloat16 | torch.float16 | torch.float32 -> 0) at |x| (float64), with the format's
    subnormal floor: the largest error of one round-to-nearest into `fmt` of a value of magnitude |x|."""
    if fmt == torch.float32:
        return torch.zeros_like(x)
    mant, emin = {torch.bfloat16: (8, -126), torch.float16: (11, -14)}[fmt]
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** (emin - 1))))
    return torch.exp2(torch.clamp(e, min=emin) - mant)


def _sigmoid(z):
    return torch.sigmoid(z)


def _act(x: torch.Tensor, act: int):
    """(value, |d value / dx|, evaluation error bound) of the exact activation at fp64 x."""
    if act == ACT_NONE:
        return x, torch.ones_like(x), torch.zeros_like(x)
    if act == ACT_GELU:
        phi = 0.5 * torch.special.erfc(-x / math.sqrt(2.0))
        dens = torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
        y = x * phi
        # a few ulps per operation, and the rounding of erfc's exponent argument -z^2 + P (z = |x| / sqrt 2, ~ z^2 ulps,
        # plus z's own rounding carried by d log erfc / dz ~ 2 z): 3 x^2 ulps
        return y, (phi + x * dens).abs(), U * (EPI_ULPS * 6 + 3 * x * x) * y.abs()
    a = 1.702 if act == ACT_QUICK_GELU else 1.0
    z = a * x
    s = _sigmoid(z)
    y = x * s
    d = (s + z * s * (1 - s)).abs()
    sig_rel = U * (5.0 + 1.2 * z.abs()) * 2  # (5 + 1.2|z|) ulps of 2^-23
    return y, d, (EPI_ULPS * U * 2 + sig_rel) * y.abs() + EPI_ULPS * U * (x.abs() * d)


@dataclass
class Ref:
    value: torch.Tensor   # fp64, in the layout of the stored output (rows, cols) of each batch entry
    bar: torch.Tensor     # fp64, same shape


def gemm_ref(*, A: torch.Tensor, B: torch.Tensor, a_mn_major: bool = False, b_mn_major: bool = False,
             out_fmt=torch.bfloat16, epi: int = EPI_STD, act: int = ACT_NONE, alpha: float = 1.0,
             bias: Optional[torch.Tensor] = None, row_scale: Optional[torch.Tensor] = None,
             rs_sumsq: Optional[torch.Tensor] = None, rs_eps: float = 0.0,
             residual: Optional[torch.Tensor] = None, res_row_mod: int = 0,
             bias_rs: Optional[torch.Tensor] = None, bias2: Optional[torch.Tensor] = None,
             bias2_rs: Optional[torch.Tensor] = None,
             rope_cos: Optional[torch.Tensor] = None, rope_sin: Optional[torch.Tensor] = None, rope_T: int = 1,
             rope_cols: int = 0, rope_pos: int = 0, c_trans: bool = False, kappa: float = KAPPA) -> Ref:
    """fp64 value and error bar of C = epilogue(alpha A B^T) as mm_gemm_fwd defines it.

    Operands are batched views: A (..., M, K) (a_mn_major: (..., K, M), as gemm_dw reads dy), B (..., N, K)
    (b_mn_major: (..., K, N), as gemm_dx / gemm_dw read w and x); leading dimensions broadcast, so a B with one batch
    entry is the shared B of b_bs = 0.  Per-output tensors are given in the output's broadcast shape:
      bias (..., N)            per column (bias_bs: its leading dimension), or per OUTPUT FEATURE with c_trans
      row_scale (..., M)       fp32, per row of A (with c_trans: per activation row, the kernel's tile column)
      rs_sumsq (M, parts)      fp32 partial sums of squares: row scale rsqrt(sum / K + rs_eps) (in fp64)
      residual (..., M, N)     added after the activation (res_row_mod: rows m % res_row_mod of a (..., mod, N) tensor)
      bias_rs / bias2_rs (..., M) fp32 and bias2 (..., N): out += bias_rs * bias + bias2_rs * bias2
      rope_cos / rope_sin (T, 64) fp32: pairs (i, i + 64) of every 128-column head below rope_cols rotated at position
                               m % rope_T + rope_pos
    c_trans: A is the weight (N_out, K), B the activation rows (M_act, K); the result is (M_act, N_out), as linear_thin
    stores it.  The returned value has the stored output's shape: (..., M, N), (..., M, N / 2) for SwiGLU."""
    f = torch.float64
    a = A.to(f)
    b = B.to(f)
    if a_mn_major:
        a = a.transpose(-1, -2)
    if b_mn_major:
        b = b.transpose(-1, -2)
    K = a.shape[-1]
    acc = torch.matmul(a, b.transpose(-1, -2))
    mag = torch.matmul(a.abs(), b.abs().transpose(-1, -2))
    e_acc = kappa * U * math.sqrt(K) * mag
    if c_trans:  # kernel tile: rows = output features, columns = activation rows; restate in the stored layout
        acc, e_acc = acc.transpose(-1, -2), e_acc.transpose(-1, -2)
    M = acc.shape[-2]

    rs = torch.full(acc.shape[:-1] + (1,), float(alpha), dtype=f, device=acc.device)
    e_rs_rel = 0.0
    if row_scale is not None:
        rs = rs * row_scale.to(f)[..., None]
        e_rs_rel = EPI_ULPS * U
    if rs_sumsq is not None:
        rs = rs * torch.rsqrt(rs_sumsq.to(f).sum(-1) / K + float(rs_eps))[..., None]
        e_rs_rel = EPI_ULPS * U * (2 + rs_sumsq.shape[-1] / 4)  # fp32 sum of the partials, divide, rsqrtf
    v = acc * rs
    e = e_acc * rs.abs() + (e_rs_rel + EPI_ULPS * U) * v.abs()

    if epi == EPI_SWIGLU:
        N = v.shape[-1]
        g = v.reshape(v.shape[:-1] + (N // 64, 2, 32))
        eg = e.reshape(g.shape)
        gate, up = g[..., 0, :], g[..., 1, :]
        s = _sigmoid(gate)
        silu = gate * s
        out = silu * up
        d_gate = (s + gate * s * (1 - s)).abs() * up.abs()
        sig_rel = U * (5.0 + 1.2 * gate.abs()) * 2
        err = (d_gate * eg[..., 0, :] + silu.abs() * eg[..., 1, :]
               + (EPI_ULPS * U * 3 + sig_rel) * out.abs())
        value, err = out.reshape(v.shape[:-1] + (N // 2,)), err.reshape(v.shape[:-1] + (N // 2,))
    elif epi == EPI_ROPE:
        N = v.shape[-1]
        pos = (torch.arange(M, device=v.device) % rope_T) + int(rope_pos)
        c = rope_cos.to(f)[pos][:, None, :]  # (M, 1, 64)
        sn = rope_sin.to(f)[pos][:, None, :]
        h = v.reshape(v.shape[:-1] + (N // 128, 2, 64))
        eh = e.reshape(h.shape)
        x1, x2 = h[..., 0, :], h[..., 1, :]
        o1 = x1 * c - x2 * sn
        o2 = x2 * c + x1 * sn
        e1 = eh[..., 0, :] * c.abs() + eh[..., 1, :] * sn.abs() + EPI_ULPS * U * 2 * ((x1 * c).abs() + (x2 * sn).abs())
        e2 = eh[..., 1, :] * c.abs() + eh[..., 0, :] * sn.abs() + EPI_ULPS * U * 2 * ((x2 * c).abs() + (x1 * sn).abs())
        rot = (torch.arange(N // 128, device=v.device) * 128 < rope_cols)[:, None]
        value = torch.stack([torch.where(rot, o1, x1), torch.where(rot, o2, x2)], -2).reshape(v.shape)
        err = torch.stack([torch.where(rot, e1, eh[..., 0, :]), torch.where(rot, e2, eh[..., 1, :])], -2).reshape(v.shape)
    else:
        if bias_rs is not None or bias2 is not None:
            s1 = bias_rs.to(f)[..., None] if bias_rs is not None else 1.0
            s2 = bias2_rs.to(f)[..., None] if bias2_rs is not None else 1.0
            t1 = s1 * bias.to(f)[..., None, :] if bias is not None else torch.zeros_like(v)
            t2 = s2 * bias2.to(f)[..., None, :] if bias2 is not None else torch.zeros_like(v)
            v = v + t1 + t2
            e = e + EPI_ULPS * U * (v.abs() + t1.abs() + t2.abs())
        elif bias is not None:
            v = v + bias.to(f)[..., None, :]  # per stored column: the output feature, also with c_trans
            e = e + EPI_ULPS * U * v.abs()
        value, d, e_act = _act(v, act)
        err = e * d + e_act
        if residual is not None:
            r = residual.to(f)
            if res_row_mod:
                r = r[..., torch.arange(M, device=v.device) % res_row_mod, :]
            value = value + r
            err = err + EPI_ULPS * U * (value.abs() + r.abs())
    return Ref(value, err + half_ulp(value.abs() + err, out_fmt))


def ratio(got: torch.Tensor, ref: Ref) -> torch.Tensor:
    """|got - ref| / bar per element (fp64); a non-finite output is an infinite ratio."""
    g = got.to(torch.float64)
    r = (g - ref.value).abs() / ref.bar
    return torch.where(torch.isfinite(g), r, torch.full_like(r, float("inf")))


def worst(got: torch.Tensor, ref: Ref):
    """(max ratio, index of the worst element, got there, ref there)."""
    r = ratio(got, ref)
    i = int(torch.argmax(r.reshape(-1)))
    idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), r.shape))
    return float(r.reshape(-1)[i]), idx, float(got.reshape(-1)[i]), float(ref.value.reshape(-1)[i])


def sumsq_ref(stored: torch.Tensor) -> torch.Tensor:
    """fp64 per-(row, 32-column chunk) sums of squares of the outputs AS STORED (M, N) -> (M, ceil(N / 32))."""
    x = stored.to(torch.float64)
    M, N = x.shape
    pad = (-N) % 32
    if pad:
        x = torch.nn.functional.pad(x, (0, pad))
    return (x * x).reshape(M, -1, 32).sum(-1)


def sumsq_bar(stored: torch.Tensor) -> torch.Tensor:
    """Bound on an fp32 fused-multiply-add chain over each chunk of 32 squares: 32 roundings of the running sum."""
    return 32 * U * sumsq_ref(stored) + 1e-300
