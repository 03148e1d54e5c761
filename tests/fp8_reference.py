"""The per-row e4m3 rule and the e4m3 GEMM restated on any device, for the FP8 tests.

Rule (weights and activation rows alike): v = fp32(x) * fp32(g), s = fp32(max |v|) / 448 (IEEE division),
q = e4m3(v / s) rounded to nearest even and saturated, q = 0 where s = 0.  Inside |v / s| <= 448 (up to one rounding)
torch's float8_e4m3fn cast is that rounding, so the restatement uses it.
"""
from __future__ import annotations

import torch

E4M3 = torch.float8_e4m3fn


def quantize_ref(x: torch.Tensor, gain: torch.Tensor | None = None):
    """-> (q float8_e4m3fn (rows, K), s fp32 (rows,))."""
    v = x.float()
    if gain is not None:
        v = v * gain.float()[None, :]
    s = v.abs().amax(1) / torch.tensor(448.0, dtype=torch.float32, device=v.device)
    zero = s == 0
    q = torch.where(zero[:, None], 0.0, v / torch.where(zero, 1.0, s)[:, None]).clamp(-448.0, 448.0).to(E4M3)
    return q, s


def gemm_ref(qx, sx, qw, sw):
    """fp64 (q_x s_x)(q_w s_w)^T and the magnitude (|q_x| s_x)(|q_w| s_w)^T of the bound."""
    a = qx.double() * sx.double()[:, None]
    b = qw.double() * sw.double()[:, None]
    return a @ b.T, a.abs() @ b.abs().T


def half_ulp(y: torch.Tensor, dt) -> torch.Tensor:
    """Half an ulp of dt at |y| (fp16's subnormal floor included)."""
    y = y.abs().clamp_min(torch.finfo(dt).tiny if dt == torch.bfloat16 else 2.0 ** -14)
    e = torch.floor(torch.log2(y))
    p = {torch.bfloat16: 8, torch.float16: 11, torch.float32: 24}[dt]
    return torch.pow(2.0, e - p)
