"""CPU tier: the fp64 GEMM restatement (tests/gemm_reference.py) against plain torch fp64 ops, its output-rounding bar
against round-to-nearest, and the fp64 case table's coverage of every GEMM kernel instance (tests/gemm_cases.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import gemm_cases as G
from tests import gemm_reference as R
from tests.decode_reference import CachedDecoder, rope_tables

D = torch.float64


def _rnd(*s, dt=torch.bfloat16, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(dt)


@pytest.mark.parametrize("act,fn", [(R.ACT_NONE, lambda x: x), (R.ACT_GELU, F.gelu), (R.ACT_SILU, F.silu),
                                    (R.ACT_QUICK_GELU, lambda x: x * torch.sigmoid(1.702 * x))])
def test_standard_epilogue_matches_torch(act, fn):
    A, B = _rnd(3, 37, 72, seed=1), _rnd(3, 29, 72, seed=2, scale=0.3)
    bias, res = _rnd(3, 29, seed=3), _rnd(3, 37, 29, seed=4)
    rs = torch.rand(3, 37, dtype=torch.float32) + 0.5
    got = R.gemm_ref(A=A, B=B, act=act, alpha=0.7, bias=bias, row_scale=rs, residual=res).value
    want = fn(torch.bmm(A.to(D), B.to(D).transpose(1, 2)) * 0.7 * rs.to(D)[..., None] + bias.to(D)[:, None]) + res.to(D)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)


def test_mn_major_ctrans_shared_b_and_row_mod():
    dy, w = _rnd(40, 24, seed=5), _rnd(24, 56, seed=6)
    assert torch.allclose(R.gemm_ref(A=dy, B=w, b_mn_major=True).value, dy.to(D) @ w.to(D))             # gemm_dx
    x = _rnd(40, 56, seed=7)
    assert torch.allclose(R.gemm_ref(A=dy, B=x, a_mn_major=True, b_mn_major=True).value, dy.to(D).T @ x.to(D))  # gemm_dw
    xt, wt, b, r = _rnd(8, 64, seed=8), _rnd(96, 64, seed=9), _rnd(96, seed=10), _rnd(8, 96, seed=11)
    rs = torch.rand(8) + 0.5
    got = R.gemm_ref(A=wt, B=xt, c_trans=True, bias=b, row_scale=rs, residual=r, act=R.ACT_SILU).value  # linear_thin
    want = F.silu(xt.to(D) @ wt.to(D).T * rs.to(D)[:, None] + b.to(D)) + r.to(D)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)
    A4, Bs = _rnd(2, 3, 16, 32, seed=12), _rnd(40, 32, seed=13)   # batch2 x batch, shared B (b_bs = 0)
    bias = _rnd(3, 40, seed=14)                                   # bias_bs = N
    res = _rnd(5, 40, seed=15)                                    # res_row_mod = 5
    got = R.gemm_ref(A=A4, B=Bs, bias=bias, residual=res, res_row_mod=5).value
    want = A4.to(D) @ Bs.to(D).T + bias.to(D)[:, None, :] + res.to(D)[torch.arange(16) % 5]
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)


def test_alignment_bias_pair_and_rms_statistic():
    H, M, hd, K = 4, 10, 16, 48
    A, B = _rnd(H, M, K, seed=16, dt=torch.float16), _rnd(H, hd, K, seed=17, dt=torch.float16)
    b1, b2 = _rnd(H, hd, seed=18, dt=torch.float16), _rnd(H, hd, seed=19, dt=torch.float16)
    s1, s2 = torch.rand(H, M), torch.rand(H, M)
    got = R.gemm_ref(A=A, B=B, out_fmt=torch.float16, bias=b1, bias_rs=s1, bias2=b2, bias2_rs=s2).value
    want = torch.bmm(A.to(D), B.to(D).transpose(1, 2)) + s1.to(D)[..., None] * b1.to(D)[:, None] + \
        s2.to(D)[..., None] * b2.to(D)[:, None]
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)
    x, w = _rnd(6, 64, seed=20), _rnd(12, 64, seed=21)
    parts = torch.rand(6, 8) * 10
    got = R.gemm_ref(A=x, B=w, rs_sumsq=parts, rs_eps=1e-5).value
    want = (x.to(D) @ w.to(D).T) / torch.sqrt(parts.to(D).sum(-1, keepdim=True) / 64 + 1e-5)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)


def test_swiglu_and_rope_epilogues():
    x, w = _rnd(5, 64, seed=22), _rnd(128, 64, seed=23, scale=0.5)
    got = R.gemm_ref(A=x, B=w, epi=R.EPI_SWIGLU).value
    h = (x.to(D) @ w.to(D).T).view(5, 2, 2, 32)            # [32 gate | 32 up] per 64-column unit
    assert torch.allclose(got, (F.silu(h[:, :, 0]) * h[:, :, 1]).reshape(5, 64), rtol=1e-13, atol=1e-13)
    M, T, pos0 = 7, 4, 3
    x, w = _rnd(M, 64, seed=24), _rnd(3 * 128, 64, seed=25)
    cos, sin = rope_tables(T + pos0, 128)                  # the oracle's fp32 tables
    got = R.gemm_ref(A=x, B=w, epi=R.EPI_ROPE, rope_cos=cos, rope_sin=sin, rope_T=T, rope_cols=256, rope_pos=pos0).value
    y = (x.to(D) @ w.to(D).T).view(M, 3, 128)
    ppos = torch.arange(M) % T + pos0
    c = torch.cat([cos, cos], -1).to(D)[ppos][:, None]
    s = torch.cat([sin, sin], -1).to(D)[ppos][:, None]
    q = y[:, :2]
    rot = CachedDecoder._rot(type("H", (), {"hd": 128})(), q)  # the decode reference's rotate-half
    want = torch.cat([q * c + rot * s, y[:, 2:]], 1).reshape(M, 384)
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)


def _round_bf16(x: torch.Tensor) -> torch.Tensor:
    """float64 -> bf16 rounded once, to nearest (ties to even), for normal values."""
    m, e = torch.frexp(x)                         # x = m 2^e, 0.5 <= |m| < 1: bf16 keeps 8 significant bits of m
    return torch.ldexp(torch.round(torch.ldexp(m, torch.full_like(e, 8))), e - 8).to(torch.bfloat16)


@pytest.mark.parametrize("fmt", [torch.bfloat16, torch.float16])
def test_output_rounding_bar_is_exact_for_round_to_nearest(fmt):
    g = torch.Generator().manual_seed(26)
    ref = torch.randn(20000, generator=g, dtype=D) * torch.exp2(torch.randint(-30, 12, (20000,), generator=g).to(D))
    if fmt == torch.float16:
        ref = ref.clamp(-60000, 60000)
    bar = R.half_ulp(ref.abs(), fmt)
    if fmt == torch.float16:  # numpy rounds float64 to half once (torch goes through fp32: a double rounding)
        r = torch.from_numpy(ref.numpy().astype(np.float16))
    else:  # bf16: fp64 -> fp32 is exact for these values' 8-bit significands only after the second step; round by hand
        r = _round_bf16(ref)
    assert bool((((r.to(D) - ref).abs() / bar) <= 1).all())           # one rounding: ratio <= 1
    bits = r.view(torch.int16)
    for step in (1, -1):                                              # either 16-bit neighbour: ratio > 1
        nb = (bits + step).view(fmt).to(D)
        ok = torch.isfinite(nb) & (r != 0)
        assert bool((((nb - ref).abs() / bar)[ok] > 1).all())


def test_case_table_covers_every_instance():
    """Planned with the no-device SM count, the table reaches all 42 kernel instances, stream-K with each epilogue and
    with MN-major operands, and the scalar epilogue with bias, residual, fp32 output and a partial last chunk."""
    from macaw_llm_b200 import ops

    if torch.cuda.is_available():
        pytest.skip("the device's own SM count is covered by test_gemm_fp64_gpu.py::test_coverage_at_device_sm_count")
    seen, sk, scalar = {}, set(), set()
    for c in G.CASES:
        ops.set_act_format(torch.float16 if c.fmt == G.F16 else torch.bfloat16)
        pl = G.plan(c, G.fake_ptrs())
        inst = G.instance(c, pl)
        seen.setdefault(inst, []).append(c.name)
        if pl["streamk_tiles"] > 0:
            sk.add(c.epi)
            if c.kind in ("dx", "dw"):
                sk.add("mn_major")
        if not pl["vectorised_epilogue"]:
            scalar.update(k for k, on in (("bias", c.bias), ("residual", c.residual), ("fp32", c.out == "fp32"),
                                          ("partial_chunk", c.n_out % 32 != 0)) if on)
    ops.set_act_format(torch.bfloat16)
    for inst in sorted(seen, key=str):
        print(inst, seen[inst])
    missing = G.all_instances() - set(seen)
    assert not missing, f"no case launches {sorted(missing, key=str)}"
    assert len(G.all_instances()) == 42
    assert sk == {ops.EPI_STD, ops.EPI_SWIGLU, ops.EPI_ROPE, "mn_major"}, sk
    assert scalar == {"bias", "residual", "fp32", "partial_chunk"}, scalar
