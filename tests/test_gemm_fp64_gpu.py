"""Every GEMM kernel instance against the fp64 restatement, element by element (tests/gemm_reference.py).

Each case of tests/gemm_cases.py sets its modes and activation format, launches through the public wrapper (ops.linear,
linear_thin, gemm_dx, gemm_dw) or gemm_raw (batched and alignment layouts), checks from the profiler's kernel name that
the launched template equals the plan's prediction, and requires |got - ref| <= bar at every element.  The worst ratio
and where it sits are printed.  The coverage test re-plans the table at the device's SM count.
"""
import math
import re
import zlib

import pytest
import torch

from tests import gemm_cases as G
from tests import gemm_reference as R

DEV = "cuda"


def _ops():
    from macaw_llm_b200 import ops

    return ops


def _lib():
    from macaw_llm_b200 import _lib

    return _lib.load()


def _launched():
    """Context: the template arguments of every GEMM kernel launched inside, parsed from the profiler's names."""
    from torch.profiler import ProfilerActivity, profile

    return profile(activities=[ProfilerActivity.CUDA])


def _parse(prof):
    def b(s):
        return s.strip() == "true"

    out = set()
    for ev in prof.events():
        m = re.search(r"gemm_wide_kernel<([^>]*)>", ev.name)
        if m:
            a = [s.strip() for s in m.group(1).split(",")]
            out.add(("wide", int(a[0].rstrip("u")), b(a[1])))
        m = re.search(r"gemm_bf16_kernel<([^>]*)>", ev.name)
        if m:
            a = [s.strip() for s in m.group(1).split(",")]
            out.add(("tile", int(a[0].rstrip("u")), int(a[1].rstrip("u")), b(a[2]), b(a[3]), b(a[4]), b(a[5])))
    return out


def _inputs(c: G.Case, seed: int):
    """Device tensors of case c (16-bit operands, fp32 side inputs) and their base addresses for raw_args()."""
    ops = _ops()
    dt = torch.float16 if c.fmt == G.F16 else torch.bfloat16
    g = torch.Generator(device=DEV).manual_seed(seed)

    def rn(*s, scale=1.0):
        return (torch.randn(*s, device=DEV, generator=g) * scale).to(dt)

    t = {}
    n_out = c.n_out
    odt = torch.float32 if c.out == "fp32" else dt
    if c.kind in ("linear", "thin"):
        t["x"] = rn(c.M, c.K)
        t["w"] = rn(c.N, c.K, scale=c.gate_std / math.sqrt(c.K))
        rows = c.M
        t["outbuf"] = torch.zeros(rows, c.ldc, device=DEV, dtype=odt)
        t["out"] = t["outbuf"][:, c.c_off:c.c_off + n_out]
    elif c.kind == "dx":  # dy (M, N), w (N, K) -> (M, K)
        t["x"] = rn(c.M, c.N)
        t["w"] = rn(c.N, c.K, scale=1 / math.sqrt(c.N))
        t["out"] = rn(c.M, c.K) if c.residual else torch.zeros(c.M, c.K, device=DEV, dtype=dt)
    elif c.kind == "dw":  # dy (M, N), x (M, K) -> (N, K)
        t["x"] = rn(c.M, c.N, scale=1 / math.sqrt(c.M))
        t["w"] = rn(c.M, c.K)
        t["out"] = rn(c.N, c.K) if c.residual else torch.zeros(c.N, c.K, device=DEV, dtype=dt)
    elif c.kind == "batched":
        t["x"] = rn(c.batch2, c.batch, c.M, c.K)
        t["w"] = rn(c.N, c.K, scale=1 / math.sqrt(c.K))
        t["out"] = torch.zeros(c.batch2, c.batch, c.M, c.N, device=DEV, dtype=dt)
        t["bias"] = rn(c.batch, c.N)
        t["res"] = rn(c.batch2, c.batch, c.M, c.N)
    elif c.kind == "align":
        H, hd = c.batch, c.N
        t["x"] = rn(H, c.M, c.K)
        t["w"] = rn(H * hd, c.K, scale=1 / math.sqrt(c.K))
        t["out"] = torch.zeros(c.M, H * hd, device=DEV, dtype=dt)
        t["bias"] = rn(H * hd)
        t["bias2"] = rn(H * hd)
        t["brs"] = torch.rand(H, c.M, device=DEV, generator=g)
        t["b2rs"] = torch.rand(H, c.M, device=DEV, generator=g)
    if c.kind in ("linear", "thin"):
        feat = c.N if c.kind == "thin" else n_out
        if c.bias:
            t["biasbuf"] = rn(feat + c.bias_off)
            t["bias"] = t["biasbuf"][c.bias_off:]
        if c.residual:
            rows = c.M
            if c.res_row_mod:
                rows = c.res_row_mod
            t["resbuf"] = rn(rows, n_out + 2 * c.res_off)
            t["res"] = t["resbuf"][:, c.res_off:c.res_off + n_out]
        if c.row_scale:
            t["rs"] = torch.rand(c.M, device=DEV, generator=g) + 0.5
        if c.rms:  # partial sums giving row scales in [0.5, 2]
            target = torch.rand(c.M, device=DEV, generator=g) * 1.5 + 0.5
            t["ssq"] = (c.K / target ** 2 / 32)[:, None].expand(c.M, 32).contiguous()
        if c.sumsq:
            t["ss"] = torch.full((c.M, n_out // 32), float("nan"), device=DEV)
        if c.epi == ops.EPI_ROPE:
            T = c.rope_T + c.rope_pos
            pos = torch.arange(T, device=DEV, dtype=torch.float32)[:, None]
            fr = pos * (1.0 / 10000 ** (torch.arange(0, 128, 2, device=DEV).float() / 128))[None]
            t["cos"], t["sin"] = fr.cos().contiguous(), fr.sin().contiguous()
            if c.rope_pos:
                t["pos"] = torch.tensor([c.rope_pos], device=DEV, dtype=torch.int32)
        if c.cancel and c.residual:  # residual ~ -(the product): the sum cancels to a few ulps of either
            with torch.no_grad():
                prod = (t["x"].double() @ t["w"].double().T)[:, :n_out]
                if c.res_row_mod:
                    prod = prod[:c.res_row_mod]
                noise = torch.randn(prod.shape, device=DEV, generator=g, dtype=torch.float64) * 0.01
                t["res"].copy_((-prod + noise).to(dt))
    if c.streamk:
        t["ws"] = ops.streamk_workspace(torch.device(DEV, torch.cuda.current_device()))
    p = {k: v.data_ptr() for k, v in t.items()}
    for k, buf in (("out", "outbuf"), ("bias", "biasbuf"), ("res", "resbuf")):  # raw_args() adds the case's offsets
        if buf in t:
            p[k] = t[buf].data_ptr()
    if c.streamk:
        p["ws_bytes"] = t["ws"].numel() * 4
    return t, p


def _launch(c: G.Case, t: dict):
    """Run case c through its public entry point."""
    ops = _ops()
    if c.kind == "linear":
        kw = {}
        if c.residual:
            kw.update(residual=t["res"], res_row_mod=c.res_row_mod)
        if c.rms:
            kw.update(rms_from=(t["ssq"], 1e-6))
        if c.sumsq:
            kw.update(sumsq_out=t["ss"])
        if c.epi == ops.EPI_ROPE:
            kw.update(rope=(t["cos"], t["sin"], c.rope_T, c.rope_cols, t.get("pos")))
        ops.STREAMK = t.get("ws")
        try:
            ops.linear(t["x"], t["w"], t.get("bias"), act=c.act, out=t["out"], alpha=c.alpha, row_scale=t.get("rs"),
                       epi=c.epi, **kw)
        finally:
            ops.STREAMK = None
    elif c.kind == "thin":
        ops.linear_thin(t["x"], t["w"], t["bias"], act=c.act, residual=t["res"], out=t["out"], row_scale=t["rs"])
    elif c.kind == "dx":
        ops.STREAMK = None
        if c.streamk:  # gemm_dx takes no workspace: the raw call is the same launch with one
            ops.gemm_raw(**G.raw_args(c, {**{k: v.data_ptr() for k, v in t.items()}, "ws_bytes": t["ws"].numel() * 4}))
        else:
            ops.gemm_dx(t["x"], t["w"], out=t["out"], accumulate=c.residual)
    elif c.kind == "dw":
        ops.gemm_dw(t["x"], t["w"], t["out"], accumulate=c.residual)
    else:
        ops.gemm_raw(**G.raw_args(c, {k: v.data_ptr() for k, v in t.items()}))


def _reference(c: G.Case, t: dict, t0: dict):
    ops = _ops()
    dt = torch.float16 if c.fmt == G.F16 else torch.bfloat16
    fmt = torch.float32 if c.out == "fp32" else dt
    kw = dict(out_fmt=fmt, epi=c.epi, act=c.act, alpha=c.alpha)
    if c.kind == "linear":
        kw.update(A=t["x"], B=t["w"])
        if c.bias:
            kw.update(bias=t["bias"])
        if c.residual:
            kw.update(residual=t0["res"], res_row_mod=c.res_row_mod)
        if c.row_scale:
            kw.update(row_scale=t["rs"])
        if c.rms:
            kw.update(rs_sumsq=t["ssq"], rs_eps=1e-6)
        if c.epi == ops.EPI_ROPE:
            kw.update(rope_cos=t["cos"], rope_sin=t["sin"], rope_T=c.rope_T, rope_cols=c.rope_cols, rope_pos=c.rope_pos)
    elif c.kind == "thin":
        kw.update(A=t["w"], B=t["x"], c_trans=True, bias=t["bias"], residual=t0["res"], row_scale=t["rs"])
    elif c.kind == "dx":
        kw.update(A=t["x"], B=t["w"], b_mn_major=True, residual=t0["out"] if c.residual else None)
    elif c.kind == "dw":
        kw.update(A=t["x"], B=t["w"], a_mn_major=True, b_mn_major=True, residual=t0["out"] if c.residual else None)
    elif c.kind == "batched":
        kw.update(A=t["x"], B=t["w"], bias=t["bias"], residual=t["res"])
    elif c.kind == "align":
        H, hd = c.batch, c.N
        kw.update(A=t["x"], B=t["w"].view(H, hd, c.K), bias=t["bias"].view(H, hd), bias_rs=t["brs"],
                  bias2=t["bias2"].view(H, hd), bias2_rs=t["b2rs"])
    return R.gemm_ref(**kw)


def _stored(c: G.Case, t: dict):
    if c.kind == "align":
        return t["out"].view(c.M, c.batch, c.N).transpose(0, 1)
    return t["out"]


def _run_case(c: G.Case, seed: int):
    ops, lib = _ops(), _lib()
    dt = torch.float16 if c.fmt == G.F16 else torch.bfloat16
    ops.set_act_format(dt)
    prev_o, prev_s = lib.mm_gemm_overlap_mode(c.overlap), lib.mm_gemm_streamk_mode(c.streamk)
    try:
        t, p = _inputs(c, seed)
        t0 = {k: v.clone() for k, v in t.items() if k in ("res", "out")}
        want = G.instance(c, G.plan(c, p))
        # The profiler's trace occasionally lacks a kernel that ran (its plan is recorded, the trace holds no GEMM):
        # only then is the launch repeated, from the original in-place output; a trace naming any other kernel fails.
        for _ in range(3):
            if c.kind in ("dx", "dw") and c.residual:  # accumulates into `out`
                t["out"].copy_(t0["out"])
            ops.PLANS = []
            try:
                with _launched() as prof:
                    _launch(c, t)
                    torch.cuda.synchronize()
            finally:
                plans, ops.PLANS = ops.PLANS, None
            got_inst = _parse(prof)
            if got_inst:
                break
        assert len(plans) == 1 and got_inst == {want} == {G.instance(c, plans[0])}, (c.name, got_inst, want, plans)
        ref = _reference(c, t, t0)
        got = _stored(c, t)
        w, idx, gv, rv = R.worst(got, ref)
        print(f"[fp64] {c.name}: {want} sk={plans[0]['streamk_tiles']} vec={plans[0]['vectorised_epilogue']} "
              f"worst ratio {w:.3f} at {idx}: got {gv:.6g} ref {rv:.6g}")
        assert w <= 1.0, (c.name, w, idx, gv, rv)
        if c.sumsq:
            want_ss = R.sumsq_ref(got)
            err = (t["ss"].double() - want_ss).abs() / R.sumsq_bar(got)
            print(f"[fp64] {c.name}: sumsq_out worst ratio {float(err.max()):.3f}")
            assert float(err.max()) <= 1.0
        if c.kind in ("linear", "thin") and (c.c_off or c.ldc_pad):  # nothing written outside the view
            buf = t["outbuf"]
            mask = torch.ones_like(buf, dtype=torch.bool)
            mask[:, c.c_off:c.c_off + c.n_out] = False
            assert bool((buf[mask] == 0).all())
        return w
    finally:
        lib.mm_gemm_overlap_mode(prev_o)
        lib.mm_gemm_streamk_mode(prev_s)
        ops.set_act_format(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize("case", G.CASES, ids=[c.name for c in G.CASES])
def test_gemm_case_against_fp64(case):
    _run_case(case, seed=zlib.crc32(case.name.encode()) % 1000)


@pytest.mark.gpu
def test_coverage_at_device_sm_count():
    """The table reaches all 42 instances when planned with this device's SM count."""
    ops, lib = _ops(), _lib()
    got = {}
    for c in G.CASES:
        dt = torch.float16 if c.fmt == G.F16 else torch.bfloat16
        ops.set_act_format(dt)
        got.setdefault(G.instance(c, G.plan(c, G.fake_ptrs())), []).append(c.name)
    ops.set_act_format(torch.bfloat16)
    assert G.all_instances() - set(got) == set(), sorted(G.all_instances() - set(got))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [G.BF16, G.F16])
@pytest.mark.parametrize("act", ["silu", "quick_gelu", "gelu", "swiglu"])
def test_activation_sweep(act, fmt):
    """The activation epilogues at pre-activations x in [-30, 30]: A's first column holds x, B selects it exactly."""
    ops = _ops()
    dt = torch.float16 if fmt == G.F16 else torch.bfloat16
    ops.set_act_format(dt)
    try:
        xs = torch.linspace(-30, 30, 60001, device=DEV).to(dt)
        M, K = xs.numel(), 64
        A = torch.zeros(M, K, device=DEV, dtype=dt)
        A[:, 0] = xs
        A[:, 1] = 1
        if act == "swiglu":
            N = 64
            B = torch.zeros(N, K, device=DEV, dtype=dt)
            B[:32, 0] = 1   # gate = x
            B[32:, 1] = 1   # up = 1
            out = ops.linear(A, B, epi=ops.EPI_SWIGLU)
            ref = R.gemm_ref(A=A, B=B, out_fmt=dt, epi=R.EPI_SWIGLU)
        else:
            a = {"silu": ops.ACT_SILU, "quick_gelu": ops.ACT_QUICK_GELU, "gelu": ops.ACT_GELU}[act]
            B = torch.zeros(32, K, device=DEV, dtype=dt)
            B[:, 0] = 1
            out = ops.linear(A, B, act=a)
            ref = R.gemm_ref(A=A, B=B, out_fmt=dt, act=a)
        torch.cuda.synchronize()
        err = (out.double() - ref.value).abs()
        units = err / R.half_ulp(ref.value.abs(), dt)
        i = int(torch.argmax(units[:, 0]))
        w, idx, gv, rv = R.worst(out, ref)
        print(f"[sweep] {act} {fmt}: worst error {float(units[i, 0]):.3f} output roundings at x = {float(xs[i]):.4g}; "
              f"worst bar ratio {w:.3f} at x = {float(xs[idx[0]]):.4g} (got {gv:.6g}, ref {rv:.6g})")
        assert w <= 1.0
    finally:
        ops.set_act_format(torch.bfloat16)
