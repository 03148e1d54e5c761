"""CPU tier of the FP8 decoder (quant.quantize_llm_fp8, mm_quantize_rows_e4m3, mm_gemm_e4m3_*): the rounding rule
restated against torch's float8_e4m3fn, the Fp8Linear state, every refusal on a CPU model, and the e4m3 GEMM's launch plan
and argument errors at the decoder's shapes — none of it needs a GPU."""
import pytest
import torch

from tests import helpers as H
from tests.fp8_reference import E4M3, quantize_ref


def crafted_rows(K: int = 64) -> torch.Tensor:
    """Scale exactly 1 (max 448) on rows 0 and 5, so v / s = v: ties between e4m3 neighbours, values just under and at
    448, subnormals of e4m3 (2^-9 .. 2^-7), +-0; a zero row; a negative maximum; a tiny row."""
    rows = torch.zeros(6, K)
    # e4m3 neighbours 1, 1.125 (tie at 1.0625 -> 1, even), 1.125, 1.25 (tie 1.1875 -> 1.25, even), 416, 448 (tie 432 -> 448)
    rows[0, :10] = torch.tensor([448.0, 1.0625, 1.1875, 432.0, 447.9, -0.0, 0.0, 2.0 ** -9, 3 * 2.0 ** -10, -2.0 ** -11])
    rows[2, 17] = -3.75
    rows[3, 5] = 1e-30
    rows[4] = torch.linspace(-5.0, 4.0, K)
    rows[5, :4] = torch.tensor([-448.0, 240.0, 248.0, -0.0009765625])
    return rows


def test_rounding_rule_on_crafted_rows():
    w = crafted_rows()
    q, s = quantize_ref(w)
    assert q.dtype == E4M3 and s.dtype == torch.float32
    assert s[0] == 1.0 and s[5] == 1.0
    assert q[0, :10].float().tolist() == [448.0, 1.0, 1.25, 448.0, 448.0, 0.0, 0.0, 2.0 ** -9, 2.0 ** -8, 0.0]
    assert q[5, :4].float().tolist() == [-448.0, 240.0, 256.0, 0.0]  # 248 and -2^-10 are ties: to even
    assert s[1] == 0 and not q[1].float().any()                            # zero row: s = 0, q = 0
    assert q[2, 17].float() == -448.0 and q[2].float().abs().sum() == 448.0
    assert q[3, 5].float() == 448.0 and float(s[3]) == float(torch.tensor(1e-30) / 448)
    assert q[4, 0].float() == -448.0 and q[4].float().max() < 448.0
    # the e4m3 values of the restatement are torch's cast of v / s (nearest even inside the range)
    v = w / torch.where(s == 0, 1.0, s)[:, None]
    assert torch.equal(q.float(), torch.where((s == 0)[:, None], 0.0, v.to(E4M3).float()))
    # a scale that underflows to 0 makes a zero row
    qz, sz = quantize_ref(torch.full((1, 16), 1e-44))
    assert sz[0] == 0 and not qz.float().any()
    # bf16 / fp16 inputs go through fp32 exactly; the gain multiplies in fp32 before the row maximum
    for dt in (torch.bfloat16, torch.float16):
        q2, s2 = quantize_ref(w.to(dt))
        q3, s3 = quantize_ref(w.to(dt).float())
        assert torch.equal(q2.float(), q3.float()) and torch.equal(s2, s3)
    g = torch.linspace(0.5, 2.0, 64).to(torch.bfloat16)
    qg, sg = quantize_ref(w.to(torch.bfloat16), g)
    q4, s4 = quantize_ref(w.to(torch.bfloat16).float() * g.float())
    assert torch.equal(qg.float(), q4.float()) and torch.equal(sg, s4)


def _cpu_model():
    model, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    return model, spec


def _fake_quantize(model):
    """An FP8 model's module structure built on the CPU with the restated rule (the device kernel cannot run here)."""
    from macaw_llm_b200 import quant

    for l in model.llm.model.layers:
        for parent, name in quant.PROJECTIONS:
            mod = getattr(l, parent)
            q, s = quantize_ref(getattr(mod, name).weight.detach())
            setattr(mod, name, quant.Fp8Linear(q, s))


def test_refusals_on_a_cpu_model():
    from macaw_llm_b200.lora import LoraConfig

    model, spec = _cpu_model()
    with pytest.raises(RuntimeError, match="quantize_llm_fp8: .*CPU"):
        model.quantize_llm_fp8()
    model.add_lora(LoraConfig(r=8, target_modules=["q_proj"]))
    with pytest.raises(RuntimeError, match="quantize_llm_fp8: .*merge_lora"):
        model.quantize_llm_fp8()
    model.merge_lora()
    _fake_quantize(model)
    with pytest.raises(RuntimeError, match="quantize_llm_fp8: the decoder is already quantized"):
        model.quantize_llm_fp8()
    with pytest.raises(RuntimeError, match="quantize_llm_int8: the decoder is already quantized"):
        model.quantize_llm_int8()
    with pytest.raises(RuntimeError, match="FP8-quantized"):
        model.add_lora(LoraConfig(r=8))
    model.train()
    inp = H.case_inputs(spec, H.load_case("text"))
    with pytest.raises(RuntimeError, match="FP8-quantized .*cannot be trained"):
        model(inp)
    # an int8 model refuses FP8 quantization
    from tests.test_quant_cpu import _fake_quantize as fake_int8

    m8, _ = _cpu_model()
    fake_int8(m8)
    with pytest.raises(RuntimeError, match="quantize_llm_fp8: the decoder is already quantized"):
        m8.quantize_llm_fp8()


def test_fp8_layer_state_and_dtype_casts():
    from macaw_llm_b200 import quant

    model, _ = _cpu_model()
    _fake_quantize(model)
    assert quant.quant_format(model) == "fp8" and quant.is_quantized(model)
    sd = model.state_dict()
    k = "llm.model.layers.0.self_attn.q_proj"
    assert sd[k + ".weight"].dtype == E4M3 and sd[k + ".weight_scale"].dtype == torch.float32
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        model.to(dt)
        lin = model.llm.model.layers[0].self_attn.q_proj
        assert lin.weight.dtype == E4M3 and lin.weight_scale.dtype == torch.float32
        assert torch.equal(lin.weight.float(), sd[k + ".weight"].float())
        assert torch.equal(lin.weight_scale, sd[k + ".weight_scale"])
        assert model.llm.model.layers[0].input_layernorm.weight.dtype == dt
    other, _ = _cpu_model()
    _fake_quantize(other)
    with torch.no_grad():
        other.llm.model.layers[0].self_attn.q_proj.weight_scale.zero_()
    other.load_state_dict(sd)
    assert torch.equal(other.llm.model.layers[0].self_attn.q_proj.weight_scale, sd[k + ".weight_scale"])
    bad = dict(sd)
    bad[k + ".weight"] = bad[k + ".weight"].to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="e4m3-quantized"):
        other.load_state_dict(bad)
    with pytest.raises(RuntimeError):
        other.llm.model.layers[0].self_attn.q_proj(torch.zeros(1, 4))
    with pytest.raises(TypeError):
        quant.Fp8Linear(torch.zeros(4, 4, dtype=torch.int8), torch.zeros(4))


# the decoder's GEMMs: (M rows of a prefill or decode batch) x (N, K, epilogue, source rows)
E, I = 4096, 11008
DECODER = [(3 * E, E, 2, [E] * 3), (E, E, 0, [E]), (2 * I, E, 1, [I] * 2), (E, I, 0, [E])]


@pytest.mark.parametrize("M", [264, 2112, 16896])
def test_e4m3_plan_at_the_decoder_shapes(M):
    from macaw_llm_b200 import ops

    for N, K, epi, rows in DECODER:
        p = ops.gemm_e4m3_plan(M=M, N=N, K=K, epi=epi, rows=rows)
        tiles = -(-M // 128) * (N // 128)
        assert p["block_n"] == 128 and p["kernel"] == ops.GEMM_CONSUMER_EPILOGUE and p["threads"] == 288
        assert p["k_blocks"] == K // 128 and p["n_tiles"] == N // 128 and p["units"] == tiles
        assert p["streamk_tiles"] == 0 and p["grid"] == min(tiles, p["workers"])
        assert p["smem_bytes"] <= 227 * 1024 and p["vectorised_epilogue"] == 1


def test_e4m3_plan_argument_errors():
    from macaw_llm_b200 import ops

    ok = dict(M=13, N=4096, K=4096)
    ops.gemm_e4m3_plan(**ok)
    for kw, msg in ((dict(K=4000), "K % 128"), (dict(N=4032), "N % 128"), (dict(lda=4104), "lda % 16"),
                    (dict(lda=4000), "lda >= K"), (dict(a_scale=False), "null A scales"),
                    (dict(w_scale=False), "non-null scales"), (dict(rows=[4096, 48]), "multiple of 32 rows")):
        with pytest.raises(RuntimeError, match=msg):
            ops.gemm_e4m3_plan(**{**ok, **kw})
    with pytest.raises(RuntimeError, match="weight is"):
        _plan_mismatch()


def _plan_mismatch():
    """A weight whose N differs from the problem's."""
    import ctypes as C

    from macaw_llm_b200 import _lib, ops

    fake = 1 << 20
    a = _lib.GemmArgs(M=8, N=256, K=256, batch=1, batch2=1, A=fake, lda=256, B=fake, ldb=256, C=fake, ldc=256, alpha=1.0)
    e = _lib.GemmE4m3Args()
    e.a_scale = fake
    e.w.q[0], e.w.scale[0], e.w.rows[0], e.w.chunks, e.w.N, e.w.K = fake, fake, 128, fake, 128, 256
    return ops._plan_of(a, e)


def test_the_case_table_reaches_every_fp8_instance():
    """tests/test_fp8_gpu.py's GEMM cases launch every gemm_e4m3_kernel instance the library has: the three epilogues
    promoted, and the standard epilogue unpromoted."""
    from tests.test_fp8_gpu import GEMM_CASES

    seen = {(c["epi"], c.get("unpromoted", False)) for c in GEMM_CASES}
    assert seen == {(0, False), (1, False), (2, False), (0, True)}


def test_fp8_kernels_are_hopper_native_sass():
    """Static check of the shipped cubin (cuobjdump, no GPU): every gemm_e4m3_kernel instance and every e4m3 instance of
    w8_thin_kernel carries wgmma (HGMMA / QGMMA), TMA loads and mbarrier operations, and none spills."""
    import os
    import re
    import shutil
    import subprocess
    import sys

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from macaw_llm_b200 import _lib

    _lib.load()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "sass_inventory.py")], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.splitlines()
    cols = next(l for l in lines if l.startswith("kernel ")).split()[1:]
    rows = {}
    for l in lines:
        m = re.match(r"(\S.*?)\s+((?:\d+\s+){%d}\d+)\s*$" % (len(cols) - 1), l)
        if m and not l.startswith(("#", "TOTAL")):
            rows[m.group(1).strip()] = dict(zip(cols, map(int, m.group(2).split())))
    e4m3 = {k: v for k, v in rows.items() if k.startswith("gemm_e4m3_kernel<")}
    thin = {k: v for k, v in rows.items() if re.fullmatch(r"w8_thin_kernel<\w+, \d+, \w+, true>", k)}
    assert len(e4m3) == 4 and len(thin) == 16, (sorted(e4m3), sorted(thin))
    for k, v in {**e4m3, **thin}.items():
        assert v["HGMMA"] > 0 and v["UTMALDG"] > 0 and v["SYNCS"] > 0 and v["HMMA"] == 0 and v["LOCAL"] == 0, (k, v)
