"""CPU tier of the int8 decoder weights (quant.py, csrc/quant.cu): the quantization rule restated on the CPU, the fused
chunk maps against the permutations the engine's 16-bit weights use, the refusals, and argument errors of the ops
wrappers and the C entry points — none of it needs a GPU."""
import ctypes

import pytest
import torch

from tests import helpers as H


def quantize_ref(w: torch.Tensor):
    """The rule, restated: s = fp32(max |w|) / 127 (IEEE), q = clamp(rint(fp32(w) / s), -127, 127) with ties to even,
    q = 0 where s = 0.  -> (q int8, s fp32)."""
    wf = w.float()
    s = wf.abs().amax(1) / torch.tensor(127.0, dtype=torch.float32)
    zero = s == 0
    q = torch.clamp(torch.round(wf / torch.where(zero, 1.0, s)[:, None]), -127, 127)
    q = torch.where(zero[:, None], 0.0, q)
    return q.to(torch.int8), s


def crafted_rows(K: int = 64) -> torch.Tensor:
    """Rows that pin the rule: .5 ties (scale exactly 1), an all-zero row, a single non-zero, negative maxima."""
    rows = torch.zeros(6, K)
    rows[0, :8] = torch.tensor([127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5])
    rows[2, 17] = -3.75
    rows[3, 5] = 1e-3
    rows[4] = torch.linspace(-5.0, 4.0, K)
    rows[5, :4] = torch.tensor([-127.0, 63.5, 64.5, -0.49])
    return rows


def test_rounding_rule_on_crafted_rows():
    w = crafted_rows()
    q, s = quantize_ref(w)
    assert s[0] == 1.0 and s[5] == 1.0
    assert q[0, :8].tolist() == [127, 0, 2, 2, 0, -2, -2, 126]        # ties to even
    assert q[5, :4].tolist() == [-127, 64, 64, 0]
    assert s[1] == 0 and not q[1].any()                               # all-zero row: s = 0, q = 0
    assert q[2, 17] == -127 and q[2].abs().sum() == 127               # single non-zero maps to -127
    assert q[3, 5] == 127 and float(s[3]) == float(torch.tensor(1e-3) / 127)
    assert q[4, 0] == -127 and q[4].max() < 127                       # the row maximum (here negative) maps to -127
    # bf16 / fp16 inputs go through fp32 exactly
    for dt in (torch.bfloat16, torch.float16):
        q2, s2 = quantize_ref(w.to(dt))
        q3, s3 = quantize_ref(w.to(dt).float())
        assert torch.equal(q2, q3) and torch.equal(s2, s3)


def test_chunk_maps_match_the_fused_layouts():
    from macaw_llm_b200 import ops

    E, I = 256, 512
    ids = [torch.arange(r) + 1000 * j for j, r in enumerate((E, E, E))]  # distinct ids per (source, row)
    cat = torch.cat(ids, 0)
    m = ops.w8_chunk_map([E, E, E])
    assert m.dtype == torch.int32 and tuple(m.shape) == (3 * E // 32, 2)
    got = torch.cat([ids[int(j)][int(r):int(r) + 32] for j, r in m])
    assert torch.equal(got, cat)
    # the engine's [gate | up]: torch.stack of 32-row groups, reshaped (engine._llama_weights)
    g, u = torch.arange(I), torch.arange(I) + 100000
    inter = torch.stack([g.view(I // 32, 32), u.view(I // 32, 32)], 1).reshape(2 * I)
    m = ops.w8_chunk_map([I, I], interleave=True)
    got = torch.cat([(g, u)[int(j)][int(r):int(r) + 32] for j, r in m])
    assert torch.equal(got, inter)
    with pytest.raises(ValueError):
        ops.w8_chunk_map([E, 48])
    with pytest.raises(ValueError):
        ops.w8_chunk_map([I, 2 * I], interleave=True)


def _cpu_model():
    model, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    return model, spec


def _fake_quantize(model):
    """A quantized model's module structure built on the CPU with the reference rule (the device kernel cannot run here)."""
    from macaw_llm_b200 import quant

    for l in model.llm.model.layers:
        for parent, name in quant.PROJECTIONS:
            mod = getattr(l, parent)
            q, s = quantize_ref(getattr(mod, name).weight.detach())
            setattr(mod, name, quant.Int8Linear(q, s))


def test_refusals_on_a_cpu_model():
    from macaw_llm_b200.lora import LoraConfig

    model, spec = _cpu_model()
    with pytest.raises(RuntimeError, match="CPU"):
        model.quantize_llm_int8()
    model.add_lora(LoraConfig(r=8, target_modules=["q_proj"]))
    with pytest.raises(RuntimeError, match="merge_lora"):
        model.quantize_llm_int8()
    model.merge_lora()
    _fake_quantize(model)
    with pytest.raises(RuntimeError, match="already quantized"):
        model.quantize_llm_int8()
    with pytest.raises(RuntimeError, match="int8"):
        model.add_lora(LoraConfig(r=8))
    model.train()
    inp = H.case_inputs(spec, H.load_case("text"))
    with pytest.raises(RuntimeError, match="cannot be trained"):
        model(inp)


def test_int8_layer_state_and_dtype_casts():
    from macaw_llm_b200 import quant

    model, _ = _cpu_model()
    _fake_quantize(model)
    sd = model.state_dict()
    k = "llm.model.layers.0.self_attn.q_proj"
    assert sd[k + ".weight"].dtype == torch.int8 and sd[k + ".weight_scale"].dtype == torch.float32
    for dt in (torch.float16, torch.bfloat16):
        model.to(dt)
        lin = model.llm.model.layers[0].self_attn.q_proj
        assert lin.weight.dtype == torch.int8 and lin.weight_scale.dtype == torch.float32
        assert torch.equal(lin.weight_scale, sd[k + ".weight_scale"])
    other, _ = _cpu_model()
    _fake_quantize(other)
    with torch.no_grad():
        other.llm.model.layers[0].self_attn.q_proj.weight.zero_()
    other.load_state_dict(sd)
    assert torch.equal(other.llm.model.layers[0].self_attn.q_proj.weight, sd[k + ".weight"])
    # a 16-bit weight is not silently truncated into an int8 layer
    bad = dict(sd)
    bad[k + ".weight"] = bad[k + ".weight"].to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="int8-quantized"):
        other.load_state_dict(bad)
    assert quant.is_quantized(other)
    with pytest.raises(RuntimeError):
        other.llm.model.layers[0].self_attn.q_proj(torch.zeros(1, 4))


def test_ops_argument_errors_without_a_gpu():
    from macaw_llm_b200 import _lib, ops

    with pytest.raises(RuntimeError, match="CUDA"):
        ops.quantize_rows_int8(torch.zeros(64, 64, dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        ops.quantize_rows_int8(torch.zeros(64, 64, dtype=torch.int32))
    q, s = torch.zeros(64, 64, dtype=torch.int8), torch.zeros(64)
    with pytest.raises(TypeError):
        ops.W8Matrix([q.float()], [s])
    with pytest.raises(TypeError):
        ops.W8Matrix([q], [s.double()])
    with pytest.raises(ValueError, match="N % 64"):
        ops.W8Matrix([q[:32]], [s[:32]])
    with pytest.raises(ValueError, match="K % 16"):
        ops.W8Matrix([torch.zeros(64, 40, dtype=torch.int8)], [s])
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.W8Matrix([q], [s])
    # the C entry points validate before touching the device
    lib = _lib.load()
    assert lib.mm_dequant_rows(None, None, 0, None) != 0 and b"null args" in lib.mm_last_error()
    m = _lib.W8Matrix()
    m.N, m.K = 96, 64
    assert lib.mm_gemm_w8_thin(ctypes.byref(m), None, 64, 1, None, 1, 4, None, None) != 0 and b"bad shape" in lib.mm_last_error()
    assert lib.mm_quantize_rows_int8(None, 64, 0, 4, 64, None, None, None) != 0


def test_decode_split_choice_fills_the_sms():
    """w8_thin_splits: every decode shape gets splits within [1, K / 128] and at least two 64-row CTAs per SM where K
    allows; the choice does not depend on the number of activation rows."""
    from macaw_llm_b200 import ops

    for N, K in ((12288, 4096), (22016, 4096), (4096, 4096), (4096, 11008), (768, 256), (1024, 256), (256, 256), (256, 512)):
        S = ops.w8_thin_splits(N, K, 132)
        ns = (K + 127) // 128
        assert 1 <= S <= ns
        assert S == ns or ((N // 64) * S >= 264 and S >= 2)
