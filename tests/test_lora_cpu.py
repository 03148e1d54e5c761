"""CPU tier: the LoRA surface (lora.py) on the tiny model — configuration checks, target resolution, PEFT's initialisation
and adapter file layout, the trainable set, the gradient-buffer layout with a frozen base, and the dropout stream ids."""
import json
import os
import re

import pytest
import torch

from tests import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# run_clm_llms.py:498-508 (the reference's LoRA recipe)
REFERENCE_TARGETS = ["q_proj", "k_proj", "v_proj", "out_proj", "fc_in", "fc_out", "wte", "embed_tokens", "lm_head"]


@pytest.fixture
def tiny():
    model, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    return model


def _L():
    from macaw_llm_b200 import lora

    return lora


def test_config_validation():
    L = _L()
    c = L.LoraConfig()
    assert (c.r, c.lora_alpha, c.lora_dropout, c.bias) == (8, 16, 0.0, "none")
    assert c.target_modules == ["q_proj", "v_proj"] and c.scaling == 2.0
    assert L.LoraConfig(r=16, lora_alpha=8).scaling == 0.5
    for r in (0, 4, 12, 72, 8.5, True):
        with pytest.raises(ValueError, match="r must be"):
            L.LoraConfig(r=r)
    for bias in ("all", "lora_only"):
        with pytest.raises(NotImplementedError, match="bias"):
            L.LoraConfig(bias=bias)
    for field, v in (("use_rslora", True), ("use_dora", True), ("fan_in_fan_out", True), ("modules_to_save", ["x"])):
        with pytest.raises(NotImplementedError, match=field):
            L.LoraConfig(**{field: v})
    with pytest.raises(ValueError):
        L.LoraConfig(lora_dropout=1.0)


def test_reference_targets_resolve(tiny):
    L = _L()
    with pytest.raises(NotImplementedError, match="embed_tokens"):
        L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=REFERENCE_TARGETS))
    names = L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=[t for t in REFERENCE_TARGETS if t != "embed_tokens"]))
    n = tiny.llm.config.num_hidden_layers
    want = {f"model.layers.{i}.self_attn.{p}" for i in range(n) for p in ("q_proj", "k_proj", "v_proj")} | {"lm_head"}
    assert set(names) == want
    with pytest.raises(ValueError, match="match no module"):
        L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=["out_proj", "fc_in"]))
    with pytest.raises(ValueError, match="cannot be adapted"):
        L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=["input_layernorm"]))


def test_add_lora_init_trainable_set_and_keys(tiny):
    from macaw_llm_b200.training import trainable_parameters

    L = _L()
    base_keys = set(tiny.state_dict())
    torch.manual_seed(0)
    tiny.add_lora(L.LoraConfig(r=16, lora_alpha=32, target_modules=["q_proj", "v_proj", "down_proj", "lm_head"]))
    sd = tiny.state_dict()
    added = set(sd) - base_keys
    assert base_keys <= set(sd)
    n = tiny.llm.config.num_hidden_layers
    want = {f"llm.model.layers.{i}.{m}.lora_{ab}.weight" for i in range(n)
            for m in ("self_attn.q_proj", "self_attn.v_proj", "mlp.down_proj") for ab in "AB"}
    want |= {"llm.lm_head.lora_A.weight", "llm.lm_head.lora_B.weight"}
    assert added == want
    q = tiny.llm.model.layers[0].self_attn.q_proj
    assert q.lora_A.weight.shape == (16, q.in_features) and q.lora_B.weight.shape == (q.out_features, 16)
    assert q.lora_A.weight.dtype == torch.bfloat16 and not torch.any(tiny.llm.lm_head.lora_B.weight != 0)
    bound = 1.0 / q.in_features ** 0.5  # kaiming_uniform(a = sqrt(5)) on (r, in): U(-1/sqrt(in), 1/sqrt(in))
    a = q.lora_A.weight.detach().float()
    assert float(a.abs().max()) <= bound * 1.01 and float(a.std()) > 0.4 * bound
    assert tiny.llm.model.embed_tokens is tiny.llm.get_input_embeddings()  # model.llm is not wrapped
    names = {nm for nm, _ in trainable_parameters(tiny)}
    assert {nm for nm in names if nm.startswith("llm.")} == want
    align = {nm for nm in names if not nm.startswith("llm.")}
    assert align and all(nm.startswith(("project_", "transform_", "image_align", "audio_align", "video_align",
                                        "video_long_self_attention.")) for nm in align)
    assert not any(p.requires_grad for nm, p in tiny.named_parameters() if "encoder" in nm)
    with pytest.raises(RuntimeError, match="already"):
        tiny.add_lora(L.LoraConfig())


def test_save_load_roundtrip_peft_layout(tiny, tmp_path):
    L = _L()
    cfg = L.LoraConfig(r=8, lora_alpha=16, lora_dropout=0.05, target_modules=["q_proj", "k_proj", "v_proj", "lm_head"])
    tiny.add_lora(cfg)
    with torch.no_grad():
        for lin in L.adapted_modules(tiny).values():
            lin.lora_B.weight.normal_(0, 0.1)
    tiny.save_lora(str(tmp_path))
    conf = json.load(open(tmp_path / "adapter_config.json"))
    assert conf == dict(peft_type="LORA", task_type="CAUSAL_LM", r=8, lora_alpha=16, lora_dropout=0.05,
                        target_modules=["q_proj", "k_proj", "v_proj", "lm_head"], bias="none", fan_in_fan_out=False)
    sd = torch.load(tmp_path / "adapter_model.bin", weights_only=True)
    assert "base_model.model.model.layers.0.self_attn.q_proj.lora_A.weight" in sd
    assert "base_model.model.lm_head.lora_B.weight" in sd
    assert all(re.fullmatch(r"base_model\.model\.(model\.layers\.\d+\.self_attn\.[qkv]_proj|lm_head)\.lora_[AB]\.weight", k)
               for k in sd)
    fresh, _, _, _ = H.build_tiny_model("cpu", torch.bfloat16)
    fresh.load_lora(str(tmp_path))  # no adapters yet: added with the stored config
    assert L.lora_config(fresh).to_dict() == conf
    got = L.lora_state_dict(fresh)
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


def test_merge_lora(tiny):
    L = _L()
    tiny.add_lora(L.LoraConfig(target_modules=["v_proj"]))
    v = tiny.llm.model.layers[1].self_attn.v_proj
    with torch.no_grad():
        v.lora_B.weight.normal_(0, 0.05)
    want = (v.weight.float() + 2.0 * v.lora_B.weight.float() @ v.lora_A.weight.float()).to(torch.bfloat16)
    tiny.merge_lora()
    assert not L.adapted_modules(tiny) and L.lora_config(tiny) is None
    assert torch.equal(v.weight, want) and "lora_A" not in v._modules


def test_grad_buffer_layout_with_frozen_base(tiny):
    from macaw_llm_b200.training import GradBuffer, trainable_parameters

    L = _L()
    tiny.add_lora(L.LoraConfig(target_modules=["q_proj", "v_proj", "o_proj", "gate_proj", "down_proj", "lm_head"]))
    gb = GradBuffer(tiny)
    n = tiny.llm.config.num_hidden_layers
    assert len(gb.buckets) == n + 2
    # contiguous buckets covering the buffer, in order
    assert gb.buckets[0][0] == 0 and gb.buckets[-1][1] == gb.flat.numel()
    assert all(a[1] == b[0] for a, b in zip(gb.buckets, gb.buckets[1:]))
    # exactly the trainable set, no slot for a frozen parameter
    assert {id(p) for p in gb.params} == {id(p) for _, p in trainable_parameters(tiny)}
    for nm, p in tiny.llm.named_parameters():
        assert (id(p) in gb.views) == p.requires_grad, nm
    assert id(tiny.llm.model.embed_tokens.weight) not in gb.views and id(tiny.llm.lm_head.weight) not in gb.views

    def span(p):
        v = gb.views[id(p)]
        return v.storage_offset(), v.storage_offset() + v.numel()

    lm = tiny.llm.lm_head
    assert [id(p) for p in gb.params[:2]] == [id(lm.lora_B.weight), id(lm.lora_A.weight)]
    for li, layer in enumerate(tiny.llm.model.layers):
        s, e = gb.buckets[n - li]  # backward order: layer L-1 first
        ad = [layer.mlp.down_proj, layer.mlp.gate_proj, layer.self_attn.o_proj, layer.self_attn.q_proj,
              layer.self_attn.v_proj]
        spans = [span(p) for lin in ad for p in (lin.lora_B.weight, lin.lora_A.weight)]
        assert all(s <= a and b <= e for a, b in spans)
        assert [a for a, _ in spans] == sorted(a for a, _ in spans)  # down, gate, o, q, v: backward order
        assert e - s == sum(b - a for a, b in spans)
    for p in gb.params:
        assert gb.views[id(p)].storage_offset() % 8 == 0  # 16-byte aligned views


def test_dropout_stream_ids_are_distinct():
    L = _L()
    src = open(os.path.join(ROOT, "macaw-llm_b200", "csrc", "philox.cuh")).read()
    consts = {k: int(v) for k, v in re.findall(r"constexpr uint32_t (SID_\w+) = (\d+)u;", src)}
    assert consts["SID_LORA_LM_HEAD"] == L.SID_LORA_LM_HEAD and consts["SID_LORA0"] == L.SID_LORA0
    src_e = open(os.path.join(ROOT, "macaw-llm_b200", "engine.py")).read()
    existing = set(map(int, re.findall(r'"(?:image|audio|video|video_long)": (\d+)', src_e.split("DROPOUT_SID", 1)[1].split("\n")[0])))
    existing |= {consts["SID_SAMPLE"]}
    assert existing == {1, 2, 3, 4, 16}
    ids = [L.lora_sid(l, t) for l in range(32) for t in L.TARGETS] + [L.lora_sid(None, "lm_head")]
    assert len(set(ids)) == len(ids) and not set(ids) & existing


def test_peft_config_fields_that_change_the_adapter_are_refused(tiny, tmp_path):
    L = _L()
    base = L.LoraConfig(r=8, lora_alpha=16, target_modules=["v_proj"]).to_dict()
    # what PEFT writes by default loads
    ok = dict(base, use_rslora=False, use_dora=False, rank_pattern={}, alpha_pattern={}, layers_to_transform=None,
              modules_to_save=None, init_lora_weights=True, base_model_name_or_path="x", inference_mode=True)
    assert L.LoraConfig.from_dict(ok).to_dict() == base
    for field, v in (("use_rslora", True), ("use_dora", True), ("rank_pattern", {"q_proj": 16}),
                     ("alpha_pattern", {"v_proj": 8}), ("layers_to_transform", [0]), ("modules_to_save", ["lm_head"]),
                     ("fan_in_fan_out", True)):
        with pytest.raises(NotImplementedError, match=field):
            L.LoraConfig.from_dict(dict(base, **{field: v}))
    # loading onto a model whose adapters have another scaling is refused
    tiny.add_lora(L.LoraConfig(r=8, lora_alpha=16, target_modules=["v_proj"]))
    tiny.save_lora(str(tmp_path))
    conf = json.load(open(tmp_path / "adapter_config.json"))
    json.dump(dict(conf, lora_alpha=32), open(tmp_path / "adapter_config.json", "w"))
    with pytest.raises(ValueError, match="lora_alpha"):
        tiny.load_lora(str(tmp_path))


def test_string_target_is_a_full_match_regex(tiny):
    L = _L()
    names = L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=r".*\.1\.self_attn\.(q|v)_proj"))
    assert set(names) == {"model.layers.1.self_attn.q_proj", "model.layers.1.self_attn.v_proj"}
    assert not L.resolve_targets(tiny.llm, L.LoraConfig(target_modules="q_proj|lm_head")).keys() - {"lm_head"}
    with pytest.raises(NotImplementedError, match="embed_tokens"):
        L.resolve_targets(tiny.llm, L.LoraConfig(target_modules=r"model\.embed_tokens|lm_head"))


def test_add_and_merge_drop_a_stale_gradient_buffer(tiny):
    from macaw_llm_b200.training import GradBuffer

    L = _L()
    ts = tiny.train_step
    ts.llama.grads = GradBuffer(tiny)  # as an earlier backward of the fully trainable model leaves it
    tiny.add_lora(L.LoraConfig(target_modules=["q_proj"]))
    assert ts.llama.grads is None
    ts.llama.grads = GradBuffer(tiny)
    tiny.merge_lora()
    assert ts.llama.grads is None


def test_reference_unmerged_lora_equals_merged_weights_fp64():
    """The tests' LoRA reference (the oracle's forward with x W^T + s (x A^T) B^T on the adapted projections) against the
    oracle's forward on merged weights W + s B A, in fp64; and with dropout multipliers of 1 it is the same formula."""
    from oracle import macaw_oracle as O
    from tests import lora_reference as R
    from tests.golden import gen

    spec, hp, shapes = H.load_shapes()
    sd = {k: v.double() if v.is_floating_point() else v for k, v in gen.make_weights(shapes, seed=0).items()}
    g = torch.Generator().manual_seed(5)
    names = [f"model.layers.{i}.{m}" for i in range(hp["llama"]["layers"])
             for m in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
                       "mlp.up_proj", "mlp.down_proj")] + ["lm_head"]
    adapters = {}
    for n in names:
        W = sd[f"llm.{n}.weight"]
        adapters[n] = (torch.randn(8, W.shape[1], generator=g, dtype=torch.float64) * 0.05,
                       torch.randn(W.shape[0], 8, generator=g, dtype=torch.float64) * 0.05, 2.0)
    merged = dict(sd)
    for n, (A, B, s) in adapters.items():
        merged[f"llm.{n}.weight"] = sd[f"llm.{n}.weight"] + s * B @ A
    E = hp["llama"]["hidden"]
    embeds = torch.randn(2, 9, E, generator=g, dtype=torch.float64) * 0.5
    mask = torch.ones(2, 9, dtype=torch.int64)
    mask[1, -2:] = 0
    want = O.llama_forward(embeds, mask, O._SD(merged, torch.float64), hp)
    got = R.llama_forward(embeds, mask, sd, hp, adapters)
    ones = R.llama_forward(embeds, mask, sd, hp, adapters, mask_fn=lambda n, r, c: torch.ones(r, c, dtype=torch.float64))
    base = O.llama_forward(embeds, mask, O._SD(sd, torch.float64), hp)
    e = float((got - want).norm() / want.norm())
    assert e < 1e-12 and torch.equal(got, ones) and float((base - want).norm() / want.norm()) > 1e-3, e
