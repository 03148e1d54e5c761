"""End-to-end parity of the CUDA path on the H100 against (a) the golden vectors minted from the unmodified reference
and (b) the CPU oracle run on the SAME bf16-rounded weights and inputs.

Tolerances (norm-wise relative error, ||ours - ref|| / ||ref||):
  * int64 attention-mask / label prefix and the sequence layout: bit-exact.
  * embeds (prefix + text) and logits vs the fp32 oracle on bf16-rounded weights: the CUDA path stores activations in
    bf16 (one rounding = 2^-9 ~ 2e-3 per element, ~1.1e-3 norm-wise), so a chain of k bf16-stored stages cannot be
    better than ~sqrt(k) * 1.1e-3.  Bars: 1e-2 on the aligned prefix rows, 3e-2 on logits; the measured values are
    printed and recorded in DESIGN.md.
  * vs the golden fixtures (fp32 reference, unrounded weights) the bf16 weight rounding adds to that; bar 5e-2.
"""
import pytest
import torch

from tests import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    model, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    return model, spec, hp, weights


def _to_bf16_inputs(inp):
    out = {}
    for k, v in inp.items():
        if isinstance(v, torch.Tensor) and v.is_floating_point():
            out[k] = v.to(torch.bfloat16)
        else:
            out[k] = v
    return out


@pytest.mark.parametrize("name", ["all3", "image", "audio", "text"])
def test_forward_vs_golden_and_oracle(tiny, name):
    from oracle import macaw_oracle as O

    model, spec, hp, weights = tiny
    case = H.load_case(name)
    inp = _to_bf16_inputs(H.case_inputs(spec, case))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    out = model(dev_inp)
    emb, mask, labels = model.prepare_inputs_for_generation(dev_inp)
    torch.cuda.synchronize()

    # ---- layout / integer side: bit-exact against the reference fixture
    g_emb = torch.from_numpy(case["embeds"])
    assert tuple(emb.shape) == tuple(g_emb.shape)
    assert torch.equal(mask.cpu(), torch.from_numpy(case["attention_mask"]))
    if int(case["with_labels"]):
        assert torch.equal(labels.cpu(), torch.from_numpy(case["labels"]))
    else:
        assert labels is None and out.loss is None
    # text rows of the splice are pure gathers of bf16 table rows: bit-exact vs the bf16-rounded table
    table = weights["llm.model.embed_tokens.weight"].to(torch.bfloat16)
    n_prefix = emb.shape[1] - int(case["L"])
    ids = inp["input_ids"]
    assert torch.equal(emb[:, 0].cpu(), table[ids[:, 0]])
    assert torch.equal(emb[:, 1 + n_prefix:].cpu(), table[ids[:, 1:]])

    # ---- floating point: oracle on the same bf16-rounded weights / inputs
    sd = H.bf16_round(weights)
    o = O.forward({k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
                  sd, hp, dtype=torch.float32)
    e_emb = H.rel_err(emb, o["embeds"])
    e_pre = H.rel_err(emb[:, 1:1 + n_prefix], o["embeds"][:, 1:1 + n_prefix]) if n_prefix else 0.0
    valid = torch.from_numpy(case["attention_mask"]).bool()
    e_log = H.rel_err(out.logits.cpu()[valid], o["logits"][valid])
    e_gold = H.rel_err(out.logits.cpu()[valid], torch.from_numpy(case["logits"])[valid])
    # the reference algorithm's OWN bf16 arithmetic on the same inputs (oracle run in bf16 on the CPU) as the yardstick
    ob = O.forward({k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
                   sd, hp, dtype=torch.bfloat16)
    r_log = H.rel_err(ob["logits"][valid], o["logits"][valid])
    r_pre = H.rel_err(ob["embeds"][:, 1:1 + n_prefix], o["embeds"][:, 1:1 + n_prefix]) if n_prefix else 0.0
    print(f"\n[parity:{name}] prefix {e_pre:.3e}  embeds {e_emb:.3e}  logits {e_log:.3e}  logits-vs-golden {e_gold:.3e}"
          f"  | reference algorithm in bf16: prefix {r_pre:.3e} logits {r_log:.3e}")
    # prefix: the block output is rounded to bf16 once (1.1e-3 norm-wise); encoder features (bf16-stored CLIP / Whisper
    # layers) feed it, so the bar is 2.5e-3 here and 1.5e-3 for the alignment block alone (test_real_width_alignment_block)
    assert e_pre < 2.5e-3 and e_emb < 2.5e-3
    assert e_log < 1e-2 and e_log < 2.0 * max(r_log, 2e-3)
    assert e_gold < 2e-2
    if int(case["with_labels"]):
        assert abs(float(out.loss) - float(o["loss"])) < 2e-2 * abs(float(o["loss"]))


def test_one_token_forward_vs_oracle(tiny):
    """A text-only forward of L = 1 (T == 1, B <= 64, no KV cache) runs the same wide GEMMs as any other forward; only a
    decode step with a cache takes the thin tails."""
    from oracle import macaw_oracle as O

    model, spec, hp, weights = tiny
    inp = H.gen.make_inputs(spec, 4, 1, seed=105, modalities=(), with_labels=False)
    inp["input_ids"] = torch.tensor([[1], [7], [300], [55]])
    out = model({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    torch.cuda.synchronize()
    assert tuple(out.logits.shape) == (4, 1, spec["llama"]["vocab_size"]) and out.loss is None
    sd = H.bf16_round(weights)
    o = O.forward(inp, sd, hp, dtype=torch.float32)
    ob = O.forward(inp, sd, hp, dtype=torch.bfloat16)
    e_log = H.rel_err(out.logits.cpu(), o["logits"])
    r_log = H.rel_err(ob["logits"], o["logits"])
    print(f"\n[parity:T=1] logits {e_log:.3e} | reference algorithm in bf16: logits {r_log:.3e}")
    assert e_log < 1e-2 and e_log < 2.0 * max(r_log, 2e-3)


def test_encoders_vs_oracle(tiny):
    from oracle import macaw_oracle as O

    model, spec, hp, weights = tiny
    sd = O._SD(H.bf16_round(weights))
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    img = model.encode_image(inp["images"].cuda())
    aud = model.encode_audio(inp["audios"].cuda())
    vid = model.encode_video_long(inp["videos"].cuda())
    torch.cuda.synchronize()
    r_img = O.clip_tokens(inp["images"].float(), sd.sub("image_encoder."), hp)
    r_aud = O.whisper_encode(inp["audios"].float(), sd.sub("audio_encoder.encoder."), hp)
    r_vid = O.encode_video_long(inp["videos"].float(), sd, hp)
    e = (H.rel_err(img, r_img), H.rel_err(aud, r_aud), H.rel_err(vid, r_vid))
    print(f"\n[parity:encoders] image {e[0]:.3e} audio {e[1]:.3e} video {e[2]:.3e}")
    assert max(e) < 1e-2


def test_video_pe_matches_reference_loop(tiny):
    import numpy as np
    import os

    model = tiny[0]
    pe = model.engine.video_pe(40, 24, torch.device("cuda"))
    ref = torch.from_numpy(np.load(os.path.join(H.GOLDEN, "video_pe_40x24.npz"))["pe"])
    assert torch.equal(pe.cpu(), ref.to(torch.bfloat16))


def test_no_cpu_fallback():
    model, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    inp = H.case_inputs(spec, H.load_case("text"))
    with pytest.raises(RuntimeError, match="no CPU"):
        model(inp)


def test_real_width_alignment_block():
    """BASELINE config 1 shape on the GPU: 1 x 50 x 768 visual feats against a 32000 x 4096 table, 16 heads."""
    from macaw_llm_b200 import ops
    from macaw_llm_b200.engine import Engine
    from oracle import macaw_oracle as O

    torch.manual_seed(0)
    E, V, C, H = 4096, 32000, 768, 16

    class M(torch.nn.Module):
        pass

    m = M()
    m.project_image = torch.nn.Conv1d(C, C, 48, 36)
    m.transform_image_to_hidden = torch.nn.Linear(C, E)
    m.image_align_attention = torch.nn.MultiheadAttention(E, H, dropout=0.1, add_bias_kv=True, add_zero_attn=True)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() > 1:
                p.normal_(0, 0.02)
            else:
                p.normal_(0, 0.02)
    m = m.cuda().to(torch.bfloat16).eval()
    table = (torch.randn(V, E) * 0.5).cuda().to(torch.bfloat16)
    feats = torch.randn(1, 50, C).cuda().to(torch.bfloat16)
    eng = Engine(m)
    prefix = torch.zeros(1, 3, E, device="cuda", dtype=torch.bfloat16)
    Lq = eng.align(feats, "image", table, prefix, 1)
    torch.cuda.synchronize()
    assert Lq == 1
    sd = O._SD({k: v.detach().float().cpu() for k, v in m.state_dict().items()})
    ref = O.align_block(feats.float().cpu(), table.float().cpu(), sd.sub("project_image."),
                        sd.sub("transform_image_to_hidden."), sd.sub("image_align_attention."), 36, H)
    e = H_rel(prefix[:, 1:2], ref)
    # yardstick measured here: the EXACT fp32 result rounded once to bf16 (the block's output lands in the bf16
    # inputs_embeds, so no implementation can do better than this)
    e_round = H_rel(ref.to(torch.bfloat16), ref)
    print(f"\n[parity:align 32000x4096] {e:.3e}   (one bf16 rounding of the exact result: {e_round:.3e})")
    # fp16 activation chain inside the block: one bf16 rounding of the output + ~8 fp16-stored stages (1.9e-4 each)
    assert e < 2e-3 and e < 1.35 * e_round
    assert float(prefix[:, 0].abs().max()) == 0 and float(prefix[:, 2].abs().max()) == 0


def H_rel(a, b):
    return H.rel_err(a, b)


def test_real_width_reduced_depth_video_audio():
    """BASELINE config 5 shapes at REAL widths (CLIP-L/14 width, Whisper-base width, LLaMA-7B width, V=32000, 16 frames
    -> 4096 video tokens -> Lq=136, head_dim 96 video self-attention) with the DEPTHS cut to 2/1/1 layers so the CPU
    oracle finishes in seconds.  Exercises every real-width code path of video + audio + text, B=2, L=64."""
    import bench
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from oracle import macaw_oracle as O

    (clip, whisper, llama), hyper = bench.real_configs()
    clip.vision_config.num_hidden_layers = 2
    whisper.encoder_layers = 1
    llama.num_hidden_layers = 1
    hyper = dict(hyper, n_frames=16)
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device="cuda", dtype=torch.bfloat16, seed=1)
    g = torch.Generator().manual_seed(5)
    B, L, V = 2, 64, llama.vocab_size
    inp = dict(images=None,
               audios=torch.randn(B, 80, 3000, generator=g).to(torch.bfloat16),
               videos=torch.randn(B, 16, 3, 224, 224, generator=g).to(torch.bfloat16),
               input_ids=torch.randint(3, V - 6, (B, L), generator=g), attention_mask=torch.ones(B, L, dtype=torch.int64))
    inp["input_ids"][:, 0] = 1
    for i, name in enumerate(("image", "audio", "video")):
        inp[f"{name}_starts"] = torch.full((B,), V - 6 + 2 * i, dtype=torch.int32)
        inp[f"{name}_ends"] = torch.full((B,), V - 5 + 2 * i, dtype=torch.int32)
    out = model({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    emb, mask, _ = model.prepare_inputs_for_generation({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    torch.cuda.synchronize()
    T = 8 + 138 + L  # audio block 6+2, video block 136+2
    assert tuple(out.logits.shape) == (B, T, V) and tuple(emb.shape) == (B, T, 4096)
    assert torch.equal(mask.cpu(), torch.ones(B, T, dtype=torch.int64))
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    hp = O.hp_from_config(cfg)
    o = O.forward({k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
                  sd, hp, dtype=torch.float32)
    e_pre = H.rel_err(emb[:, 1:147], o["embeds"][:, 1:147])
    e_log = H.rel_err(out.logits, o["logits"])
    print(f"\n[parity:real-width video+audio] prefix {e_pre:.3e} logits {e_log:.3e}")
    assert e_pre < 1e-2 and e_log < 3e-2


def test_cuda_graph_replay_matches_eager(tiny):
    model, spec, hp, weights = tiny
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    ref = model(dev_inp)
    ref_logits, ref_loss = ref.logits.clone(), float(ref.loss)
    model.engine.enable_cuda_graphs(True)
    try:
        for _ in range(3):  # capture, then two replays
            out = model(inp)  # host tensors: copied into the graph's static inputs
            torch.cuda.synchronize()
            assert torch.equal(out.logits, ref_logits), float((out.logits.float() - ref_logits.float()).abs().max())
            assert abs(float(out.loss) - ref_loss) < 1e-5 * abs(ref_loss)  # CE uses float atomics: order-dependent last bits
        # different values, same signature -> same graph, new result
        inp2 = dict(inp)
        inp2["input_ids"] = inp["input_ids"].clone()
        inp2["input_ids"][:, 3] = 7
        out2 = model(inp2)
        torch.cuda.synchronize()
        assert not torch.equal(out2.logits, ref_logits)
    finally:
        model.engine.enable_cuda_graphs(False)
    eager2 = model({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp2.items()})
    assert torch.equal(eager2.logits, out2.logits), float((eager2.logits.float() - out2.logits.float()).abs().max())


def test_encoder_side_stream_option_is_bit_identical(tiny):
    """`engine.overlap_encoders = True` (Whisper tower on a side stream, joined before the alignment blocks) changes only
    the schedule: logits are bit-identical to the single-stream run, eagerly and under CUDA-graph capture."""
    model, spec, hp, weights = tiny
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    ref = model(dev_inp).logits.clone()
    model.engine.overlap_encoders = True
    try:
        assert torch.equal(model(dev_inp).logits, ref)
        model.engine.enable_cuda_graphs(True)
        for _ in range(2):
            out = model(inp)
            torch.cuda.synchronize()
            assert torch.equal(out.logits, ref)
    finally:
        model.engine.enable_cuda_graphs(False)
        model.engine.overlap_encoders = False


def test_resized_vocab_not_multiple_of_8():
    """The real pipeline resizes the table to 32007 rows (run_clm_llms.py:495): V % 8 != 0 exercises the padded score
    buffer, the ragged-K P.table GEMM and the unaligned (scalar-store) lm_head epilogue.  Tiny model, V = 512 + 7."""
    from oracle import macaw_oracle as O

    model, spec, hp, weights = H.build_tiny_model("cpu", torch.float32)
    model.llm.resize_token_embeddings(519)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        model.llm.model.embed_tokens.weight[512:].copy_(torch.randn(7, 256, generator=g) * 0.5)
        model.llm.lm_head.weight[512:].copy_(torch.randn(7, 256, generator=g) / 16)
    model = model.cuda().to(torch.bfloat16).eval()
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    for i, name in enumerate(("image", "audio", "video")):  # modal tokens live in the appended rows, as in the reference
        inp[f"{name}_starts"] = torch.full((2,), 513 + 2 * i, dtype=torch.int32)
        inp[f"{name}_ends"] = torch.full((2,), 514 + 2 * i, dtype=torch.int32)
    out = model({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    torch.cuda.synchronize()
    assert out.logits.shape[-1] == 519
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    hp2 = dict(hp, llama=dict(hp["llama"], vocab=519))
    o = O.forward({k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
                  sd, hp2, dtype=torch.float32)
    valid = o["attention_mask"].bool()
    e = H.rel_err(out.logits.cpu()[valid], o["logits"][valid])
    print(f"\n[parity:V=519] logits {e:.3e} loss {float(out.loss):.4f} vs {float(o['loss']):.4f}")
    assert e < 3e-2 and abs(float(out.loss) - float(o["loss"])) < 2e-2 * abs(float(o["loss"]))


def test_batch1_no_mask_no_labels(tiny):
    """Smallest call shapes: B=1, no attention_mask key, no labels (reference returns mask=None, labels=None)."""
    from oracle import macaw_oracle as O

    model, spec, hp, weights = tiny
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("image")))
    inp.pop("attention_mask")
    inp.pop("labels", None)
    emb, mask, labels = model.prepare_inputs_for_generation({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    out = model({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()})
    torch.cuda.synchronize()
    assert mask is None and labels is None and out.loss is None
    o = O.forward({k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
                  H.bf16_round(weights), hp, dtype=torch.float32)
    assert o["attention_mask"] is None
    assert H.rel_err(out.logits, o["logits"]) < 3e-2


def test_generate_greedy_vs_oracle(tiny):
    """inputs['inference'] = True (reference modeling.py:954-960): greedy decoding with the KV cache.  bf16 vs fp32 can
    flip an argmax between near-tied logits, so the check is teacher-forced: feeding the GPU's tokens to the oracle, every
    GPU-chosen token must be the oracle's top-1 or within a small margin of it, and the first token must match exactly
    when the oracle's top-2 gap is not a near-tie."""
    from oracle import macaw_oracle as O

    model, spec, hp, weights = tiny
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    inp.pop("labels", None)
    n_new = 6
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    toks = model(dict(dev_inp, inference=True, max_new_tokens=n_new))
    torch.cuda.synchronize()
    assert toks.dtype == torch.int64 and toks.shape[0] == 2 and 1 <= toks.shape[1] <= n_new
    f32 = {k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}
    o_toks, o_logits = O.generate_greedy(f32, H.bf16_round(weights), hp, max_new_tokens=toks.shape[1],
                                         forced_tokens=toks.cpu())
    for b in range(toks.shape[0]):
        for s_ in range(toks.shape[1]):
            t = int(toks[b, s_])
            if t == 32006:  # pad after EOS
                continue
            row = o_logits[b, s_]
            gap = float(row.max() - row[t])
            assert gap <= 0.05 * float(row.std()) + 1e-3, (b, s_, t, int(row.argmax()), gap)


def test_decode_step_matches_full_recompute(tiny):
    """KV-cache consistency on the GPU itself: logits of a cached decode step == logits of a fresh prefill over the
    extended sequence (both bf16 kernels; differences only from tile shapes / accumulation order)."""
    from macaw_llm_b200 import ops

    model, spec, hp, weights = tiny
    eng = model.engine
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("audio")))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items() if k not in ("labels", "attention_mask")}
    with torch.no_grad():
        embeds, _, _ = eng.prepare_inputs(dev_inp)
        B, T, E = embeds.shape
        table = eng.w(model.llm.model.embed_tokens.weight, "llm.embed")
        nxt = torch.tensor([5, 9], device="cuda")
        ext = torch.cat([embeds, table[nxt].unsqueeze(1)], dim=1)
        full = eng.llama_forward(ext.clone(), None)[:, -1, :]
        cache = [torch.empty((B, T + 4, 2, E), device="cuda", dtype=torch.bfloat16) for _ in model.llm.model.layers]
        x = embeds.reshape(B * T, E).clone()
        eng._llama_layers(x, B, T, None, 0, cache, T + 4)
        x1 = ops.embed_gather(table, nxt)
        x1 = eng._llama_layers(x1, B, 1, None, T, cache, T + 4)
        step = eng._lm_head(x1)
    torch.cuda.synchronize()
    assert H.rel_err(step, full) < 1e-2


def test_alignment_row_chunking(tiny):
    """The alignment scores buffer is chunked over query rows (video at large batch); force tiny chunks and compare."""
    model, spec, hp, weights = tiny
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("all3")))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    ref, _, _ = model.prepare_inputs_for_generation(dev_inp)
    model.engine.align_max_rows = 5  # video: Nq = 32 rows -> 7 chunks; image / audio: 12 rows -> 3 chunks
    try:
        got, _, _ = model.prepare_inputs_for_generation(dev_inp)
    finally:
        model.engine.align_max_rows = None
    torch.cuda.synchronize()
    assert H.rel_err(got, ref) < 2e-3


def test_fp32_and_fp16_parameter_models_use_bf16_shadows():
    """Reference users call model.half() (llm_trainer.py:366-368): non-bf16 parameters are shadowed to bf16 once per
    weight version; results equal the bf16 model built from the same (bf16-representable) weights."""
    model_bf16, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    model_f32, _, _, _ = H.build_tiny_model("cuda", torch.float32)
    with torch.no_grad():
        for (n, p32), (_, p16) in zip(model_f32.named_parameters(), model_bf16.named_parameters()):
            p32.copy_(p16.float())
    inp = _to_bf16_inputs(H.case_inputs(spec, H.load_case("image")))
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    a = model_bf16(dev_inp).logits
    b = model_f32(dev_inp).logits
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    # an in-place weight update must invalidate the shadow
    with torch.no_grad():
        model_f32.llm.lm_head.weight.mul_(2.0)
    c = model_f32(dev_inp).logits
    torch.cuda.synchronize()
    assert H.rel_err(c, 2.0 * a.float()) < 1e-2


def test_left_padding_does_not_leak_into_valid_positions(tiny):
    """DESIGN.md "unspecified rows": a query position whose own key is padding has every key masked; the reference then
    attends uniformly (additive finfo.min clamp), this implementation emits zeros for that row.  Those rows are never
    read by valid positions (padded keys are masked for everyone), so with LEFT padding — where such rows exist — the
    logits at all valid positions must still match the oracle."""
    from oracle import macaw_oracle as O
    from tests.golden import gen

    model, spec, hp, weights = tiny
    inp = gen.make_inputs(spec, 2, 14, seed=91, modalities=(), with_labels=False)
    mask = torch.ones(2, 14, dtype=torch.int64)
    mask[0, :5] = 0        # left padding in sample 0 (text-only: no prefix in front of it)
    inp["attention_mask"] = mask
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    out = model(dev_inp)
    o = O.forward(inp, H.bf16_round(weights), hp, dtype=torch.float32)
    valid = mask.bool()
    e = H.rel_err(out.logits.cpu()[valid], o["logits"][valid])
    print(f"\n[parity:left padding] logits at valid positions {e:.3e}")
    assert e < 1e-2
    assert torch.isfinite(out.logits.float()).all()   # the masked rows are zeros / finite, never NaN
