"""CPU tier: the drop-in class surface (SURVEY.md §8b) — constructor kwargs, attribute / state_dict names,
config round trip, loud failure without CUDA, batch sharding under a world_size-2 gloo group."""
import os
import sys

import pytest
import torch

from tests import helpers as H
from tests.golden import gen


def _tiny_cfg():
    from macaw_llm_b200.modeling import MM_LLMs_Config

    clip, whisper, llama = gen.build_configs(gen.TINY)
    return MM_LLMs_Config(n_frames=2, attention_heads=2, clip_config=clip, whisper_config=whisper, llm_config=llama)


def test_state_dict_keys_and_shapes_match_reference():
    from macaw_llm_b200.modeling import MM_LLMs

    _, _, shapes = H.load_shapes()  # keys/shapes of the live reference model (tests/golden/make_golden.py)
    sd = MM_LLMs(_tiny_cfg()).state_dict()
    assert set(sd) == set(shapes)
    assert all(tuple(sd[k].shape) == shapes[k] for k in shapes)


def test_config_surface_roundtrip(tmp_path):
    import modeling  # root-level drop-in module name used by the reference's callers

    cfg = _tiny_cfg()
    assert modeling.MM_LLMs_Config is modeling.MM_LLMsConfig
    assert cfg.model_type == "mm_llms" and cfg.hidden_size == 256
    d = cfg.to_dict()
    for k in ("image_config", "audio_config", "llm_config", "n_frames", "attention_heads", "image_conv_kernel",
              "image_conv_stride", "video_conv_kernel", "video_conv_stride", "audio_conv_kernel", "audio_conv_stride",
              "hidden_size", "model_type"):
        assert k in d
    cfg.save_pretrained(tmp_path)
    c2 = modeling.MM_LLMs_Config.from_pretrained(tmp_path)
    assert (c2.n_frames, c2.attention_heads, c2.audio_conv_kernel) == (2, 2, 240)
    assert c2.llm_config.hidden_size == 256 and c2.image_config.projection_dim == 192
    dflt = modeling.MM_LLMs_Config(clip_config=cfg.image_config, whisper_config=cfg.audio_config, llm_config=cfg.llm_config)
    assert (dflt.n_frames, dflt.attention_heads, dflt.image_conv_kernel, dflt.image_conv_stride, dflt.video_conv_kernel,
            dflt.video_conv_stride, dflt.audio_conv_kernel, dflt.audio_conv_stride) == (6, 8, 48, 36, 36, 30, 240, 220)


def test_reference_caller_surface():
    """What run_clm_llms.py / llm_trainer.py reach for (SURVEY.md §8b)."""
    from macaw_llm_b200.modeling import MM_LLMs

    m = MM_LLMs(_tiny_cfg())
    for attr in ("image_encoder", "video_encoder", "audio_encoder", "llm", "prepare_inputs_for_generation",
                 "encode_image", "encode_audio", "encode_video_long"):
        assert hasattr(m, attr)
    m.llm.resize_token_embeddings(512 + 7)  # run_clm_llms.py:495
    assert m.llm.model.embed_tokens.weight.shape[0] == 519 and m.llm.lm_head.weight.shape[0] == 519
    frozen = [n for n, _ in m.named_parameters() if "encoder" in n]  # run_clm_llms.py:390-393 name test
    assert frozen and all(n.split(".")[0] in ("image_encoder", "video_encoder", "audio_encoder") or "encoder" in n for n in frozen)
    with pytest.raises(RuntimeError, match="no CPU"):  # the generate branch exists, but nothing executes on the CPU
        m({"inference": True, "input_ids": torch.ones(1, 4, dtype=torch.long), "images": None, "audios": None,
           "videos": None})


def test_cpu_parameters_raise():
    model, spec, hp, _ = H.build_tiny_model("cpu", torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU"):
        model(H.case_inputs(spec, H.load_case("text")))


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from macaw_llm_b200 import dist as D

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    inp = gen.make_inputs(gen.TINY, 5, 9, seed=3, modalities=("image",))
    sh = D.shard_inputs(inp, rank, world)
    lo, hi = D.shard_range(5, rank, world)
    ok = torch.equal(sh["input_ids"], inp["input_ids"][lo:hi]) and sh["images"].shape[0] == hi - lo and sh["videos"] is None
    ms = D.max_over_ranks(10.0 + rank)
    loss = D.weighted_mean_loss(float(rank + 1) * (hi - lo), hi - lo)
    q.put((rank, ok, lo, hi, ms, loss))
    dist.destroy_process_group()


def test_sharding_and_reductions_world2_gloo():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = sorted(q.get(timeout=120) for _ in ps)
    [p.join(60) for p in ps]
    assert [r[1] for r in res] == [True, True]
    assert (res[0][2], res[0][3], res[1][2], res[1][3]) == (0, 3, 3, 5)      # contiguous cover of the global batch
    assert res[0][4] == res[1][4] == 11.0                                      # max over ranks
    assert abs(res[0][5] - (1 * 3 + 2 * 2) / 5) < 1e-12                        # token-weighted global mean


def _gloo_grad_worker(rank, world, port, q):
    """Each rank differentiates ITS shard with the CPU gradient oracle, deposits the gradients in the flat GradBuffer and
    all-reduces it; rank 0 reports a few entries."""
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from macaw_llm_b200 import dist as D
    from macaw_llm_b200.training import GradBuffer, allreduce_grads
    from oracle import macaw_oracle as O

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    model, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    inp = gen.make_inputs(spec, 4, 12, seed=11, modalities=(), with_labels=True)
    sh = D.shard_inputs(inp, rank, world)
    _, grads, _ = O.llama_loss_and_grads(sh, H.bf16_round(weights), hp)
    gb = GradBuffer(model)
    gb.attach()
    named = dict(model.named_parameters())
    for k, g in grads.items():
        named[k].grad.copy_(g)
    for i in range(len(gb.buckets)):  # bucket by bucket, as the backward pass issues them
        allreduce_grads(gb, world, bucket=i)
    # numpy arrays are pickled by value (torch tensors would travel as shared-memory handles that die with the worker)
    q.put((rank, {k: named[k].grad.float().numpy().copy() for k in ("llm.lm_head.weight", "llm.model.layers.0.mlp.up_proj.weight",
                                                                    "llm.model.norm.weight")}))
    dist.destroy_process_group()


def test_allreduced_gradient_equals_single_process_gradient_world2_gloo():
    """SURVEY.md §4 / §8e: the all-reduced (averaged) gradient of the per-rank mean losses equals the single-process
    gradient of their mean — through the flat GradBuffer buckets the training step uses."""
    import torch.multiprocessing as mp

    from macaw_llm_b200 import dist as D
    from oracle import macaw_oracle as O

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + os.getpid() % 1000
    ps = [ctx.Process(target=_gloo_grad_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = dict(q.get(timeout=300) for _ in ps)
    [p.join(60) for p in ps]
    _, spec, hp, weights = H.build_tiny_model("cpu", torch.bfloat16)
    inp = gen.make_inputs(spec, 4, 12, seed=11, modalities=(), with_labels=True)
    sd = H.bf16_round(weights)
    g0 = O.llama_loss_and_grads(D.shard_inputs(inp, 0, 2), sd, hp)[1]
    g1 = O.llama_loss_and_grads(D.shard_inputs(inp, 1, 2), sd, hp)[1]
    for k, got in res[0].items():
        got = torch.from_numpy(got)
        want = 0.5 * (g0[k] + g1[k])
        assert H.rel_err(got, want) < 1e-2, k                       # bf16 storage of the gradient buffer
        assert torch.equal(got, torch.from_numpy(res[1][k]))        # both ranks hold the same averaged gradient


def test_grad_buffer_layout_and_reference_freezing():
    """Host logic of the training step (reference run_clm_llms.py:390-393, llm_trainer.py:184-188): the trainable set is
    everything whose name lacks 'encoder' that the step differentiates; the flat gradient buffer lists it in BACKWARD order
    (lm_head, final norm, layers L-1 .. 0, then table + alignment modules) in contiguous, 16-byte aligned buckets."""
    from macaw_llm_b200.training import GradBuffer, freeze_like_reference, trainable_parameters

    model, spec, hp, _ = H.build_tiny_model("cpu", torch.bfloat16)
    freeze_like_reference(model)
    frozen = {n for n, p in model.named_parameters() if not p.requires_grad}
    assert frozen and all("encoder" in n for n in frozen)
    assert all(p.requires_grad for n, p in model.named_parameters() if "encoder" not in n)
    train = dict(trainable_parameters(model))
    assert not (set(train) & frozen)
    gb = GradBuffer(model)
    assert {id(p) for p in gb.params} == {id(p) for p in train.values()}, "buffer covers exactly the differentiated set"
    L = len(model.llm.model.layers)
    assert len(gb.buckets) == L + 2
    # buckets tile the flat buffer in order, every view is 16-byte aligned and views do not overlap
    assert gb.buckets[0][0] == 0 and gb.buckets[-1][1] == gb.flat.numel()
    assert all(gb.buckets[i][1] == gb.buckets[i + 1][0] for i in range(len(gb.buckets) - 1))
    spans = sorted((v.data_ptr(), v.numel() * 2) for v in gb.views.values())
    assert all(a % 16 == 0 for a, _ in spans)
    assert all(spans[i][0] + spans[i][1] <= spans[i + 1][0] for i in range(len(spans) - 1))
    assert sum(n for _, n in spans) == gb.flat.numel() * 2
    # backward order: lm_head first, layer L-1 before layer 0, the embedding table in the last bucket
    off = {id(p): (gb.views[id(p)].data_ptr() - gb.flat.data_ptr()) // 2 for p in gb.params}
    llm = model.llm
    assert off[id(llm.lm_head.weight)] == 0
    assert off[id(llm.model.layers[L - 1].mlp.down_proj.weight)] < off[id(llm.model.layers[0].mlp.down_proj.weight)]
    s, e = gb.buckets[-1]
    assert s <= off[id(llm.model.embed_tokens.weight)] < e and s <= off[id(model.image_align_attention.in_proj_weight)] < e
    # attach(): p.grad views the buffer; a second attach reports "accumulate", zero() detaches
    fresh = gb.attach(skip=gb.align_params["video"])
    assert all(fresh.values()) and model.video_align_attention.in_proj_weight.grad is None
    assert llm.lm_head.weight.grad.data_ptr() == gb.flat.data_ptr()
    again = gb.attach(skip=gb.align_params["video"])
    assert not again[id(llm.lm_head.weight)] and again[id(model.video_align_attention.in_proj_weight)]
    gb.zero()
    assert llm.lm_head.weight.grad is None


def test_grad_buffer_with_frozen_decoder_layers():
    """freeze_llama_layers (bench.py --mode train): frozen decoder layers leave the trainable set and the flat gradient
    buffer (their bucket is empty, so no optimizer state either); every other parameter keeps its slot and order."""
    from macaw_llm_b200.training import GradBuffer, freeze_like_reference, freeze_llama_layers, trainable_parameters

    model, spec, hp, _ = H.build_tiny_model("cpu", torch.bfloat16)
    freeze_like_reference(model)
    full = GradBuffer(model)
    freeze_llama_layers(model, 1)
    frozen = {n for n, p in model.named_parameters() if n.startswith("llm.model.layers.0.")}
    assert frozen and all(not p.requires_grad for n, p in model.named_parameters() if n in frozen)
    assert all(p.requires_grad for n, p in model.named_parameters() if n.startswith("llm.model.layers.1."))
    train = dict(trainable_parameters(model))
    assert not (set(train) & frozen)
    gb = GradBuffer(model)
    assert {id(p) for p in gb.params} == {id(p) for p in train.values()}
    L = len(model.llm.model.layers)
    assert len(gb.buckets) == L + 2 and gb.buckets[L][0] == gb.buckets[L][1]  # layer 0 = the last layer bucket: empty
    n_frozen = sum(p.numel() for n, p in model.named_parameters() if n in frozen)
    assert gb.flat.numel() == full.flat.numel() - n_frozen
    with pytest.raises(ValueError):
        freeze_llama_layers(model, L + 1)
    freeze_llama_layers(model, 0)
    assert all(p.requires_grad for p in model.llm.parameters())
