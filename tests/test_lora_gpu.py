"""GPU tier: LoRA adapters — the four adapter kernels (csrc/lora.cu) against fp64 torch, the tiny model's training step
with adapters against autograd of the fp32 oracle, graph replay, and inference / generation on the folded weights."""
import copy

import pytest
import torch

from tests import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16
# storage-rounding bars of a 16-bit result (test_train_gpu.py / test_train_fp16_gpu.py use 8e-3 / 1e-3 for single kernels)
BAR16 = {BF16: 8e-3, F16: 1e-3}


def _ops(fmt=BF16):
    from macaw_llm_b200 import ops

    ops.set_act_format(fmt)
    return ops


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def rope_ref(y, cos, sin, T):
    """rotate-half RoPE over 128-wide heads, position = row % T (fp64)."""
    M, N = y.shape
    pos = torch.arange(M, device=y.device) % T
    c, s = cos[pos].double().repeat(1, N // 128), sin[pos].double().repeat(1, N // 128)
    y = y.view(M, N // 128, 2, 64)
    lo, hi = y[:, :, 0].reshape(M, -1), y[:, :, 1].reshape(M, -1)
    return torch.stack([(lo * c - hi * s).view(M, -1, 64), (hi * c + lo * s).view(M, -1, 64)], 2).reshape(M, N)


# (M, K, N, r, adapters sharing x, RoPE): q/k/v, gate/up, down, lm_head (ragged M)
# + a 32007-row lm_head (odd row stride, column tail) with a K that is not a multiple of the 64-column chunk
CASES = [(2112, 4096, 4096, 8, 3, True), (2112, 4096, 11008, 16, 2, False), (2112, 11008, 4096, 64, 1, False),
         (1000, 4096, 32000, 8, 1, False), (600, 4104, 32007, 8, 1, False)]


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "M{}_K{}_N{}_r{}_n{}{}".format(*c[:5], "_rope" if c[5] else ""))
@pytest.mark.parametrize("fmt", [BF16, F16], ids=["bf16", "fp16"])
def test_lora_kernels_vs_fp64(fmt, case, dropout):
    """u = drop(x) A^T, y <- rope(y + s u B^T), g = s dy B, dB (+)= s dy^T u, dA (+)= g^T drop(x), dx += drop(g A) against
    fp64 torch on the same 16-bit operands and the masks of ops.dropout_mask; two launches are bit-identical.  The
    dropout cases accumulate into existing gradients, the others overwrite them."""
    ops = _ops(fmt)
    try:
        M, K, N, r, n, rope = case
        g = torch.Generator(device=DEV).manual_seed(M + K + N + r)
        rn = lambda *s, scale=1.0: (torch.randn(*s, device=DEV, generator=g) * scale).to(fmt)  # noqa: E731
        x = rn(M, K)
        As = [rn(r, K, scale=K ** -0.5) for _ in range(n)]
        Bs = [rn(N, r, scale=0.5) for _ in range(n)]
        s, p = 2.0, 0.05
        seed = torch.tensor([(3 << 32) | 77], dtype=torch.int64, device=DEV)
        sids = [40 + j for j in range(n)]
        drop = (p, seed, sids) if dropout else None
        masks = [ops.dropout_mask(M, K, (p, seed, sid), DEV).double() if dropout else torch.ones(M, K, device=DEV,
                                                                                               dtype=torch.float64)
                 for sid in sids]
        xd = x.double()
        errs = {}
        # ---- down
        us = ops.lora_down(x, As, dropout=drop)
        us2 = ops.lora_down(x, As, dropout=drop)
        assert all(torch.equal(a, b) for a, b in zip(us, us2))
        for j in range(n):
            errs[f"u{j}"] = rel(us[j], (xd * masks[j]) @ As[j].double().t())
        # ---- up (in place, RoPE for the q / k case)
        ys = [rn(M, N) for _ in range(n)]
        y0 = [y.clone() for y in ys]
        cos, sin = _rope_tables(528)
        ops.lora_up(ys, us, Bs, s, rope=(cos, sin, 528) if rope else None)
        ys2 = [y.clone() for y in y0]
        ops.lora_up(ys2, us, Bs, s, rope=(cos, sin, 528) if rope else None)
        assert all(torch.equal(a, b) for a, b in zip(ys, ys2))
        for j in range(n):
            ref = y0[j].double() + s * us[j].double() @ Bs[j].double().t()
            if rope:
                ref = rope_ref(ref, cos, sin, 528)
            errs[f"y{j}"] = rel(ys[j], ref)
        # ---- backward through dy
        dys = [rn(M, N) for _ in range(n)]
        acc = [dropout] * n
        dB0 = [rn(N, r) if dropout else torch.full((N, r), float("nan"), device=DEV, dtype=fmt) for _ in range(n)]
        dBs = [d.clone() for d in dB0]
        gs = ops.lora_bwd_dy(dys, us, Bs, dBs, s, acc)
        dBs2 = [d.clone() for d in dB0]
        gs2 = ops.lora_bwd_dy(dys, us, Bs, dBs2, s, acc)
        assert all(torch.equal(a, b) for a, b in zip(gs + dBs, gs2 + dBs2))
        for j in range(n):
            errs[f"g{j}"] = rel(gs[j], s * dys[j].double() @ Bs[j].double())
            ref = s * dys[j].double().t() @ us[j].double() + (dB0[j].double() if dropout else 0.0)
            errs[f"dB{j}"] = rel(dBs[j], ref)
        # ---- backward through x
        dA0 = [rn(r, K, scale=10.0) if dropout else torch.full((r, K), float("nan"), device=DEV, dtype=fmt) for _ in range(n)]
        dAs, dx = [d.clone() for d in dA0], rn(M, K)
        dx0 = dx.clone()
        ops.lora_bwd_x(x, gs, As, dAs, dx, acc, dropout=drop)
        dAs2, dx2 = [d.clone() for d in dA0], dx0.clone()
        ops.lora_bwd_x(x, gs, As, dAs2, dx2, acc, dropout=drop)
        assert all(torch.equal(a, b) for a, b in zip(dAs + [dx], dAs2 + [dx2]))
        ref_dx = dx0.double()
        for j in range(n):
            gd = gs[j].double()
            ref = gd.t() @ (xd * masks[j]) + (dA0[j].double() if dropout else 0.0)
            errs[f"dA{j}"] = rel(dAs[j], ref)
            ref_dx = ref_dx + (gd @ As[j].double()) * masks[j]
        errs["dx"] = rel(dx, ref_dx)
        print(f"\n[lora {fmt} {case} dropout={dropout}] " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
        for k, v in errs.items():
            assert v < (1e-5 if k[0] in "ug" else BAR16[fmt]), (k, v)
    finally:
        _ops(BF16)


def _rope_tables(T, hd=128):
    inv = (1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))).to(DEV)
    fr = torch.arange(T, device=DEV, dtype=torch.float32)[:, None] * inv[None, :]
    return fr.cos().contiguous(), fr.sin().contiguous()


def test_lora_refuses_bad_arguments():
    ops = _ops()
    x = torch.zeros(64, 256, device=DEV, dtype=BF16)
    with pytest.raises(RuntimeError, match="r must be a multiple of 8"):
        ops.lora_down(x, [torch.zeros(12, 256, device=DEV, dtype=BF16)])


# ---------------------------------------------------------------------------------------------------- tiny model
ALL_TARGETS = ["q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj", "lm_head"]


def _lora_model(fmt, targets=ALL_TARGETS, dropout=0.0, unit_gains=False):
    from macaw_llm_b200.lora import LoraConfig

    model, spec, hp, weights = H.build_tiny_model(DEV, fmt)
    if unit_gains:  # the folded gain is then exact, so attached and merged adapters give the same derived weights
        with torch.no_grad():
            for n, p in model.llm.named_parameters():
                if "norm" in n:
                    p.fill_(1.0)
    torch.manual_seed(3)
    model.add_lora(LoraConfig(r=8, lora_alpha=16, lora_dropout=dropout, target_modules=targets))
    return model, spec, hp


def _randomise_B(model, std=0.05):
    from macaw_llm_b200 import lora

    g = torch.Generator(device=DEV).manual_seed(11)
    with torch.no_grad():
        for lin in lora.adapted_modules(model).values():
            lin.lora_B.weight.copy_(torch.randn(lin.lora_B.weight.shape, device=DEV, generator=g) * std)


def _inputs(spec, fmt, modalities=("image", "audio"), seed=78, B=2, L=14):
    from tests.golden import gen

    inp = gen.make_inputs(spec, B, L, seed=seed, modalities=modalities, pad_tail=2, with_labels=True)
    return {k: (v.to(fmt).to(DEV) if isinstance(v, torch.Tensor) and v.is_floating_point() else
                (v.to(DEV) if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()}


def _effective_state(model):
    """fp32 CPU state dict with every adapter merged in fp32 (W + s B A): the oracle's weights."""
    from macaw_llm_b200 import lora

    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items() if ".lora_" not in k}
    for name, lin in lora.adapted_modules(model).items():
        sd[f"llm.{name}.weight"] = lora.merged_weight(lin).cpu()
    return sd


@pytest.mark.parametrize("lora_dropout", [0.0, 0.05], ids=["p0", "p0.05"])
@pytest.mark.parametrize("fmt", [BF16, F16], ids=["bf16", "fp16"])
def test_training_step_gradients_vs_oracle(fmt, lora_dropout):
    """Loss and the gradient of every adapter and alignment parameter against autograd of the fp32 oracle with the LoRA
    term (tests/lora_reference.py), with the adapters' input dropout off and at the reference's p = 0.05 (the reference
    applies the masks ops.dropout_mask regenerates from the step's seed and each adapter's stream id); the base
    parameters get no gradient and are bit-unchanged by the optimizer step; a few steps lower the loss.  fp16 runs with
    DynamicLossScaler."""
    from macaw_llm_b200 import lora
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, trainable_parameters
    from tests import lora_reference as R

    from macaw_llm_b200 import ops

    model, spec, hp = _lora_model(fmt, dropout=lora_dropout)
    _randomise_B(model)
    inp = _inputs(spec, fmt)
    scaler = DynamicLossScaler(initial_scale_power=12) if fmt == F16 else None
    model.train()
    model.train_step.attention_dropout = False
    try:
        out = model(inp)
        (scaler.scale(out.loss) if scaler else out.loss).backward()
        torch.cuda.synchronize()
    finally:
        model.eval()
    S = scaler.loss_scale if scaler else 1.0
    mask_fn = None
    if lora_dropout > 0:
        seed = model.train_step.last_seed

        def mask_fn(name, rows, cols):
            layer = None if name == "lm_head" else int(name.split(".")[2])
            sid = lora.lora_sid(layer, name.rsplit(".", 1)[-1])
            return ops.dropout_mask(rows, cols, (lora_dropout, seed, sid), DEV).cpu()

    adapters = {n: (lin.lora_A.weight, lin.lora_B.weight, lin.lora_scaling) for n, lin in lora.adapted_modules(model).items()}
    sd = {k: v for k, v in model.state_dict().items() if ".lora_" not in k}
    loss_ref, gref = R.loss_and_grads({k: (v.float().cpu() if isinstance(v, torch.Tensor) and v.is_floating_point()
                                           else (v.cpu() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()},
                                      sd, hp, adapters, mask_fn)
    assert abs(float(out.loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    named = dict(model.named_parameters())
    errs = {k: rel(named[k].grad.double().cpu() / S, gr) for k, gr in gref.items()
            if ".lora_" in k or k.startswith(("project_image", "project_audio", "transform_image", "transform_audio",
                                               "image_align", "audio_align"))}
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print(f"\n[lora train {fmt} p={lora_dropout}] loss {float(out.loss):.5f} vs {float(loss_ref):.5f}; worst: "
          + ", ".join(f"{k}={v:.2e}" for k, v in top))
    for k, v in errs.items():
        assert v < (3e-2 if ".lora_" in k else 5e-2), (k, v)  # the whole-model bars of test_train_gpu.py
    for n, p in model.named_parameters():
        if n.startswith("llm.") and ".lora_" not in n:
            assert p.grad is None, n
    # optimizer steps: base bit-unchanged, loss goes down
    base = {n: p.detach().clone() for n, p in model.named_parameters() if n.startswith("llm.") and ".lora_" not in n}
    opt = FusedAdamW([p for _, p in trainable_parameters(model)], lr=3e-3, weight_decay=0.0, max_grad_norm=1.0)
    model.train()
    losses = []
    try:
        for _ in range(6):
            opt.zero_grad()
            out = model(inp)
            (scaler.scale(out.loss) if scaler else out.loss).backward()
            opt.step(loss_scaler=scaler)
            losses.append(float(out.loss))
    finally:
        model.eval()
    print(f"[lora train {fmt}] losses {['%.4f' % v for v in losses]}")
    assert losses[-1] < losses[0] - 0.02
    assert all(torch.equal(p, base[n]) for n, p in model.named_parameters() if n in base)


def test_training_step_graph_replay_matches_eager():
    """The whole step (forward with the adapters' input dropout live, backward, AdamW) captured once and replayed, against
    eager steps from the same state: bit-identical adapters (every adapter reduction is a fixed-order sum; text-only
    inputs keep the alignment blocks' atomics out)."""
    from macaw_llm_b200 import lora
    from macaw_llm_b200.training import FusedAdamW, trainable_parameters

    model0, spec, hp = _lora_model(BF16, dropout=0.05)
    inp = _inputs(spec, BF16, modalities=(), seed=5, B=2, L=24)
    k = 4
    runs = {}
    for mode in ("eager", "graph"):
        m = copy.deepcopy(model0)
        opt = FusedAdamW([p for _, p in trainable_parameters(m)], lr=1e-3, weight_decay=0.0)
        m.train()

        def step():
            opt.zero_grad()
            m(inp).loss.backward()
            opt.step()

        try:
            if mode == "graph":
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    step()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    step()
                for _ in range(k - 1):
                    graph.replay()
            else:
                for _ in range(k):
                    step()
            torch.cuda.synchronize()
        finally:
            m.eval()
        runs[mode] = {n: p.detach().clone() for n, p in m.named_parameters() if ".lora_" in n}
        assert int(m.train_step._seed) == m.train_step.dropout_base_seed + k  # one fresh dropout seed per step
    assert runs["eager"].keys() == runs["graph"].keys() and len(runs["eager"]) == 2 * len(lora.adapted_modules(model0))
    for n in runs["eager"]:
        assert torch.equal(runs["eager"][n], runs["graph"][n]), n


def _train_once(model, inp, lr=2e-2):
    from macaw_llm_b200.training import FusedAdamW, trainable_parameters

    opt = FusedAdamW([p for _, p in trainable_parameters(model)], lr=lr, weight_decay=0.0)
    model.train()
    try:
        opt.zero_grad()
        model(inp).loss.backward()
        opt.step()
        torch.cuda.synchronize()
    finally:
        model.eval()


def test_inference_with_adapters():
    """B = 0: eval logits byte-identical to the model without adapters.  After training: eval logits match the fp32 oracle
    of the adapted model; generate with attached adapters gives the tokens of the merged model; generate, a training step,
    generate: the second call (and a forward replayed through enable_cuda_graphs) reflects the new adapters."""
    from oracle import macaw_oracle as O
    from macaw_llm_b200.lora import LoraConfig

    plain, spec, hp, _ = H.build_tiny_model(DEV, BF16)
    inp = _inputs(spec, BF16, seed=21)
    with torch.no_grad():
        want = plain(inp).logits.clone()
    plain.add_lora(LoraConfig(target_modules=ALL_TARGETS))
    with torch.no_grad():
        got = plain(inp).logits
    assert torch.equal(got, want)

    model, spec, hp = _lora_model(BF16, unit_gains=True)
    _train_once(model, inp)
    _train_once(model, inp)
    with torch.no_grad():
        logits = model(inp).logits.float().cpu()
    ref = O.forward({k: (v.float().cpu() if isinstance(v, torch.Tensor) and v.is_floating_point()
                         else (v.cpu() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()},
                    _effective_state(model), hp)["logits"]
    e = rel(logits, ref)
    print(f"\n[lora eval] logits vs oracle rel {e:.2e}")
    assert e < 2e-2
    gen_in = {k: v for k, v in inp.items() if k not in ("labels",)}
    gen_in["inference"], gen_in["max_new_tokens"] = True, 8
    t1 = model(gen_in)
    merged = copy.deepcopy(model)
    merged.merge_lora()
    assert torch.equal(t1, merged(gen_in))
    # generate -> train -> generate, and the graphed forward
    model.engine.enable_cuda_graphs(True)
    try:
        with torch.no_grad():
            g1 = model(inp).logits.clone()
        _train_once(model, inp)
        t2 = model(gen_in)
        with torch.no_grad():
            g2 = model(inp).logits.clone()
    finally:
        model.engine.enable_cuda_graphs(False)
    with torch.no_grad():
        eager = model(inp).logits
    merged = copy.deepcopy(model)
    merged.merge_lora()
    assert torch.equal(t2, merged(gen_in))
    assert torch.equal(g2, eager) and not torch.equal(g1, g2)


def test_two_forwards_then_one_backward_keep_their_own_dropout_masks():
    """Each forward keeps its adapters' dropout seed with its saved activations: (loss_a + loss_b).backward() gives the
    gradients of backward(a) followed by backward(b), forwards in the same order (seeds s + 1, s + 2 either way)."""
    from macaw_llm_b200 import lora

    model0, spec, hp = _lora_model(BF16, dropout=0.05)
    _randomise_B(model0)
    a = _inputs(spec, BF16, modalities=(), seed=31, B=2, L=20)
    b = _inputs(spec, BF16, modalities=(), seed=32, B=2, L=20)
    grads = {}
    for mode in ("joint", "separate"):
        m = copy.deepcopy(model0)
        m.train()
        try:
            if mode == "joint":
                (m(a).loss + m(b).loss).backward()
            else:
                m(a).loss.backward()
                m(b).loss.backward()
            torch.cuda.synchronize()
        finally:
            m.eval()
        grads[mode] = {n: lin.lora_A.weight.grad.float().clone() for n, lin in lora.adapted_modules(m).items()}
    worst = max(rel(grads["joint"][n], grads["separate"][n]) for n in grads["joint"])
    print(f"\n[lora two forwards] worst adapter-gradient rel diff {worst:.2e}")
    assert worst < 1e-2
