"""Training step on the H100 (SURVEY.md §8f rank 1): every backward kernel against torch autograd of the same op, the
whole decoder's gradients against autograd of the CPU oracle (fp32, same bf16-rounded weights), the fused AdamW against
torch.optim.AdamW, and a few optimisation steps through the public `model(inputs).loss.backward()` path.

Gradients are bf16 tensors produced from bf16-stored activations: per-op bars are 6e-3 (one bf16 rounding of the result
+ bf16 inputs), whole-model gradient bars 3e-2 norm-wise per parameter tensor (measured values are printed)."""
import math

import pytest
import torch

from tests import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from macaw_llm_b200 import ops

    return ops


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(torch.bfloat16)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


@pytest.mark.parametrize("M,N,K", [(2112, 4096, 4096), (300, 1000, 520), (528, 512, 256), (70, 11008, 4096)])
def test_gemm_dx_dw(M, N, K):
    """dX = dY W (MN-major B) and dW = dY^T X (MN-major A and B), with and without accumulation."""
    ops = _ops()
    x, w, dy = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(M, N, seed=3)
    dx = ops.gemm_dx(dy, w)
    assert rel(dx, dy.float() @ w.float()) < 4e-3
    dw = torch.empty(N, K, device=DEV, dtype=torch.bfloat16)
    ops.gemm_dw(dy, x, dw, accumulate=False)
    ref = dy.float().t() @ x.float()
    assert rel(dw, ref) < 4e-3
    ops.gemm_dw(dy, x, dw, accumulate=True)
    assert rel(dw, 2 * ref) < 6e-3
    ops.gemm_dx(dy, w, out=dx, accumulate=True)
    assert rel(dx, 2 * (dy.float() @ w.float())) < 6e-3


def test_rmsnorm_swiglu_backward():
    ops = _ops()
    rows, cols = 300, 4096
    x, g, dy, dres = rnd(rows, cols, seed=4), (1 + 0.1 * rnd(cols, seed=5).float()).to(torch.bfloat16), rnd(rows, cols, seed=6), rnd(rows, cols, seed=7)
    xf = x.float().requires_grad_(True)
    gf = g.float().requires_grad_(True)
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * gf
    y.backward(dy.float())
    rstd = ops.rms_rstd(x, 1e-6)
    dg = torch.zeros(cols, device=DEV)
    dx = ops.rmsnorm_bwd(dy, x, rstd, g, dres, dg)
    assert rel(dx, xf.grad + dres.float()) < 4e-3 and rel(dg, gf.grad) < 2e-3
    # narrow rows (tiny models) and no residual branch
    x2, dy2 = rnd(37, 256, seed=8), rnd(37, 256, seed=9)
    g2 = torch.ones(256, device=DEV, dtype=torch.bfloat16)
    x2f = x2.float().requires_grad_(True)
    (x2f * torch.rsqrt(x2f.pow(2).mean(-1, keepdim=True) + 1e-6)).backward(dy2.float())
    assert rel(ops.rmsnorm_bwd(dy2, x2, ops.rms_rstd(x2, 1e-6), g2, None, None), x2f.grad) < 4e-3
    # SwiGLU
    gt, up, dh = rnd(64, 1024, seed=10), rnd(64, 1024, seed=11), rnd(64, 1024, seed=12)
    gtf, upf = gt.float().requires_grad_(True), up.float().requires_grad_(True)
    h = torch.nn.functional.silu(gtf) * upf
    h.backward(dh.float())
    assert rel(ops.swiglu_fwd(gt, up), h) < 4e-3
    dgt, dup = ops.swiglu_bwd(dh, gt, up)
    assert rel(dgt, gtf.grad) < 4e-3 and rel(dup, upf.grad) < 4e-3


@pytest.mark.parametrize("B,H,T,hd,causal,masked", [(2, 4, 528, 128, True, False), (2, 2, 200, 128, True, True),
                                                    (1, 2, 300, 64, False, False)])
def test_attention_backward(B, H, T, hd, causal, masked):
    ops = _ops()
    q, k, v, do = (rnd(B, T, H, hd, seed=20 + i) for i in range(4))
    km = None
    if masked:
        km = torch.ones(B, T, dtype=torch.int32, device=DEV)
        km[0, T - 37:] = 0
    scale = hd ** -0.5
    qf, kf, vf = (t.float().permute(0, 2, 1, 3).requires_grad_(True) for t in (q, k, v))
    s = (qf @ kf.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(T, T, device=DEV, dtype=torch.bool), 1), float("-inf"))
    if km is not None:
        s = s.masked_fill(km[:, None, None, :] == 0, float("-inf"))
    o = torch.softmax(s, -1) @ vf
    o.backward(do.float().permute(0, 2, 1, 3))
    dq, dk, dv = ops.attention_bwd(q, k, v, do, scale=scale, causal=causal, key_mask=km)
    e = [rel(a, b.grad.permute(0, 2, 1, 3)) for a, b in ((dq, qf), (dk, kf), (dv, vf))]
    print(f"\n[attention bwd B{B} H{H} T{T} hd{hd}] dq {e[0]:.2e} dk {e[1]:.2e} dv {e[2]:.2e}")
    assert max(e) < 8e-3


def test_ce_backward_scatter_colsum():
    ops = _ops()
    B, T, V = 2, 9, 519
    logits = rnd(B, T, V, scale=2.0, seed=30)
    labels = torch.randint(0, V, (B, T), generator=torch.Generator().manual_seed(1)).to(DEV)
    labels[0, :3] = -100
    lf = logits.float().requires_grad_(True)
    loss_ref = torch.nn.functional.cross_entropy(lf[:, :-1].reshape(-1, V), labels[:, 1:].reshape(-1), ignore_index=-100)
    loss_ref.backward()
    loss, cnt = ops.ce_loss_with_count(logits.clone(), labels)
    assert abs(float(loss) - float(loss_ref)) < 2e-3 * abs(float(loss_ref)) and int(cnt) == int((labels[:, 1:] != -100).sum())
    d = ops.ce_bwd(logits.clone(), labels, cnt, 0.5)
    assert rel(d, 0.5 * lf.grad) < 6e-3
    # embedding scatter-add with repeated ids
    table_g = torch.zeros(50, 64, device=DEV, dtype=torch.bfloat16)
    ids = torch.tensor([3, 7, 3, 49, 3, -1], device=DEV)
    dx = rnd(6, 64, seed=31)
    ops.embed_scatter_add(dx, ids, table_g)
    ref = torch.zeros(50, 64, device=DEV)
    ref.index_add_(0, ids[:5], dx[:5].float())
    assert rel(table_g, ref) < 8e-3
    cs = torch.zeros(64, device=DEV)
    ops.colsum(dx, cs)
    assert rel(cs, dx.float().sum(0)) < 1e-5


def test_fused_adamw_matches_torch():
    from macaw_llm_b200.training import FusedAdamW

    torch.manual_seed(0)
    p = torch.nn.Parameter(torch.randn(1000, 64, device=DEV).to(torch.bfloat16))
    ref = torch.nn.Parameter(p.detach().float().clone())
    opt = FusedAdamW([p], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    topt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    for i in range(3):
        g = torch.randn(1000, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(i)).to(torch.bfloat16)
        p.grad = g.clone()
        ref.grad = g.float()
        v0 = p._version
        opt.step()
        topt.step()
        assert p._version > v0  # the engine's weight caches key on the version counter
    assert rel(opt.state[id(p)][0], ref) < 1e-6 and rel(p, ref) < 3e-3


def test_dropout_mask_matches_philox_restatement():
    """mm_dropout_mask (the multipliers every dropout kernel regenerates) vs the numpy Philox4x32-10 restatement pinned to
    the published known-answer vectors (tests/test_oracle.py): bit-exact; a different seed / stream id gives a different
    mask; the forward and backward softmax kernels of a dropout attention apply exactly this mask."""
    ops = _ops()
    seed = torch.tensor([(9 << 32) | 1234567], dtype=torch.int64, device=DEV)
    m = ops.dropout_mask(67, 131, (0.1, seed, 3), DEV).cpu().numpy()
    want = H.dropout_multipliers(67, 131, 0.1, seed=(9 << 32) | 1234567, sid=3)
    assert (m == want).all()
    assert (ops.dropout_mask(67, 131, (0.1, seed, 4), DEV).cpu().numpy() != want).any()
    assert (ops.dropout_mask(67, 131, (0.1, seed + 1, 3), DEV).cpu().numpy() != want).any()
    # attention_train_fwd / attention_bwd against autograd with this mask
    B, Hh, T, hd, pd = 2, 3, 37, 96, 0.1
    q, k, v, do = (rnd(B, T, Hh, hd, scale=0.7, seed=s) for s in (1, 2, 3, 4))
    drop = (pd, seed, 7)
    o = ops.attention_train_fwd(q, k, v, scale=hd ** -0.5, dropout=drop)
    dq, dk, dv = ops.attention_bwd(q, k, v, do, scale=hd ** -0.5, causal=False, dropout=drop)
    mult = ops.dropout_mask(B * Hh * T, T, drop, DEV).view(B, Hh, T, T).double().cpu()
    qf, kf, vf = (t.double().cpu().permute(0, 2, 1, 3).requires_grad_(True) for t in (q, k, v))
    p = torch.softmax(qf @ kf.transpose(-1, -2) * hd ** -0.5, dim=-1) * mult
    of = p @ vf
    of.backward(do.double().cpu().permute(0, 2, 1, 3))
    assert rel(o.permute(0, 2, 1, 3), of.detach()) < 6e-3
    for got, ref in ((dq, qf.grad), (dk, kf.grad), (dv, vf.grad)):
        assert rel(got.permute(0, 2, 1, 3), ref) < 8e-3


@pytest.fixture(scope="module")
def tiny_train():
    model, spec, hp, weights = H.build_tiny_model("cuda", torch.bfloat16)
    return model, spec, hp, weights


def _oracle_dropout_masks(model, spec, present, B):
    """The attention-dropout multipliers the device kernels applied in the latest training forward (regenerated from its
    Philox seed through mm_dropout_mask), in the oracle's layout: (B*H, Lq, S+2) with batch-head index b*H + h."""
    ops = _ops()
    eng, ts = model.engine, model.train_step
    masks = {}
    V = model.llm.model.embed_tokens.weight.shape[0]
    for n in present:
        mha = getattr(model, f"{n}_align_attention")
        Hh, Lq = mha.num_heads, eng.last_lens[n]
        m = ops.dropout_mask(Hh * B * Lq, V + 2, (mha.dropout, ts.last_seed, eng.DROPOUT_SID[n]), DEV)
        masks[n] = m.view(Hh, B, Lq, V + 2).permute(1, 0, 2, 3).reshape(B * Hh, Lq, V + 2).cpu()
        keep = float((m != 0).float().mean())
        assert abs(keep - (1 - mha.dropout)) < 0.01, (n, keep)
        assert torch.all((m == 0) | ((m - 1 / (1 - mha.dropout)).abs() < 1e-6))
    if "video" in present:
        mha = model.video_long_self_attention
        Hh = mha.num_heads
        N = eng._video_long_len
        m = ops.dropout_mask(B * Hh * N, N + 2, (mha.dropout, ts.last_seed, eng.DROPOUT_SID["video_long"]), DEV)
        masks["video_long"] = m.view(B * Hh, N, N + 2).cpu()
    return masks


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("name", ["text_labels", "image_audio", "all3"])
def test_gradients_vs_oracle_autograd(tiny_train, name, dropout):
    """`model.train(); model(inputs).loss.backward()` vs autograd of the fp32 CPU oracle on the same bf16-rounded weights
    (dropout=True: with the MHAs' attention dropout live, as in the reference's train() mode — the oracle applies the SAME
    Philox mask, exported from the device; dropout=False: `train_step.attention_dropout = False`):
    every LLaMA parameter AND the alignment modules (Conv1d, Linear, MHA in/out projections, bias_k / bias_v), the embedding
    table through the gathered rows and as the alignment attention's keys / values.  text_labels / image_audio: the oracle
    gradient is the reference's FULL gradient (encoders frozen, dropout off); all3 adds the video path incl.
    `video_long_self_attention` (through the Conv1d data gradient)."""
    from oracle import macaw_oracle as O
    from tests.golden import gen

    model, spec, hp, weights = tiny_train
    if name == "all3":
        inp = H.case_inputs(spec, H.load_case("all3"))
    elif name == "image_audio":
        inp = gen.make_inputs(spec, 2, 14, seed=78, modalities=("image", "audio"), pad_tail=2, with_labels=True)
    else:
        inp = gen.make_inputs(spec, 3, 24, seed=77, modalities=(), pad_tail=4, with_labels=True)
    inp = {k: (v.to(torch.bfloat16) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}
    dev_inp = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    if dropout and name == "text_labels":
        pytest.skip("no MHA on the text-only path")
    present = {"text_labels": (), "image_audio": ("image", "audio"), "all3": ("image", "audio", "video")}[name]
    model.train()
    model.train_step.attention_dropout = bool(dropout)
    try:
        for p in model.parameters():
            p.grad = None
        out = model(dev_inp)
        assert out.loss.requires_grad and out.logits is None
        out.loss.backward()
        torch.cuda.synchronize()
        masks = _oracle_dropout_masks(model, spec, present, inp["input_ids"].shape[0]) if dropout else None
    finally:
        model.train_step.attention_dropout = True
        model.eval()
    sd = H.bf16_round(weights)
    loss_ref, grads_ref = O.full_loss_and_grads(
        {k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}, sd, hp,
        dropout=masks)
    assert abs(float(out.loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    named = dict(model.named_parameters())
    worst, worst_align = ("", 0.0), ("", 0.0)
    errs = {k: rel(named[k].grad, gr) for k, gr in grads_ref.items() if named[k].grad is not None}
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:8]
    print(f"\n[train:{name}] largest gradient errors: " + ", ".join(f"{k}={e:.2e}" for k, e in top))
    tg, tr = named["llm.model.embed_tokens.weight"].grad.float().cpu(), grads_ref["llm.model.embed_tokens.weight"]
    row_err = (tg - tr).norm(dim=1)
    worst_rows = row_err.topk(5).indices.tolist()
    ids_l = inp["input_ids"].reshape(-1).tolist()
    print(f"[train:{name}] table grad: |ours| {float(tg.norm()):.4e} |ref| {float(tr.norm()):.4e}; worst rows "
          + ", ".join(f"{r}(|d|={float(row_err[r]):.2e},|ref|={float(tr[r].norm()):.2e},|ours|={float(tg[r].norm()):.2e},count={ids_l.count(r)})" for r in worst_rows))
    for k, gr in grads_ref.items():
        is_align = not k.startswith("llm.")
        if is_align and not any(k.startswith((f"project_{m}.", f"transform_{m}_to_hidden.", f"{m}_align_attention.") +
                                             (("video_long_self_attention.",) if m == "video" else ())) for m in present):
            assert named[k].grad is None, k  # modality absent from the batch: no gradient, as in torch
            continue
        g = named[k].grad
        assert g is not None, k
        e = rel(g, gr)
        if is_align and e > worst_align[1]:
            worst_align = (k, e)
        if not is_align and e > worst[1]:
            worst = (k, e)
        assert e < (5e-2 if is_align else 3e-2), (k, e)
    assert (named["video_long_self_attention.in_proj_weight"].grad is not None) == ("video" in present)
    assert named["temporal_self_attention.in_proj_weight"].grad is None    # never reached by forward (dead in the reference too)
    assert named["image_encoder.visual_projection.weight"].grad is None    # encoders are frozen (run_clm_llms.py:390-393)
    print(f"\n[train:{name}{'+dropout' if dropout else ''}] loss {float(out.loss):.5f} vs oracle {float(loss_ref):.5f}; worst gradient rel err: llm "
          f"{worst[1]:.3e} ({worst[0]}), alignment {worst_align[1]:.3e} ({worst_align[0]})")


def test_gradient_accumulation_and_optimizer_steps(tiny_train):
    """Two backward passes without zero_grad accumulate (2x the gradient); a few FusedAdamW steps lower the loss and the
    inference path picks the updated weights up (derived-weight caches follow the version counters)."""
    from macaw_llm_b200.training import FusedAdamW, trainable_parameters
    from tests.golden import gen
    import copy

    model0, spec, hp, weights = tiny_train
    model = copy.deepcopy(model0)
    inp = gen.make_inputs(spec, 2, 16, seed=5, modalities=("image",), with_labels=True)
    inp = {k: (v.to(torch.bfloat16).cuda() if isinstance(v, torch.Tensor) and v.is_floating_point() else
               (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()}
    params = [p for _, p in trainable_parameters(model)]
    opt = FusedAdamW(params, lr=3e-3, weight_decay=0.0)
    model.train()
    opt.zero_grad()
    model.train_step.attention_dropout = False  # identical passes: the accumulated gradient is exactly twice the first
    model(inp).loss.backward()
    g1 = model.llm.lm_head.weight.grad.float().clone()
    model(inp).loss.backward()
    assert rel(model.llm.lm_head.weight.grad, 2 * g1) < 1e-2
    model.train_step.attention_dropout = True
    s0 = int(model.train_step._seed) if model.train_step._seed is not None else None
    losses = []
    for _ in range(6):
        opt.zero_grad()
        out = model(inp)
        out.loss.backward()
        opt.step()
        losses.append(float(out.loss))
    assert int(model.train_step._seed) == (s0 + 6 if s0 is not None else model.train_step.dropout_base_seed + 6)  # one seed per step
    model.eval()
    with torch.no_grad():
        ev = float(model(inp).loss)
    print(f"\n[train loop] losses {['%.4f' % l for l in losses]}  eval after {ev:.4f}")
    assert losses[-1] < losses[0] - 0.05 and ev < losses[0]


def test_frozen_decoder_layers_get_no_gradient(tiny_train):
    """The lower decoder layers frozen (as bench.py --mode train does to fit one 80 GB GPU): they get no gradient and no
    optimizer update, the backward pass still runs through them, so every other gradient — the alignment modules' and the
    table's included — is the one the fully trainable step computes."""
    from macaw_llm_b200.training import FusedAdamW, freeze_llama_layers, trainable_parameters
    from tests.golden import gen
    import copy

    model0, spec, hp, weights = tiny_train
    inp = gen.make_inputs(spec, 2, 16, seed=9, modalities=("image", "audio"), with_labels=True)
    inp = {k: (v.to(torch.bfloat16).cuda() if isinstance(v, torch.Tensor) and v.is_floating_point() else
               (v.cuda() if isinstance(v, torch.Tensor) else v)) for k, v in inp.items()}

    def grads(m):
        m.train()
        m.train_step.attention_dropout = False
        try:
            for p in m.parameters():
                p.grad = None
            m(inp).loss.backward()
            torch.cuda.synchronize()
        finally:
            m.train_step.attention_dropout = True
            m.eval()
        return {n: (p.grad.float().clone() if p.grad is not None else None) for n, p in m.named_parameters()}

    full = grads(copy.deepcopy(model0))
    model = copy.deepcopy(model0)
    freeze_llama_layers(model, 1)
    part = grads(model)
    frozen = {n for n, _ in model.named_parameters() if n.startswith("llm.model.layers.0.")}
    assert frozen and not ({n for n, _ in trainable_parameters(model)} & frozen)
    for n, g in full.items():
        if n in frozen:
            assert part[n] is None, n
        elif g is not None:
            assert part[n] is not None and rel(part[n], g) < 2e-3, n  # bf16 atomics in the table scatter may reorder sums
    w0 = model.llm.model.layers[0].mlp.down_proj.weight.detach().clone()
    w1 = model.llm.model.layers[1].mlp.down_proj.weight.detach().clone()
    opt = FusedAdamW([p for _, p in trainable_parameters(model)], lr=1e-3, weight_decay=0.0)
    model.train()
    try:
        model(inp).loss.backward()
        opt.step()
        torch.cuda.synchronize()
    finally:
        model.eval()
    assert torch.equal(model.llm.model.layers[0].mlp.down_proj.weight, w0)
    assert not torch.equal(model.llm.model.layers[1].mlp.down_proj.weight, w1)
