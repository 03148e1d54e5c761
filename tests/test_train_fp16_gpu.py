"""fp16 training on the H100: the training kernels in the fp16 format against fp32 autograd (the bf16 cases of
tests/test_train_gpu.py, same bars or tighter), the gradient-norm pass (mm_grad_sumsq) and the device loss scaler
(mm_loss_scale_update) against an fp64 sum and the host restatement of tests/test_loss_scaler_cpu.py, whole-model
gradients of an fp16 model (loss-scaled) against autograd of the fp32 oracle, overflow-skipped steps, gradient clipping
against torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW, and the whole fp16 step replayed from a CUDA graph."""
import copy
import math

import numpy as np
import pytest
import torch

from tests import helpers as H
from tests.test_loss_scaler_cpu import ScaleRef

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16


def _ops():
    from macaw_llm_b200 import ops

    return ops


@pytest.fixture
def fp16_format():
    ops = _ops()
    ops.set_act_format(F16)
    try:
        yield ops
    finally:
        ops.set_act_format(BF16)


def rnd(*shape, scale=1.0, seed=0, dtype=F16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


# ---------------------------------------------------------------------------------------------------- per-kernel checks
@pytest.mark.parametrize("M,N,K", [(2112, 4096, 4096), (300, 1000, 520), (528, 512, 256), (70, 11008, 4096)])
def test_gemm_dx_dw_fp16(fp16_format, M, N, K):
    ops = fp16_format
    x, w, dy = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(M, N, seed=3)
    dx = ops.gemm_dx(dy, w)
    dw = torch.empty(N, K, device=DEV, dtype=F16)
    ops.gemm_dw(dy, x, dw, accumulate=False)
    ref_dx, ref_dw = dy.float() @ w.float(), dy.float().t() @ x.float()
    e = [rel(dx, ref_dx), rel(dw, ref_dw)]
    ops.gemm_dw(dy, x, dw, accumulate=True)
    ops.gemm_dx(dy, w, out=dx, accumulate=True)
    e += [rel(dw, 2 * ref_dw), rel(dx, 2 * ref_dx)]
    print(f"\n[fp16 gemm M{M} N{N} K{K}] dx {e[0]:.2e} dw {e[1]:.2e} acc dw {e[2]:.2e} acc dx {e[3]:.2e}")
    assert e[0] < 4e-3 and e[1] < 4e-3 and e[2] < 6e-3 and e[3] < 6e-3


def test_rmsnorm_swiglu_backward_fp16(fp16_format):
    ops = fp16_format
    rows, cols = 300, 4096
    x, dy, dres = rnd(rows, cols, seed=4), rnd(rows, cols, seed=6), rnd(rows, cols, seed=7)
    g = (1 + 0.1 * rnd(cols, seed=5).float()).to(F16)
    xf, gf = x.float().requires_grad_(True), g.float().requires_grad_(True)
    (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * gf).backward(dy.float())
    dg = torch.zeros(cols, device=DEV)
    dx = ops.rmsnorm_bwd(dy, x, ops.rms_rstd(x, 1e-6), g, dres, dg)
    e_dx, e_dg = rel(dx, xf.grad + dres.float()), rel(dg, gf.grad)
    x2, dy2 = rnd(37, 256, seed=8), rnd(37, 256, seed=9)
    x2f = x2.float().requires_grad_(True)
    (x2f * torch.rsqrt(x2f.pow(2).mean(-1, keepdim=True) + 1e-6)).backward(dy2.float())
    e_dx2 = rel(ops.rmsnorm_bwd(dy2, x2, ops.rms_rstd(x2, 1e-6), torch.ones(256, device=DEV, dtype=F16), None, None), x2f.grad)
    gt, up, dh = rnd(64, 1024, seed=10), rnd(64, 1024, seed=11), rnd(64, 1024, seed=12)
    gtf, upf = gt.float().requires_grad_(True), up.float().requires_grad_(True)
    h = torch.nn.functional.silu(gtf) * upf
    h.backward(dh.float())
    dgt, dup = ops.swiglu_bwd(dh, gt, up)
    e_h, e_dg_, e_du = rel(ops.swiglu_fwd(gt, up), h), rel(dgt, gtf.grad), rel(dup, upf.grad)
    print(f"\n[fp16 rmsnorm bwd] dx {e_dx:.2e} dg {e_dg:.2e} narrow dx {e_dx2:.2e}; [swiglu] h {e_h:.2e} dgate {e_dg_:.2e} "
          f"dup {e_du:.2e}")
    assert e_dx < 4e-3 and e_dg < 2e-3 and e_dx2 < 4e-3 and max(e_h, e_dg_, e_du) < 4e-3


@pytest.mark.parametrize("B,H,T,hd,causal,masked", [(2, 4, 528, 128, True, False), (2, 2, 200, 128, True, True),
                                                    (1, 2, 300, 64, False, False)])
def test_attention_backward_fp16(fp16_format, B, H, T, hd, causal, masked):
    ops = fp16_format
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
    (torch.softmax(s, -1) @ vf).backward(do.float().permute(0, 2, 1, 3))
    dq, dk, dv = ops.attention_bwd(q, k, v, do, scale=scale, causal=causal, key_mask=km)
    e = [rel(a, b.grad.permute(0, 2, 1, 3)) for a, b in ((dq, qf), (dk, kf), (dv, vf))]
    print(f"\n[fp16 attention bwd B{B} H{H} T{T} hd{hd}] dq {e[0]:.2e} dk {e[1]:.2e} dv {e[2]:.2e}")
    assert max(e) < 8e-3


def test_ce_backward_scatter_colsum_fp16(fp16_format):
    ops = fp16_format
    B, T, V = 2, 9, 519
    logits = rnd(B, T, V, scale=2.0, seed=30)
    labels = torch.randint(0, V, (B, T), generator=torch.Generator().manual_seed(1)).to(DEV)
    labels[0, :3] = -100
    lf = logits.float().requires_grad_(True)
    torch.nn.functional.cross_entropy(lf[:, :-1].reshape(-1, V), labels[:, 1:].reshape(-1), ignore_index=-100).backward()
    _, cnt = ops.ce_loss_with_count(logits.clone(), labels)
    gs = torch.tensor([1024.0], device=DEV)  # a loss scale, read from the device
    d = ops.ce_bwd(logits.clone(), labels, cnt, gs)
    e_ce = rel(d, 1024.0 * lf.grad)
    table_g = torch.zeros(50, 64, device=DEV, dtype=F16)
    ids = torch.tensor([3, 7, 3, 49, 3, -1], device=DEV)
    dx = rnd(6, 64, seed=31)
    ops.embed_scatter_add(dx, ids, table_g)
    ref = torch.zeros(50, 64, device=DEV)
    ref.index_add_(0, ids[:5], dx[:5].float())
    e_sc = rel(table_g, ref)
    cs = torch.zeros(64, device=DEV)
    ops.colsum(dx, cs)
    e_cs = rel(cs, dx.float().sum(0))
    print(f"\n[fp16 ce bwd (device scale)] {e_ce:.2e}; scatter-add {e_sc:.2e}; colsum {e_cs:.2e}")
    assert e_ce < 6e-3 and e_sc < 8e-3 and e_cs < 1e-5


def test_dropout_attention_fp16(fp16_format):
    ops = fp16_format
    seed = torch.tensor([(9 << 32) | 1234567], dtype=torch.int64, device=DEV)
    B, Hh, T, hd, pd = 2, 3, 37, 96, 0.1
    q, k, v, do = (rnd(B, T, Hh, hd, scale=0.7, seed=s) for s in (1, 2, 3, 4))
    drop = (pd, seed, 7)
    mult_np = H.dropout_multipliers(B * Hh * T, T, pd, seed=(9 << 32) | 1234567, sid=7)
    assert (ops.dropout_mask(B * Hh * T, T, drop, DEV).cpu().numpy() == mult_np).all()
    o = ops.attention_train_fwd(q, k, v, scale=hd ** -0.5, dropout=drop)
    dq, dk, dv = ops.attention_bwd(q, k, v, do, scale=hd ** -0.5, causal=False, dropout=drop)
    mult = torch.from_numpy(mult_np).view(B, Hh, T, T).double()
    qf, kf, vf = (t.double().cpu().permute(0, 2, 1, 3).requires_grad_(True) for t in (q, k, v))
    of = (torch.softmax(qf @ kf.transpose(-1, -2) * hd ** -0.5, dim=-1) * mult) @ vf
    of.backward(do.double().cpu().permute(0, 2, 1, 3))
    e = [rel(o.permute(0, 2, 1, 3), of.detach())] + [rel(g.permute(0, 2, 1, 3), r) for g, r in
                                                     ((dq, qf.grad), (dk, kf.grad), (dv, vf.grad))]
    print(f"\n[fp16 dropout attention] o {e[0]:.2e} dq {e[1]:.2e} dk {e[2]:.2e} dv {e[3]:.2e}")
    assert e[0] < 6e-3 and max(e[1:]) < 8e-3


def test_fused_adamw_fp16_matches_torch():
    from macaw_llm_b200.training import FusedAdamW

    torch.manual_seed(0)
    p = torch.nn.Parameter(torch.randn(1000, 64, device=DEV).to(F16))
    ref = torch.nn.Parameter(p.detach().float().clone())
    opt = FusedAdamW([p], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    topt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    try:
        for i in range(3):
            g = torch.randn(1000, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(i)).to(F16)
            p.grad = g.clone()
            ref.grad = g.float()
            opt.step()
            topt.step()
    finally:
        _ops().set_act_format(BF16)
    e_master, e_p = rel(opt.state[id(p)][0], ref), rel(p, ref)
    print(f"\n[fp16 adamw] master {e_master:.2e} param {e_p:.2e}")
    assert e_master < 1e-6 and e_p < 3e-3


# ---------------------------------------------------------------------------------------------------- gradient norm pass
@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("n", [1, 7, 4096 + 3, 3_000_001])
def test_grad_sumsq_vs_fp64(dtype, n):
    ops = _ops()
    g = rnd(n, scale=3.0, seed=n % 97, dtype=dtype)
    out = torch.zeros(1, device=DEV)
    ops.grad_sumsq(g, out)
    out2 = torch.zeros(1, device=DEV)
    ops.grad_sumsq(g, out2)
    want = float(g.double().pow(2).sum())
    e = abs(float(out) - want) / max(want, 1e-30)
    print(f"\n[grad_sumsq {dtype} n={n}] rel err {e:.2e}")
    assert e < 1e-5
    assert torch.equal(out, out2)  # deterministic: bit-identical across calls
    ops.grad_sumsq(g, out)  # adds into the scalar
    assert abs(float(out) - 2 * float(out2)) <= 1e-6 * float(out2)


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_grad_sumsq_non_finite(bad):
    ops = _ops()
    for dtype in (F16, BF16):
        g = rnd(100_003, seed=5, dtype=dtype)
        g[77_777] = bad
        out = torch.zeros(1, device=DEV)
        ops.grad_sumsq(g, out)
        assert not math.isfinite(float(out)), (dtype, bad)
        g = rnd(100_003, seed=5, dtype=dtype)
        g[-1] = bad  # in the n % 8 tail
        out.zero_()
        ops.grad_sumsq(g, out)
        assert not math.isfinite(float(out)), (dtype, bad, "tail")


def test_grad_sumsq_beyond_2_31_elements():
    """More than 2^31 elements (64-bit indexing; the bench's trainable set is 2.21 B): 4.3 GB of fp16."""
    ops = _ops()
    n = (1 << 31) + 4099
    g = torch.full((n,), 0.5, device=DEV, dtype=F16)
    hot = torch.tensor([5, (1 << 31) - 1, 1 << 31, n - 4096, n - 1], device=DEV)
    g[hot] = 100.0
    out = torch.zeros(1, device=DEV)
    ops.grad_sumsq(g, out)
    want = (n - 5) * 0.25 + 5 * 1e4
    e = abs(float(out) - want) / want
    print(f"\n[grad_sumsq n=2^31+4099] {float(out):.6e} vs {want:.6e}: rel err {e:.2e}")
    assert e < 1e-5
    g[n - 8] = float("inf")  # beyond 2^31, in the 128-bit body (the last n % 8 = 3 elements are the tail)
    out.zero_()
    ops.grad_sumsq(g, out)
    assert not math.isfinite(float(out))
    del g
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- device loss scaler
@pytest.mark.parametrize("max_norm", [None, 1.0])
def test_loss_scale_update_matches_restatement(max_norm):
    """A few thousand steps of a seeded pattern of finite and non-finite sums of squares: every field of the device state
    equals the host restatement's, the multiplier bit for bit."""
    from macaw_llm_b200.training import DynamicLossScaler, _new_scale_state

    ops = _ops()
    sc = DynamicLossScaler(initial_scale_power=12, loss_scale_window=7, hysteresis=2, min_loss_scale=2.0 ** -3)
    st = sc._state(torch.device(DEV))
    ref = ScaleRef(initial_scale_power=12, window=7, hysteresis=2, min_scale=2.0 ** -3, max_norm=max_norm)
    rng = np.random.default_rng(1234)
    sumsq = torch.zeros(1, device=DEV)
    n_ovf = 0
    for i in range(3000):
        u = rng.random()
        if u < 0.25:
            v = [float("inf"), float("nan")][int(rng.integers(2))]
            n_ovf += 1
        else:
            v = float(np.float32((float(ref.scale) * rng.uniform(0.05, 4.0)) ** 2))
        sumsq.fill_(v)
        ops.loss_scale_update(st, sumsq, max_norm=max_norm, dynamic=True, window=7, hysteresis=2, min_scale=2.0 ** -3)
        ref.update(v)
        got = sc.state_dict()
        want = ref.fields()
        for k in ("scale", "cur_iter", "last_overflow_iter", "cur_hysteresis", "skip", "skipped", "step"):
            assert got[k] == want[k], (i, k, got[k], want[k])
        assert np.float32(got["grad_mult"]) == np.float32(want["grad_mult"]), (i, got["grad_mult"], want["grad_mult"])
        assert float(sumsq) == 0.0  # consumed
    assert 0 < ref.skipped == n_ovf and sc.skipped_steps == n_ovf
    print(f"\n[loss scaler, max_norm={max_norm}] 3000 steps, {n_ovf} overflows, final scale {sc.loss_scale}")
    # clipping alone: fixed unit scale
    cs = _new_scale_state(torch.device(DEV), 1.0, 1)
    sumsq.fill_(16.0)
    ops.loss_scale_update(cs, sumsq, max_norm=1.0, dynamic=False, window=1, hysteresis=1, min_scale=1.0)
    assert float(cs.view(torch.float32)[0]) == 1.0 and int(cs[8]) == 1
    assert np.float32(float(cs.view(torch.float32)[6])) == np.float32(1.0) / (np.float32(4.0) + np.float32(1e-6))


# ---------------------------------------------------------------------------------------------------- whole model, fp16
@pytest.fixture(scope="module")
def tiny_fp16():
    return H.build_tiny_model("cuda", F16)


def fp16_round(sd: dict) -> dict:
    return {k: (v.to(F16).float() if v.is_floating_point() else v) for k, v in sd.items()}


def _inputs(spec, name):
    from tests.golden import gen

    if name == "all3":
        inp = H.case_inputs(spec, H.load_case("all3"))
    elif name == "image_audio":
        inp = gen.make_inputs(spec, 2, 14, seed=78, modalities=("image", "audio"), pad_tail=2, with_labels=True)
    else:
        inp = gen.make_inputs(spec, 3, 24, seed=77, modalities=(), pad_tail=4, with_labels=True)
    return {k: (v.to(F16) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}


def _dev(inp):
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("name", ["text_labels", "image_audio", "all3"])
def test_fp16_gradients_vs_oracle_autograd(tiny_fp16, name, dropout):
    """The fp16 model, loss-scaled backward (`DynamicLossScaler.scale(loss).backward()`): p.grad / S against autograd of
    the fp32 oracle on the same fp16-rounded weights and inputs, the attention-dropout masks exported from the device."""
    from macaw_llm_b200.training import DynamicLossScaler
    from oracle import macaw_oracle as O
    from tests.test_train_gpu import _oracle_dropout_masks

    model, spec, hp, weights = tiny_fp16
    if dropout and name == "text_labels":
        pytest.skip("no MHA on the text-only path")
    inp = _inputs(spec, name)
    present = {"text_labels": (), "image_audio": ("image", "audio"), "all3": ("image", "audio", "video")}[name]
    scaler = DynamicLossScaler(initial_scale_power=10)
    model.train()
    model.train_step.attention_dropout = bool(dropout)
    try:
        for p in model.parameters():
            p.grad = None
        out = model(_dev(inp))
        scaler.scale(out.loss).backward()
        torch.cuda.synchronize()
        masks = _oracle_dropout_masks(model, spec, present, inp["input_ids"].shape[0]) if dropout else None
    finally:
        model.train_step.attention_dropout = True
        model.eval()
    S = scaler.loss_scale
    loss_ref, grads_ref = O.full_loss_and_grads(
        {k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()},
        fp16_round(weights), hp, dropout=masks)
    assert abs(float(out.loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    named = dict(model.named_parameters())
    worst, worst_align = ("", 0.0), ("", 0.0)
    for k, gr in grads_ref.items():
        is_align = not k.startswith("llm.")
        if is_align and not any(k.startswith((f"project_{m}.", f"transform_{m}_to_hidden.", f"{m}_align_attention.") +
                                             (("video_long_self_attention.",) if m == "video" else ())) for m in present):
            assert named[k].grad is None, k
            continue
        g = named[k].grad
        assert g is not None and g.dtype == F16, k
        assert torch.isfinite(g).all(), k
        e = rel(g.float() / S, gr)
        if is_align and e > worst_align[1]:
            worst_align = (k, e)
        if not is_align and e > worst[1]:
            worst = (k, e)
        assert e < (5e-2 if is_align else 3e-2), (k, e)
    print(f"\n[fp16 train:{name}{'+dropout' if dropout else ''}] S={S:g} loss {float(out.loss):.5f} vs oracle "
          f"{float(loss_ref):.5f}; worst gradient rel err: llm {worst[1]:.3e} ({worst[0]}), alignment {worst_align[1]:.3e} "
          f"({worst_align[0]})")


def _train_inputs(spec, seed=5):
    from tests.golden import gen

    inp = gen.make_inputs(spec, 2, 16, seed=seed, modalities=("image",), with_labels=True)
    return _dev({k: (v.to(F16) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()})


def test_skipped_steps_end_to_end(tiny_fp16):
    """initial_scale_power=40: every gradient overflows fp16 at first.  Skipped steps leave parameters, master weights,
    moments and the step counter bit-identical; the scale follows the restatement; once it fits, steps resume and the
    loss falls."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, trainable_parameters

    model0, spec, hp, weights = tiny_fp16
    model = copy.deepcopy(model0)
    inp = _train_inputs(spec)
    params = [p for _, p in trainable_parameters(model)]
    opt = FusedAdamW(params, lr=3e-3, weight_decay=0.0, max_grad_norm=1.0)
    scaler = DynamicLossScaler(initial_scale_power=40, loss_scale_window=1000, hysteresis=2)
    ref = ScaleRef(initial_scale_power=40, window=1000, hysteresis=2, max_norm=1.0)
    model.train()
    model.train_step.attention_dropout = False
    losses, n_skip = [], 0
    try:
        for it in range(60):
            opt.zero_grad()
            out = model(inp)
            scaler.scale(out.loss).backward()
            snap_p = [p.detach().clone() for p in params]
            snap_st = {k: tuple(t.clone() for t in v) for k, v in opt.state.items()}
            opt.step(loss_scaler=scaler)
            d = scaler.state_dict()
            ref.update(float("inf") if d["skip"] else 1.0)  # the device's overflow verdict drives the restatement
            assert d["scale"] == float(ref.scale) and d["skipped"] == ref.skipped and d["step"] == ref.step, (it, d)
            if d["skip"]:
                n_skip += 1
                assert all(torch.equal(a, p) for a, p in zip(snap_p, params)), it
                for k, v in snap_st.items():
                    assert all(torch.equal(a, b) for a, b in zip(v, opt.state[k])), it
                assert not losses, "a skip after steps resumed"  # S only grows back after 1000 clean steps
            else:
                losses.append(float(out.loss))
    finally:
        model.train_step.attention_dropout = True
        model.eval()
    print(f"\n[fp16 skipped steps] {n_skip} skipped, final scale {scaler.loss_scale:g}, losses "
          f"{['%.4f' % l for l in losses[:3]]} .. {losses[-1]:.4f}")
    # 2^40 halves once per skipped step after the first (hysteresis 2) down to the first scale that fits
    assert n_skip >= 20 and scaler.skipped_steps == n_skip and scaler.loss_scale == 2.0 ** (40 - (n_skip - 1))
    assert len(losses) >= 10 and losses[-1] < losses[0] - 0.05


def _clip_case(dtype, max_norm, scale_power, gscale):
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW

    torch.manual_seed(0)
    shapes = [(300, 64), (64,), (17, 8)]
    ps = [torch.nn.Parameter(torch.randn(*s, device=DEV).to(dtype)) for s in shapes]
    refs = [torch.nn.Parameter(p.detach().float().clone()) for p in ps]
    opt = FusedAdamW(ps, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, max_grad_norm=max_norm)
    topt = torch.optim.AdamW(refs, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    scaler = DynamicLossScaler(initial_scale_power=scale_power) if scale_power is not None else None
    S = 2.0 ** scale_power if scale_power is not None else 1.0
    norms = []
    try:
        for i in range(3):
            gen = torch.Generator(device=DEV).manual_seed(10 + i)
            gs = [torch.randn(*s, device=DEV, generator=gen) * gscale for s in shapes]
            if scaler is not None:
                scaler._state(torch.device(DEV))
            for p, r, g in zip(ps, refs, gs):
                p.grad = (g * S).to(dtype)
                r.grad = p.grad.float() / S
            norms.append(float(torch.nn.utils.clip_grad_norm_(refs, max_norm)))
            opt.step(loss_scaler=scaler)
            topt.step()
    finally:
        _ops().set_act_format(BF16)
    e_master = max(rel(opt.state[id(p)][0], r) for p, r in zip(ps, refs))
    e_p = max(rel(p, r) for p, r in zip(ps, refs))
    return e_master, e_p, norms


@pytest.mark.parametrize("dtype,max_norm,scale_power,gscale", [
    (BF16, 1.0, None, 1.0),      # clipped
    (F16, 1.0, None, 1.0),       # clipped, fp16 parameters
    (BF16, 1e3, None, 1.0),      # below the threshold: no clipping
    (F16, 1.0, 8, 1.0),          # fp16 with a loss scale: unscale + clip in one multiplier
])
def test_clipping_matches_torch(dtype, max_norm, scale_power, gscale):
    e_master, e_p, norms = _clip_case(dtype, max_norm, scale_power, gscale)
    print(f"\n[clip {dtype} max_norm={max_norm} S=2^{scale_power}] norms {['%.3f' % n for n in norms]}: master "
          f"{e_master:.2e} param {e_p:.2e}")
    assert (min(norms) > max_norm) == (max_norm < 10)
    assert e_master < 1e-5 and e_p < 3e-3


# ---------------------------------------------------------------------------------------------------- CUDA graph
def test_fp16_step_cuda_graph_matches_eager(tiny_fp16):
    """The whole fp16 step (forward, scaled backward, gradient norm, scaler update, AdamW) captured once and replayed k
    times, against k eager steps from an identical initial state (dropout off): the same loss-scale trajectory and skip
    decisions, parameters within the tolerance of the frozen-layer test (the table scatter's atomics may reorder sums)."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, trainable_parameters

    model0, spec, hp, weights = tiny_fp16
    inp = _train_inputs(spec, seed=9)
    k = 12

    def setup():
        m = copy.deepcopy(model0)
        ps = [p for _, p in trainable_parameters(m)]
        # S = 2^20: the first steps overflow fp16 and are skipped (the logits' gradient alone is ~S / n_valid), the scale
        # halves until the gradients fit and the later steps are taken
        return m, ps, FusedAdamW(ps, lr=1e-3, weight_decay=0.0, max_grad_norm=1.0), DynamicLossScaler(initial_scale_power=20,
                                                                                                        hysteresis=1)

    def make_step(m, opt, sc):
        def step():
            opt.zero_grad()
            out = m(inp)
            sc.scale(out.loss).backward()
            m.train_step.llama.finish_allreduce()
            opt.step(loss_scaler=sc)
            return out.loss
        return step

    runs = {}
    for mode in ("eager", "graph"):
        m, ps, opt, sc = setup()
        m.train()
        m.train_step.attention_dropout = False
        traj = []
        try:
            step = make_step(m, opt, sc)
            if mode == "graph":
                # warm-up on a side stream (one real step, counted), then capture one step and replay it k - 1 times
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    step()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                d = sc.state_dict()
                traj.append((d["scale"], d["skip"], d["skipped"], d["step"]))
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    step()
                # capture recorded the step without running it
                for _ in range(k - 1):
                    graph.replay()
                    torch.cuda.synchronize()
                    d = sc.state_dict()
                    traj.append((d["scale"], d["skip"], d["skipped"], d["step"]))
            else:
                for _ in range(k):
                    step()
                    torch.cuda.synchronize()
                    d = sc.state_dict()
                    traj.append((d["scale"], d["skip"], d["skipped"], d["step"]))
        finally:
            m.train_step.attention_dropout = True
            m.eval()
        runs[mode] = (traj, {n: p.detach().float().clone() for n, p in m.named_parameters()})
    (te, pe), (tg, pg) = runs["eager"], runs["graph"]
    print(f"\n[fp16 graph vs eager] trajectory eager {te}\n                      graph {tg}")
    assert te == tg
    assert any(t[1] for t in te) and not te[-1][1]  # both skipped and taken steps were exercised
    worst = max(rel(pg[n], pe[n]) for n in pe)
    print(f"[fp16 graph vs eager] worst parameter rel diff {worst:.2e}")
    assert worst < 2e-3
