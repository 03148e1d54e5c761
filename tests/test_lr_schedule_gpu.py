"""The learning-rate schedule on the H100 (mm_lr_schedule, `FusedAdamW(lr_schedule=LRSchedule(...))`): the kernel against
the host restatement over every step, the scheduled optimizer against torch.optim.AdamW driven by transformers'
get_cosine_schedule_with_warmup, overflow-skipped fp16 steps that do not advance the schedule, host-resident state bit
for bit with device state under a schedule, and a whole tiny fp16 step replayed from a CUDA graph whose lr changes from
replay to replay."""
import copy

import numpy as np
import pytest
import torch

from tests import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16
SHAPES = [(300, 64), (37,), (17, 8)]  # 37 % 8 != 0: the 8-wide and the scalar kernel both run


def _ops():
    from macaw_llm_b200 import ops

    return ops


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


# Tolerance policy: an lr the device computed against the host restatement (LRSchedule.lr_of_update, or fp32 of HF's lr)
# may differ by 1 fp32 ulp, since the device's double cos may differ from the host libm's in the last bit of the double
# before the rounding to fp32.  Device results against device results (eager vs graph, host vs device state, with vs
# without skipped steps) run the same kernels on the same inputs and must be bit-identical.
def ulps(a, b) -> int:
    """Distance in fp32 units in the last place between two finite fp32 values."""
    ia, ib = (int(np.array([x], dtype=np.float32).view(np.int32)[0]) for x in (a, b))
    return abs(ia - ib)


def lr_close(got, want) -> bool:
    return ulps(got, want) <= 1


# ---------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("name", ["linear", "cosine", "constant_with_warmup"])
def test_lr_schedule_kernel_matches_restatement(name):
    """mm_lr_schedule for t = 0 .. N + 50 (one launch per t, each writing its own slot) against
    numpy.float32(base * lr_lambda(max(t - 1, 0))): at most 1 fp32 ulp apart (the device's double cos may differ from the
    host's in the last bit of the double); the bit-exact count is printed."""
    from macaw_llm_b200.training import LRSchedule

    ops = _ops()
    base = 3e-5
    exact = total = 0
    for W, N in ((0, 1), (1, 1), (0, 10), (3, 10), (10, 10), (3, 100), (30, 1000), (1, 1000), (1000, 1000)):
        s = LRSchedule(name, W, N)
        ts = torch.arange(0, N + 51, dtype=torch.int32, device=DEV)
        out = torch.full((ts.numel(),), float("nan"), dtype=torch.float32, device=DEV)
        for i in range(ts.numel()):
            ops.lr_schedule(ts[i:i + 1], out[i:i + 1], base_lr=base, kind=name, warmup_steps=W, training_steps=N)
        got = out.cpu().numpy()
        want = np.array([np.float32(base * s.lr_lambda(max(int(t) - 1, 0))) for t in ts.cpu()], dtype=np.float32)
        ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert np.isfinite(got).all() and int(ulps.max()) <= 1, (W, N, int(ulps.argmax()), got[ulps.argmax()],
                                                                 want[ulps.argmax()])
        exact += int((ulps == 0).sum())
        total += ulps.size
    print(f"\n[lr_schedule {name}] {exact} of {total} values bit-exact, the rest within 1 ulp")


# ---------------------------------------------------------------------------------------------------- optimizer
def test_scheduled_adamw_matches_torch_and_hf_cosine():
    """FusedAdamW(lr_schedule=cosine) against torch.optim.AdamW + transformers.get_cosine_schedule_with_warmup over 30
    steps spanning warmup, decay and the rise past N, at the tolerance of test_fused_adamw_matches_torch; the lr of each
    step is the fp32 of HF's; the first step (lr 0) moves m and v but leaves master and parameters bit-unchanged."""
    from transformers import get_cosine_schedule_with_warmup

    from macaw_llm_b200.training import FusedAdamW, LRSchedule

    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(*s, device=DEV).to(BF16)) for s in SHAPES]
    refs = [torch.nn.Parameter(p.detach().float().clone()) for p in ps]
    W, N, base = 5, 25, 1e-2
    opt = FusedAdamW(ps, lr=base, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, lr_schedule=LRSchedule("cosine", W, N))
    topt = torch.optim.AdamW(refs, lr=base, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    sched = get_cosine_schedule_with_warmup(topt, num_warmup_steps=W, num_training_steps=N)
    for i in range(30):
        gen = torch.Generator(device=DEV).manual_seed(i)
        for p, r in zip(ps, refs):
            p.grad = torch.randn(p.shape, device=DEV, generator=gen).to(BF16)
            r.grad = p.grad.float()
        hf_lr = topt.param_groups[0]["lr"]
        before = [p.detach().clone() for p in ps]
        opt.step()
        topt.step()
        sched.step()
        assert lr_close(opt.last_lr(), float(np.float32(hf_lr))), (i, opt.last_lr(), hf_lr)
        if i == 0:
            assert hf_lr == 0.0
            for p, p0 in zip(ps, before):
                w, m, v = opt.state[id(p)]
                assert torch.equal(p, p0) and torch.equal(w, p0.float())
                assert m.abs().max() > 0 and v.abs().max() > 0
    e_master = max(rel(opt.state[id(p)][0], r) for p, r in zip(ps, refs))
    e_p = max(rel(p, r) for p, r in zip(ps, refs))
    print(f"\n[scheduled AdamW vs torch + HF cosine, 30 steps] master {e_master:.2e} param {e_p:.2e}")
    assert e_master < 1e-6 and e_p < 3e-3


def _scheduled_fp16_run(grad_steps, inf_steps=(), budget=None):
    """fp16 parameters, DynamicLossScaler (hysteresis 100: an overflow does not change the scale) + clipping, cosine
    schedule W = 3, N = 10.  grad_steps: the seeds of the gradients fed, in order; on inf_steps (indices into it) one
    gradient element is +inf.  -> (parameters, (master, m, v) per parameter, per-step log of (skip, step, lr))."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, LRSchedule

    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(*s, device=DEV).to(F16)) for s in SHAPES]
    opt = FusedAdamW(ps, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, max_grad_norm=1.0,
                     device_state_bytes=budget, lr_schedule=LRSchedule("cosine", 3, 10))
    scaler = DynamicLossScaler(initial_scale_power=8, hysteresis=100)
    S = 2.0 ** 8
    log = []
    try:
        for i, seed in enumerate(grad_steps):
            gen = torch.Generator(device=DEV).manual_seed(100 + seed)
            for p in ps:
                p.grad = (torch.randn(p.shape, device=DEV, generator=gen) * S).to(F16)
            if i in inf_steps:
                ps[1].grad[5] = float("inf")
            snap = [p.detach().clone() for p in ps], {k: tuple(t.clone() for t in v) for k, v in opt.state.items()}
            opt.step(loss_scaler=scaler)
            d = scaler.state_dict()
            log.append((d["skip"], d["step"], opt.last_lr()))
            if d["skip"]:  # a skipped step writes nothing
                assert all(torch.equal(a, p) for a, p in zip(snap[0], ps)), i
                for k, v in snap[1].items():
                    assert all(torch.equal(a, b) for a, b in zip(v, opt.state[k])), i
    finally:
        _ops().set_act_format(BF16)
    states = [tuple(t.detach().cpu().clone() for t in opt.state[id(p)]) for p in ps]
    return [p.detach().cpu().clone() for p in ps], states, log


SKIPS = (0, 4, 5, 9)  # the very first step (before any applied one), a pair, and one inside the decay


def test_skipped_steps_do_not_advance_the_schedule():
    """Overflow-skipped steps write nothing and do not advance the schedule: the lrs of the applied steps are
    fp32(base * lambda(0)), lambda(1), ... with no gaps, and the run ends bit-identical to one fed only the gradients of
    the applied steps."""
    from macaw_llm_b200.training import LRSchedule

    s = LRSchedule("cosine", 3, 10)
    steps = list(range(16))
    ps, st, log = _scheduled_fp16_run(steps, SKIPS)
    assert [i for i, (skip, _, _) in enumerate(log) if skip] == list(SKIPS)
    applied = [(t, lr) for skip, t, lr in log if not skip]
    assert [t for t, _ in applied] == list(range(1, len(applied) + 1))
    assert all(lr_close(lr, s.lr_of_update(1e-2, t)) for t, (_, lr) in enumerate(applied, 1)), applied
    print(f"\n[schedule over skips] (skip, step, lr): {log}")
    ps2, st2, log2 = _scheduled_fp16_run([i for i in steps if i not in SKIPS])
    assert [lr for _, _, lr in log2] == [lr for _, lr in applied]
    assert all(torch.equal(a, b) for a, b in zip(ps, ps2))
    assert all(torch.equal(a, b) for x, y in zip(st, st2) for a, b in zip(x, y))


@pytest.mark.parametrize("budget", [0, 12 * 300 * 64])
def test_host_state_bit_identical_under_a_schedule(budget):
    """The scheduled run (skips included) with every state in host memory (budget 0) and with a budget that keeps only
    the first tensor on the device: parameters, master weights and moments bit-identical to device state."""
    ps, st, log = _scheduled_fp16_run(list(range(16)), SKIPS)
    ps_h, st_h, log_h = _scheduled_fp16_run(list(range(16)), SKIPS, budget=budget)
    assert log_h == log
    assert all(torch.equal(a, b) for a, b in zip(ps, ps_h))
    assert all(torch.equal(a, b) for x, y in zip(st, st_h) for a, b in zip(x, y))


# ---------------------------------------------------------------------------------------------------- CUDA graph
@pytest.fixture(scope="module")
def tiny_fp16():
    return H.build_tiny_model("cuda", F16)


def test_scheduled_fp16_step_cuda_graph_matches_eager(tiny_fp16):
    """The whole fp16 step with a cosine schedule (forward, scaled backward, gradient norm, scaler update, lr schedule,
    AdamW) captured once and replayed, against eager steps from the same initial state (the pattern of
    test_fp16_step_cuda_graph_matches_eager): the same (scale, skip, step, lr) trajectory, parameters within that test's
    tolerance, and an lr that changes from replay to replay as the warmup ends and the decay runs."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, LRSchedule, trainable_parameters
    from tests.test_train_fp16_gpu import _train_inputs

    model0, spec, hp, weights = tiny_fp16
    inp = _train_inputs(spec, seed=9)
    k, base = 16, 1e-3
    sched = LRSchedule("cosine", 3, 10)

    def setup():
        m = copy.deepcopy(model0)
        ps = [p for _, p in trainable_parameters(m)]
        # S = 2^20: the first steps overflow and are skipped, then the scale fits and the schedule starts
        return m, FusedAdamW(ps, lr=base, weight_decay=0.0, max_grad_norm=1.0, lr_schedule=sched), \
            DynamicLossScaler(initial_scale_power=20, hysteresis=1)

    def make_step(m, opt, sc):
        def step():
            opt.zero_grad()
            out = m(inp)
            sc.scale(out.loss).backward()
            m.train_step.llama.finish_allreduce()
            opt.step(loss_scaler=sc)
            return out.loss
        return step

    def record(traj, sc, opt):
        d = sc.state_dict()
        traj.append((d["scale"], d["skip"], d["step"], opt.last_lr()))

    runs = {}
    for mode in ("eager", "graph"):
        m, opt, sc = setup()
        m.train()
        m.train_step.attention_dropout = False
        traj = []
        try:
            step = make_step(m, opt, sc)
            if mode == "graph":
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    step()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                record(traj, sc, opt)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    step()
                for _ in range(k - 1):
                    graph.replay()
                    torch.cuda.synchronize()
                    record(traj, sc, opt)
            else:
                for _ in range(k):
                    step()
                    torch.cuda.synchronize()
                    record(traj, sc, opt)
        finally:
            m.train_step.attention_dropout = True
            m.eval()
        runs[mode] = (traj, {n: p.detach().float().clone() for n, p in m.named_parameters()})
    (te, pe), (tg, pg) = runs["eager"], runs["graph"]
    print(f"\n[scheduled fp16 graph vs eager] trajectory (scale, skip, step, lr)\n  eager {te}\n  graph {tg}")
    assert te == tg
    assert any(t[1] for t in te) and not te[-1][1]
    applied = 0
    for scale, skip, t, lr in tg:  # the applied steps counted from the skip flags alone; the lr is that of their count
        applied += 0 if skip else 1
        assert t == applied and lr_close(lr, sched.lr_of_update(base, max(applied, 1))), (t, applied, lr)
    replay_lrs = [t[3] for t in tg[1:] if not t[1]]
    assert len(set(replay_lrs)) >= 4, replay_lrs  # warmup ends and the decay runs across replays
    assert max(replay_lrs) > 0.0 and lr_close(max(replay_lrs), sched.lr_of_update(base, 4))  # the peak, after W = 3
    worst = max(rel(pg[n], pe[n]) for n in pe)
    print(f"[scheduled fp16 graph vs eager] worst parameter rel diff {worst:.2e}")
    assert worst < 2e-3
