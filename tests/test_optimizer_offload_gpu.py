"""AdamW state in page-locked host memory, updated by the GPU over PCIe (mm_host_alloc + mm_adamw_host,
`FusedAdamW(device_state_bytes=...)`), on the H100: the host-state kernel against mm_adamw on device copies of the same
inputs (bit for bit), the optimizer under every placement with clipping and overflow-skipped fp16 steps (bit for bit),
and a whole tiny fp16 training step with host state replayed from a CUDA graph against eager steps with device state.
Host allocations stay under 2 GB."""
import copy

import pytest
import torch

from tests import helpers as H

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16


def _ops():
    from macaw_llm_b200 import ops

    return ops


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-20))


def _host_state(ops, n):
    """(block, master, m, v) over one exact-size host block, laid out as FusedAdamW lays it out."""
    sz = (4 * n + 15) // 16 * 16
    blk = ops.host_alloc(3 * sz)
    return (blk,) + tuple(blk.view(o, n) for o in (0, sz, 2 * sz))


# ---------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("n", [1, 7, 128, 4099, 32000 * 4096])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_adamw_host_kernel_bit_identical(dtype, n):
    """mm_adamw_host on host state against mm_adamw on device copies: plain steps, a device step counter, a device
    gradient multiplier and a skipped step (skip_dev = 1 writes no byte of host state)."""
    ops = _ops()
    ops.set_act_format(dtype)
    blk = None
    try:
        gen = torch.Generator(device=DEV).manual_seed(n % 1009)
        p_d = torch.randn(n, device=DEV, generator=gen).to(dtype)
        p_h = p_d.clone()
        w_d, m_d, v_d = p_d.float(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        blk, w_h, m_h, v_h = _host_state(ops, n)
        w_h.copy_(w_d)
        m_h.zero_()
        v_h.zero_()
        step_dev = torch.zeros(1, device=DEV, dtype=torch.int32)
        mult = torch.tensor([0.37], device=DEV)
        skip = torch.ones(1, device=DEV, dtype=torch.int32)
        hyper = dict(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1)
        cases = [dict(step=1), dict(step=2, grad_scale=0.5), dict(step=0, step_dev=step_dev),
                 dict(step=0, step_dev=step_dev, grad_mult_dev=mult), dict(step=0, step_dev=step_dev, skip_dev=skip),
                 dict(step=0, step_dev=step_dev, grad_mult_dev=mult)]
        for i, kw in enumerate(cases):
            g = (torch.randn(n, device=DEV, generator=gen) * (0.1 + i)).to(dtype)
            step_dev.fill_(i + 1)
            torch.cuda.synchronize()
            before = (w_h.clone(), m_h.clone(), v_h.clone()) if "skip_dev" in kw else None
            ops.adamw(p_d, g, w_d, m_d, v_d, **hyper, **kw)
            ops.adamw_host(p_h, g, w_h, m_h, v_h, block=blk, **hyper, **kw)
            torch.cuda.synchronize()  # the host views are read by the CPU below
            assert torch.equal(p_h, p_d), (i, kw)
            assert torch.equal(w_h, w_d.cpu()) and torch.equal(m_h, m_d.cpu()) and torch.equal(v_h, v_d.cpu()), (i, kw)
            if before is not None:
                assert all(torch.equal(a, b) for a, b in zip(before, (w_h, m_h, v_h))), "a skipped step wrote host state"
        assert float(m_h.abs().max()) > 0  # the state really moved
    finally:
        ops.set_act_format(BF16)
        if blk is not None:
            blk.free()


# ---------------------------------------------------------------------------------------------------- optimizer
@pytest.mark.parametrize("dtype", [F16, BF16])
def test_fused_adamw_placements_bit_identical(dtype):
    """FusedAdamW with device_state_bytes None / 0 / a budget that splits the set, fed the same synthetic gradients
    (the shapes of test_train_fp16_gpu._clip_case) with clipping and, for fp16, a DynamicLossScaler whose first steps
    overflow: parameters and all states are identical across placements after every step, and skipped steps leave them
    untouched."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW

    shapes = [(300, 64), (64,), (17, 8)]
    torch.manual_seed(0)
    init = [torch.randn(*s, device=DEV).to(dtype) for s in shapes]
    budgets = [None, 0, 12 * (64 + 17 * 8)]  # the last one: the large tensor on the host, the two small ones on the device
    runs = []
    for b in budgets:
        ps = [torch.nn.Parameter(t.clone()) for t in init]
        opt = FusedAdamW(ps, lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1, max_grad_norm=1.0,
                         device_state_bytes=b)
        sc = DynamicLossScaler(initial_scale_power=18, hysteresis=1) if dtype == F16 else None
        runs.append((ps, opt, sc))
    assert [r[1].host_state_bytes for r in runs] == [0, 3 * (4 * 300 * 64 + 256 + 544), 3 * 4 * 300 * 64]
    n_skip = 0
    try:
        for i in range(10):
            gen = torch.Generator(device=DEV).manual_seed(100 + i)
            gs = [torch.randn(*s, device=DEV, generator=gen) for s in shapes]
            snaps = []
            for ps, opt, sc in runs:
                S = sc.loss_scale if sc is not None else 1.0
                for p, g in zip(ps, gs):
                    p.grad = (g * S).to(dtype)
                torch.cuda.synchronize()
                snaps.append(([p.detach().clone() for p in ps],
                              {k: tuple(t.clone() for t in v) for k, v in opt.state.items()}))
                opt.step(loss_scaler=sc)
            torch.cuda.synchronize()
            skipped = runs[0][2] is not None and runs[0][2].state_dict()["skip"]
            n_skip += int(bool(skipped))
            (ps0, opt0, _) = runs[0]
            for ps, opt, sc in runs[1:]:
                if sc is not None:
                    assert sc.state_dict() == runs[0][2].state_dict(), i
                for p0, p in zip(ps0, ps):
                    assert torch.equal(p0, p), (i, opt.device_state_bytes)
                    s0, s = opt0.state[id(p0)], opt.state[id(p)]
                    assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(s0, s)), (i, opt.device_state_bytes)
                assert any(t.device.type == "cpu" for v in opt.state.values() for t in v)
            if skipped:
                for (ps, opt, _), (sp, sst) in zip(runs, snaps):
                    assert all(torch.equal(a, p) for a, p in zip(sp, ps)), i
                    for k, v in sst.items():
                        assert all(torch.equal(a, b) for a, b in zip(v, opt.state[k])), i
    finally:
        _ops().set_act_format(BF16)
    if dtype == F16:
        assert 0 < n_skip < 10, n_skip  # both skipped and taken steps were exercised
    print(f"\n[offload placements {dtype}] 10 steps, {n_skip} skipped, identical across {budgets}")


# ---------------------------------------------------------------------------------------------------- whole model
def test_fp16_step_host_state_cuda_graph_matches_eager():
    """The whole fp16 step (forward, scaled backward, clipping, scaler, AdamW) with every AdamW state in host memory,
    captured once and replayed k times, against k eager steps with device state: the same scale and skip trajectory,
    parameters within the tolerance of test_fp16_step_cuda_graph_matches_eager (the table scatter's atomics may reorder
    sums), and the state really in the host block."""
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, trainable_parameters
    from tests.test_train_fp16_gpu import _train_inputs

    model0, spec, hp, weights = H.build_tiny_model("cuda", F16)
    inp = _train_inputs(spec, seed=9)
    k = 12

    def make_step(m, opt, sc):
        def step():
            opt.zero_grad()
            out = m(inp)
            sc.scale(out.loss).backward()
            m.train_step.llama.finish_allreduce()
            opt.step(loss_scaler=sc)
            return out.loss
        return step

    def record(sc, traj):
        torch.cuda.synchronize()
        d = sc.state_dict()
        traj.append((d["scale"], d["skip"], d["skipped"], d["step"]))

    runs = {}
    for mode in ("eager", "graph"):
        m = copy.deepcopy(model0)
        ps = [p for _, p in trainable_parameters(m)]
        opt = FusedAdamW(ps, lr=1e-3, weight_decay=0.0, max_grad_norm=1.0,
                         device_state_bytes=None if mode == "eager" else 0)
        sc = DynamicLossScaler(initial_scale_power=20, hysteresis=1)
        m.train()
        m.train_step.attention_dropout = False
        traj = []
        try:
            step = make_step(m, opt, sc)
            if mode == "graph":
                # the first step runs eagerly on a side stream (it allocates the host block), then one step is captured
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    step()
                torch.cuda.current_stream().wait_stream(side)
                record(sc, traj)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    step()
                for _ in range(k - 1):
                    graph.replay()
                    record(sc, traj)
                assert opt.host_state_bytes > 0 and opt.host_state_bytes == opt._host_block.nbytes
                states = [t for v in opt.state.values() for t in v]
                assert len(states) == 3 * len(ps) and all(t.device.type == "cpu" for t in states)
            else:
                for _ in range(k):
                    step()
                    record(sc, traj)
                assert opt.host_state_bytes == 0 and all(t.is_cuda for v in opt.state.values() for t in v)
        finally:
            m.train_step.attention_dropout = True
            m.eval()
        runs[mode] = (traj, {n: p.detach().float().clone() for n, p in m.named_parameters()})
        del opt
    (te, pe), (tg, pg) = runs["eager"], runs["graph"]
    print(f"\n[host-state graph vs eager] trajectory eager {te}\n                           graph {tg}")
    assert te == tg
    assert any(t[1] for t in te) and not te[-1][1]
    worst = max(rel(pg[n], pe[n]) for n in pe)
    print(f"[host-state graph vs eager] worst parameter rel diff {worst:.2e}")
    assert worst < 2e-3
