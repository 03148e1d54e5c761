#!/usr/bin/env python
"""Training with AdamW state in page-locked host memory, updated by the GPU over PCIe (`FusedAdamW(device_state_bytes=…)`,
the equivalent of DeepSpeed's offload_optimizer {device: cpu, pin_memory: true} in the reference's
configs/deepspeed_config.json).  Setup of tools/bench_train_precision.py: cfg4 shape, micro-batch 4, L = 512 -> T = 528,
fp16 with DynamicLossScaler() and max_grad_norm = 1.0, CUDA-graph replay of the whole optimizer step.

Runs (one JSON line each):
  A   top 8 decoder layers trained, every state on the device (the default path; run first and again last)
  C1  all 32 layers, the largest device_state_bytes that fits next to the step (value reported)
  C3  as C1, with 3 micro-batches per optimizer step (train.sh: gradient_accumulation_steps 3) in one graph
  B   top 8 layers, device_state_bytes = 0: every state in host memory

Each line: ms per optimizer step (mean over the timed steps that were not overflow-skipped), tokens/s, the optimizer
step alone (CUDA events), host-state bytes and the PCIe rate 2 * host bytes / optimizer time, peak device memory, the
loss trajectory, skipped steps, and the duration of the first step (which pins and fills the host state).  Before these, the update kernels are compared on one host-resident state (mm_adamw on the device alias against
mm_adamw_host) beside a copy-engine reference (1 GiB pinned H2D and D2H copies, alone and concurrent), and the card, its
power limit and PCIe link are read with one query-only nvidia-smi call.

Host memory is checked before anything is pinned: if the state plus an 8 GiB margin exceeds MemAvailable, the script
exits with a message (no fall-back, no swapping).  Not the benchmark of record (bench.py is)."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

GiB = 1 << 30
HOST_MARGIN = 8 * GiB


def card() -> dict:
    q = "name,power.limit,pcie.link.gen.current,pcie.link.width.current"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power, gen, width = (s.strip() for s in out[0].split(","))
        return {"gpu": name, "power_limit": power, "pcie_link": f"gen {gen} x{width}"}
    except Exception as e:  # the numbers stay usable, the card is then unknown
        return {"gpu": f"unknown ({e})", "power_limit": "unknown", "pcie_link": "unknown"}


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("MemAvailable not found in /proc/meminfo")


def require_host(nbytes: int, what: str) -> None:
    avail = mem_available()
    if nbytes + HOST_MARGIN > avail:
        print(json.dumps({"run": what, "error": f"needs {nbytes / GiB:.1f} GiB of page-locked host memory + "
                                                f"{HOST_MARGIN / GiB:.0f} GiB margin, MemAvailable is {avail / GiB:.1f} GiB"}),
              flush=True)
        sys.exit(3)


def _time(fn, reps: int) -> float:
    """ms per call (CUDA events around `reps` calls, after one warm-up call)."""
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(n: int, reps: int) -> dict:
    """mm_adamw (the HBM-laid-out vec8 kernel) and mm_adamw_host on the same host-resident state of n elements (bf16 p, g
    in HBM); rates are host bytes moved (24 B per element) per second."""
    from macaw_llm_b200 import _lib, ops

    sz = (4 * n + 15) // 16 * 16
    require_host(3 * sz, "kernels")
    blk = ops.host_alloc(3 * sz)
    try:
        w, m, v = (blk.view(o, n) for o in (0, sz, 2 * sz))
        p = torch.randn(n, device="cuda").to(torch.bfloat16)
        g = (torch.randn(n, device="cuda") * 1e-2).to(torch.bfloat16)
        w.copy_(p.float())
        m.zero_()
        v.zero_()
        lib = _lib.load()
        args = lambda: (p.data_ptr(), g.data_ptr(), blk.dev_ptr(w), blk.dev_ptr(m), blk.dev_ptr(v), n, 1e-5, 0.9,  # noqa: E731
                        0.999, 1e-8, 0.0, 1, None, 1.0, None, None, None, ops._stream())
        old = lambda: ops._check(lib.mm_adamw(*args()), "mm_adamw")  # noqa: E731
        new = lambda: ops._check(lib.mm_adamw_host(*args()), "mm_adamw_host")  # noqa: E731
        t = {"mm_adamw_on_alias": [], "mm_adamw_host": []}
        for _ in range(2):  # interleaved, so that drift affects both alike
            t["mm_adamw_on_alias"].append(_time(old, reps))
            t["mm_adamw_host"].append(_time(new, reps))
        res = {"elements": n, "host_bytes_per_call": 24 * n}
        for k, ms in t.items():
            res[k] = {"ms": ms, "GB_per_s": [24 * n / (x / 1e3) / 1e9 for x in ms]}
        return res
    finally:
        blk.free()


def copy_engine(reps: int) -> dict:
    """Copy-engine reference: a 1 GiB pinned host tensor copied H2D and D2H, alone and concurrently on two streams."""
    require_host(2 * GiB, "copy_engine")
    h1 = torch.empty(GiB, dtype=torch.uint8, pin_memory=True)
    h2 = torch.empty(GiB, dtype=torch.uint8, pin_memory=True)
    d1 = torch.empty(GiB, dtype=torch.uint8, device="cuda")
    d2 = torch.empty(GiB, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def both():
        cur = torch.cuda.current_stream()
        s1.wait_stream(cur)
        s2.wait_stream(cur)
        with torch.cuda.stream(s1):
            d1.copy_(h1, non_blocking=True)
        with torch.cuda.stream(s2):
            h2.copy_(d2, non_blocking=True)
        cur.wait_stream(s1)
        cur.wait_stream(s2)

    h2d = _time(lambda: d1.copy_(h1, non_blocking=True), reps)
    d2h = _time(lambda: h2.copy_(d2, non_blocking=True), reps)
    dup = _time(both, reps)
    res = {"bytes": GiB, "h2d_GB_per_s": GiB / (h2d / 1e3) / 1e9, "d2h_GB_per_s": GiB / (d2h / 1e3) / 1e9,
           "concurrent_GB_per_s": 2 * GiB / (dup / 1e3) / 1e9}
    del h1, h2, d1, d2
    return res


def _free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def run(name: str, train_layers: int, budget, accum: int, args) -> dict:
    """budget: None (device state), an int (bytes), or "max" (the largest that fits, found with a probe step)."""
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from macaw_llm_b200.training import (DynamicLossScaler, FusedAdamW, _host_layout, _state_placement,
                                         freeze_like_reference, freeze_llama_layers, trainable_parameters)

    _free()
    dt = torch.float16
    (clip, whisper, llama), hyper = bench.real_configs()
    dev = torch.device("cuda", 0)
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=dev, dtype=dt, seed=0)
    freeze_like_reference(model)
    n_layers = len(model.llm.model.layers)
    freeze_llama_layers(model, n_layers - train_layers)
    host = bench.synth_inputs(args.micro_batch, args.seq_len, llama.vocab_size, clip.vision_config.image_size,
                              2 * whisper.max_source_positions, 1234, dtype=dt)
    host["labels"] = host["input_ids"].clone()
    inp = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    params = [p for _, p in trainable_parameters(model)]
    numels = [p.numel() for p in params]
    model.train()
    res = {"run": name}
    if budget == "max":
        # probe: one forward + backward (gradient buffer included) without the optimizer; the captured graph keeps a
        # second copy of the activations in its private pool, so the state budget leaves room for both plus a margin
        base = torch.cuda.memory_allocated()
        out = model(inp)
        out.loss.backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        kept = torch.cuda.memory_allocated()
        del out
        for p in params:
            p.grad = None
        total = torch.cuda.get_device_properties(dev).total_memory
        act = peak - kept
        budget = max(0, (total - peak - act - args.margin_gib * GiB) // GiB * GiB)
        res.update(probe={"weights_gb": base / 1e9, "after_backward_gb": kept / 1e9, "peak_gb": peak / 1e9,
                          "activations_gb": act / 1e9, "margin_gib": args.margin_gib})
        _free()
    if budget is not None:
        offs, host_bytes = _host_layout(numels, _state_placement(numels, budget))
        require_host(host_bytes, name)
    scaler = DynamicLossScaler()
    opt = FusedAdamW(params, lr=2e-5, weight_decay=0.0, max_grad_norm=1.0, device_state_bytes=budget)

    def step():
        opt.zero_grad()
        for _ in range(accum):
            out = model(inp)
            scaler.scale(out.loss / accum if accum > 1 else out.loss).backward()
        model.train_step.llama.finish_allreduce()
        opt.step(loss_scaler=scaler)
        return out.loss

    t0 = time.perf_counter()
    losses = [float(step())]  # the first step allocates (and pins) the optimizer state
    first_step_s = time.perf_counter() - t0
    for _ in range(args.eager_steps - 1):
        losses.append(float(step()))
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        losses.append(float(step()))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    static = {}
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        static["loss"] = step()
    graph.replay()
    losses.append(float(static["loss"]))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times, skips = [], []
    for _ in range(args.steps):  # one event pair per step: the loss and the skip flag are read after each
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        skips.append(int(scaler.state[5]))
        losses.append(float(static["loss"]))
    taken = [t for t, s in zip(times, skips) if not s] or times  # a skipped step writes no state: it is faster
    ms = sum(taken) / len(taken)
    # the optimizer step alone (gradient norm, scaler update, AdamW launches) on the last replay's gradients: a real step
    opt_ms = []
    for _ in range(2):
        e0.record()
        opt.step(loss_scaler=scaler)
        e1.record()
        torch.cuda.synchronize()
        opt_ms.append(e0.elapsed_time(e1))
    d = scaler.state_dict()
    tokens = args.micro_batch * (args.seq_len + 16) * accum
    hb = opt.host_state_bytes
    res.update(ms_per_step=ms, ms_per_step_each=times, skipped_each=skips, tokens_per_s=tokens / (ms / 1e3), optimizer_ms=opt_ms,
               device_state_bytes=budget, host_state_bytes=hb,
               pcie_GB_per_s=(2 * hb / (min(opt_ms) / 1e3) / 1e9) if hb else None,
               peak_device_gb=torch.cuda.max_memory_allocated() / 1e9, trainable_params=sum(numels),
               trained_layers=f"{train_layers} of {n_layers}", micro_batches_per_step=accum,
               first_step_s=first_step_s, loss_trajectory=losses, loss_scale=d["scale"], skipped_steps=d["skipped"],
               optimizer_steps=d["step"],
               config=f"cfg4 fp16, micro-batch {args.micro_batch} x {accum}, L={args.seq_len} -> T={args.seq_len + 16}, "
                      "DynamicLossScaler() + max_grad_norm=1.0, CUDA-graph replay of the whole optimizer step")
    blk = opt._host_block
    del graph, static, model, opt, params, inp, scaler, step
    _free()
    if blk is not None and blk.host:  # the optimizer's finalizer frees the block when the optimizer is collected
        res["host_block_outlived_optimizer"] = True
        blk.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed graph replays per run")
    ap.add_argument("--eager-steps", type=int, default=5, help="eager steps before the captured one")
    ap.add_argument("--micro-batch", type=int, default=4)
    ap.add_argument("--seq-len", type=int, default=512)
    ap.add_argument("--runs", default="kernels,copy,A,C1,C3,B,A")
    ap.add_argument("--kernel-elements", type=int, default=1 << 28)
    ap.add_argument("--margin-gib", type=int, default=4, help="device memory left free beside the state budget of C")
    ap.add_argument("--budget", type=int, default=None, help="device_state_bytes for C (default: the largest that fits)")
    args = ap.parse_args()
    c = card()
    print(json.dumps(dict(c, mem_available_gib=mem_available() / GiB)), flush=True)
    budget_c = args.budget if args.budget is not None else "max"
    for r in args.runs.split(","):
        if r == "kernels":
            out = {"run": "kernels", **kernels(args.kernel_elements, 3)}
        elif r == "copy":
            out = {"run": "copy_engine", **copy_engine(5)}
        elif r == "A":
            out = run("A", 8, None, 1, args)
        elif r == "B":
            out = run("B", 8, 0, 1, args)
        elif r in ("C1", "C3"):
            out = run(r, 32, budget_c, int(r[1]), args)
            budget_c = out["device_state_bytes"]  # C3 reuses C1's budget
        else:
            raise SystemExit(f"unknown run {r}")
        print(json.dumps(dict(out, **c)), flush=True)


if __name__ == "__main__":
    main()
