#!/usr/bin/env python
"""The learning-rate schedule on the device (`FusedAdamW(lr_schedule=LRSchedule(...))`, mm_lr_schedule) at the training
bench's configuration: cfg4 shape, fp16 with DynamicLossScaler() and max_grad_norm = 1.0, micro-batch 4, L = 512 ->
T = 528, the top 8 decoder layers trained, CUDA-graph replay of the whole optimizer step.

Three JSON lines:
  card        the card's name and power limit (one query-only nvidia-smi call)
  cost        ms per optimizer step without a schedule and with cosine (W = 3, N = 100), one graph each over the same
              model and optimizer (the second graph shares the first's memory pool), replayed in alternating blocks, at
              least 2 rounds each; per-step CUDA events, the mean over the steps that were not overflow-skipped, and the
              spread.  Also mm_lr_schedule alone (CUDA events over back-to-back launches).
  trajectory  train.sh's recipe for 100 optimizer steps: 3 micro-batches per step (gradient_accumulation_steps 3), lr
              3e-5, warmup_ratio 0.03 (W = 3), cosine, on a freshly built model.  The first steps run eagerly (the
              capture needs them), the rest are graph replays.  After every step, lr, loss scale, skip flag, step counter
              and loss are copied into a device log; it is read once, after the timed window.  The applied steps are
              counted on the host from the skip flags alone; the device's step counter must equal that count, and
              every step's lr fp32(3e-5 * lambda(applied steps before it)) from the host restatement
              (LRSchedule.lr_lambda) within 1 fp32 ulp, across the overflow-skipped steps too (the bit-exact count is
              reported); the script exits non-zero on a mismatch.

Not the benchmark of record (bench.py is)."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

BASE_LR = 3e-5


def ulps(a: float, b: float) -> int:
    """Distance in fp32 units in the last place.  The device's lr may differ from the host restatement by 1: its double
    cos may differ from the host libm's in the last bit of the double before the rounding to fp32."""
    ia, ib = (int(torch.tensor([x], dtype=torch.float32).view(torch.int32)) for x in (a, b))
    return abs(ia - ib)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stay usable, the card is then unknown
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def _free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def setup(args):
    """The bench's fp16 training model (top `train_layers` decoder layers trained), its inputs and its parameters."""
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from macaw_llm_b200.training import freeze_like_reference, freeze_llama_layers, trainable_parameters

    dt = torch.float16
    (clip, whisper, llama), hyper = bench.real_configs()
    dev = torch.device("cuda", 0)
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=dev, dtype=dt, seed=0)
    freeze_like_reference(model)
    n_layers = len(model.llm.model.layers)
    freeze_llama_layers(model, n_layers - args.train_layers)
    host = bench.synth_inputs(args.micro_batch, args.seq_len, llama.vocab_size, clip.vision_config.image_size,
                              2 * whisper.max_source_positions, 1234, dtype=dt)
    host["labels"] = host["input_ids"].clone()
    inp = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    model.train()
    return model, inp, [p for _, p in trainable_parameters(model)], n_layers


def make_step(model, inp, opt, scaler, accum: int):
    def step():
        opt.zero_grad()
        for _ in range(accum):
            out = model(inp)
            scaler.scale(out.loss / accum if accum > 1 else out.loss).backward()
        model.train_step.llama.finish_allreduce()
        opt.step(loss_scaler=scaler)
        return out.loss
    return step


def warm_and_capture(step, pool=None, after_warm=None):
    """One eager step on a side stream (the warm-up a capture needs; `after_warm(loss)` sees its loss), then the capture
    of one step, which records it without running it.  -> (graph, the captured step's loss, detached).

    No loss with its autograd graph may outlive its step: the graph keeps the anchor leaf's gradient accumulator alive,
    with the stream it was created on, and the next step's backward would then wait on that stream — under capture, an
    uncaptured one."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        loss = step()
        if after_warm is not None:
            after_warm(loss)
        float(loss)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    del loss
    gc.collect()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, pool=pool, capture_error_mode="thread_local"):
        static_loss = step()
    return g, static_loss.detach()


def log_row(log: torch.Tensor, i: int, lr: torch.Tensor, scaler, loss: torch.Tensor) -> None:
    """log[i] = (lr, loss scale, skip, step, loss): device copies only, no sync."""
    st = scaler.state
    log[i].copy_(torch.cat([lr.reshape(1).float(), st.view(torch.float32)[0:1], st[5:6].float(), st[8:9].float(),
                            loss.detach().reshape(1).float()]))


def cost(args) -> dict:
    from macaw_llm_b200 import ops
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, LRSchedule

    _free()
    model, inp, params, n_layers = setup(args)
    sched = LRSchedule("cosine", 3, 100)
    scaler = DynamicLossScaler()
    opt = FusedAdamW(params, lr=BASE_LR, weight_decay=0.0, max_grad_norm=1.0)
    step = make_step(model, inp, opt, scaler, 1)
    for _ in range(args.warmup):  # past the early overflow-skipped steps
        float(step())
    graphs, loss_src = {}, {}
    graphs["none"], loss_src["none"] = warm_and_capture(step)
    opt.lr_schedule = sched  # the same optimizer and state, now scheduled: warm up, then capture into the same pool
    graphs["cosine"], loss_src["cosine"] = warm_and_capture(step, pool=graphs["none"].pool())
    const_lr = torch.full((1,), BASE_LR, device="cuda", dtype=torch.float32)
    lr_src = {"none": const_lr, "cosine": opt._lr_dev}
    for name in ("none", "cosine"):
        graphs[name].replay()
    torch.cuda.synchronize()
    per = {"none": [], "cosine": []}
    skipped = {"none": 0, "cosine": 0}
    rounds = []
    for r in range(args.rounds):
        order = ("none", "cosine") if r % 2 == 0 else ("cosine", "none")
        for name in order:
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            log = torch.zeros((args.steps, 5), device="cuda", dtype=torch.float32)
            for i in range(args.steps):
                ev[i][0].record()
                graphs[name].replay()
                ev[i][1].record()
                log_row(log, i, lr_src[name], scaler, loss_src[name])
            torch.cuda.synchronize()
            ms = [a.elapsed_time(b) for a, b in ev]
            skip = log[:, 2].cpu().tolist()
            taken = [t for t, s in zip(ms, skip) if not s]
            skipped[name] += len(ms) - len(taken)
            per[name].append(statistics.mean(taken or ms))
            rounds.append({"round": r, "schedule": name, "ms_mean": per[name][-1], "ms_each": ms,
                           "skipped": int(sum(skip))})
    # mm_lr_schedule alone: back-to-back launches on the scaler's step counter, into a scratch scalar
    reps = 2000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st_step = scaler.state[8:9]
    scratch = torch.zeros((1,), device="cuda", dtype=torch.float32)
    for _ in range(10):
        ops.lr_schedule(st_step, scratch, base_lr=BASE_LR, kind="cosine", warmup_steps=3, training_steps=100)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        ops.lr_schedule(st_step, scratch, base_lr=BASE_LR, kind="cosine", warmup_steps=3, training_steps=100)
    e1.record()
    torch.cuda.synchronize()
    kern_us = e0.elapsed_time(e1) / reps * 1e3
    res = {"run": "cost", "schedule": "cosine W=3 N=100", "rounds": rounds}
    for name in ("none", "cosine"):
        v = per[name]
        res[name] = {"ms_per_step_by_round": v, "mean": statistics.mean(v), "min": min(v), "max": max(v),
                     "skipped_steps_in_timed_window": skipped[name]}
    res["cosine_minus_none_ms"] = res["cosine"]["mean"] - res["none"]["mean"]
    res["spread_ms"] = {"none": max(per["none"]) - min(per["none"]), "cosine": max(per["cosine"]) - min(per["cosine"])}
    res["mm_lr_schedule_alone_us"] = kern_us
    res.update(trainable_params=sum(p.numel() for p in params), peak_device_gb=torch.cuda.max_memory_allocated() / 1e9,
               config=f"cfg4 fp16, micro-batch {args.micro_batch}, L={args.seq_len} -> T={args.seq_len + 16}, top "
                      f"{args.train_layers} of {n_layers} decoder layers trained, DynamicLossScaler() + max_grad_norm=1.0, "
                      f"CUDA-graph replay, {args.steps} steps per block, blocks alternated")
    del graphs, model, opt, params, inp, scaler, step, lr_src, loss_src
    _free()
    return res


def trajectory(args) -> dict:
    from macaw_llm_b200.training import DynamicLossScaler, FusedAdamW, LRSchedule

    _free()
    model, inp, params, n_layers = setup(args)
    n_steps, accum = args.trajectory_steps, 3
    sched = LRSchedule.from_warmup_ratio("cosine", 0.03, n_steps)
    scaler = DynamicLossScaler()
    opt = FusedAdamW(params, lr=BASE_LR, weight_decay=0.0, max_grad_norm=1.0, lr_schedule=sched)
    step = make_step(model, inp, opt, scaler, accum)
    log = torch.zeros((n_steps, 5), device="cuda", dtype=torch.float32)
    n_eager = 2  # optimizer steps 1 and 2 run eagerly, the second on the side stream the capture needs
    loss = step()
    log_row(log, 0, opt._lr_dev, scaler, loss)
    float(loss)
    del loss
    graph, static_loss = warm_and_capture(step, after_warm=lambda l: log_row(log, 1, opt._lr_dev, scaler, l))
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_steps - n_eager)]
    torch.cuda.synchronize()
    w0, w1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0.record()
    for j, i in enumerate(range(n_eager, n_steps)):
        ev[j][0].record()
        graph.replay()
        ev[j][1].record()
        log_row(log, i, opt._lr_dev, scaler, static_loss)
    w1.record()
    torch.cuda.synchronize()  # the timed window ends here; everything below reads the device log
    ms = [a.elapsed_time(b) for a, b in ev]
    rows = log.cpu().tolist()
    lr, scale, skip, t, loss = ([r[c] for r in rows] for c in range(5))
    skip, t = [int(s) for s in skip], [int(x) for x in t]
    mismatches, applied, exact = [], 0, 0
    for i in range(n_steps):
        # the applied steps are counted on the host from the skip flags alone.  An applied step is update number
        # `applied`, with applied - 1 before it; a skipped one leaves the device counter and rewrites the lr of the
        # latest applied update (that of the first before any), which its AdamW launches do not use
        applied += 0 if skip[i] else 1
        want32 = sched.lr_of_update(BASE_LR, max(applied, 1))
        if t[i] != applied or ulps(lr[i], want32) > 1:
            mismatches.append({"step": i + 1, "lr": lr[i], "want": want32, "counter": t[i], "applied": applied})
        exact += lr[i] == want32
    taken = [m for m, s in zip(ms, skip[n_eager:]) if not s]
    res = {"run": "trajectory", "recipe": "train.sh: lr 3e-5, warmup_ratio 0.03, cosine, 3 micro-batches per step, fp16 "
                                          "DynamicLossScaler() + max_grad_norm=1.0",
           "schedule": repr(sched), "optimizer_steps": n_steps, "eager_steps": n_eager, "replayed_steps": n_steps - n_eager,
           "ms_per_step_replayed": statistics.mean(taken) if taken else None,
           "window_ms": w0.elapsed_time(w1), "skipped_steps": sum(skip), "applied_steps": t[-1],
           "lr_check": "pass" if not mismatches else "FAIL", "lr_mismatches": mismatches, "lr_bit_exact": exact,
           "lr": lr, "loss_scale": scale, "skip": skip, "step_counter": t, "loss": loss,
           "peak_device_gb": torch.cuda.max_memory_allocated() / 1e9,
           "config": f"cfg4 fp16, micro-batch {args.micro_batch} x {accum}, L={args.seq_len} -> T={args.seq_len + 16}, top "
                     f"{args.train_layers} of {n_layers} decoder layers trained, CUDA-graph replay"}
    del graph, static_loss, model, opt, params, inp, scaler, step
    _free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="graph replays per timed block of the cost run")
    ap.add_argument("--rounds", type=int, default=3, help="blocks per schedule in the cost run (alternated)")
    ap.add_argument("--warmup", type=int, default=8, help="eager steps before the cost run's captures")
    ap.add_argument("--trajectory-steps", type=int, default=100)
    ap.add_argument("--micro-batch", type=int, default=4)
    ap.add_argument("--seq-len", type=int, default=512)
    ap.add_argument("--train-layers", type=int, default=8)
    ap.add_argument("--runs", default="cost,trajectory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_schedule: needs a CUDA device (an H100); there is no CPU path")
    if args.rounds < 2:
        raise SystemExit("bench_train_schedule: --rounds must be >= 2 (the spread needs repeated blocks)")
    c = card()
    print(json.dumps(dict(run="card", **c)), flush=True)
    rc = 0
    for r in args.runs.split(","):
        if r == "cost":
            out = cost(args)
        elif r == "trajectory":
            out = trajectory(args)
            rc = rc or (out["lr_check"] != "pass")
        else:
            raise SystemExit(f"unknown run {r}")
        print(json.dumps(dict(out, **c)), flush=True)
    sys.exit(int(rc))


if __name__ == "__main__":
    main()
