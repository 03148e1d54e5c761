#!/usr/bin/env python
"""Training step in both 16-bit formats at the training bench's configuration (bench.py --mode train: cfg4 shape,
micro-batch 4, L = 512 -> T = 528, the top 8 decoder layers trained, synthetic inputs from bench.synth_inputs):

  fp16  the reference's recipe (train.sh --fp16 True): DynamicLossScaler with DeepSpeed's defaults, FusedAdamW with
        max_grad_norm = 1.0 — one gradient-norm pass + the loss-scale update before AdamW
  bf16  as bench.py --mode train runs it (no scaler, no clipping)

One JSON line per format: ms per step (CUDA events over graph replays of the whole step, after warm-up), the loss
trajectory, the final loss scale and skipped steps, and — fp16 only — the isolated time of mm_grad_sumsq +
mm_loss_scale_update over the flat gradient buffer with the bytes/s it reaches against the H100 SXM's 3.35 TB/s.  The
card name and power limit are read once (nvidia-smi, query only).  Not the benchmark of record (bench.py is)."""
import argparse
import gc
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stay usable, the card is then unknown
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def run(fmt: str, args) -> dict:
    from macaw_llm_b200 import ops
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from macaw_llm_b200.training import (DynamicLossScaler, FusedAdamW, freeze_like_reference, freeze_llama_layers,
                                         trainable_parameters)

    dt = torch.float16 if fmt == "fp16" else torch.bfloat16
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
    params = [p for _, p in trainable_parameters(model)]
    scaler = DynamicLossScaler() if fmt == "fp16" else None
    opt = FusedAdamW(params, lr=2e-5, weight_decay=0.0, max_grad_norm=1.0 if fmt == "fp16" else None)
    model.train()

    def step():
        opt.zero_grad()
        out = model(inp)
        (scaler.scale(out.loss) if scaler is not None else out.loss).backward()
        model.train_step.llama.finish_allreduce()
        opt.step(loss_scaler=scaler)
        return out.loss

    losses = [float(step()) for _ in range(3)]
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
    for _ in range(2):
        graph.replay()
        losses.append(float(static["loss"]))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    losses.append(float(static["loss"]))
    n_train = sum(p.numel() for p in params)
    res = {"format": fmt, "ms_per_step": ms, "steps": args.steps, "warmup": 6, "loss_trajectory": losses,
           "trainable_params": n_train, "optimizer": "FusedAdamW" + (" max_grad_norm=1.0 + DynamicLossScaler()" if scaler else ""),
           "config": f"cfg4, micro-batch {args.micro_batch}, L={args.seq_len} -> T={args.seq_len + 16}, top "
                     f"{args.train_layers} of {n_layers} decoder layers trained, CUDA-graph replay of the whole step"}
    if scaler is not None:
        d = scaler.state_dict()
        res.update(loss_scale=d["scale"], skipped_steps=d["skipped"], optimizer_steps=d["step"], grad_norm=d["grad_norm"])
        # the norm pass + scaler update alone, on the same flat buffer (state on a scratch copy: the run's state is kept)
        flat = model.train_step.llama.grads.flat
        st = scaler.state.clone()
        sumsq = torch.zeros(1, device=dev)
        parts = torch.empty(ops.grad_sumsq_parts(flat.numel()), device=dev)
        for _ in range(3):
            ops.grad_sumsq(flat, sumsq, parts)
            ops.loss_scale_update(st, sumsq, max_norm=1.0, dynamic=True, window=1000, hysteresis=2, min_scale=1.0)
        reps = 20
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            ops.grad_sumsq(flat, sumsq, parts)
            ops.loss_scale_update(st, sumsq, max_norm=1.0, dynamic=True, window=1000, hysteresis=2, min_scale=1.0)
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / reps
        nbytes = flat.numel() * flat.element_size()
        res.update(norm_pass={"elements": flat.numel(), "bytes": nbytes, "ms": t, "bytes_per_s": nbytes / (t / 1e3),
                              "fraction_of_3.35TB/s": nbytes / (t / 1e3) / HBM_PEAK,
                              "fraction_of_step": t / ms})
    res["mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    del graph, static, model, opt, params, inp, scaler
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--micro-batch", type=int, default=4)
    ap.add_argument("--seq-len", type=int, default=512)
    ap.add_argument("--train-layers", type=int, default=8)
    ap.add_argument("--formats", default="fp16,bf16")
    args = ap.parse_args()
    c = card()
    for fmt in args.formats.split(","):
        print(json.dumps(dict(run(fmt, args), **c)), flush=True)


if __name__ == "__main__":
    main()
