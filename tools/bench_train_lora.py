#!/usr/bin/env python
"""LoRA fine-tuning of the 7B model at the training bench's configuration (cfg4: micro-batch 4, L = 512 -> T = 528,
image + audio + text, synthetic inputs from bench.synth_inputs), fp16 with the reference's recipe (DynamicLossScaler,
FusedAdamW max_grad_norm = 1.0, cosine LRSchedule):

  lora   every decoder layer adapted with the reference's targets (run_clm_llms.py:498-508: q/k/v/lm_head, r = 8,
         alpha = 16, dropout 0.05; the GPT-J names and embed_tokens dropped), base frozen
  top8   the existing partial full fine-tune: the top 8 decoder layers trained (bench.py --mode train)

The two are alternated over `--rounds` rounds in this process (a fresh model each time).  One JSON line per run: ms per
step (CUDA events over graph replays of the whole step, after warm-up), tokens/s, peak device memory, trainable
parameters, loss trajectory.  Then each LoRA kernel alone at the production shapes of one layer (M = 2112, E = 4096,
V = 32000, r = 8): bytes moved (the operands and results each launch must read or write once; the fp32 partials of the
reductions are reported separately), time (CUDA events over 50 launches) and GB/s against the H100 SXM's 3.35 TB/s.
Card name, power limit and the median SM clock over the timed windows (nvidia-smi, query only) are read in the same call.
Not the benchmark of record (bench.py is)."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
REFERENCE_TARGETS = ["q_proj", "k_proj", "v_proj", "lm_head"]


def smi(query: str) -> str:
    return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits"], capture_output=True,
                          text=True, timeout=30).stdout.strip().splitlines()[0]


class ClockSampler:
    """SM clock samples (MHz) every 200 ms while active."""

    def __init__(self):
        self.samples, self._on, self._t = [], False, None

    def __enter__(self):
        self._on = True
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        import time

        while self._on:
            try:
                self.samples.append(int(smi("clocks.sm")))
            except Exception:
                pass
            time.sleep(0.2)

    def __exit__(self, *exc):
        self._on = False
        self._t.join()


CLOCKS = []


def run_step(variant: str, args) -> dict:
    from macaw_llm_b200.lora import LoraConfig
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from macaw_llm_b200.training import (DynamicLossScaler, FusedAdamW, LRSchedule, freeze_like_reference,
                                         freeze_llama_layers, trainable_parameters)

    dt = torch.float16
    (clip, whisper, llama), hyper = bench.real_configs()
    dev = torch.device("cuda", 0)
    torch.cuda.reset_peak_memory_stats()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=dev, dtype=dt, seed=0)
    freeze_like_reference(model)
    n_layers = len(model.llm.model.layers)
    if variant == "lora":
        model.add_lora(LoraConfig(r=8, lora_alpha=16, lora_dropout=0.05, target_modules=REFERENCE_TARGETS))
    else:
        freeze_llama_layers(model, n_layers - args.train_layers)
    host = bench.synth_inputs(args.micro_batch, args.seq_len, llama.vocab_size, clip.vision_config.image_size,
                              2 * whisper.max_source_positions, 1234, dtype=dt)
    host["labels"] = host["input_ids"].clone()
    inp = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    params = [p for _, p in trainable_parameters(model)]
    scaler = DynamicLossScaler()
    opt = FusedAdamW(params, lr=3e-5, weight_decay=0.0, max_grad_norm=1.0,
                     lr_schedule=LRSchedule.from_warmup_ratio("cosine", 0.03, 1000))
    model.train()

    def step():
        opt.zero_grad()
        out = model(inp)
        scaler.scale(out.loss).backward()
        opt.step(loss_scaler=scaler)
        return out.loss

    losses = [float(step()) for _ in range(2)]
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
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler() as cs:
        e0.record()
        for _ in range(args.steps):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
    CLOCKS.extend(cs.samples)
    ms = e0.elapsed_time(e1) / args.steps
    losses.append(float(static["loss"]))
    T = args.seq_len + 16
    res = {"variant": variant, "ms_per_step": ms, "tokens_per_s": args.micro_batch * T / (ms / 1e3), "steps": args.steps,
           "trainable_params": sum(p.numel() for p in params), "peak_mem_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
           "loss_trajectory": losses, "loss_scale": scaler.loss_scale, "skipped_steps": scaler.skipped_steps,
           "config": f"cfg4 fp16, micro-batch {args.micro_batch}, L={args.seq_len} -> T={T}, "
                     + ("LoRA r=8 alpha=16 p=0.05 on q/k/v of all " + f"{n_layers} layers + lm_head, base frozen"
                        if variant == "lora" else f"top {args.train_layers} of {n_layers} decoder layers trained")
                     + "; DynamicLossScaler, max_grad_norm=1.0, cosine schedule; CUDA-graph replay of the whole step"}
    del graph, static, model, opt, params, inp, scaler
    gc.collect()
    torch.cuda.empty_cache()
    return res


def time_launch(fn, reps=50):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler() as cs:
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
    CLOCKS.extend(cs.samples)
    return e0.elapsed_time(e1) / reps


def kernels(args) -> list:
    from macaw_llm_b200 import lora, ops

    ops.set_act_format(torch.float16)
    dev = "cuda"
    M, E, V, r, p = args.micro_batch * (args.seq_len + 16), 4096, 32000, 8, 0.05
    f16 = torch.float16
    rn = lambda *s, scale=1.0: (torch.randn(*s, device=dev) * scale).to(f16)  # noqa: E731
    seed = torch.tensor([12345], dtype=torch.int64, device=dev)
    out = []

    def rec(name, fn, nbytes, partial_bytes=0):
        ms = time_launch(fn)
        out.append({"kernel": name, "ms": ms, "bytes": nbytes, "partials_bytes": partial_bytes,
                    "GB_per_s": nbytes / (ms / 1e3) / 1e9, "fraction_of_3.35TB/s": nbytes / (ms / 1e3) / HBM_PEAK})

    sids3 = [lora.lora_sid(0, t) for t in ("q_proj", "k_proj", "v_proj")]
    for label, n, N, K, sids in (("q/k/v (3 adapters)", 3, E, E, sids3), ("lm_head", 1, V, E, [lora.SID_LORA_LM_HEAD])):
        x = rn(M, K)
        As = [rn(r, K, scale=K ** -0.5) for _ in range(n)]
        Bs = [rn(N, r, scale=0.02) for _ in range(n)]
        drop = (p, seed, sids)
        us = ops.lora_down(x, As, dropout=drop)
        ys = [rn(M, N) for _ in range(n)]
        dys = [rn(M, N, scale=1e-3) for _ in range(n)]
        dAs, dBs, dx = [torch.zeros(r, K, device=dev, dtype=f16) for _ in range(n)], \
            [torch.zeros(N, r, device=dev, dtype=f16) for _ in range(n)], rn(M, K)
        gs = ops.lora_bwd_dy(dys, us, Bs, dBs, 2.0, [True] * n)
        w16 = n * r * K * 2
        rec(f"mm_lora_down {label} M={M} K={K} r={r}", lambda: ops.lora_down(x, As, dropout=drop),
            M * K * 2 + w16 + n * M * r * 4)
        if n == 3:
            cos = torch.rand(args.seq_len + 16, 64, device=dev)
            rec(f"mm_lora_up q/k + RoPE M={M} N={N} r={r}",
                lambda: ops.lora_up(ys[:2], us[:2], Bs[:2], 2.0, rope=(cos, cos, args.seq_len + 16)),
                2 * (2 * M * N * 2 + N * r * 2 + M * r * 4))
        else:
            rec(f"mm_lora_up {label} M={M} N={N} r={r}", lambda: ops.lora_up(ys, us, Bs, 2.0),
                n * (2 * M * N * 2 + N * r * 2 + M * r * 4))
        nt, mt = (N + 127) // 128, (M + 127) // 128
        rec(f"mm_lora_bwd_dy {label} M={M} N={N} r={r}", lambda: ops.lora_bwd_dy(dys, us, Bs, dBs, 2.0, [True] * n),
            n * (M * N * 2 + 2 * N * r * 2 + N * r * 2 + M * r * 4 + M * r * 4),
            n * 4 * r * (nt * M + mt * N) * 2)
        rec(f"mm_lora_bwd_x {label} M={M} K={K} r={r}",
            lambda: ops.lora_bwd_x(x, gs, As, dAs, dx, [True] * n, dropout=drop),
            M * K * 2 + 2 * M * K * 2 + n * (M * r * 4 + r * K * 2 + 2 * r * K * 2), n * 4 * r * mt * K * 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--micro-batch", type=int, default=4)
    ap.add_argument("--seq-len", type=int, default=512)
    ap.add_argument("--train-layers", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_lora: needs a CUDA device (an H100); nothing is measured without one")
    card = {"gpu": smi("name"), "power_limit_w": smi("power.limit")}
    print(json.dumps(card), flush=True)
    for rnd in range(args.rounds):
        for variant in ("lora", "top8"):
            print(json.dumps(dict(run_step(variant, args), round=rnd)), flush=True)
    for k in kernels(args):
        print(json.dumps(k), flush=True)
    print(json.dumps(dict(card, median_sm_clock_mhz=statistics.median(CLOCKS) if CLOCKS else None,
                          clock_samples=len(CLOCKS))), flush=True)


if __name__ == "__main__":
    main()
