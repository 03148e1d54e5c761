#!/usr/bin/env python
"""FP8 prefill against 16-bit in one process: a 7B model (random weights, bf16 by default) and its twin from the same seed
after quantize_llm_fp8(), alternated over --rounds rounds.

Per round and model: the eval forward of cfg4 (image + audio + text, L = 512 -> T = 528) at B = 4 (the per-GPU batch of
the 8-GPU run) and B = 32, and of cfg2 (image + text, L = 256) at B = 1: ms/step and tokens/s (CUDA events around the
forward, graphs off); then decode ms/step at B = 1, 8, 64, 96 (image + text, L = 256), one batch size at a time, each
from the medians of five alternated generate(new) / generate(1) calls.  Once per model at cfg4 B = 4 and B = 32, with
ops.PROFILE set: the in-step rate of every LLaMA GEMM (2 M N K over its CUDA-event time, mean per projection), the
GEMMs' summed time and that of the FP8 activation quantizations.  Also the peak memory of each
model's warm-up, the norm-wise relative difference of the FP8 logits from the 16-bit logits, and the card, its power limit
and the median SM clock sampled during the timed rounds."""
import argparse
import os
import statistics
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402


def _smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


class Clock:
    """SM clock samples (nvidia-smi, every 0.5 s) while running."""

    def __init__(self):
        self.v, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            s = _smi("clocks.sm")
            if s.isdigit():
                self.v.append(int(s))
            self._stop.wait(0.5)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()


def _inputs(B, L, V, audio):
    host = bench.synth_inputs(B, L, V, 224, 3000, 1234)
    if not audio:
        host["audios"] = None
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}


def _forward_ms(model, inp, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        model(inp)
        e0.record()
        for _ in range(n):
            out = model(inp)
        e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n, out.logits


def _decode_ms(eng, inp, new, reps=5):
    """ms per decode step: (generate(new) - generate(1)) / (new - 1), from the medians of `reps` alternated calls of each
    (one pair alone is at the mercy of the prefill's own variation)."""
    times = {1: [], new: []}
    for _ in range(reps):
        for n in (1, new):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.generate(inp, max_new_tokens=n, eos_token_id=-1)
            torch.cuda.synchronize()
            times[n].append(time.perf_counter() - t0)
    return (statistics.median(times[new]) - statistics.median(times[1])) / (new - 1) * 1e3


def _gemm_rates(model, inp):
    """Mean TFLOP/s of each LLaMA projection GEMM in one forward, from CUDA events around each launch."""
    from macaw_llm_b200 import ops

    ops.PROFILE = []
    try:
        with torch.no_grad():
            model(inp)
        torch.cuda.synchronize()
        rec = [(tag, fl, e0.elapsed_time(e1)) for tag, fl, e0, e1 in ops.PROFILE if tag.startswith("llama")]
    finally:
        ops.PROFILE = None
    gemms = [r for r in rec if r[0] == "llama"]
    names = ("qkv", "o_proj", "gate_up", "down_proj")
    out = {}
    for i, n in enumerate(names):
        r = gemms[i::4]
        out[n] = sum(f for _, f, _ in r) / sum(t for _, _, t in r) / 1e9
    quant = [t for tag, _, t in rec if tag == "llama.quantize"]
    return out, sum(t for _, _, t in gemms), sum(quant), len(quant)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--new", type=int, default=16)
    ap.add_argument("--dtype", choices=("bf16", "fp16"), default="bf16")
    a = ap.parse_args()
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[a.dtype]
    (clip, whisper, llama), hyper = bench.real_configs()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    V = llama.vocab_size
    work = {"cfg4 B=4": _inputs(4, 512, V, True), "cfg4 B=32": _inputs(32, 512, V, True), "cfg2 B=1": _inputs(1, 256, V, False)}
    dec = {B: _inputs(B, 256, V, False) for B in (1, 8, 64, 96)}
    card = f"{torch.cuda.get_device_name()}, power limit {_smi('power.limit') or 'unknown'} W"
    print(f"[bench_fp8] {card}; {dtype}; rounds {a.rounds}, {a.steps} forwards per measurement, decode new={a.new}")
    models = {}
    for name in ("fp8", "16-bit"):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m = MM_LLMs.build_random(cfg, device="cuda", dtype=dtype, seed=0)
        if name == "fp8":
            m.quantize_llm_fp8()
        with torch.no_grad():
            for inp in work.values():
                m(inp)
        torch.cuda.synchronize()
        print(f"[bench_fp8] {name:6s} peak memory above the start (model + cfg4 B=32 forward): "
              f"{(torch.cuda.max_memory_allocated() - base) / 2 ** 30:.2f} GiB")
        models[name] = m
    for wname, inp in work.items():
        la = _forward_ms(models["fp8"], inp, 1)[1].float()
        lb = _forward_ms(models["16-bit"], inp, 1)[1].float()
        print(f"[bench_fp8] {wname}: FP8 logits vs 16-bit, norm-wise relative difference "
              f"{float((la - lb).norm() / lb.norm()):.4f}")
        del la, lb
    for wname in ("cfg4 B=4", "cfg4 B=32"):
        for name, m in models.items():
            rates, t_gemm, t_q, n_q = _gemm_rates(m, work[wname])
            print(f"[bench_fp8] {name:6s} {wname} in-step GEMM rate (2MNK / CUDA-event time): "
                  + ", ".join(f"{k} {v:.0f} TFLOP/s" for k, v in rates.items())
                  + f"; LLaMA GEMMs {t_gemm:.1f} ms" + (f", {n_q} activation quantizations {t_q:.1f} ms" if n_q else ""))
    with Clock() as clk:
        for r in range(a.rounds):
            for wname, inp in work.items():
                B, T = inp["input_ids"].shape[0], None
                res = {}
                for name, m in models.items():
                    ms, lg = _forward_ms(m, inp, a.steps)
                    T = lg.shape[1]
                    res[name] = ms
                    del lg
                print(f"[bench_fp8] round {r} {wname} T={T}: " + "; ".join(
                    f"{n} {ms:.1f} ms/step, {B * T / ms * 1e3:.0f} tokens/s" for n, ms in res.items())
                    + f"; 16-bit / FP8 {res['16-bit'] / res['fp8']:.3f}")
        # one batch size at a time: the KV caches of both models at B = 96 alone take 32 GB
        for B, inp in dec.items():
            for m in models.values():
                m.engine.generate(inp, max_new_tokens=a.new, eos_token_id=-1)
            for r in range(a.rounds):
                res = {name: _decode_ms(m.engine, inp, a.new) for name, m in models.items()}
                print(f"[bench_fp8] round {r} decode B={B}: " + "; ".join(f"{n} {v:.3f} ms/step" for n, v in res.items()))
            for m in models.values():
                m.engine._decode.clear()
            torch.cuda.empty_cache()
    print(f"[bench_fp8] {card}; median SM clock during the rounds {statistics.median(clk.v) if clk.v else 'n/a'} MHz "
          f"({len(clk.v)} samples)")


if __name__ == "__main__":
    main()
