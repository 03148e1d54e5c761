#!/usr/bin/env python
"""Decode-path measurement (row 8f-2): image+text prefill then decoding at LLaMA-7B width.
Prints prefill ms and ms per decode step / tokens per second.  Not the benchmark of record (bench.py is).

--sample: greedy and sampled decoding (--temperature / --top-k / --top-p / --repetition-penalty, Vicuna's
generation_config by default) in one process, alternated over three rounds, then mm_sample_rows alone against
mm_argmax_rows (CUDA events, V = 32007) at 1, 8 and 64 rows.  Runs in fp16 unless --dtype says otherwise."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402


def _card() -> str:
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return f"{torch.cuda.get_device_name()}, power limit {pl or 'unknown'}"


def _decode_ms(eng, dev_in, new, **kw):
    """(prefill ms, ms per decode step) from a prefill-only call and a call with `new` tokens."""
    times = {}
    for n in (1, new):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        toks = eng.generate(dev_in, max_new_tokens=n, eos_token_id=-1, **kw)  # eos -1: never stop early
        torch.cuda.synchronize()
        times[n] = time.perf_counter() - t0
        assert toks.shape[1] == n
    return times[1] * 1e3, (times[new] - times[1]) / (new - 1) * 1e3


def _kernel_us(ops, rows, V, launches, cfg):
    g = torch.Generator(device="cuda").manual_seed(rows)
    logits = (torch.randn((rows, V), device="cuda", generator=g) * 3.0).to(ops.ACT())
    seen = torch.zeros((rows, (V + 31) // 32), device="cuda", dtype=torch.int32)
    seed = torch.tensor([12345], device="cuda", dtype=torch.int64)
    step = torch.zeros((1,), device="cuda", dtype=torch.int32)
    out = {}
    for name, fn in (("argmax_rows", lambda: ops.argmax_rows(logits)),
                     ("sample_rows", lambda: ops.sample_rows(logits, seen, seed_dev=seed, step_dev=step, **cfg))):
        for _ in range(20):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        e1.synchronize()
        out[name] = e0.elapsed_time(e1) / launches * 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seq-len", type=int, default=256)
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--sample", action="store_true", help="compare greedy and sampled decoding, and time the sampler")
    ap.add_argument("--temperature", type=float, default=0.9)
    ap.add_argument("--top-k", type=int, default=50)
    ap.add_argument("--top-p", type=float, default=0.6)
    ap.add_argument("--repetition-penalty", type=float, default=1.0)
    ap.add_argument("--dtype", choices=("bf16", "fp16"), default=None, help="default: fp16 with --sample, else bf16")
    a = ap.parse_args()
    from macaw_llm_b200 import ops
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[a.dtype or ("fp16" if a.sample else "bf16")]
    (clip, whisper, llama), hyper = bench.real_configs()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device="cuda", dtype=dtype, seed=0)
    host = bench.synth_inputs(a.batch, a.seq_len, llama.vocab_size, 224, 3000, 1234)
    host["audios"] = None
    dev_in = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    eng = model.engine
    if a.sample:
        scfg = dict(do_sample=True, temperature=a.temperature, top_k=a.top_k, top_p=a.top_p,
                    repetition_penalty=a.repetition_penalty)
        print(f"[bench_decode] {_card()}; B={a.batch} T={a.seq_len + 8} new={a.new} {dtype}; sampling {scfg}")
        for kw in ({}, dict(scfg, seed=1)):  # warm-up: weight caches, both decode graphs
            eng.generate(dev_in, max_new_tokens=a.new, eos_token_id=-1, **kw)
        for rnd in range(3):
            for name, kw in (("greedy", {}), ("sampled", dict(scfg, seed=rnd))):
                pre, step = _decode_ms(eng, dev_in, a.new, **kw)
                print(f"[bench_decode] round {rnd} {name:7s}: prefill {pre:.1f} ms, decode {step:.3f} ms/step")
        for rows in (1, 8, 64):
            us = _kernel_us(ops, rows, 32007, 2000, scfg)
            print(f"[bench_decode] kernel rows={rows} V=32007 (2000 launches): argmax_rows {us['argmax_rows']:.1f} us, "
                  f"sample_rows {us['sample_rows']:.1f} us")
        return
    for n in (2, a.new, 1, a.new):  # warm-up, then: prefill + (new-1) steps, prefill only, again
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        toks = eng.generate(dev_in, max_new_tokens=n, eos_token_id=-1)  # eos -1: never stop early (random weights)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        print(f"[bench_decode] B={a.batch} new={n}: {dt * 1e3:.1f} ms, out {tuple(toks.shape)}")
        if n == 1:
            t_prefill = dt
        last = dt
    per_step = (last - t_prefill) / (a.new - 1)
    print(f"[bench_decode] prefill {t_prefill * 1e3:.1f} ms (T={a.seq_len + 8}); decode {per_step * 1e3:.2f} ms/step -> "
          f"{a.batch / per_step:.0f} tokens/s at B={a.batch} (weight streaming floor 13.5 GB / 6.57 TB/s = 2.05 ms)")


if __name__ == "__main__":
    main()
