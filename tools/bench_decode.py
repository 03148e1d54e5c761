#!/usr/bin/env python
"""Decode-path measurement (row 8f-2): image+text prefill then decoding at LLaMA-7B width.
Prints prefill ms and ms per decode step / tokens per second.  Not the benchmark of record (bench.py is).

--sample: greedy and sampled decoding (--temperature / --top-k / --top-p / --repetition-penalty, Vicuna's
generation_config by default) in one process, alternated over three rounds, then mm_sample_rows alone against
mm_argmax_rows (CUDA events, V = 32007) at 1, 8 and 64 rows.  Runs in fp16 unless --dtype says otherwise.

--int8: the 16-bit model and a twin built from the same seed and quantized (quantize_llm_int8), fp16 unless --dtype says
otherwise: peak device memory of each (measured with only that model's working set counted), five alternated rounds of
prefill ms and decode ms/step at B = 1, 8, 64 and two at B = 96, then each decode GEMM with its tail alone (one call per
layer captured in a CUDA graph and replayed between CUDA events, so no host time is counted and, with the weights of all
32 layers in turn, nothing is served from L2): the 16-bit linear_thin_fused against the int8 linear_w8_thin_fused at
M = 1, 8, 64, with the weight bytes each streams per second as a share of 3.35 TB/s.

--kv-int8: the 16-bit KV cache against the int8 one (Engine.enable_int8_kv_cache), bf16 unless --dtype says otherwise.
First the decode attention alone: ops.attention (fa_wgmma_kernel at Tq = 1) over 16-bit caches against
ops.attention_decode_i8 over int8 caches, one call per layer over 32 layers' caches captured in a CUDA graph and replayed
between CUDA events (nothing served from L2), at Tk = 264 of 320 rows for B = 1, 8, 64, 96 and Tk = 2048 of 2112 at B = 8,
with the cache bytes each reads per second as a share of 3.35 TB/s.  Then generate() with 16-bit and with int8 decoder
weights: per weight format, the peak device memory of a B = 64 call with each cache, and three alternated rounds of
prefill ms and decode ms/step at T = 264, B = 1, 8, 64, 96, and at T = 2048, B = 8 (two engines on one model, sharing its
derived weights, so that neither re-captures its decode graph between rounds)."""
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


HBM_BPS = 3.35e12  # H100 SXM data sheet


def _gemm_us(fn, n_layers, replays):
    """Kernel time of fn(i) (a GEMM + tail on layer i's weights) per call: one call per layer captured in a CUDA graph,
    the graph replayed `replays` times between CUDA events (no host launch cost in the window)."""
    for i in range(n_layers):  # warm-up: function attributes, allocator pool
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(n_layers):
            fn(i)
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / (replays * n_layers) * 1e3


def _int8(a, cfg, dtype):
    from macaw_llm_b200 import ops
    from macaw_llm_b200.modeling import MM_LLMs

    llama = cfg.llm_config
    batches = (1, 8, 64)
    inputs = {}
    for B in batches:
        host = bench.synth_inputs(B, a.seq_len, llama.vocab_size, 224, 3000, 1234)
        host["audios"] = None
        inputs[B] = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    print(f"[bench_decode] {_card()}; int8 decoder vs 16-bit, {dtype}, T={a.seq_len + 8}, new={a.new}, B={batches}")
    # the quantized twin first: its peak is measured alone; the 16-bit model's peak is measured above the twin's residency
    models = {}
    qm = MM_LLMs.build_random(cfg, device="cuda", dtype=dtype, seed=0)
    qm.quantize_llm_int8()
    for name, m in (("int8", qm), ("16-bit", None)):
        if m is None:
            m = MM_LLMs.build_random(cfg, device="cuda", dtype=dtype, seed=0)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = 0 if name == "int8" else resident_q
        for B in batches:  # warm-up: weight caches, KV caches and decode graphs of every batch size
            m.engine.generate(inputs[B], max_new_tokens=a.new, eos_token_id=-1)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        if name == "int8":
            resident_q = torch.cuda.memory_allocated()
        models[name] = m
        print(f"[bench_decode] {name:6s} peak memory allocated with B = {batches} warmed up: {peak / 2 ** 30:.2f} GiB")
    for rnd in range(5):
        for B in batches:
            res = {name: _decode_ms(m.engine, inputs[B], a.new) for name, m in models.items()}
            print(f"[bench_decode] round {rnd} B={B:2d}: " + "; ".join(
                f"{n} prefill {p:.1f} ms, decode {s:.3f} ms/step" for n, (p, s) in res.items()))
    # B > 64: no thin decode path; the int8 model dequantizes every layer in every step.  The KV caches of the smaller
    # batches are dropped first to make room.
    big = 96
    host = bench.synth_inputs(big, a.seq_len, llama.vocab_size, 224, 3000, 1234)
    host["audios"] = None
    inp_big = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    for m in models.values():
        m.engine._decode.clear()
    torch.cuda.empty_cache()
    for m in models.values():
        m.engine.generate(inp_big, max_new_tokens=a.new, eos_token_id=-1)
    for rnd in range(2):
        res = {name: _decode_ms(m.engine, inp_big, a.new) for name, m in models.items()}
        print(f"[bench_decode] round {rnd} B={big}: " + "; ".join(
            f"{n} prefill {p:.1f} ms, decode {s:.3f} ms/step" for n, (p, s) in res.items()))
    for m in models.values():
        m.engine._decode.clear()
    del inp_big
    torch.cuda.empty_cache()
    # each decode GEMM with its tail, over the weights of all layers in turn
    m16, eng16, engq = models["16-bit"], models["16-bit"].engine, models["int8"].engine
    eng16.set_format()
    E, I = llama.hidden_size, llama.intermediate_size
    L = len(m16.llm.model.layers)
    w16 = [eng16._llama_weights(i, l, E, I) for i, l in enumerate(m16.llm.model.layers)]
    w8 = [engq._w8_layer(i, l) for i, l in enumerate(models["int8"].llm.model.layers)]
    cos, sin = eng16.rope_tables(64, 128, "cuda")
    for M in batches:
        g = torch.Generator(device="cuda").manual_seed(M)
        x = (torch.randn((M, E), device="cuda", generator=g)).to(dtype)
        h = (torch.randn((M, I), device="cuda", generator=g)).to(dtype)
        rs = torch.ones((M,), device="cuda")
        cache = torch.zeros((M, 64, 2, E), device="cuda", dtype=dtype)
        pos = torch.tensor([3], device="cuda", dtype=torch.int32)
        gemms = (("qkv", 0, x, dict(mode=ops.THIN_QKV, row_scale=rs, rope=(cos, sin, pos), cache=cache, t0_dev=pos)),
                 ("o_proj", 2, x, dict(mode=ops.THIN_RES, residual=x)),
                 ("gate_up", 1, x, dict(mode=ops.THIN_SWIGLU, row_scale=rs)),
                 ("down_proj", 3, h, dict(mode=ops.THIN_RES, residual=x)))
        for name, j, inp, kw in gemms:
            kw = dict(kw)
            mode = kw.pop("mode")
            N, K = w16[0][j].shape
            t16 = _gemm_us(lambda i: ops.linear_thin_fused(inp, w16[i][j], mode, **kw), L, 20)
            t8 = _gemm_us(lambda i: ops.linear_w8_thin_fused(inp, w8[i][j], mode, **kw), L, 20)
            b16, b8 = 2 * N * K, N * K + 4 * N
            print(f"[bench_decode] gemm {name:9s} {N}x{K} M={M:2d}: 16-bit {t16:7.1f} us ({b16 / t16 / 1e6:.2f} TB/s, "
                  f"{b16 / t16 / 1e6 / HBM_BPS * 1e12:.0%}); int8 {t8:7.1f} us ({b8 / t8 / 1e6:.2f} TB/s, "
                  f"{b8 / t8 / 1e6 / HBM_BPS * 1e12:.0%}); {t16 / t8:.2f}x")


def _kv_int8(a, cfg, dtype):
    from macaw_llm_b200 import ops
    from macaw_llm_b200.engine import Engine, KVCacheInt8
    from macaw_llm_b200.modeling import MM_LLMs

    llama = cfg.llm_config
    E, Hh, L = llama.hidden_size, llama.num_attention_heads, llama.num_hidden_layers
    print(f"[bench_decode] {_card()}; 16-bit vs int8 KV cache, {dtype}")
    ops.set_act_format(dtype)
    scale = 128 ** -0.5
    for B, tk, t_max in ((1, 264, 320), (8, 264, 320), (64, 264, 320), (96, 264, 320), (8, 2048, 2112)):
        g = torch.Generator(device="cuda").manual_seed(B + tk)
        q = torch.randn((B, 1, Hh, 128), device="cuda", generator=g).to(dtype)
        c16 = [torch.randn((B, t_max, 2, E), device="cuda", generator=g).to(dtype) for _ in range(L)]
        c8 = KVCacheInt8.allocate(B, t_max, L, E, "cuda")
        qkv = torch.empty((B, 3 * E), device="cuda", dtype=dtype)
        for i in range(L):
            for t in range(0, t_max, 64):  # the int8 caches hold the quantized 16-bit ones
                qkv.view(B, 3, E)[:, 1:] = c16[i][:, t]
                ops.kv_append_i8(qkv, B, 1, c8.layers[i], c8.ks[i], t)
        tk_dev = torch.tensor([tk], device="cuda", dtype=torch.int32)
        kv = [c.unflatten(-1, (Hh, 128)) for c in c16]
        t16 = _gemm_us(lambda i: ops.attention(q, kv[i][:, :, 0], kv[i][:, :, 1], scale=scale, tk_dev=tk_dev), L, 20)
        t8 = _gemm_us(lambda i: ops.attention_decode_i8(q, c8.layers[i], c8.ks[i], scale=scale, tk_dev=tk_dev), L, 20)
        b16, b8 = B * Hh * tk * 2 * 128 * 2, B * Hh * tk * 2 * (128 + 4)
        print(f"[bench_decode] attention B={B:2d} Tk={tk} of {t_max}: 16-bit fa_wgmma {t16:7.1f} us "
              f"({b16 / t16 / 1e6:.2f} TB/s, {b16 / t16 / 1e6 / HBM_BPS * 1e12:.0%}); int8 decode {t8:7.1f} us "
              f"({b8 / t8 / 1e6:.2f} TB/s, {b8 / t8 / 1e6 / HBM_BPS * 1e12:.0%}); {t16 / t8:.2f}x")
        del c16, c8, kv
        torch.cuda.empty_cache()

    def inputs(B, seq_len):
        host = bench.synth_inputs(B, seq_len, llama.vocab_size, 224, 3000, 1234)
        host["audios"] = None
        return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}

    for wname in ("16-bit", "int8"):
        m = MM_LLMs.build_random(cfg, device="cuda", dtype=dtype, seed=0)
        if wname == "int8":
            m.quantize_llm_int8()
        engs = {"16-bit cache": m.engine, "int8 cache": Engine(m)}
        engs["int8 cache"]._cache = m.engine._cache  # the derived weights are the same: keep one copy
        engs["int8 cache"].enable_int8_kv_cache(True)
        inp = inputs(64, a.seq_len)
        for name, eng in engs.items():
            eng.generate(inp, max_new_tokens=a.new, eos_token_id=-1)
            eng._decode.clear()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            eng.generate(inp, max_new_tokens=a.new, eos_token_id=-1)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            print(f"[bench_decode] {wname} weights, {name}: peak memory of a B = 64, T = {a.seq_len + 8}, "
                  f"new = {a.new} call above the resident model: {peak / 2 ** 30:.2f} GiB")
            eng._decode.clear()
        for B, seq_len in ((1, a.seq_len), (8, a.seq_len), (64, a.seq_len), (96, a.seq_len), (8, 2040)):
            inp = inputs(B, seq_len)
            for eng in engs.values():  # warm-up: KV caches and the decode graph of this shape
                eng.generate(inp, max_new_tokens=a.new, eos_token_id=-1)
            for rnd in range(3):
                res = {name: _decode_ms(eng, inp, a.new) for name, eng in engs.items()}
                print(f"[bench_decode] {wname} weights round {rnd} B={B:2d} T={seq_len + 8}: " + "; ".join(
                    f"{n} prefill {p:.1f} ms, decode {st:.3f} ms/step" for n, (p, st) in res.items()))
            for eng in engs.values():
                eng._decode.clear()
            del inp
            torch.cuda.empty_cache()
        del engs, m
        torch.cuda.empty_cache()


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
    ap.add_argument("--int8", action="store_true", help="compare the 16-bit decoder with its int8-quantized twin")
    ap.add_argument("--kv-int8", action="store_true", help="compare the 16-bit KV cache with the int8 one")
    ap.add_argument("--dtype", choices=("bf16", "fp16"), default=None, help="default: fp16 with --sample / --int8, else bf16")
    a = ap.parse_args()
    from macaw_llm_b200 import ops
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}[a.dtype or ("fp16" if a.sample or a.int8 else "bf16")]
    (clip, whisper, llama), hyper = bench.real_configs()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    if a.int8:
        return _int8(a, cfg, dtype)
    if a.kv_int8:
        return _kv_int8(a, cfg, dtype)
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
