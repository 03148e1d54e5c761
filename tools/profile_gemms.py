#!/usr/bin/env python
"""Run the GEMMs of ONE layer of a model family at BASELINE shapes between cudaProfilerStart/Stop (for ncu).

  ncu --set full --clock-control none --profile-from-start off -o prof_gemms_llama \
      python tools/profile_gemms.py --family llama --batch 32
Families: llama (qkv+RoPE, o_proj+res, gate/up+SwiGLU, down+res at M = batch*528), clip (qkv, out+res, fc1+quick_gelu, fc2+res
at M = batch*257, d=1024), whisper (same four at M = batch*1500, d=512).  Prints CUDA-event TFLOP/s per GEMM (not a bench value
when run under ncu)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--family", default="llama", choices=["llama", "clip", "whisper"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--streamk", type=int, default=0, help="1: hand the GEMMs a stream-K workspace (mm_gemm_args.sk_workspace)")
    a = ap.parse_args()
    from macaw_llm_b200 import ops

    dt = torch.float16 if a.dtype == "fp16" else torch.bfloat16
    ops.set_act_format(dt)
    dev = "cuda"
    if a.streamk:
        ops.STREAMK = ops.streamk_workspace(torch.device("cuda", 0))
    g = torch.Generator(device=dev).manual_seed(0)

    def r(*s, scale=1.0):
        return (torch.randn(*s, device=dev, generator=g) * scale).to(dt)

    if a.family == "llama":
        M, E, I = a.batch * 528, 4096, 11008
        x, wqkv, wo, wgu, wd = r(M, E), r(3 * E, E, scale=0.02), r(E, E, scale=0.02), r(2 * I, E, scale=0.02), r(E, I, scale=0.02)
        fr = torch.arange(528, device=dev, dtype=torch.float32)[:, None] * (1.0 / 10000 ** (torch.arange(0, 128, 2, device=dev).float() / 128))[None]
        rope = (fr.cos().contiguous(), fr.sin().contiguous(), 528, 2 * E)
        rstd = torch.rand(M, device=dev) + 0.5
        att = r(M, E)
        ss = torch.empty(M, E // 32, device=dev, dtype=torch.float32)
        calls = [
            ("qkv+rope", 2.0 * M * 3 * E * E, lambda: ops.linear(x, wqkv, epi=ops.EPI_ROPE, rope=rope, row_scale=rstd)),
            ("o_proj+res", 2.0 * M * E * E, lambda: ops.linear(att, wo, residual=x, out=x, sumsq_out=ss)),
            ("gate_up+swiglu", 2.0 * M * 2 * I * E, lambda: ops.linear(x, wgu, epi=ops.EPI_SWIGLU, rms_from=(ss, 1e-6))),
        ]
        h = r(M, I)
        calls.append(("down+res", 2.0 * M * E * I, lambda: ops.linear(h, wd, residual=x, out=x, sumsq_out=ss)))
    else:
        D, F, T = (1024, 4096, 257) if a.family == "clip" else (512, 2048, 1500)
        act = ops.ACT_QUICK_GELU if a.family == "clip" else ops.ACT_GELU
        M = a.batch * T
        x, wqkv, bqkv, wo, bo = r(M, D), r(3 * D, D, scale=0.03), r(3 * D), r(D, D, scale=0.03), r(D)
        w1, b1, w2, b2 = r(F, D, scale=0.03), r(F), r(D, F, scale=0.03), r(D)
        att, hmid = r(M, D), r(M, F)
        calls = [
            ("qkv", 2.0 * M * 3 * D * D, lambda: ops.linear(x, wqkv, bqkv)),
            ("out+res", 2.0 * M * D * D, lambda: ops.linear(att, wo, bo, residual=x, out=x)),
            ("fc1+act", 2.0 * M * F * D, lambda: ops.linear(x, w1, b1, act=act)),
            ("fc2+res", 2.0 * M * D * F, lambda: ops.linear(hmid, w2, b2, residual=x, out=x)),
        ]
    for _, _, f in calls:
        f()
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    res = []
    for name, fl, f in calls:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            f()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        res.append(f"{name}: {ms * 1e3:.1f} us, {fl / ms / 1e9:.0f} TFLOP/s")
    torch.cuda.cudart().cudaProfilerStop()
    print(f"[profile_gemms {a.family} B={a.batch} {a.dtype}{' streamk' if a.streamk else ''}] " + "; ".join(res))


if __name__ == "__main__":
    main()
