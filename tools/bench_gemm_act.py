#!/usr/bin/env python
"""Time the GEMMs whose epilogue evaluates a sigmoid (SwiGLU, quick-GELU) and one GELU control, with CUDA events.

  python tools/bench_gemm_act.py [--root DIR] [--iters 50] [--out FILE]

--root: the checkout whose macaw_llm_b200 is imported (default: this one), so that two builds of the library can be
timed alternately in separate processes.  Prints one JSON line per GEMM: median and min milliseconds per launch over
five windows of --iters launches, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=50)
ap.add_argument("--tag", default="")
ap.add_argument("--out", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import torch  # noqa: E402

from macaw_llm_b200 import ops  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                       str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
dt = torch.float16
ops.set_act_format(dt)
g = torch.Generator(device="cuda").manual_seed(0)


def r(*s, scale=1.0):
    return (torch.randn(*s, device="cuda", generator=g) * scale).to(dt)


E, I = 4096, 11008
cases = []
for M in (4 * 528, 32 * 528):  # the LLaMA gate/up + SwiGLU at per-GPU batch 4 and 32
    x, w = r(M, E), r(2 * I, E, scale=E ** -0.5)
    ss = torch.rand(M, E // 32, device="cuda", generator=g) * 32 + 1
    out = torch.empty(M, I, device="cuda", dtype=dt)
    cases.append((f"swiglu_{M}x{2 * I}x{E}", 2.0 * M * 2 * I * E,
                  lambda x=x, w=w, ss=ss, out=out: ops.linear(x, w, epi=ops.EPI_SWIGLU, rms_from=(ss, 1e-6), out=out)))
for name, M, N, K, act in (("clip_fc1", 32 * 257, 4096, 1024, ops.ACT_QUICK_GELU),
                           ("whisper_fc1", 32 * 1500, 2048, 512, ops.ACT_GELU)):
    x, w, b = r(M, K), r(N, K, scale=K ** -0.5), r(N)
    out = torch.empty(M, N, device="cuda", dtype=dt)
    cases.append((f"{name}_{M}x{N}x{K}", 2.0 * M * N * K,
                  lambda x=x, w=w, b=b, out=out, act=act: ops.linear(x, w, b, act=act, out=out)))

lines = []
for name, flops, fn in cases:
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / args.iters)
    ms.sort()
    d = dict(tag=args.tag, gemm=name, ms_median=round(ms[2], 4), ms_min=round(ms[0], 4),
             tflops_median=round(flops / ms[2] / 1e9, 1), card=card)
    lines.append(json.dumps(d))
    print(lines[-1], flush=True)
if args.out:
    with open(args.out, "a") as f:
        f.write("\n".join(lines) + "\n")
