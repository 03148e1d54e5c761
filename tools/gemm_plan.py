#!/usr/bin/env python
"""Schedules the GEMM dispatcher picks for the dense GEMMs of the BASELINE configs at every per-GPU batch of the 1/2/4/8-GPU
run (mm_gemm_plan: the host side of mm_gemm_fwd without a launch — no GPU needed, the library assumes the 132 SMs of an H100 SXM).

Explains the strong-scaling curve from the schedule alone: `fill` = share of the scheduled tile slots that carry work
(wave quantisation), next to the padded-row share of the last M tile.
Usage: python tools/gemm_plan.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from macaw_llm_b200 import ops  # noqa: E402

def row(name, M, N, K, **kw):
    p = ops.gemm_plan(M=M, N=N, K=K, **kw)
    pad = 1.0 - M / (p["m_tiles"] * 128.0)
    eff = p["fill"] * (1.0 - pad) if p["streamk_tiles"] == 0 else (1.0 - pad)  # stream-K shares the tail over all CTAs
    flops = 2.0 * M * N * K
    wide = p["kernel"] == ops.GEMM_TILE_PAIRS  # N-neighbouring tile pairs (overlap mode 2, the default)
    return (f"  {name:22s} M={M:6d} N={N:6d} K={K:6d}  BN={p['block_n']:3d} units={p['units']:5d} "
            f"waves={p['waves']:3d} fill={p['fill']:.3f} pad={pad:.3f} group_m={p['group_m']:2d} streamk_tiles={p['streamk_tiles']:3d} "
            f"-> useful share of the scheduled MMA slots {eff:.3f}{'  [128x256 main loop]' if wide else ''}"), flops, eff


def family(title, rows):
    print(title)
    tot = w = 0.0
    for r in rows:
        line, flops, eff = r
        print(line)
        tot += flops
        w += flops / eff
    print(f"  {'FLOP-weighted':22s} {tot / w:.3f}")
    return tot, w


def main():
    E, I, V = 4096, 11008, 32000
    print("# tools/gemm_plan.py — schedules from mm_gemm_plan (host-side dispatch of mm_gemm_fwd, 132 SMs, fp16 operands)")
    print("# fill = units / (waves x workers); pad = padded rows of the last 128-row M tile; stream-K launches count the tail as")
    print("# fully shared.  cfg4: T = 528 positions per sample, 257 CLIP tokens per image, 1500 Whisper frames per clip.")
    for B in (32, 16, 8, 4):
        print(f"\n## cfg4, per-GPU batch {B}  (the {32 // B}-GPU point of the strong-scaling run)")
        M = B * 528
        family(f"LLaMA-7B layer (x32) + lm_head, M = {M}", [
            row("qkv + RoPE", M, 3 * E, E, epi=ops.EPI_ROPE, fp16=True, streamk=True),
            row("o_proj (+res)", M, E, E, fp16=True, streamk=True),
            row("gate-up + SwiGLU", M, 2 * I, E, epi=ops.EPI_SWIGLU, fp16=True, streamk=True),
            row("down_proj (+res)", M, E, I, fp16=True, streamk=True),
        ])
        print(row("lm_head", M, V, E, fp16=True, streamk=True)[0])
        Mc = B * 257
        family(f"CLIP ViT-L/14 layer (x24), M = {Mc}", [
            row("qkv", Mc, 3072, 1024, fp16=True), row("out (+res)", Mc, 1024, 1024, fp16=True),
            row("fc1 + quick_gelu", Mc, 4096, 1024, fp16=True), row("fc2 (+res)", Mc, 1024, 4096, fp16=True),
        ])
        Mw = B * 1500
        family(f"Whisper-base encoder layer (x6), M = {Mw}", [
            row("qkv", Mw, 1536, 512, fp16=True), row("out (+res)", Mw, 512, 512, fp16=True),
            row("fc1 + gelu", Mw, 2048, 512, fp16=True), row("fc2 (+res)", Mw, 512, 2048, fp16=True),
        ])
    print("\n## decode step (B = 8 rows, swapped operands: the weight fills the 128-row MMA tile; split-K of 4 through batch=4)")
    for name, N, K in (("qkv", 3 * E, E), ("o_proj", E, E), ("gate-up", 2 * I, E), ("down_proj", E, I)):
        p = ops.gemm_plan(M=N, N=8, K=K // 4, batch=4, c_fp32=True)
        print(f"  {name:22s} weight rows={N:6d} K/4={K // 4:5d}  BN={p['block_n']:3d} units={p['units']:4d} grid={p['grid']:3d} "
              f"waves={p['waves']} fill={p['fill']:.3f}")


if __name__ == "__main__":
    main()
