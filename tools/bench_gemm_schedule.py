#!/usr/bin/env python
"""Time the GEMM kernel per epilogue-overlap mode (`mm_gemm_overlap_mode`) in one process, with CUDA events.

  python tools/bench_gemm_schedule.py [--modes 0,1] [--rounds 3] [--iters 20] [--dtype fp16] [--out FILE]

Modes: 0 consumer epilogue, 1 epilogue warpgroup, 2 epilogue warpgroup + the 128 x 256 main loop for launches whose N
tiles pair up (the LLaMA and lm_head rows, CLIP / Whisper fc2, the K sweep from K = 2048); e.g. `--modes 1,2`.

Two tables; every measurement is repeated once per mode for `--rounds` rounds, and per GEMM the modes alternate within
each round, in swapped order every other round (median and min..max reported):
  K sweep   M = 16896, N = 4096, the o_proj epilogue (residual + sumsq_out), K in {512 .. 8192}.  Time per tile of one CTA
            is fitted as a + b * k_blocks: `a` is the per-tile overhead (epilogue, pipeline fill), `b` the main-loop cost
            per 64-deep k-block (512 tensor-core cycles at the ideal rate).  Both are reported in cycles at the median
            SM clock nvidia-smi sampled during the run.
  bench     the GEMMs of the benchmark's forward at global batch 32, called as Engine calls them: LLaMA QKV + RoPE,
            o_proj + residual, gate/up + SwiGLU, down + residual (RMSNorm statistics through rms_from / sumsq_out, stream-K
            workspace set), lm_head, CLIP's and Whisper's four layer GEMMs, and one LLaMA launch with a stream-K tail.
Every mode's outputs are compared with the first mode's, bit for bit, at the timed sizes.  Card name, power limit and
the sampled SM clocks are printed beside the numbers.  Residual GEMMs write a separate output tensor (same traffic as the
in-place call) so that repeated launches see the same inputs."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


class Clocks:
    """nvidia-smi samples of the SM clock and board power while the measurements run."""

    def __init__(self):
        self.rows, self.proc, self.thread = [], None, None

    def __enter__(self):
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits",
                                      "-i", str(torch.cuda.current_device()), "-lms", "200"],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)

        def pump():
            for line in self.proc.stdout:
                try:
                    mhz, w = (float(v) for v in line.split(","))
                    self.rows.append((mhz, w))
                except ValueError:
                    pass

        self.thread = threading.Thread(target=pump, daemon=True)
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.proc.terminate()
        self.proc.wait(timeout=10)
        self.thread.join(timeout=10)

    def summary(self):
        busy = [r for r in self.rows if r[1] > 150.0] or self.rows  # samples under load
        if not busy:
            return {"sm_mhz_median": None}
        mhz = sorted(r[0] for r in busy)
        return {"sm_mhz_median": statistics.median(mhz), "sm_mhz_min": mhz[0], "sm_mhz_max": mhz[-1],
                "power_w_median": statistics.median(r[1] for r in busy), "samples": len(busy)}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="0,1", help="comma-separated overlap modes out of 0, 1, 2")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--dtype", default="fp16", choices=["bf16", "fp16"])
    ap.add_argument("--out", default=None, help="also append the result lines to this file")
    a = ap.parse_args()
    from macaw_llm_b200 import _lib, ops

    modes = [int(m) for m in a.modes.split(",")]
    assert modes and all(m in (0, 1, 2) for m in modes), "--modes takes overlap modes 0, 1 and 2"
    lib = _lib.load()
    dt = torch.float16 if a.dtype == "fp16" else torch.bfloat16
    ops.set_act_format(dt)
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    g = torch.Generator(device=dev).manual_seed(0)
    sk_ws = ops.streamk_workspace(dev)
    lines = []

    def emit(obj):
        s = json.dumps(obj)
        print(s, flush=True)
        lines.append(s)

    def r(*s, scale=1.0):
        return (torch.randn(*s, device=dev, generator=g) * scale).to(dt)

    def ss_parts(M, E):  # plausible per-(row, 32-column) sums of squares of a residual stream
        return torch.rand(M, E // 32, device=dev, generator=g) * 32 + 1.0

    cases = []  # (table, name, flops, tiles_per_cta, k_blocks, streamk, fn -> output tensors)

    def case(table, name, M, N, K, fn, streamk=False, kb=None):
        plan = ops.gemm_plan(M=M, N=N, K=K, fp16=dt == torch.float16, streamk=streamk)
        cases.append(dict(table=table, name=name, flops=2.0 * M * N * K, plan=plan, streamk=streamk, fn=fn))

    # ---- K sweep: o_proj epilogue at M = 16896, N = 4096
    M, N = 32 * 528, 4096
    res = r(M, N)
    for K in (512, 1024, 2048, 4096, 8192):
        x, w = r(M, K), r(N, K, scale=K ** -0.5)
        out, ss = torch.empty(M, N, device=dev, dtype=dt), torch.empty(M, N // 32, device=dev)
        case("ksweep", f"K={K}", M, N, K,
             lambda x=x, w=w, out=out, ss=ss: (ops.linear(x, w, residual=res, out=out, sumsq_out=ss), ss), streamk=True)

    # ---- the bench's GEMMs at global batch 32
    E, I, V, T = 4096, 11008, 32000, 528
    M = 32 * T
    x, wqkv, wo, wgu, wd, wl = (r(M, E), r(3 * E, E, scale=0.02), r(E, E, scale=0.02), r(2 * I, E, scale=0.02),
                                r(E, I, scale=0.02), r(V, E, scale=0.02))
    fr = torch.arange(T, device=dev, dtype=torch.float32)[:, None] * (
        1.0 / 10000 ** (torch.arange(0, 128, 2, device=dev).float() / 128))[None]
    rope = (fr.cos().contiguous(), fr.sin().contiguous(), T, 2 * E)
    ssx = ss_parts(M, E)
    att, h = r(M, E), r(M, I)
    o_qkv, o_o, o_gu, o_d = (torch.empty(M, 3 * E, device=dev, dtype=dt), torch.empty(M, E, device=dev, dtype=dt),
                             torch.empty(M, I, device=dev, dtype=dt), torch.empty(M, E, device=dev, dtype=dt))
    o_l = torch.empty(M, V, device=dev, dtype=dt)
    ss1, ss2 = torch.empty(M, E // 32, device=dev), torch.empty(M, E // 32, device=dev)
    case("bench", "llama qkv+rope", M, 3 * E, E,
         lambda: (ops.linear(x, wqkv, epi=ops.EPI_ROPE, rope=rope, rms_from=(ssx, 1e-6), out=o_qkv),), streamk=True)
    case("bench", "llama o_proj+res", M, E, E,
         lambda: (ops.linear(att, wo, residual=x, out=o_o, sumsq_out=ss1), ss1), streamk=True)
    case("bench", "llama gate_up+swiglu", M, 2 * I, E,
         lambda: (ops.linear(x, wgu, epi=ops.EPI_SWIGLU, rms_from=(ssx, 1e-6), out=o_gu),), streamk=True)
    case("bench", "llama down+res", M, E, I,
         lambda: (ops.linear(h, wd, residual=x, out=o_d, sumsq_out=ss2), ss2), streamk=True)
    case("bench", "lm_head", M, V, E, lambda: (ops.linear(x, wl, rms_from=(ssx, 1e-6), out=o_l),), streamk=True)
    Ms = 31 * T  # 128 M tiles x 32 N tiles = 4096 tiles: a partial last wave, split by the stream-K tail
    o_s, ss3 = torch.empty(Ms, E, device=dev, dtype=dt), torch.empty(Ms, E // 32, device=dev)
    case("bench", "llama o_proj+res B=31 (stream-K)", Ms, E, E,
         lambda: (ops.linear(att[:Ms], wo, residual=x[:Ms], out=o_s, sumsq_out=ss3), ss3), streamk=True)
    for fam, (D, F, Tf, act) in (("clip", (1024, 4096, 257, ops.ACT_QUICK_GELU)), ("whisper", (512, 2048, 1500, ops.ACT_GELU))):
        Mf = 32 * Tf
        xf, wq, bq, wo_, bo = r(Mf, D), r(3 * D, D, scale=0.03), r(3 * D), r(D, D, scale=0.03), r(D)
        w1, b1, w2, b2 = r(F, D, scale=0.03), r(F), r(D, F, scale=0.03), r(D)
        af, hf = r(Mf, D), r(Mf, F)
        oq, oo, o1, o2 = (torch.empty(Mf, 3 * D, device=dev, dtype=dt), torch.empty(Mf, D, device=dev, dtype=dt),
                          torch.empty(Mf, F, device=dev, dtype=dt), torch.empty(Mf, D, device=dev, dtype=dt))
        case("bench", f"{fam} qkv", Mf, 3 * D, D, lambda xf=xf, wq=wq, bq=bq, oq=oq: (ops.linear(xf, wq, bq, out=oq),))
        case("bench", f"{fam} out+res", Mf, D, D,
             lambda af=af, wo_=wo_, bo=bo, xf=xf, oo=oo: (ops.linear(af, wo_, bo, residual=xf, out=oo),))
        case("bench", f"{fam} fc1+act", Mf, F, D,
             lambda xf=xf, w1=w1, b1=b1, o1=o1, act=act: (ops.linear(xf, w1, b1, act=act, out=o1),))
        case("bench", f"{fam} fc2+res", Mf, D, F,
             lambda hf=hf, w2=w2, b2=b2, xf=xf, o2=o2: (ops.linear(hf, w2, b2, residual=xf, out=o2),))

    def run(c):
        ops.STREAMK = sk_ws if c["streamk"] else None
        try:
            return c["fn"]()
        finally:
            ops.STREAMK = None

    prev_mode = lib.mm_gemm_overlap_mode(-1)
    emit({"card": card(), "library_source_hash": lib.mm_build_hash().decode(), "dtype": a.dtype, "modes": modes, "rounds": a.rounds, "iters": a.iters, "sms": sms})
    try:
        # outputs: every mode against the first, bit for bit
        ref = {}
        for m in modes:
            lib.mm_gemm_overlap_mode(m)
            for c in cases:
                got = [t.clone() for t in run(c)]
                if m == modes[0]:
                    ref[c["name"]] = got
                else:
                    same = all(torch.equal(u, v) for u, v in zip(ref[c["name"]], got))
                    c.setdefault("identical", {})[m] = same
        torch.cuda.synchronize()
        ref.clear()
        times = {(c["name"], m): [] for c in cases for m in modes}
        with Clocks() as clk:
            for m in modes:  # warm-up of every shape and mode
                lib.mm_gemm_overlap_mode(m)
                for c in cases:
                    for _ in range(3):
                        run(c)
            torch.cuda.synchronize()
            # per case, the modes alternate within each round and swap order every round: both see the same
            # predecessor work and the same share of the card's power-limited clock
            for c in cases:
                for rnd in range(a.rounds):
                    for m in (modes if rnd % 2 == 0 else modes[::-1]):
                        lib.mm_gemm_overlap_mode(m)
                        run(c)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.iters):
                            run(c)
                        e1.record()
                        torch.cuda.synchronize()
                        times[(c["name"], m)].append(e0.elapsed_time(e1) / a.iters)
        clocks = clk.summary()
    finally:
        lib.mm_gemm_overlap_mode(prev_mode)
    mhz = clocks.get("sm_mhz_median")
    emit({"clocks": clocks})
    for c in cases:
        p = c["plan"]
        row = {"table": c["table"], "gemm": c["name"], "block_n": p["block_n"], "tiles": p["units"], "grid": p["grid"],
               "k_blocks": p["k_blocks"], "streamk_tiles": p["streamk_tiles"]}
        for m in modes:
            ms = times[(c["name"], m)]
            tf = [c["flops"] / (t * 1e-3) / 1e12 for t in ms]
            row[f"mode{m}"] = {"ms_median": round(statistics.median(ms), 4), "ms_min": round(min(ms), 4),
                               "ms_max": round(max(ms), 4), "tflops_median": round(statistics.median(tf), 1),
                               "tflops_min": round(min(tf), 1), "tflops_max": round(max(tf), 1)}
        if "identical" in c:
            row["bit_identical_to_mode%d" % modes[0]] = c["identical"]
        c["row"] = row
        emit(row)
    # K sweep fit: time per tile of one CTA = a + b * k_blocks (least squares over the sweep), in SM cycles
    sweep = [c for c in cases if c["table"] == "ksweep"]
    for m in modes:
        xs = [c["plan"]["k_blocks"] for c in sweep]
        ys = []
        for c in sweep:
            per_cta = c["plan"]["units"] / c["plan"]["grid"]
            ys.append(statistics.median(times[(c["name"], m)]) * 1e-3 / per_cta)  # seconds per tile
        n = len(xs)
        mx, my = sum(xs) / n, sum(ys) / n
        b = sum((u - mx) * (v - my) for u, v in zip(xs, ys)) / sum((u - mx) ** 2 for u in xs)
        a0 = my - b * mx
        fit = {"fit": f"mode{m}", "a_us": round(a0 * 1e6, 3), "b_us_per_kblock": round(b * 1e6, 4)}
        if mhz:
            fit.update(a_cycles=round(a0 * mhz * 1e6), b_cycles_per_kblock=round(b * mhz * 1e6, 1),
                       b_ideal_cycles=512, at_sm_mhz=mhz)
        emit(fit)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
