"""Per-kernel time of the greedy-decode step (bench.py --mode decode workload: image+text, B=8, LLaMA-7B) from the CUPTI
activity trace (torch.profiler) of graph-replayed steps.  Usage on an H100:

    python tools/profile_decode.py [--new 32] > decode_kernels.txt

Prints one row per kernel: launches per decode step, average duration, total per step, share.  Timings taken under the
profiler are for ATTRIBUTION only (they explain bench.py's ms_per_decode_step, they are not a bench value)."""
import argparse
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32)
    args = ap.parse_args()
    import bench
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    (clip, whisper, llama), hyper = bench.real_configs()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    V, B, L = llama.vocab_size, 8, 256
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device=dev, dtype=torch.bfloat16, seed=0)
    host = bench.synth_inputs(B, L, V, clip.vision_config.image_size, 2 * whisper.max_source_positions, 1234)
    inp = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    inp["audios"] = None
    inp["inference"] = True
    for _ in range(2):
        model.engine.generate(dict(inp), max_new_tokens=args.new, eos_token_id=-1)
    torch.cuda.synchronize()

    def trace(n):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model.engine.generate(dict(inp), max_new_tokens=n, eos_token_id=-1)
            torch.cuda.synchronize()
        acc = collections.defaultdict(lambda: [0, 0.0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                a = acc[ev.name]
                a[0] += 1
                a[1] += ev.device_time  # us
        return acc

    a1, an = trace(1), trace(args.new)
    steps = args.new - 1
    rows = []
    for name, (cnt, us) in an.items():
        c1, u1 = a1.get(name, (0, 0.0))
        dc, du = cnt - c1, us - u1
        if dc > 0:
            rows.append((du / steps, dc / steps, du / dc, name))
    rows.sort(reverse=True)
    total = sum(r[0] for r in rows)
    print(f"decode step = {args.new - 1} replayed steps averaged; kernel time per step {total:.1f} us")
    print(f"{'kernel':70s} {'launch/step':>11s} {'avg us':>9s} {'us/step':>9s} {'share':>6s}")
    for per_step, lps, avg, name in rows:
        print(f"{name[:70]:70s} {lps:11.1f} {avg:9.2f} {per_step:9.1f} {per_step / total:6.1%}")


if __name__ == "__main__":
    main()
