#!/usr/bin/env python
"""Minimal driver for profiler runs (ncu): build the cfg4 model, run `--warm` untimed forwards, then `--steps`
forwards.  Numbers printed under a profiler are never bench values (bench.py is the benchmark of record).

  ncu --metrics gpu__time_duration.sum --clock-control none -k regex:mm:: -c 1200 --csv --log-file launches.csv \
      python tools/profile_forward.py --batch 32 --warm 1 --steps 1
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq-len", type=int, default=512)
    ap.add_argument("--warm", type=int, default=1)
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--layers", type=int, default=0, help="truncate LLaMA depth (profiling convenience only)")
    ap.add_argument("--video-frames", type=int, default=0, help="add a video of F frames per sample and drop the image (BASELINE config 5: F=16)")
    ap.add_argument("--kernels", action="store_true", help="print a per-kernel time table from the CUPTI trace (torch.profiler)")
    a = ap.parse_args()
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config

    (clip, whisper, llama), hyper = bench.real_configs()
    if a.layers:
        llama.num_hidden_layers = a.layers
    if a.video_frames:
        hyper = dict(hyper, n_frames=a.video_frames)
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    model = MM_LLMs.build_random(cfg, device="cuda", dtype=torch.bfloat16, seed=0)
    host = bench.synth_inputs(a.batch, a.seq_len, llama.vocab_size, 224, 3000, 1234)
    if a.video_frames:
        host["images"] = None
        host["videos"] = torch.randn(a.batch, a.video_frames, 3, 224, 224).to(torch.bfloat16)
    dev_in = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host.items()}
    for _ in range(a.warm):
        model(dev_in)
    torch.cuda.synchronize()
    if a.kernels:
        import collections

        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                model(dev_in)
            torch.cuda.synchronize()
        acc = collections.defaultdict(lambda: [0, 0.0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                acc[ev.name][0] += 1
                acc[ev.name][1] += ev.device_time
        tot = sum(v[1] for v in acc.values())
        print(f"[profile_forward --kernels] B={a.batch}: kernel time {tot / a.steps / 1e3:.2f} ms/step")
        for name, (cnt, us) in sorted(acc.items(), key=lambda kv: -kv[1][1])[:16]:
            print(f"{name[:72]:72s} {cnt / a.steps:8.1f} {us / cnt:9.1f} us {us / a.steps / 1e3:8.3f} ms {us / tot:6.1%}")
        return
    torch.cuda.cudart().cudaProfilerStart()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        out = model(dev_in)
    e1.record()
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStop()
    print(f"[profile_forward] {a.steps} step(s), {e0.elapsed_time(e1) / a.steps:.2f} ms/step, logits {tuple(out.logits.shape)}")


if __name__ == "__main__":
    main()
