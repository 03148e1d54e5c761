"""Device JPEG decode of one training step's media against Pillow on one host core.

The batch is the reference's micro-batch of 4 samples, each with 1 image and 6 pre-extracted video frames: 28 files of
640x480 `gen.synth_image` content written by Pillow at q75 4:2:0, q95 4:2:0 and q95 4:4:4, each without and with restart
markers (one per MCU row).  Per variant, one JSON line:
  device    the three kernels of mm_jpeg_decode by torch.profiler (CUDA activity), and the whole decode (host parse + pack,
            two copies, kernels, status read) by CUDA events / wall clock, median over `--iters` runs
  host      get_self_inputs given the 28 files as bytes (decode + resize / crop / normalise on the device; wall time to a
            synchronise) against Pillow decoding the same 28 files serially on one core, both in this process
Needs Pillow (the baseline) and an H100; prints the card name and power limit first.  Writes nothing but stdout.

  python tools/bench_jpeg.py [--iters 20]
"""
from __future__ import annotations

import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = [("q75_420", dict(quality=75, subsampling=2)), ("q95_420", dict(quality=95, subsampling=2)),
            ("q95_444", dict(quality=95, subsampling=0))]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def files(kw: dict, restart: bool):
    import numpy as np
    from PIL import Image

    from tests.golden import gen

    out = []
    for s in range(28):
        buf = io.BytesIO()
        extra = dict(restart_marker_rows=1) if restart else {}
        Image.fromarray(gen.synth_image(480, 640, seed=100 + s)).save(buf, "JPEG", **kw, **extra)
        out.append(buf.getvalue())
    assert all(np.asarray(Image.open(io.BytesIO(b))).shape == (480, 640, 3) for b in out)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image

    from macaw_llm_b200 import jpeg
    from macaw_llm_b200.inputs import DeviceInputPipeline

    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg: needs a CUDA device")
    print(json.dumps(dict(card(), torch=torch.__version__, pillow=Image.__version__, batch="4 x (1 image + 6 frames)")),
          flush=True)
    pipe = DeviceInputPipeline("cuda", torch.bfloat16, n_frames=6)
    ids = torch.randint(3, 32000, (4, 64))
    batch = dict(input_ids=ids, attention_mask=torch.ones(4, 64, dtype=torch.int64), labels=ids.clone())
    for vname, kw in VARIANTS:
        for restart in (False, True):
            data = files(kw, restart)
            ref = [np.asarray(Image.open(io.BytesIO(b))) for b in data]
            got = pipe.decode_jpegs(data)
            exact = all(np.array_equal(g.cpu().numpy(), r) for g, r in zip(got, ref))
            # host side alone: parse + pack
            t_host = []
            for _ in range(args.iters):
                t0 = time.perf_counter()
                jpeg.pack([jpeg.parse(b) for b in data])
                t_host.append(time.perf_counter() - t0)
            # whole decode: events on the stream, wall clock to the status read
            ev, wall = [], []
            for _ in range(args.iters):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                pipe.decode_jpegs(data)
                e1.record()
                wall.append(time.perf_counter() - t0)
                torch.cuda.synchronize()
                ev.append(e0.elapsed_time(e1))
            # per kernel, in a profiled run of its own
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    pipe.decode_jpegs(data)
                torch.cuda.synchronize()
            stages = {}
            for e in prof.key_averages():
                for k in ("jpeg_entropy_kernel", "jpeg_idct_kernel", "jpeg_color_kernel"):
                    if k in e.key:
                        stages[k] = round(e.device_time_total / max(e.count, 1) / 1e3, 4)
            # the step's input pipeline given bytes, against Pillow decoding serially on this core
            frames = [[data[7 * i + 1 + j] for j in range(6)] for i in range(4)]
            imgs = [data[7 * i] for i in range(4)]
            gsi, pil = [], []
            for _ in range(max(3, args.iters // 4)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pipe.get_self_inputs(batch, imgs, [None] * 4, frames)
                torch.cuda.synchronize()
                gsi.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                for b in data:
                    np.asarray(Image.open(io.BytesIO(b)))
                pil.append(time.perf_counter() - t0)
            med = lambda xs: round(statistics.median(xs) * 1e3, 3)  # noqa: E731
            print(json.dumps(dict(
                variant=vname, restart_markers=restart, files=len(data), mean_file_kb=round(sum(map(len, data)) / 28 / 1024, 1),
                segments=sum(len(jpeg.parse(b).segments) for b in data), bit_exact_vs_pillow=exact,
                device=dict(kernel_ms=stages, decode_events_ms=round(statistics.median(ev), 3), decode_wall_ms=med(wall),
                            host_parse_pack_ms=med(t_host)),
                host=dict(get_self_inputs_bytes_ms=med(gsi), pillow_decode_one_core_ms=med(pil),
                          pillow_ms_per_file=round(statistics.median(pil) * 1e3 / 28, 3)))), flush=True)


if __name__ == "__main__":
    main()
