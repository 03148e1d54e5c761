#!/usr/bin/env python
"""Yardstick for the full-depth fp16 parity numbers (CPU only, no GPU, no kernel library): how far does the REFERENCE
ALGORITHM's own fp16 arithmetic drift from its fp32 evaluation on the benchmarked model?

The oracle (oracle/macaw_oracle.py, a restatement of the reference pinned against the unmodified module) is run twice on
the same fp16-representable random-init weights and inputs of the FULL-DEPTH model (CLIP ViT-L/14 x24, Whisper-base x6,
LLaMA-7B x32, V = 32000): once in fp32, once with every activation and matmul in fp16 (torch CPU half kernels, fp32
accumulation inside a matmul, 16-bit storage between ops — what the reference's `.half()` model does on its GPU).  The
norm-wise difference is the floor any fp16 implementation of this model sits on; the GPU path's measured error
(tests/test_fp16_gpu.py prints it) is read against it.

Lives under tests/ because it drives the oracle (test infrastructure: only tests/, smoke() and bench.py's CPU arm may).
Usage: python tests/golden/fp16_yardstick.py [--configs cfg2,cfg4] [--layers 32] [--dtype fp16|bf16]
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg4")
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"], help="16-bit format of the model and of the low-precision run")
    a = ap.parse_args()
    import bench
    from macaw_llm_b200.modeling import MM_LLMs, MM_LLMs_Config
    from oracle import macaw_oracle as O

    torch.set_num_threads(os.cpu_count())
    (clip, whisper, llama), hyper = bench.real_configs()
    cfg = MM_LLMs_Config(clip_config=clip, whisper_config=whisper, llm_config=llama, **hyper)
    t0 = time.time()
    lp = torch.float16 if a.dtype == "fp16" else torch.bfloat16
    model = MM_LLMs.build_random(cfg, device="cpu", dtype=lp, seed=0)
    sd = {k: v.detach() for k, v in model.state_dict().items() if not k.startswith("video_encoder")}
    hp = O.hp_from_config(cfg)
    hp["llama"]["layers"] = a.layers
    print(f"# model built on the CPU in {time.time() - t0:.0f} s ({a.dtype} random init, seed 0; {os.cpu_count()} threads)", flush=True)
    for config in a.configs.split(","):
        L = 256 if config == "cfg2" else 512
        inp = bench.synth_inputs(1, L, llama.vocab_size, 224, 3000, a.seed, pin=False)
        if config == "cfg2":
            inp["audios"] = None
        # inputs as the fp16 model receives them (llm_trainer.py:366-368 `.half()`), handed to both evaluations
        f = {k: (v.to(lp).float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}
        t1 = time.time()
        with torch.no_grad():
            x32 = O.forward(f, sd, hp, dtype=torch.float32)
            t2 = time.time()
            x16 = O.forward(f, sd, hp, dtype=lp)
        t3 = time.time()
        n_prefix = x32["embeds"].shape[1] - L
        # layout: BOS | per modality: start token row, 6 aligned rows, end token row | text — the aligned rows only
        idx = [1 + 8 * m + 1 + r for m in range(n_prefix // 8) for r in range(6)]
        e_pre = rel(x16["embeds"][:, idx], x32["embeds"][:, idx])
        e_log = rel(x16["logits"], x32["logits"])
        agree = float((x16["logits"].float().argmax(-1) == x32["logits"].argmax(-1)).float().mean())
        what = "cfg2 image+text, B=1, T=264" if config == "cfg2" else "cfg4 sample image+audio+text, B=1, T=528"
        print(f"[reference algorithm, {a.dtype} vs fp32, FULL depth ({a.layers} LLaMA layers), {what}] aligned prefix rows {e_pre:.3e}  "
              f"logits {e_log:.3e}  argmax agreement {agree:.4f}   (fp32 {t2 - t1:.0f} s, {a.dtype} {t3 - t2:.0f} s)", flush=True)


if __name__ == "__main__":
    main()
