"""Backward of one LLaMA attention layer at the training bench's shape (B=4, H=32, T=528, hd=128, causal + key mask) between
cudaProfilerStart/Stop, with CUDA-event timing of the whole op and of the softmax-backward kernel alone.

    ncu --set full --clock-control none --profile-from-start off -k regex:softmax_bwd -c 1 -o prof_softmax_bwd \
        python tools/profile_attn_bwd.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from macaw_llm_b200 import _lib, ops

    ops.set_act_format(torch.bfloat16)
    dev = "cuda"
    B, H, T, hd = 4, 32, 528, 128
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v, do = ((torch.randn(B, T, H, hd, device=dev, generator=g) * 0.5).to(torch.bfloat16) for _ in range(4))
    km = torch.ones(B, T, device=dev, dtype=torch.int32)

    def run():
        return ops.attention_bwd(q, k, v, do, scale=hd ** -0.5, causal=True, key_mask=km)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    Tp = (T + 7) // 8 * 8
    S = torch.randn(B, H, T, Tp, device=dev)
    dP = torch.randn(B, H, T, Tp, device=dev)
    P = torch.empty(B, H, T, Tp, device=dev, dtype=torch.bfloat16)
    dS = torch.empty_like(P)

    def soft():
        ops._check(_lib.load().mm_attn_softmax_bwd(S.data_ptr(), dP.data_ptr(), P.data_ptr(), dS.data_ptr(), B, H, T, T, Tp,
                                                   hd ** -0.5, 1, km.data_ptr(), 0.0, None, 0, ops._stream()), "softmax_bwd")

    soft()
    torch.cuda.synchronize()
    torch.cuda.cudart().cudaProfilerStart()
    for name, f, n in (("attention_bwd (7 launches)", run, 10), ("softmax_bwd kernel", soft, 20)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            f()
        e1.record()
        torch.cuda.synchronize()
        print(f"[profile_attn_bwd] {name}: {e0.elapsed_time(e1) / n * 1e3:.1f} us")
    torch.cuda.cudart().cudaProfilerStop()
    byts = S.numel() * 4 * 2 + P.numel() * 2 * 2
    print(f"[profile_attn_bwd] softmax_bwd algorithmic bytes {byts / 1e6:.0f} MB")


if __name__ == "__main__":
    main()
