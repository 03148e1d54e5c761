"""Overlap mode 2 (two N-neighbouring 128 x 128 tiles under one 128 x 256 main loop, gemm_wide_kernel) computes the bits
of mode 1.

The wide kernel walks the same tiles with the same k-order and runs the same epilogue code per tile, so every output must
equal mode 1's exactly (torch.equal): the decoder's and lm_head's GEMMs at the benchmark's 16896 rows, at 17 M tiles and
at ragged M / N / K, in both activation formats, over repeated launches and a CUDA-graph replay.  Each case checks from
the profiler's kernel names that mode 2 really ran the wide kernel, as mm_gemm_plan predicted; launches that do not
qualify (odd number of N tiles, fewer than 32 k-blocks, a stream-K tail, MN-major operands) must keep the kernel modes
0 / 1 run."""
import pytest
import torch

from tests.test_gemm_overlap_gpu import E, I, M32, T, V, _case, _launched, _lib, _ops, _planned, run_mode

pytestmark = pytest.mark.gpu


WIDE = [
    ("rope_rms", M32, 3 * E, E),          # LLaMA QKV + RoPE + RMSNorm statistic
    ("res_sumsq", M32, E, E),             # o_proj + residual + sumsq_out
    ("swiglu_rms", M32, 2 * I, E),        # gate/up + SwiGLU
    ("res_sumsq", M32, E, I),             # down + residual
    ("plain_fp32", M32, V, E),            # lm_head, fp32 logits
    ("row_scale_alpha", M32, V, E),       # lm_head's shape, 16-bit out
    ("rope_rms", 4 * T, 3 * E, E),        # 17 M tiles: the last wave of pairs is partial
    ("swiglu_rms", 4 * T, 2 * I, E),
    ("res_sumsq", 4000, E, E),            # ragged M
    ("bias_gelu", 4000, 4000, 2120),      # ragged M, N (32 tiles, the last one partial) and K
]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("kind,M,N,K", WIDE, ids=[f"{s[0]}-{s[1]}x{s[2]}x{s[3]}" for s in WIDE])
def test_wide_bit_identical_to_mode_1(kind, M, N, K, dt):
    fn = _case(kind, M, N, K, dt, seed=M + N + K)
    want = run_mode(fn, 1)
    got = run_mode(fn, 2)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert all(torch.isfinite(t.float()).all() for t in want)
    ops, lib = _ops(), _lib()
    prev = lib.mm_gemm_overlap_mode(2)
    try:
        assert _launched(fn) == {_planned(kind, M, N, K, dt)} == {ops.GEMM_TILE_PAIRS}
        lib.mm_gemm_overlap_mode(1)
        assert _launched(fn) == {_planned(kind, M, N, K, dt)} == {ops.GEMM_EPILOGUE_WARPGROUP}
    finally:
        lib.mm_gemm_overlap_mode(prev)


@pytest.mark.parametrize("kind,M,N,K,streamk", [("bias_gelu", M32, E + 128, 2048, False),        # 33 N tiles
                                                ("bias_quick_gelu_res", M32, E, 1024, False),    # 16 k-blocks
                                                ("res_sumsq", 31 * T, E, E, True),               # stream-K tail
                                                ("res_sumsq", 100, E, E, False),                 # less than a wave of pairs
                                                ("dx", 4 * T, E, I, False)])                     # MN-major B
def test_unqualified_launches_keep_the_narrow_kernel(kind, M, N, K, streamk):
    ops, lib = _ops(), _lib()
    fn = _case(kind, M, N, K, torch.float16)
    want = run_mode(fn, 1) if not streamk else None
    prev = lib.mm_gemm_overlap_mode(2)
    prev_sk = lib.mm_gemm_streamk_mode(2) if streamk else None
    ops.STREAMK = ops.streamk_workspace(torch.device("cuda", 0)) if streamk else None
    try:
        if streamk:
            assert ops.gemm_plan(M=M, N=N, K=K, fp16=True, streamk=True)["streamk_tiles"] > 0
        launched = _launched(fn)
        assert launched == {_planned(kind, M, N, K, torch.float16, streamk)} and ops.GEMM_TILE_PAIRS not in launched
        if want is not None:
            for a, b in zip(fn(), want):
                assert torch.equal(a, b)
    finally:
        ops.STREAMK = None
        lib.mm_gemm_overlap_mode(prev)
        if prev_sk is not None:
            lib.mm_gemm_streamk_mode(prev_sk)


def test_wide_repeat_and_graph_replay():
    """Repeated launches and a CUDA-graph replay of mode 2 reproduce mode 1's eager outputs bit for bit."""
    lib = _lib()
    fns = [_case("rope_rms", M32, 3 * E, E, torch.float16, seed=21), _case("res_sumsq", M32, E, I, torch.float16, seed=22)]
    want = [run_mode(f, 1) for f in fns]
    prev = lib.mm_gemm_overlap_mode(2)
    try:
        for _ in range(3):
            for f, w in zip(fns, want):
                for a, b in zip(f(), w):
                    assert torch.equal(a, b)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for f in fns:  # warm-up on the capture stream
                f()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        outs = []
        with torch.cuda.graph(graph):
            for f in fns:
                outs.append(f())
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            for o, w in zip(outs, want):
                for a, b in zip(o, w):
                    assert torch.equal(a, b)
    finally:
        lib.mm_gemm_overlap_mode(prev)


def test_mode_2_is_the_default_and_settable():
    import os

    lib = _lib()
    prev = lib.mm_gemm_overlap_mode(-1)
    if "MACAW_B200_GEMM_OVERLAP" not in os.environ:
        assert prev == 2
    try:
        assert lib.mm_gemm_overlap_mode(2) == prev
        assert lib.mm_gemm_overlap_mode(3) == 2  # out of range: ignored
        assert lib.mm_gemm_overlap_mode(-1) == 2
    finally:
        lib.mm_gemm_overlap_mode(prev)
