"""The GEMM's epilogue-overlap modes (mm_gemm_overlap_mode) compute the same bits.

Mode 1 (a dedicated epilogue warpgroup runs a tile's epilogue while the consumer warpgroups start the next tile's main
loop) keeps the MMA k-order and the per-element epilogue arithmetic of mode 0, so its outputs must equal mode 0's exactly
(torch.equal), for every epilogue, at the benchmark's batch-32 shapes, at ragged / odd-tile shapes and for the training
step's MN-major operands, in both activation formats, over repeated launches and a CUDA-graph replay.  Each case also
checks, from the launched kernel's name, that mode 1 really ran the epilogue warpgroup and that mm_gemm_plan predicted
the kernel that ran; launches below 32 k-blocks or with a stream-K tail keep the consumer epilogue in every mode."""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
E, I, V, T = 4096, 11008, 32000, 528
M32 = 32 * T  # the benchmark's LLaMA rows at global batch 32


def _ops():
    from macaw_llm_b200 import ops

    return ops


def _lib():
    from macaw_llm_b200 import _lib

    return _lib.load()


def run_mode(fn, mode):
    """Run `fn` in overlap mode `mode` and return cloned outputs."""
    lib = _lib()
    prev = lib.mm_gemm_overlap_mode(mode)
    try:
        out = [t.clone() for t in fn()]
        torch.cuda.synchronize()
    finally:
        lib.mm_gemm_overlap_mode(prev)
    return out


def _case(kind, M, N, K, dt, seed=0):
    """Inputs of one GEMM call and a closure making the call; returns (fn, flops)."""
    ops = _ops()
    ops.set_act_format(dt)
    g = torch.Generator(device=DEV).manual_seed(seed)

    def r(*s, scale=1.0):
        return (torch.randn(*s, device=DEV, generator=g) * scale).to(dt)

    x, w = r(M, K), r(N, K, scale=K ** -0.5)
    ssx = torch.rand(M, E // 32, device=DEV, generator=g) * 32 + 1.0
    if kind == "rope_rms":
        pos = torch.arange(T, device=DEV, dtype=torch.float32)[:, None]
        fr = pos * (1.0 / 10000 ** (torch.arange(0, 128, 2, device=DEV).float() / 128))[None]
        rope = (fr.cos().contiguous(), fr.sin().contiguous(), T, N * 2 // 3)
        return lambda: (ops.linear(x, w, epi=ops.EPI_ROPE, rope=rope, rms_from=(ssx, 1e-6)),)
    if kind == "swiglu_rms":
        return lambda: (ops.linear(x, w, epi=ops.EPI_SWIGLU, rms_from=(ssx, 1e-6)),)
    if kind == "res_sumsq":
        res = r(M, N)
        ss = torch.empty(M, N // 32, device=DEV)
        return lambda: (ops.linear(x, w, residual=res, sumsq_out=ss), ss)
    if kind == "plain_fp32":
        return lambda: (ops.linear(x, w, out_fp32=True),)
    if kind == "bias_gelu":
        b = r(N)
        return lambda: (ops.linear(x, w, b, act=ops.ACT_GELU),)
    if kind == "bias_quick_gelu_res":
        b, res = r(N), r(M, N)
        return lambda: (ops.linear(x, w, b, act=ops.ACT_QUICK_GELU, residual=res),)
    if kind == "row_scale_alpha":
        rs = torch.rand(M, device=DEV, generator=g) + 0.5
        return lambda: (ops.linear(x, w, row_scale=rs, alpha=0.37),)
    if kind == "thin":  # decode step: operands swapped, transposed epilogue
        b, res = r(N), r(M, N)
        return lambda: (ops.linear_thin(x, w, b, act=ops.ACT_GELU, residual=res),)
    if kind == "dx":  # dy (M, K) @ w (K, N): the layer's weight read as stored
        dy, wt = r(M, K), r(K, N, scale=K ** -0.5)
        return lambda: (ops.gemm_dx(dy, wt),)
    if kind == "dw":  # dw (N_out = N, K_in = K) += dy (M, N)^T @ x (M, K), accumulating into an existing gradient
        dy, g0 = r(M, N), r(N, K)
        out = torch.empty_like(g0)

        def dw():
            out.copy_(g0)
            return (ops.gemm_dw(dy, x, out, accumulate=True),)
        return dw
    raise ValueError(kind)


def _launched(fn):
    """The variant (ops.GEMM_*, as in gemm_plan()["kernel"]) of every GEMM kernel `fn` launches, from the profiler's
    kernel names: gemm_wide_kernel, or gemm_bf16_kernel with the EWG template argument (the last one) false / true."""
    from torch.profiler import ProfilerActivity, profile

    ops = _ops()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    variants = set()
    for ev in prof.events():
        if "gemm_wide_kernel<" in ev.name:
            variants.add(ops.GEMM_TILE_PAIRS)
        m = re.search(r"gemm_bf16_kernel<([^>]*)>", ev.name)
        if m:
            ewg = m.group(1).split(",")[-1].strip() == "true"
            variants.add(ops.GEMM_EPILOGUE_WARPGROUP if ewg else ops.GEMM_CONSUMER_EPILOGUE)
    assert variants, "no GEMM kernel launched"
    return variants


def _planned(kind, M, N, K, dt, streamk=False):
    """The variant ops.gemm_plan predicts, under the current modes, for the GEMM call of _case(kind, M, N, K, dt)."""
    ops = _ops()
    kw = dict(M=M, N=N, K=K, fp16=dt == torch.float16, streamk=streamk)
    if kind == "rope_rms":
        kw.update(epi=ops.EPI_ROPE)
    elif kind == "swiglu_rms":
        kw.update(epi=ops.EPI_SWIGLU)
    elif kind == "plain_fp32":
        kw.update(c_fp32=True)
    elif kind == "thin":  # linear_thin swaps the operands
        kw.update(M=N, N=M, c_trans=True)
    elif kind == "dx":
        kw.update(b_mn_major=True)
    elif kind == "dw":  # gemm_dw: dW (N x K) = dy^T x over the M rows
        kw.update(M=N, N=K, K=M, a_mn_major=True, b_mn_major=True)
    return ops.gemm_plan(**kw)["kernel"]


# (kind, M, N, K): the benchmark's batch-32 GEMMs, then odd M-tile counts, ragged edges and the training step's
# input / weight-gradient GEMMs (MN-major operands).  Every case has >= 32 k-blocks and no stream-K tail, so mode 1
# launches the epilogue warpgroup (asserted below).
SHAPES = [
    ("rope_rms", M32, 3 * E, E),              # LLaMA QKV + RoPE
    ("res_sumsq", M32, E, E),                 # o_proj + residual + next RMSNorm statistic
    ("swiglu_rms", M32, 2 * I, E),            # gate/up + SwiGLU
    ("res_sumsq", M32, E, I),                 # down + residual
    ("plain_fp32", M32, V, E),                # lm_head's shape, fp32 out
    ("bias_quick_gelu_res", 32 * 257, 4096, 2048),  # CLIP fc1 rows, M tail
    ("bias_gelu", 32 * 1500, 2048, 2048),     # Whisper fc1 rows
    ("rope_rms", 4 * T, 3 * E, E),            # per-rank batch 4: 17 M tiles
    ("swiglu_rms", 4 * T, 2 * I, E),
    ("res_sumsq", 300, 1024, 2120),           # ragged M, K % 64 != 0
    ("bias_gelu", 300, 1000, 2120),           # N % 32 != 0
    ("row_scale_alpha", 2112, 4096, 4096),
    ("thin", 8, 4096, 4096),                  # swapped operands, transposed epilogue
    ("dx", 4 * T, E, I),                      # training: dx = dy W, MN-major B
    ("dw", 4 * T, E, E),                      # training: dW += dy^T x, MN-major A and B, 33 k-blocks
]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("kind,M,N,K", SHAPES, ids=[f"{s[0]}-{s[1]}x{s[2]}x{s[3]}" for s in SHAPES])
def test_overlap_modes_bit_identical(kind, M, N, K, dt):
    fn = _case(kind, M, N, K, dt, seed=M + N + K)
    want = run_mode(fn, 0)
    got = run_mode(fn, 1)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert all(torch.isfinite(t.float()).all() for t in want)
    ops, lib = _ops(), _lib()
    prev = lib.mm_gemm_overlap_mode(0)
    try:
        assert _launched(fn) == {_planned(kind, M, N, K, dt)} == {ops.GEMM_CONSUMER_EPILOGUE}
        lib.mm_gemm_overlap_mode(1)  # the case really runs the epilogue warpgroup, as planned
        assert _launched(fn) == {_planned(kind, M, N, K, dt)} == {ops.GEMM_EPILOGUE_WARPGROUP}
    finally:
        lib.mm_gemm_overlap_mode(prev)


@pytest.mark.parametrize("kind,M,N,K,streamk", [("bias_gelu", 32 * 1500, 2048, 512, False),   # 8 k-blocks
                                                ("bias_quick_gelu_res", 32 * 257, 4096, 1024, False),  # 16
                                                ("res_sumsq", 31 * T, E, E, True)])          # stream-K tail
def test_short_k_and_streamk_keep_consumer_epilogue(kind, M, N, K, streamk):
    """Launches below 32 k-blocks or with a stream-K tail take the consumer-epilogue kernel in every mode."""
    ops, lib = _ops(), _lib()
    fn = _case(kind, M, N, K, torch.float16)
    prev = lib.mm_gemm_overlap_mode(1)
    prev_sk = lib.mm_gemm_streamk_mode(2) if streamk else None
    ops.STREAMK = ops.streamk_workspace(torch.device(DEV, 0)) if streamk else None
    try:
        if streamk:
            assert ops.gemm_plan(M=M, N=N, K=K, fp16=True, streamk=True)["streamk_tiles"] > 0
        assert _launched(fn) == {_planned(kind, M, N, K, torch.float16, streamk)} == {ops.GEMM_CONSUMER_EPILOGUE}
    finally:
        ops.STREAMK = None
        lib.mm_gemm_overlap_mode(prev)
        if prev_sk is not None:
            lib.mm_gemm_streamk_mode(prev_sk)


def test_overlap_repeat_and_graph_replay():
    """Repeated launches and a CUDA-graph replay of mode 1 reproduce mode 0's eager outputs bit for bit."""
    ops, lib = _ops(), _lib()
    fns = [_case("rope_rms", M32, 3 * E, E, torch.float16, seed=11), _case("res_sumsq", M32, E, I, torch.float16, seed=12)]
    want = [run_mode(f, 0) for f in fns]
    prev = lib.mm_gemm_overlap_mode(1)
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


def test_overlap_mode_setter():
    lib = _lib()
    prev = lib.mm_gemm_overlap_mode(0)
    try:
        assert lib.mm_gemm_overlap_mode(-1) == 0
        assert lib.mm_gemm_overlap_mode(7) == 0  # out of range: ignored
        assert lib.mm_gemm_overlap_mode(1) == 0
        assert lib.mm_gemm_overlap_mode(-1) == 1
    finally:
        lib.mm_gemm_overlap_mode(prev)
