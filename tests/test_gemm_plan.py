"""CPU tier: the host side of mm_gemm_fwd (tile width from the cost model, rasterisation group, stream-K tail, kernel
variant and launch shape, argument checks) through mm_gemm_plan — the same dispatcher run without a launch.  No GPU
involved: the library assumes the 132 SMs of an H100 SXM when no device is visible.  The decisions asserted here are the ones DESIGN.md §3 / §6 document."""
import ctypes as C
import random

import pytest

from macaw_llm_b200 import _lib, ops

E, I, V = 4096, 11008, 32000
SMS = 132
CONSUMER, EWG, PAIRS = ops.GEMM_CONSUMER_EPILOGUE, ops.GEMM_EPILOGUE_WARPGROUP, ops.GEMM_TILE_PAIRS
SMEM_128, SMEM_64, SMEM_PAIRS = 199936, 183552, 216320  # 4 stages of 128 x 128, 6 of 128 x 64, 3 of 128 x 256


def plan(**kw):
    return ops.gemm_plan(**kw)


def test_llama_gemms_at_batch_32_use_full_width_tiles():
    M = 32 * 528  # 132 M tiles: every N column of tiles is exactly one wave
    for N, K, epi in ((3 * E, E, ops.EPI_ROPE), (E, E, ops.EPI_STD), (2 * I, E, ops.EPI_SWIGLU), (E, I, ops.EPI_STD),
                      (V, E, ops.EPI_STD)):
        p = plan(M=M, N=N, K=K, epi=epi, fp16=True, streamk=True)
        assert (p["block_n"], p["grid"], p["workers"]) == (128, SMS, SMS), (N, K, p)
        assert (p["kernel"], p["threads"], p["smem_bytes"]) == (PAIRS, 384, SMEM_PAIRS), (N, K, p)
        assert p["units"] == (M // 128) * ((N + 127) // 128) and p["waves"] == (N + 127) // 128 and p["streamk_tiles"] == 0
        assert p["smem_bytes"] <= 227 * 1024 and p["vectorised_epilogue"] == 1
    # rasterisation group ~ 16 MiB of A rows: 16 M tiles at K = 4096, 6 at K = 11008
    assert plan(M=M, N=E, K=E)["group_m"] == 16 and plan(M=M, N=E, K=I)["group_m"] == 6


def test_short_k_gemms_stay_single_cta():
    # CLIP / Whisper layers (K = 1024 / 512)
    for M, N, K in ((8224, 3072, 1024), (8224, 4096, 1024), (48000, 1536, 512), (48000, 2048, 512)):
        p = plan(M=M, N=N, K=K, fp16=True)
        assert p["workers"] == SMS and p["grid"] == SMS and p["block_n"] == 128, p
        assert (p["kernel"], p["threads"], p["smem_bytes"]) == (CONSUMER, 288, SMEM_128), p  # < 32 k-blocks
    p = plan(M=8224, N=1024, K=4096, fp16=True)  # fc2: 65 x 8 = 520 tiles of 128 x 128 fill 4 waves (528 slots)
    assert (p["block_n"], p["units"], p["waves"]) == (128, 520, 4)
    assert (p["kernel"], p["grid"]) == (PAIRS, SMS)  # 260 pairs


def test_per_gpu_batch_of_the_8_gpu_run():
    """M = 2112 = 17 M tiles: the tile width that needs the fewest cost-weighted waves, stream-K where the tail pays."""
    M = 4 * 528
    qkv = plan(M=M, N=3 * E, K=E, epi=ops.EPI_ROPE, fp16=True, streamk=True)
    assert (qkv["block_n"], qkv["units"], qkv["waves"], qkv["streamk_tiles"]) == (128, 17 * 96, 13, 0)  # 48-tile tail: too small a saving
    assert (qkv["kernel"], qkv["grid"]) == (PAIRS, SMS)  # 816 pairs
    gu = plan(M=M, N=2 * I, K=E, epi=ops.EPI_SWIGLU, fp16=True, streamk=True)
    assert (gu["units"], gu["waves"], gu["streamk_tiles"], gu["grid"]) == (17 * 172, 23, (17 * 172) % SMS, SMS)
    assert (gu["kernel"], gu["threads"], gu["smem_bytes"]) == (CONSUMER, 288, SMEM_128)  # the tail takes the consumer epilogue
    o = plan(M=M, N=E, K=E, fp16=True, streamk=True)  # 64-wide tiles: 9 waves of 128 x 64 beat 5 of 128 x 128
    assert (o["block_n"], o["units"], o["waves"]) == (64, 17 * 64, 9)
    assert (o["kernel"], o["threads"], o["grid"], o["smem_bytes"]) == (EWG, 512, SMS, SMEM_64)
    head = plan(M=M, N=V, K=E, fp16=True, streamk=True)
    assert (head["block_n"], head["units"], head["waves"], head["grid"]) == (128, 17 * 250, 33, SMS)
    assert (head["streamk_tiles"], head["kernel"]) == (0, PAIRS)
    assert plan(M=M, N=2 * I, K=E, epi=ops.EPI_SWIGLU, fp16=True, streamk=False)["streamk_tiles"] == 0  # opt-in per launch


def test_policy_switches():
    lib = _lib.load()
    for mode, want in ((0, (CONSUMER, 288, SMEM_128)), (1, (EWG, 512, SMEM_128))):
        prev = lib.mm_gemm_overlap_mode(mode)
        try:
            p = plan(M=32 * 528, N=3 * E, K=E, epi=ops.EPI_ROPE, fp16=True, streamk=True)
            assert (p["kernel"], p["threads"], p["smem_bytes"], p["grid"]) == want + (SMS,), mode
        finally:
            lib.mm_gemm_overlap_mode(prev)
    prev = lib.mm_gemm_streamk_mode(0)
    try:
        assert plan(M=4 * 528, N=2 * I, K=E, epi=ops.EPI_SWIGLU, streamk=True)["streamk_tiles"] == 0
    finally:
        lib.mm_gemm_streamk_mode(prev)
    assert plan(M=4 * 528, N=2 * I, K=E, epi=ops.EPI_SWIGLU, streamk=True)["streamk_tiles"] == 20
    prev = lib.mm_gemm_streamk_mode(2)  # whenever the schedule allows
    try:
        p = plan(M=4 * 528, N=E, K=E, streamk=True)
        assert p["streamk_tiles"] == p["units"] % SMS == 32
        assert plan(M=1028, N=1024, K=1024, streamk=True)["streamk_tiles"] == 0   # needs more than one full wave
        assert plan(M=8224, N=3072, K=1024, streamk=True)["streamk_tiles"] == 1560 % SMS
    finally:
        lib.mm_gemm_streamk_mode(prev)


def test_thin_decode_gemms_use_narrow_tiles():
    # swapped operands (c_trans): the weight rows fill the 128-row MMA tile, the 8 token rows are the N extent
    p = plan(M=E, N=8, K=E, c_trans=True)
    assert p["block_n"] == 32 and p["units"] == E // 128 and p["grid"] == E // 128
    assert (p["kernel"], p["threads"], p["smem_bytes"]) == (EWG, 512, SMEM_64)  # 8 stages of 128 x 32: as many bytes
    p = plan(M=E, N=8, K=E // 4, batch=4, c_fp32=True)  # split-K of 4 through the batch dimension: 128 units
    assert p["units"] == 4 * (E // 128) and p["grid"] == 128
    assert (p["kernel"], p["threads"]) == (CONSUMER, 288)  # 16 k-blocks


def test_kernel_variant_of_narrow_and_mn_major_launches():
    p = plan(M=100, N=E, K=E)  # the cost model picks 128 tiles of 128 x 32: less than a wave
    assert (p["block_n"], p["units"], p["kernel"], p["threads"], p["grid"]) == (32, 128, EWG, 512, 128)
    dx = plan(M=4 * 528, N=E, K=I, b_mn_major=True)  # training: dx = dy W
    dw = plan(M=E, N=E, K=4 * 528, a_mn_major=True, b_mn_major=True)  # training: dW = dy^T x, 33 k-blocks
    for p in (dx, dw):
        assert (p["kernel"], p["threads"], p["grid"]) == (EWG, 512, SMS), p


def test_schedule_invariants_random_shapes():
    rng = random.Random(7)
    for _ in range(300):
        M = rng.choice([1, 7, 128, 129, 257, 1028, 2112, 4224, 6000, 16896]) + rng.choice([0, 0, 8, 64])
        N = rng.choice([8, 64, 96, 512, 768, 1024, 1536, 3072, 4096, 12288, 22016, 32000])
        K = rng.choice([64, 256, 512, 768, 1024, 2048, 4096, 11008])
        batch = rng.choice([1, 1, 1, 2, 16])
        b_mn = rng.random() < 0.2
        a_mn = b_mn and rng.random() < 0.5
        if a_mn:
            M = (M + 7) // 8 * 8  # lda = M must be a multiple of 8
        if b_mn:
            N = (N + 7) // 8 * 8
        p = plan(M=M, N=N, K=K, batch=batch, b_mn_major=b_mn, a_mn_major=a_mn, streamk=rng.random() < 0.5)
        assert p["block_n"] in (32, 64, 128) and (not b_mn or p["block_n"] >= 64)
        assert p["m_tiles"] == (M + 127) // 128 and p["n_tiles"] == (N + p["block_n"] - 1) // p["block_n"]
        assert p["k_blocks"] == (K + 63) // 64
        assert p["units"] == batch * p["m_tiles"] * p["n_tiles"]
        assert p["threads"] == {CONSUMER: 288, EWG: 512, PAIRS: 384}[p["kernel"]]
        assert p["kernel"] == CONSUMER or p["streamk_tiles"] == 0
        assert p["kernel"] != PAIRS or (batch == 1 and not b_mn and p["n_tiles"] % 2 == 0 and p["smem_bytes"] == SMEM_PAIRS)
        assert p["workers"] == SMS
        assert p["waves"] == -(-p["units"] // p["workers"]) and 0 < p["grid"] <= SMS
        assert 0 <= p["streamk_tiles"] < SMS
        assert p["smem_bytes"] <= 227 * 1024 and p["group_m"] >= 2


def test_argument_checks_raise_with_a_message():
    lib = _lib.load()
    fake = 1 << 20

    def rc(**over):
        kw = dict(M=256, N=256, K=256, batch=1, batch2=1, A=fake, lda=256, B=fake, ldb=256, C=fake, ldc=256, alpha=1.0)
        kw.update(over)
        a = _lib.GemmArgs(**kw)
        out = _lib.GemmPlan()
        r = lib.mm_gemm_plan(C.byref(a), C.byref(out))
        return r, _lib.last_error()

    assert rc()[0] == 0
    r, msg = rc(a_fp16=1, b_fp16=0)
    assert r != 0 and "mixed f16 x bf16" in msg  # wgmma takes one input type for both operands
    r, msg = rc(lda=250)
    assert r != 0 and "multiples of 8" in msg
    r, msg = rc(A=fake + 2)
    assert r != 0 and "16-byte aligned" in msg
    r, msg = rc(epi=ops.EPI_ROPE)
    assert r != 0 and "RoPE" in msg          # no cos / sin tables
    r, msg = rc(a_mn_major=1)
    assert r != 0 and "MN-major A" in msg    # needs MN-major B as well
    r, msg = rc(M=0)
    assert r != 0 and "bad shape" in msg
    with pytest.raises(RuntimeError):
        ops.gemm_plan(M=256, N=100, K=256, epi=ops.EPI_SWIGLU)  # SwiGLU epilogue needs N % 64 == 0
