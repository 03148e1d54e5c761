"""CPU tier: the pair walk of the wide GEMM kernel (`pair_coord` and the round-robin loop of `gemm_wide_kernel`,
csrc/gemm_wgmma.cu), restated in Python.  The wide kernel is a different walk over the tiles mm_gemm_plan reports, not a
different tiling, so for every launch the plan gives the tile-pair kernel:
  1. the plan still reports the 128-wide tile grid (block_n 128, units = m_tiles * n_tiles);
  2. the pairs (m_blk, 2 j), (m_blk, 2 j + 1) visited by the plan's CTAs 0 .. grid - 1 cover every tile of that grid
     exactly once;
  3. the TMA loader's cursor (one lane of a consumer warp, running ahead of the main loop) visits the same (pair, k-block)
     sequence as the consumers of its CTA;
  4. every index product formed on the device fits a signed 32-bit integer.
Test infrastructure only: a restatement of the schedule, not the kernel."""
import random

import pytest

from macaw_llm_b200 import ops

SMS = 132
E, I, V = 4096, 11008, 32000
PAIRS = ops.GEMM_TILE_PAIRS


def pair_coord(idx, m_tiles, n_tiles, group_m):
    """Line-by-line restatement of the device function."""
    n_pairs = n_tiles // 2
    in_group = group_m * n_pairs
    g = idx // in_group
    first_m = g * group_m
    gsz = min(m_tiles - first_m, group_m)
    rr = idx - g * in_group
    assert max(idx, in_group, first_m + gsz, rr) < 2 ** 31
    return first_m + rr % gsz, 2 * (rr // gsz)


def check_walk(p):
    m_tiles, n_tiles, gm = p["m_tiles"], p["n_tiles"], p["group_m"]
    pairs = m_tiles * (n_tiles // 2)
    grid = p["grid"]
    assert 0 < grid <= p["workers"]
    seen = [[0] * n_tiles for _ in range(m_tiles)]
    for worker in range(grid):
        consumer, loader = [], []
        for u in range(worker, pairs, grid):                      # consumers and epilogue warpgroup
            consumer.append(pair_coord(u, m_tiles, n_tiles, gm))
        ld_u = worker                                             # the loader's cursor, advanced k-block by k-block
        ld_kb = 0
        while ld_u < pairs:
            if ld_kb == 0:
                loader.append(pair_coord(ld_u, m_tiles, n_tiles, gm))
            ld_kb += 1
            if ld_kb == p["k_blocks"]:
                ld_kb, ld_u = 0, ld_u + grid
        assert loader == consumer
        for m_blk, n_blk in consumer:
            assert 0 <= m_blk < m_tiles and 0 <= n_blk and n_blk + 1 < n_tiles
            seen[m_blk][n_blk] += 1
            seen[m_blk][n_blk + 1] += 1
    assert all(c == 1 for row in seen for c in row), "every 128 x 128 tile of the plan exactly once"
    # TMA coordinates: m_blk * 128, (n_blk + 1) * 128, kb * 64
    assert m_tiles * 128 < 2 ** 31 and n_tiles * 128 < 2 ** 31 and p["k_blocks"] * 64 < 2 ** 31


@pytest.mark.parametrize("N,K,epi", [(3 * E, E, ops.EPI_ROPE), (E, E, ops.EPI_STD), (2 * I, E, ops.EPI_SWIGLU),
                                     (E, I, ops.EPI_STD), (V, E, ops.EPI_STD)])
@pytest.mark.parametrize("M", [32 * 528, 4 * 528])
def test_benchmark_shapes(M, N, K, epi):
    p = ops.gemm_plan(M=M, N=N, K=K, epi=epi, fp16=True)
    if M == 4 * 528 and N == E:
        assert p["block_n"] == 64 and p["kernel"] == ops.GEMM_EPILOGUE_WARPGROUP  # o_proj / down at 17 M tiles
        return
    assert (p["block_n"], p["kernel"]) == (128, PAIRS) and p["units"] == p["m_tiles"] * p["n_tiles"]
    if M == 32 * 528:
        assert (p["m_tiles"] * (p["n_tiles"] // 2)) % SMS == 0  # whole waves of pairs at the benchmark's batch
    check_walk(p)


def test_random_qualifying_shapes():
    rng = random.Random(11)
    n = 0
    while n < 150:
        M = rng.choice([2112, 4000, 4224, 6000, 16896, 33000]) + rng.choice([0, 0, 8, 64])
        N = rng.choice([1024, 1536, 3072, 4000, 4096, 12288, 22016, 32000])
        K = rng.choice([2048, 2120, 4096, 11008])
        p = ops.gemm_plan(M=M, N=N, K=K, fp16=rng.random() < 0.5)
        if p["kernel"] != PAIRS:
            continue
        n += 1
        assert p["block_n"] == 128 and p["units"] == p["m_tiles"] * p["n_tiles"]
        check_walk(p)


def test_shapes_that_do_not_qualify():
    ewg, consumer = ops.GEMM_EPILOGUE_WARPGROUP, ops.GEMM_CONSUMER_EPILOGUE
    assert ops.gemm_plan(M=16896, N=E + 128, K=E)["kernel"] == ewg                 # 33 N tiles
    assert ops.gemm_plan(M=16896, N=E, K=1024)["kernel"] == consumer               # 16 k-blocks
    assert ops.gemm_plan(M=100, N=E, K=E)["kernel"] == ewg                         # less than one wave of pairs
    assert ops.gemm_plan(M=31 * 528, N=E, K=E, streamk=True)["kernel"] == consumer  # stream-K tail
