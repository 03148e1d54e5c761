"""CPU tier: the stream-K tail schedule of the wgmma GEMM (`gemm_work`, csrc/gemm_wgmma.cu), restated in Python
and checked for the properties the kernel's hand-over relies on.  The tail shapes come from the real dispatcher
(mm_gemm_plan), so the cases are the ones the product path launches (lm_head / QKV / down_proj at the per-GPU batch of the
8-GPU run) plus random ones.  Test infrastructure only — a restatement of the schedule, not the kernel.

Properties (the comments above `struct GemmWork` state them; a violation would be a deadlock or a wrong sum on the GPU):
  1. full tiles [0, first) are each computed exactly once, whole (role 0), round-robin over the CTAs;
  2. the k-blocks of every tail tile are covered exactly once by the pieces of consecutive CTAs' equal shares;
  3. a CTA owns at most two tail pieces — at most ONE contributor piece (role 1) and it is always the CTA's FIRST unit, so a
     contributor never waits behind anything; a finisher (role 2) waits only for CTAs with a LOWER index;
  4. every tail tile has exactly one finisher, its piece ends the tile, and its contributor range [c0, c0 + nc) — minus the CTAs
     whose share is empty, which the kernel skips (`sk_has`) — is exactly the set of CTAs holding a contributor piece of it;
  5. the 32-bit arithmetic bound the host checks (SMs * num_k * (SMs + 1) < 2^31) covers every product formed.
"""
import random

import pytest

from macaw_llm_b200 import ops

SMS = 132  # the library's SM count when no device is visible (H100 SXM)


def gemm_work(worker, n_workers, total_tiles, it, sk_tiles, sk_first, num_k):
    """Line-by-line restatement of the device function (unsigned 32-bit arithmetic modelled with a range assertion)."""
    first = sk_first if sk_tiles > 0 else total_tiles
    n_full = (first - worker + n_workers - 1) // n_workers if first > worker else 0
    n_sk, has_b = 0, False
    nk, U, u0, u1, ta, end_a = 1, 0, 0, 0, 0, 0
    if sk_tiles > 0:
        nk = num_k
        U = sk_tiles * nk
        assert (worker + 1) * U < 2 ** 32  # the products formed on the device fit unsigned 32-bit
        u0 = worker * U // n_workers
        u1 = (worker + 1) * U // n_workers
        if u0 < u1:
            ta = u0 // nk
            end_a = min(u1, (ta + 1) * nk)
            has_b = u1 > end_a
            n_sk = 2 if has_b else 1
    if it >= n_sk:
        f = it - n_sk
        if f >= n_full:
            return None
        return dict(tile=worker + f * n_workers, kb0=0, kb1=num_k, role=0, c0=0, nc=0)
    if has_b and it == 0:
        return dict(tile=first + ta + 1, kb0=0, kb1=u1 - end_a, role=1, c0=0, nc=0)
    w = dict(tile=first + ta, kb0=u0 - ta * nk, kb1=end_a - ta * nk, role=0, c0=0, nc=0)
    w["role"] = 2 if w["kb1"] == num_k else 1
    if w["role"] == 2:
        c0 = worker
        while c0 > 0 and c0 * U // n_workers > ta * nk:
            c0 -= 1
        w["c0"], w["nc"] = c0, worker - c0
    return w


def check_schedule(total_tiles, n_workers, sk_tiles, num_k):
    sk_first = total_tiles - sk_tiles
    full_seen = [0] * sk_first
    cover = {t: [0] * num_k for t in range(sk_first, total_tiles)}
    finisher, contributors = {}, {t: [] for t in range(sk_first, total_tiles)}
    for w in range(n_workers):
        it, n_role1, tail_units = 0, 0, 0
        while True:
            u = gemm_work(w, n_workers, total_tiles, it, sk_tiles, sk_first, num_k)
            if u is None:
                break
            if u["role"] == 0:
                assert 0 <= u["tile"] < sk_first and (u["kb0"], u["kb1"]) == (0, num_k)
                full_seen[u["tile"]] += 1
            else:
                tail_units += 1
                assert sk_first <= u["tile"] < total_tiles and 0 <= u["kb0"] < u["kb1"] <= num_k
                for kb in range(u["kb0"], u["kb1"]):
                    cover[u["tile"]][kb] += 1
                if u["role"] == 1:
                    n_role1 += 1
                    assert it == 0, "a contributor piece must be the CTA's first unit (it never waits)"
                    contributors[u["tile"]].append(w)
                else:
                    assert u["kb1"] == num_k and u["tile"] not in finisher
                    finisher[u["tile"]] = (w, u["c0"], u["nc"])
            it += 1
        assert n_role1 <= 1 and tail_units <= 2
    assert all(c == 1 for c in full_seen), "every full tile exactly once"
    for t, ks in cover.items():
        assert all(c == 1 for c in ks), f"tail tile {t}: k-blocks covered {ks}"
        assert t in finisher
        w, c0, nc = finisher[t]
        U = sk_tiles * num_k
        # CTAs whose share of the tail is empty (more CTAs than tail k-blocks) hold no piece: the kernel's `sk_has` skips them
        has = [c for c in range(c0, c0 + nc) if c * U // n_workers < (c + 1) * U // n_workers]
        assert has == sorted(contributors[t]), (t, finisher[t], contributors[t])
        assert all(c < w for c in contributors[t]), "finishers wait only for lower-indexed CTAs"


@pytest.mark.parametrize("M,N,K", [(2112, 32000, 4096), (2112, 12288, 4096), (2112, 4096, 11008), (8224, 3072, 1024)])
def test_product_shapes(M, N, K):
    lib_mode = ops._lib.load().mm_gemm_streamk_mode(2)  # whenever the schedule allows: exercise every shape
    try:
        p = ops.gemm_plan(M=M, N=N, K=K, streamk=True)
        total, sk, nk = p["units"], p["streamk_tiles"], p["k_blocks"]
        assert sk == total % SMS and sk > 0
    finally:
        ops._lib.load().mm_gemm_streamk_mode(lib_mode)
    assert SMS * nk * (SMS + 1) < 2 ** 31  # the host-side guard of the 32-bit arithmetic
    check_schedule(total, SMS, sk, nk)


def test_random_tails():
    rng = random.Random(5)
    for _ in range(200):
        n_workers = rng.choice([4, 7, 16, SMS])
        num_k = rng.choice([8, 9, 16, 64, 172])
        waves = rng.randint(1, 4)
        sk = rng.randint(1, n_workers - 1)
        check_schedule(waves * n_workers + sk, n_workers, sk, num_k)


def test_no_tail_is_plain_round_robin():
    for total in (1, SMS - 1, SMS, 300):
        check_schedule(total, SMS, 0, 64)
