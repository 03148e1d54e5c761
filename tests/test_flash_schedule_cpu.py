"""CPU tier: the tile walk of the wgmma flash-attention kernel (csrc/attn_wgmma.cu), restated on CPU tensors.

What is checked without a GPU is the ALGORITHM the kernel's roles agree on, not the kernel (the GPU tier does that):
  * 128-query tiles, 64-key tiles; causal query tiles are aligned to the END of the sequence, so the ragged tile sits at the
    start (rows before 0 are zero fill, never stored) and sees one key tile: T = 528 walks 25 key tiles per head, not 29;
  * key validity = Tk bound & key-padding mask, causal limit per row: key j visible to query i iff j <= i + Tk - Tq;
  * RESCALE POLICY: the accumulator and the row sum are expressed in a reference max; the kernel advances it whenever the
    running max grows (tau = 0).  A lazy policy that advances it only when the max grows by more than 2^tau gives the same
    O / l, because P and l use that same reference — probabilities may exceed 1 (up to 2^tau) in between;
  * rows with every key masked produce zeros (DESIGN.md "unspecified rows"; the reference attends uniformly there and
    nothing downstream reads those rows).
The restatement is test infrastructure; no product code routes through it.
"""
import math

import pytest
import torch

MQ, KT, TAU = 128, 64, 0.0  # kFaMQ, kFaKT of csrc/attn_wgmma.cu; its exact running-max rescale


def key_tiles_of(mt, Tq, Tk, causal):
    nq = -(-Tq // MQ)
    q_base = Tq - nq * MQ if causal else 0
    kv_end = min(Tk, q_base + mt * MQ + MQ + (Tk - Tq)) if causal else Tk
    return (-(-kv_end // KT) if kv_end > 0 else 0), q_base


def flash_walk(q, k, v, scale, causal=False, key_mask=None, tau=TAU):
    """q (Tq, hd), k / v (Tk, hd) fp64; key_mask (Tk,) bool or None -> (out (Tq, hd), key tiles walked, per-row accumulator rescales done)."""
    Tq, hd = q.shape
    Tk = k.shape[0]
    nq = -(-Tq // MQ)
    shift = Tk - Tq
    scale_log2 = scale * 1.4426950408889634
    out = torch.zeros(Tq, hd, dtype=q.dtype)
    walked = rescales = 0
    for mt in range(nq - 1, -1, -1):  # heaviest query tile first, as the CTA walks them
        n_tiles, q_base = key_tiles_of(mt, Tq, Tk, causal)
        rows = torch.arange(q_base + mt * MQ, q_base + mt * MQ + MQ)
        live = (rows >= 0) & (rows < Tq)
        qt = torch.zeros(MQ, hd, dtype=q.dtype)
        qt[live] = q[rows[live]]  # rows outside [0, Tq) are TMA zero fill
        m_used = torch.full((MQ,), -math.inf, dtype=q.dtype)
        l = torch.zeros(MQ, dtype=q.dtype)
        O = torch.zeros(MQ, hd, dtype=q.dtype)
        for j in range(n_tiles):
            walked += 1
            keys = torch.arange(j * KT, j * KT + KT)
            ok = keys < Tk
            kt = torch.zeros(KT, hd, dtype=q.dtype)
            vt = torch.zeros(KT, hd, dtype=q.dtype)
            kt[ok], vt[ok] = k[keys[ok]], v[keys[ok]]
            if key_mask is not None:
                ok = ok & torch.cat([key_mask, torch.zeros(max(0, j * KT + KT - Tk), dtype=torch.bool)])[j * KT:j * KT + KT]
            okm = ok[None, :].expand(MQ, KT)
            if causal:
                okm = okm & (keys[None, :] <= (rows[:, None] + shift))
            s = qt @ kt.T
            mx = torch.where(okm, s, torch.full_like(s, -math.inf)).max(1).values * scale_log2
            # reference max: advanced only on the first finite max or when it grew by more than tau
            adv = ((mx > m_used + tau) | torch.isinf(m_used)) & ~torch.isinf(mx)
            resc = adv & ~torch.isinf(m_used)
            alpha = torch.where(resc, torch.exp2(m_used - mx), torch.ones_like(mx))
            m_used = torch.where(adv, mx, m_used)
            m_ref = torch.where(torch.isinf(m_used), torch.zeros_like(m_used), m_used)
            p = torch.where(okm, torch.exp2(s * scale_log2 - m_ref[:, None]), torch.zeros_like(s))
            assert float(p.max()) <= 2.0 ** tau * (1 + 1e-9)  # bounded by the lazy-rescale threshold
            l = l * alpha + p.sum(1)
            rescales += int(resc.sum())  # per-row accumulator rescales
            if bool(resc.any()):
                O = O * alpha[:, None]
            O = O + p @ vt
        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        out[rows[live]] = (O * inv[:, None])[live]
    return out, walked, rescales


def reference(q, k, v, scale, causal, key_mask):
    Tq, Tk = q.shape[0], k.shape[0]
    s = (q @ k.T) * scale
    ok = torch.ones(Tq, Tk, dtype=torch.bool)
    if key_mask is not None:
        ok &= key_mask[None, :]
    if causal:
        ok &= torch.arange(Tk)[None, :] <= (torch.arange(Tq)[:, None] + (Tk - Tq))
    s = s.masked_fill(~ok, -math.inf)
    p = torch.softmax(s, dim=1)
    p = torch.where(ok.any(1, keepdim=True), p, torch.zeros_like(p))  # fully masked rows: zeros
    return p @ v


@pytest.mark.parametrize("Tq,Tk,causal,masked", [
    (528, 528, True, True),    # the LLaMA shape of cfg4: ragged first tile, padding mask
    (257, 257, False, False),  # CLIP: 257 tokens
    (130, 4098, False, False), # video-long: 4096 + 2 keys (a slice of the queries)
    (1, 300, True, False),     # one decode step over a cache
    (200, 328, True, True),    # prefill continuation: Tk > Tq
])
def test_tile_walk_is_exact(Tq, Tk, causal, masked):
    g = torch.Generator().manual_seed(Tq * 7 + Tk)
    hd = 64
    q = torch.randn(Tq, hd, generator=g, dtype=torch.float64)
    k = torch.randn(Tk, hd, generator=g, dtype=torch.float64)
    v = torch.randn(Tk, hd, generator=g, dtype=torch.float64)
    km = None
    if masked:
        km = torch.ones(Tk, dtype=torch.bool)
        km[Tk - 37:] = False  # right padding
        km[5] = False
    out, _, _ = flash_walk(q, k, v, hd ** -0.5, causal, km)
    ref = reference(q, k, v, hd ** -0.5, causal, km)
    assert float((out - ref).abs().max()) < 1e-12


def test_causal_tiles_aligned_to_the_sequence_end_walk_25_not_29_key_tiles():
    T = 528
    assert sum(key_tiles_of(mt, T, T, True)[0] for mt in range(5)) == 25
    # the start-aligned layout (ragged tile LAST, walking every key tile) would take 2 + 4 + 6 + 8 + 9 = 29
    assert sum(min(-(-T // KT), -(-(min(T, (mt + 1) * MQ)) // KT)) for mt in range(5)) == 29
    # the ragged tile holds rows -112 .. 15 and sees a single key tile
    n, q_base = key_tiles_of(0, T, T, True)
    assert (n, q_base) == (1, -112)


def test_lazy_rescale_policy_does_not_change_the_result():
    """Scores that grow along the key axis force reference-max advances; tau = 0 (rescale on every growth: the kernel) and
    tau = 8 (lazy) must agree: O and l are expressed in the same reference."""
    g = torch.Generator().manual_seed(11)
    T, hd = 384, 64
    q = torch.randn(T, hd, generator=g, dtype=torch.float64)
    k = torch.randn(T, hd, generator=g, dtype=torch.float64) * torch.linspace(0.3, 3.0, T, dtype=torch.float64)[:, None]
    v = torch.randn(T, hd, generator=g, dtype=torch.float64)
    sc = hd ** -0.5
    ref = reference(q, k, v, sc, False, None)
    eager, _, n_eager = flash_walk(q, k, v, sc, tau=0.0)
    lazy, _, n_lazy = flash_walk(q, k, v, sc, tau=8.0)
    print(f"[lazy rescale] row rescales: tau=0 {n_eager}, tau=8 {n_lazy}")
    assert 0 < n_lazy < n_eager // 2  # the threshold really skips rescales, and this input really needs some
    assert float((eager - ref).abs().max()) < 1e-10 and float((lazy - ref).abs().max()) < 1e-10


def test_fully_masked_rows_give_zeros_and_leak_nowhere():
    """Left padding: query rows whose own key is padding see no key at all under the causal rule + mask."""
    g = torch.Generator().manual_seed(3)
    T, hd = 140, 64
    q = torch.randn(T, hd, generator=g, dtype=torch.float64)
    k = torch.randn(T, hd, generator=g, dtype=torch.float64)
    v = torch.randn(T, hd, generator=g, dtype=torch.float64)
    km = torch.ones(T, dtype=torch.bool)
    km[:9] = False  # left padding
    out, _, _ = flash_walk(q, k, v, hd ** -0.5, True, km)
    assert float(out[:9].abs().max()) == 0.0
    # valid rows are independent of what the padded positions hold
    k2, v2 = k.clone(), v.clone()
    k2[:9], v2[:9] = 100.0, -100.0
    out2, _, _ = flash_walk(q, k2, v2, hd ** -0.5, True, km)
    assert float((out[9:] - out2[9:]).abs().max()) == 0.0
