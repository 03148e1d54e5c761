"""fp64 restatement of the sampled decoding step (mm_sample_rows, include/macaw_b200.h): HF's processor chain
RepetitionPenalty -> Temperature -> TopK -> TopP, softmax and the inverse-CDF draw from the Philox word.

`restate` also flags the draws whose token a last-bits difference between this fp64 arithmetic and the kernel's fp32
scores / fixed-point masses could change: a token whose top-k or top-p decision lies within TOL of its threshold, when
flipping that decision changes the drawn token, or a draw within TOL (of the total mass) of a CDF boundary."""
from __future__ import annotations

import numpy as np

from tests.helpers import philox4x32_10

SID_SAMPLE = 16  # csrc/philox.cuh
TOL = 1e-5


def uniforms(seed: int, step: int, rows: int) -> np.ndarray:
    """u = (w >> 8) * 2^-24, w = word 0 of philox(key = seed, counter = (step, row, SID_SAMPLE, 0))."""
    ctr = np.stack([np.full(rows, step, np.uint32), np.arange(rows, dtype=np.uint32),
                    np.full(rows, SID_SAMPLE, np.uint32), np.zeros(rows, np.uint32)], axis=1)
    w = philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))[:, 0]
    return (w >> np.uint32(8)).astype(np.float64) * 2.0 ** -24


def seen_mask(bits: np.ndarray, V: int) -> np.ndarray:
    """(rows, ceil(V/32)) uint32 bitmap -> (rows, V) bool."""
    b = bits.astype(np.uint32)
    return ((b[:, np.arange(V) >> 5] >> (np.arange(V) & 31).astype(np.uint32)) & 1).astype(bool)


def penalise(s: np.ndarray, seen: np.ndarray, penalty: float) -> np.ndarray:
    """RepetitionPenaltyLogitsProcessor: s < 0 ? s * p : s / p on every generated token."""
    if penalty == 1.0:
        return s
    return np.where(seen, np.where(s < 0, s * penalty, s / penalty), s)


def kept_set(s: np.ndarray, top_k: int, top_p: float):
    """Temperature-scaled scores of one row -> (kept bool, ambiguous bool).

    Top-k keeps every score >= the k-th largest.  Top-p, over the softmax of the top-k survivors, removes token i iff
    M(<= p_i) <= 1 - top_p, where M(<= p) is the kept mass of all tokens with probability <= p: HF's ascending cumsum
    rule with a tied group removed or kept as a whole.  The largest token (group) always stays."""
    V = s.shape[0]
    keep = np.ones(V, bool)
    amb = np.zeros(V, bool)
    if 0 < top_k < V:
        kth = np.partition(s, V - top_k)[V - top_k]
        keep = s >= kth
        amb |= (np.abs(s - kth) <= TOL * max(abs(kth), 1e-30)) & (s != kth)
    if top_p < 1.0:
        e = np.where(keep, np.exp(s - s.max()), 0.0)
        order = np.argsort(e, kind="stable")
        es = e[order]
        M = np.cumsum(es)[np.searchsorted(es, es, side="right") - 1] / es.sum()
        rem = M <= 1.0 - top_p
        rem[es == es[-1]] = False
        removed = np.zeros(V, bool)
        removed[order] = rem
        near = np.zeros(V, bool)
        near[order] = np.abs(M - (1.0 - top_p)) <= TOL
        amb |= near & keep
        keep &= ~removed
    return keep, amb


def inverse_cdf(w: np.ndarray, u: float):
    """First token whose cumulative (normalised) mass exceeds u, and whether u lies within TOL of a boundary."""
    c = np.cumsum(w) / w.sum()
    i = int(np.searchsorted(c, u, side="right"))
    near = abs(c[i] - u) <= TOL or (i > 0 and abs(u - c[i - 1]) <= TOL)
    return i, near


def restate(logits: np.ndarray, bits: np.ndarray, *, do_sample: bool, repetition_penalty: float = 1.0,
            temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, seed: int = 0, step: int = 0):
    """(rows, V) logits (the 16-bit values, as floats) and (rows, ceil(V/32)) bitmap -> (tokens int64, flagged bool)."""
    rows, V = logits.shape
    s_all = penalise(logits.astype(np.float64), seen_mask(bits, V), repetition_penalty)
    toks = np.zeros(rows, np.int64)
    flags = np.zeros(rows, bool)
    if not do_sample:
        for r in range(rows):
            s = s_all[r]
            toks[r] = int(np.argmax(s))
            other = s[s != s[toks[r]]]
            flags[r] = other.size > 0 and s[toks[r]] - other.max() <= TOL * max(abs(s[toks[r]]), 1e-30)
        return toks, flags
    u = uniforms(seed, step, rows)
    for r in range(rows):
        s = s_all[r] / temperature
        keep, amb = kept_set(s, top_k, top_p)
        p = np.exp(s - s.max())
        toks[r], near = inverse_cdf(np.where(keep, p, 0.0), u[r])
        if amb.any():
            alt, near_alt = inverse_cdf(np.where(keep ^ amb, p, 0.0), u[r])
            near = near or near_alt or alt != toks[r]
        flags[r] = near
    return toks, flags


def warped_probs(logits_row: np.ndarray, *, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """The exact distribution the draw samples from (one row, empty bitmap)."""
    s = logits_row.astype(np.float64) / temperature
    keep, _ = kept_set(s, top_k, top_p)
    p = np.where(keep, np.exp(s - s.max()), 0.0)
    return p / p.sum()
