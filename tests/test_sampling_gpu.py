"""GPU tier of the sampled generate branch: mm_sample_rows against the fp64 restatement (tests/sampling_ref.py), its
distribution, and Engine.generate / MM_LLMs' generate branch with sampling and a repetition penalty on the tiny model
against the CPU oracle, teacher-forced."""
import numpy as np
import pytest
import torch

from tests import helpers as H
from tests import sampling_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (do_sample, repetition_penalty, temperature, top_k, top_p)
CONFIGS = [(True, 1.0, 1.0, 0, 1.0), (True, 1.0, 0.9, 50, 0.6), (True, 1.3, 0.7, 0, 0.9), (True, 1.0, 1.5, 200, 0.95),
           (True, 1.2, 0.8, 1, 1.0), (False, 1.3, 1.0, 0, 1.0)]


def _bits_of(tokens: np.ndarray, words: int) -> np.ndarray:
    b = np.zeros((tokens.shape[0], words), np.uint32)
    b[np.arange(tokens.shape[0]), tokens >> 5] = (np.uint32(1) << (tokens & 31).astype(np.uint32))
    return b


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [519, 32000, 32007])
def test_kernel_matches_restatement(dtype, V):
    from macaw_llm_b200 import ops

    words = (V + 31) // 32
    total = flagged = 0
    mism = []
    ops.set_act_format(dtype)
    try:
        for rows in (1, 8, 64):
            g = torch.Generator().manual_seed(V * 131 + rows)
            for ci, (do_sample, pen, T, k, p) in enumerate(CONFIGS):
                # logits of std 8: the mass sits on a few tokens, so few draws fall within the tolerance of a boundary
                # between the tiny-probability tokens of a flat 32k-token tail (at std 3 about 2 % of the untruncated
                # draws do, though the kernel still matched every one of them)
                full = (torch.randn((rows, V + 5), generator=g) * 8.0).to(dtype)
                logits, lg = full[:, :V], full.to(DEV)[:, :V]  # row stride V + 5 > V
                bits0 = torch.randint(0, 2 ** 31, (rows, words), generator=g, dtype=torch.int64)
                bits0 &= torch.randint(0, 2 ** 31, (rows, words), generator=g, dtype=torch.int64)
                bits0 &= torch.randint(0, 2 ** 31, (rows, words), generator=g, dtype=torch.int64)  # ~1/8 of the bits
                bits0 = bits0.to(torch.int32)
                for seed, step in ((1234567, 0), ((99 << 32) | 5, 1), (2 ** 64 - 3, 17), (42, 2 ** 31 - 1), (7, 3),
                                   ((1 << 63) | 99, 64)):
                    seen = bits0.to(DEV).contiguous()
                    sd = torch.tensor([seed - 2 ** 64 if seed >= 2 ** 63 else seed], dtype=torch.int64, device=DEV)
                    stp = torch.tensor([step], dtype=torch.int32, device=DEV)
                    tok = ops.sample_rows(lg, seen, do_sample=do_sample, repetition_penalty=pen, temperature=T,
                                          top_k=k, top_p=p, seed_dev=sd, step_dev=stp).cpu().numpy()
                    ref, flag = R.restate(logits.float().numpy(), bits0.numpy().view(np.uint32), do_sample=do_sample,
                                          repetition_penalty=pen, temperature=T, top_k=k, top_p=p, seed=seed, step=step)
                    want_bits = bits0.numpy().view(np.uint32) | _bits_of(tok, words)
                    assert np.array_equal(seen.cpu().numpy().view(np.uint32), want_bits), (rows, ci, seed)
                    bad = (tok != ref) & ~flag
                    assert not bad.any(), (rows, ci, seed, step, np.flatnonzero(bad), tok[bad], ref[bad])
                    total += rows
                    flagged += int(flag.sum())
                    mism.append(int((tok != ref).sum()))
    finally:
        ops.set_act_format(torch.bfloat16)
    print(f"V={V} {dtype}: {total} draws, {flagged} flagged near a boundary, {sum(mism)} differ (all flagged)")
    assert flagged <= 0.001 * total, (flagged, total)


def test_distribution_chi_square():
    """2^17 copies of one row in one launch (a fresh Philox counter per row) against the exact warped distribution."""
    from scipy import stats

    from macaw_llm_b200 import ops

    V, rows, T, k, p = 519, 1 << 17, 0.8, 30, 0.9
    row = (torch.randn((V,), generator=torch.Generator().manual_seed(3)) * 2.0).to(torch.bfloat16)
    want = R.warped_probs(row.float().numpy(), temperature=T, top_k=k, top_p=p)
    support = np.flatnonzero(want > 0)
    assert 10 <= support.size <= 30, support.size
    lg = row.to(DEV).unsqueeze(0).expand(rows, V).contiguous()
    seen = torch.zeros((rows, (V + 31) // 32), dtype=torch.int32, device=DEV)
    sd = torch.tensor([(11 << 32) | 12345], dtype=torch.int64, device=DEV)
    stp = torch.tensor([7], dtype=torch.int32, device=DEV)
    tok = ops.sample_rows(lg, seen, do_sample=True, temperature=T, top_k=k, top_p=p, seed_dev=sd, step_dev=stp)
    counts = np.bincount(tok.cpu().numpy(), minlength=V)
    assert counts[want == 0].sum() == 0
    exp = want[support] * rows
    obs = counts[support].astype(np.float64)
    small = exp < 5  # pool the rare bins so that every expected count is >= 5
    if small.any():
        exp = np.r_[exp[~small], exp[small].sum()]
        obs = np.r_[obs[~small], obs[small].sum()]
    pval = stats.chisquare(obs, exp).pvalue
    print(f"chi-square over {exp.size} bins: p = {pval:.4f}")
    assert pval > 1e-4


# ---------------------------------------------------------------------------------------------------- the tiny model
@pytest.fixture(scope="module")
def tiny():
    model, spec, hp, weights = H.build_tiny_model(DEV, torch.bfloat16)
    inp = H.case_inputs(spec, H.load_case("all3"))
    inp.pop("labels", None)
    inp = {k: (v.to(torch.bfloat16) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}
    dev_inp = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}
    return model, hp, weights, inp, dev_inp


def _oracle_logits(tiny, toks):
    from oracle import macaw_oracle as O

    model, hp, weights, inp, _ = tiny
    f32 = {k: (v.float() if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in inp.items()}
    _, o_logits = O.generate_greedy(f32, H.bf16_round(weights), hp, max_new_tokens=toks.shape[1], forced_tokens=toks.cpu())
    return o_logits.double().numpy()


def _check_teacher_forced(tiny, toks, *, do_sample, repetition_penalty, temperature=1.0, top_k=0, top_p=1.0):
    """Every generated token must be the oracle's choice under the same configuration once its oracle logit is raised by
    the greedy test's bf16 margin (0.05 std + 1e-3): in the kept set when sampling, within the margin of the top score
    of the penalised logits otherwise."""
    o = _oracle_logits(tiny, toks)
    toks = toks.cpu().numpy()
    B, n = toks.shape
    V = o.shape[-1]
    for b in range(B):
        seen = np.zeros(V, bool)
        for j in range(n):
            t = int(toks[b, j])
            if t == 32006:  # pad after EOS
                continue
            row = o[b, j]
            margin = 0.05 * float(row.std()) + 1e-3
            s = R.penalise(row, seen, repetition_penalty)
            if do_sample:
                s = s / temperature
                s[t] += margin / temperature
                keep, _ = R.kept_set(s, top_k, top_p)
                assert keep[t], (b, j, t)
            else:
                assert s.max() - s[t] <= margin, (b, j, t, int(s.argmax()))
            seen[t] = True


def test_top_k_1_is_greedy(tiny):
    model, _, _, _, dev_inp = tiny
    greedy = model.engine.generate(dev_inp, max_new_tokens=6)
    sampled = model.engine.generate(dev_inp, max_new_tokens=6, do_sample=True, top_k=1, seed=5)
    assert torch.equal(greedy, sampled), (greedy, sampled)


def test_seeded_generation_is_deterministic_across_graph_replay(tiny):
    model, _, _, _, dev_inp = tiny
    eng = model.engine
    cfg = dict(max_new_tokens=12, do_sample=True, temperature=1.5, top_k=0, top_p=1.0, repetition_penalty=1.1)
    eng.generate(dev_inp, max_new_tokens=12)  # a greedy graph is cached: the sampled call below captures its own
    first = eng.generate(dev_inp, seed=77, **cfg)  # eager first step + capture
    again = eng.generate(dev_inp, seed=77, **cfg)  # graph replay
    other = eng.generate(dev_inp, seed=78, **cfg)
    assert first.shape[1] == 12
    assert torch.equal(first, again)
    assert not torch.equal(first, other)
    # the public surface: llm.generation_config, seeded by torch's default generator when no seed is given
    gc = model.llm.generation_config
    saved = (gc.do_sample, gc.temperature, gc.top_k)
    try:
        gc.do_sample, gc.temperature, gc.top_k = True, 1.5, 0
        torch.manual_seed(2024)
        a = model(dict(dev_inp, inference=True, max_new_tokens=12))
        b = model(dict(dev_inp, inference=True, max_new_tokens=12))
        torch.manual_seed(2024)
        c = model(dict(dev_inp, inference=True, max_new_tokens=12))
    finally:
        gc.do_sample, gc.temperature, gc.top_k = saved
    assert torch.equal(a, c) and not torch.equal(a, b)


def test_sampled_tokens_lie_in_the_oracle_kept_set(tiny):
    model, _, _, _, dev_inp = tiny
    cfg = dict(do_sample=True, temperature=0.9, top_k=50, top_p=0.6, repetition_penalty=1.2)
    for seed in (1, 2):
        toks = model.engine.generate(dev_inp, max_new_tokens=6, seed=seed, **cfg)
        _check_teacher_forced(tiny, toks, **cfg)


def test_greedy_with_repetition_penalty_vs_oracle(tiny):
    model, _, _, _, dev_inp = tiny
    toks = model.engine.generate(dev_inp, max_new_tokens=6, repetition_penalty=1.3)
    _check_teacher_forced(tiny, toks, do_sample=False, repetition_penalty=1.3)


def test_default_generation_config_is_todays_greedy(tiny):
    model, _, _, _, dev_inp = tiny
    from macaw_llm_b200.modeling import generation_settings

    assert generation_settings(model.llm.generation_config)["do_sample"] is False
    toks = model(dict(dev_inp, inference=True, max_new_tokens=6))
    assert torch.equal(toks, model.engine.generate(dev_inp, max_new_tokens=6))
