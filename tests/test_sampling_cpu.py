"""CPU tier of the sampled generate branch: the fp64 restatement of mm_sample_rows (tests/sampling_ref.py) against the
installed transformers' own logits processors, and the resolution of `llm.generation_config` into the decoding
arguments of Engine.generate."""
import numpy as np
import pytest
import torch
from transformers import GenerationConfig
from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                    TopKLogitsWarper, TopPLogitsWarper)

from tests import sampling_ref as R

V = 32007


def _rows(n, seed, scale):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, V)) * scale
    assert all(np.unique(r).size == V for r in x)  # tie-free
    return x


def _hf_kept(x, seen_ids, temperature, top_k, top_p, penalty):
    """The tokens HF's processor chain leaves finite, in fp64 (so that only the rule, not fp32 rounding, is compared)."""
    scores = torch.from_numpy(x)
    ids = torch.from_numpy(seen_ids)
    procs = []
    if penalty != 1.0:
        procs.append(RepetitionPenaltyLogitsProcessor(penalty))
    if temperature != 1.0:
        procs.append(TemperatureLogitsWarper(temperature))
    if top_k:
        procs.append(TopKLogitsWarper(top_k))
    if top_p < 1.0:
        procs.append(TopPLogitsWarper(top_p))
    for p in procs:
        scores = p(ids, scores)
    return torch.isfinite(scores).numpy(), scores.numpy()


@pytest.mark.parametrize("temperature,top_k,top_p,penalty", [
    (1.0, 50, 1.0, 1.0), (0.9, 50, 0.6, 1.0), (0.7, 0, 0.9, 1.0), (1.3, 200, 0.95, 1.2), (0.5, 5, 0.3, 1.0),
    (1.0, 0, 0.5, 1.5), (2.0, 1000, 0.99, 1.1), (1.0, 1, 1.0, 1.0),
])
def test_restatement_kept_sets_match_transformers(temperature, top_k, top_p, penalty):
    x = _rows(6, seed=hash((temperature, top_k, top_p, penalty)) & 0xFFFF, scale=3.0)
    rng = np.random.default_rng(7)
    seen_ids = rng.integers(0, V, (x.shape[0], 40))
    bits = np.zeros((x.shape[0], (V + 31) // 32), np.uint32)
    for r in range(x.shape[0]):
        for t in seen_ids[r]:
            bits[r, t >> 5] |= np.uint32(1 << (t & 31))
    hf_keep, hf_scores = _hf_kept(x, seen_ids, temperature, top_k, top_p, penalty)
    s = R.penalise(x, R.seen_mask(bits, V), penalty) / temperature
    for r in range(x.shape[0]):
        keep, _ = R.kept_set(s[r], top_k, top_p)
        assert np.array_equal(keep, hf_keep[r]), (r, np.flatnonzero(keep ^ hf_keep[r]))
        # and the surviving scores are HF's warped scores
        np.testing.assert_allclose(s[r][keep], hf_scores[r][keep], rtol=1e-12)


def test_inverse_cdf_draw():
    w = np.array([0.0, 1.0, 0.0, 2.0, 1.0])
    assert R.inverse_cdf(w, 0.0)[0] == 1
    assert R.inverse_cdf(w, 0.2499)[0] == 1
    assert R.inverse_cdf(w, 0.25)[0] == 3  # the first token whose cumulative mass EXCEEDS u
    assert R.inverse_cdf(w, 0.7501)[0] == 4
    assert R.inverse_cdf(w, 0.25)[1] and not R.inverse_cdf(w, 0.5)[1]


def test_uniforms_follow_the_philox_words():
    from tests.helpers import philox4x32_10

    seed, step = (5 << 32) | 77, 3
    u = R.uniforms(seed, step, 4)
    w = philox4x32_10(np.array([[step, 2, R.SID_SAMPLE, 0]], np.uint32), (77, 5))[0, 0]
    assert u[2] == (int(w) >> 8) / 2 ** 24 and np.all((0 <= u) & (u < 1))


def test_tied_group_is_kept_or_removed_whole():
    # probabilities 0.1, 0.1, 0.2, 0.6: with top_p = 0.85, 1 - top_p = 0.15 lies inside the tied pair's cumsum
    # (0.1, 0.2): HF's per-position rule would split the pair, the group rule keeps both (M(<= 0.1) = 0.2 > 0.15)
    s = np.log(np.array([0.1, 0.1, 0.2, 0.6]))
    keep, _ = R.kept_set(s, 0, 0.85)
    assert keep.tolist() == [True, True, True, True]
    keep, _ = R.kept_set(s, 0, 0.75)  # 0.25: M(<= 0.1) = 0.2 <= 0.25 -> both go
    assert keep.tolist() == [False, False, True, True]
    keep, _ = R.kept_set(s, 0, 0.0)  # the largest always stays
    assert keep.tolist() == [False, False, False, True]


# ---------------------------------------------------------------------------------------------------- generation_config
def _settings(**fields):
    from macaw_llm_b200.modeling import generation_settings

    return generation_settings(GenerationConfig(**fields))


def test_default_generation_config_is_greedy():
    from macaw_llm_b200.modeling import LlamaForCausalLM, generation_settings
    from transformers import LlamaConfig

    llm = LlamaForCausalLM(LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                       num_attention_heads=2))
    assert isinstance(llm.generation_config, GenerationConfig)
    d = GenerationConfig._get_default_generation_params()
    got = generation_settings(llm.generation_config)
    assert got == dict(do_sample=bool(d["do_sample"]), temperature=d["temperature"], top_k=d["top_k"],
                       top_p=d["top_p"], repetition_penalty=d["repetition_penalty"])
    assert got["do_sample"] is False and got["repetition_penalty"] == 1.0
    assert generation_settings(None) == got  # a model whose attribute was cleared decodes greedily too


def test_vicuna_style_generation_config():
    # a Vicuna checkpoint's generation_config.json: do_sample, temperature 0.9, top_p 0.6, top_k unset
    got = _settings(do_sample=True, temperature=0.9, top_p=0.6, max_length=4096, bos_token_id=1, eos_token_id=2,
                    pad_token_id=0)
    assert got == dict(do_sample=True, temperature=0.9, top_k=GenerationConfig._get_default_generation_params()["top_k"],
                       top_p=0.6, repetition_penalty=1.0)
    assert got["top_k"] == 50


def test_explicit_settings_pass_through():
    got = _settings(do_sample=True, temperature=0.7, top_k=0, top_p=0.95, repetition_penalty=1.3)
    assert got == dict(do_sample=True, temperature=0.7, top_k=0, top_p=0.95, repetition_penalty=1.3)


@pytest.mark.parametrize("field,value", [
    ("num_beams", 4), ("min_new_tokens", 3), ("min_length", 5), ("no_repeat_ngram_size", 3), ("typical_p", 0.9),
    ("min_p", 0.05), ("epsilon_cutoff", 3e-4), ("eta_cutoff", 3e-4), ("bad_words_ids", [[5]]),
    ("suppress_tokens", [7]), ("sequence_bias", {(5,): -1.0}), ("num_return_sequences", 2),
    ("encoder_repetition_penalty", 1.2), ("forced_eos_token_id", 2), ("renormalize_logits", True),
])
def test_unsupported_fields_are_refused(field, value):
    kw = {field: value}
    if field == "num_return_sequences":
        kw["do_sample"] = True
    with pytest.raises(NotImplementedError, match=field):
        _settings(**kw)
