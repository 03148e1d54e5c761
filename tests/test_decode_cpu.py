"""CPU tier of the decode tests: the KV-cached fp64 reference (tests/decode_reference.py) equals the oracle's full
recompute (`oracle.macaw_oracle.llama_forward` over the whole extended sequence, no mask), so the GPU tier's comparisons
against it are comparisons against the oracle.  The runs cross position 64 (the attention kernel's key tile)."""
import pytest
import torch

from oracle import macaw_oracle as O
from tests import decode_reference as R


def _random_decoder(E, H, L, I, V, seed):
    """Random decoder state dict in the MM_LLMs key layout (norm gains away from 1 so their placement matters)."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s, std=0.02: torch.randn(*s, generator=g, dtype=torch.float64) * std  # noqa: E731
    sd = {"llm.model.embed_tokens.weight": rnd(V, E, std=1.0), "llm.lm_head.weight": rnd(V, E),
          "llm.model.norm.weight": 1.0 + rnd(E, std=0.1)}
    for i in range(L):
        p = f"llm.model.layers.{i}."
        sd[p + "input_layernorm.weight"] = 1.0 + rnd(E, std=0.1)
        sd[p + "post_attention_layernorm.weight"] = 1.0 + rnd(E, std=0.1)
        for n in ("q", "k", "v", "o"):
            sd[p + f"self_attn.{n}_proj.weight"] = rnd(E, E, std=E ** -0.5)
        sd[p + "mlp.gate_proj.weight"] = rnd(I, E, std=E ** -0.5)
        sd[p + "mlp.up_proj.weight"] = rnd(I, E, std=E ** -0.5)
        sd[p + "mlp.down_proj.weight"] = rnd(E, I, std=I ** -0.5)
    hp = dict(llama=dict(hidden=E, layers=L, heads=H, eps=1e-6, vocab=V))
    return sd, hp


@pytest.mark.parametrize("E,H,L,I,V", [(256, 2, 2, 512, 512),    # the tiny golden config's decoder
                                       (512, 4, 3, 1024, 640)])  # wider, more heads, deeper
def test_cached_decode_equals_full_recompute(E, H, L, I, V):
    B, T0, n = 2, 23, 50  # the last step attends over 73 keys
    sd, hp = _random_decoder(E, H, L, I, V, seed=E + L)
    g = torch.Generator().manual_seed(7)
    prompt = torch.randint(0, V, (B, T0), generator=g)
    toks = torch.randint(0, V, (B, n), generator=g)
    toks[0, 5] = V + 6  # an id past the table (a finished row's pad) reads the last row, as generate clamps it
    table = sd["llm.model.embed_tokens.weight"]
    pre, steps = R.decode_logits(sd, hp, table[prompt], toks)
    assert pre.dtype == torch.float64 and tuple(pre.shape) == (B, T0, V) and tuple(steps.shape) == (B, n + 1, V)
    seq = torch.cat([prompt, toks.clamp(max=V - 1)], dim=1)
    with torch.no_grad():
        full = O.llama_forward(table[seq], None, O._SD(sd, torch.float64), hp)
    scale = float(full.abs().max())
    d_pre = float((pre - full[:, :T0]).abs().max()) / scale
    d_steps = float((steps - full[:, T0 - 1:T0 + n]).abs().max()) / scale
    print(f"\n[decode reference E={E}] max |cached - full| / max |full|: prefill {d_pre:.1e}, steps {d_steps:.1e}")
    assert d_pre < 1e-12 and d_steps < 1e-12


def test_rope_tables_are_the_oracles_angles():
    """The reference's fp32 tables are the oracle's cos / sin (its cos(emb) halves) bit for bit."""
    hd, T = 128, 2048
    cos, sin = R.rope_tables(T, hd)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
    freqs = torch.arange(T).float()[:, None] * inv_freq[None]
    emb = torch.cat([freqs, freqs], dim=-1)
    assert cos.dtype == torch.float32 and torch.equal(torch.cat([cos, cos], -1), emb.cos())
    assert torch.equal(torch.cat([sin, sin], -1), emb.sin())
