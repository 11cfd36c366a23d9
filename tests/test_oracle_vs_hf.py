"""Pins oracle/model_ref.py against transformers' own model classes on the same seeded
weights (the reference repo holds no model code or golden vectors — SURVEY.md §8c)."""
import pytest
import torch

from oracle.model_ref import RefModel
from sutro_b200 import modelspec as MS


def hf_config(spec):
    """(transformers config, causal-LM class) of a spec."""
    import transformers
    common = dict(vocab_size=spec.vocab_size, hidden_size=spec.d_model,
                  intermediate_size=spec.d_ff, num_hidden_layers=spec.n_layers,
                  num_attention_heads=spec.n_q_heads, num_key_value_heads=spec.n_kv_heads,
                  head_dim=spec.head_dim, max_position_embeddings=spec.max_position,
                  rms_norm_eps=spec.rms_eps, tie_word_embeddings=spec.tied_embeddings,
                  attention_bias=False, attn_implementation="eager")
    if spec.family == "qwen3":
        cfg = transformers.Qwen3Config(rope_theta=spec.rope_theta, **common)
        cls = transformers.Qwen3ForCausalLM
    else:
        rp = {"rope_type": "llama3", "rope_theta": spec.rope_theta, **spec.rope_scaling}
        cfg = transformers.LlamaConfig(rope_parameters=rp, mlp_bias=False, **common)
        cls = transformers.LlamaForCausalLM
    return cfg, cls


def hf_model(spec, weights):
    cfg, cls = hf_config(spec)
    m = cls(cfg).eval()
    sd = {k: v.float() for k, v in weights.items()}
    if spec.tied_embeddings:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in k or "inv_freq" in k for k in missing), missing
    return m


@pytest.mark.parametrize("name", ["tiny-qwen3", "tiny-qwen3-g4", "tiny-llama"])
def test_oracle_logits_match_transformers(name):
    spec = MS.get_spec(name)
    w = MS.make_weights(spec, seed=3, std=0.05)
    ids = torch.randint(0, spec.vocab_size, (40,), generator=torch.Generator().manual_seed(1))
    ref = RefModel(spec, w).logits(ids.tolist())
    m = hf_model(spec, w)
    with torch.no_grad():
        hf32 = m(ids[None]).logits[0]
    scale = hf32.std().item()
    # fp32 transformers vs bf16-rounded oracle: bf16 noise only
    assert (ref - hf32).abs().max().item() < 0.1 * scale
    assert (ref - hf32).abs().mean().item() < 0.015 * scale
    # bf16 transformers rounds at the same op boundaries as the oracle
    with torch.no_grad():
        hf16 = m.to(torch.bfloat16)(ids[None]).logits[0].float()
    assert (ref - hf16).abs().max().item() < 0.1 * scale
    # decisions agree wherever the fp32 model's top-1 margin is not tiny
    top2 = hf32.topk(2, dim=-1).values
    decided = (top2[:, 0] - top2[:, 1]) > 0.05 * scale
    assert decided.float().mean() > 0.5
    assert torch.equal(ref.argmax(-1)[decided], hf32.argmax(-1)[decided])


def test_rope_inv_freq_matches_transformers_llama3():
    spec = MS.get_spec("tiny-llama")
    m = hf_model(spec, MS.make_weights(spec, seed=0))
    assert torch.equal(m.model.rotary_emb.inv_freq.float(), MS.rope_inv_freq(spec))


@pytest.mark.parametrize("name", ["qwen-3-4b", "llama-3.1-8b"])
def test_rope_tables_match_transformers_at_every_position(name):
    """The engine's bf16 cos/sin tables (MS.rope_tables) at all 32,768 positions equal the ones
    transformers' rotary-embedding module gives a bf16 model.  The only element allowed to differ
    is one whose fp32 value lies within one fp32 ulp of a bf16 rounding midpoint, where the fp32
    cos/sin of either side may round the other way; such elements are counted."""
    import transformers
    spec = MS.get_spec(name)
    cfg, _ = hf_config(spec)
    mod = {"qwen3": transformers.models.qwen3.modeling_qwen3.Qwen3RotaryEmbedding,
           "llama": transformers.models.llama.modeling_llama.LlamaRotaryEmbedding}[spec.family]
    rot = mod(cfg)
    n, half = MS.CONTEXT_WINDOW, spec.head_dim // 2
    assert spec.max_position == n == 32768
    pos = torch.arange(n)[None]
    with torch.no_grad():
        hf32 = rot(torch.zeros(1, dtype=torch.float32), pos)
        hf16 = rot(torch.zeros(1, dtype=torch.bfloat16), pos)
    cos, sin = MS.rope_tables(spec, n)
    assert cos.shape == sin.shape == (n, half) and cos.dtype == torch.bfloat16
    near_mid = 0
    for what, mine, h32, h16 in (("cos", cos, hf32[0][0], hf16[0][0]),
                                 ("sin", sin, hf32[1][0], hf16[1][0])):
        assert h16.dtype == torch.bfloat16
        assert torch.equal(h16[:, :half], h16[:, half:])          # rotate_half layout
        diff = mine.view(torch.int16) != h16[:, :half].view(torch.int16)
        low = h32[:, :half].contiguous().view(torch.int32) & 0xFFFF
        mid = (low - 0x8000).abs() <= 1
        assert not (diff & ~mid).any(), (what, diff.nonzero()[:5].tolist())
        near_mid += int(diff.sum())
    print("ROPE_TABLES", name, f"positions={n}", f"near_midpoint_differences={near_mid}")


def test_fast_mode_is_the_same_model():
    """RefModel(fast=True) (fp32-cached weights, used by the CPU baseline) == default."""
    spec = MS.get_spec("tiny-qwen3")
    w = MS.make_weights(spec, seed=1, std=0.05)
    ids = list(range(5, 40))
    a = RefModel(spec, w).logits(ids)
    b = RefModel(spec, w, fast=True).logits(ids)
    assert torch.equal(a, b)
