"""Opt-in context windows past 32,768 tokens: which windows each model accepts, the YaRN RoPE
tables they switch Qwen3 to, the prefill budget they default to, and the config loader."""
import pytest
import torch

from oracle.model_ref import RefModel
from sutro_b200 import modelspec as MS
from sutro_b200 import pretrained as PT
from sutro_b200.engine import default_max_prefill_tokens


def _yarn(k, old):
    return {"rope_type": "yarn", "factor": float(k), "original_max_position_embeddings": old}


# --------------------------------------------------------------------------- option rules
@pytest.mark.parametrize("name", ["llama-3.1-8b", "llama-3-8b", "qwen-3-4b", "qwen-3-14b",
                                  "qwen-3-4b-thinking", "qwen-3-14b-thinking"])
def test_131072_is_accepted(name):
    base = MS.get_spec(name)
    spec = MS.with_window(base, 131072)
    assert spec.max_position == 131072
    if base.family == "llama":
        assert spec.rope_scaling == base.rope_scaling       # RoPE unchanged
    else:
        assert spec.rope_scaling == _yarn(4, 32768)
    assert default_max_prefill_tokens(spec) == 32768


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("name", ["qwen-3-4b", "qwen-3-14b"])
def test_qwen3_yarn_factor_is_the_window_multiple(name, k):
    spec = MS.with_window(MS.get_spec(name), k * 32768)
    assert spec.rope_scaling == _yarn(k, 32768) and spec.max_position == k * 32768


@pytest.mark.parametrize("name,window", [
    ("qwen-3-4b", 40000), ("qwen-3-14b", 40000), ("llama-3.1-8b", 131073),
    ("qwen-3-4b", 131073), ("qwen-3-4b", 5 * 32768), ("qwen-3-0.6b", 32769),
    ("qwen-3-0.6b", 65536), ("qwen-3-embedding-0.6b", 32769), ("qwen-3-embedding-0.6b", 131072),
    ("tiny-qwen3", 600), ("tiny-qwen3", 5 * 512), ("tiny-llama", 4 * 512 + 1),
    ("qwen-3-4b", 0)])
def test_windows_outside_the_limits_raise(name, window):
    with pytest.raises(ValueError):
        MS.with_window(MS.get_spec(name), window)


def test_the_error_names_the_limit():
    with pytest.raises(ValueError, match="131072"):
        MS.with_window(MS.get_spec("llama-3.1-8b"), 131073)
    with pytest.raises(ValueError, match="32768"):
        MS.with_window(MS.get_spec("qwen-3-0.6b"), 65536)


@pytest.mark.parametrize("name", sorted(MS.SPECS))
def test_no_option_is_the_registered_spec(name):
    spec = MS.get_spec(name)
    assert MS.with_window(spec, None) is spec
    assert MS.with_window(spec, spec.max_position) is spec


@pytest.mark.parametrize("name,window,yarn", [
    ("tiny-qwen3", 2048, 4), ("tiny-qwen3", 1024, 2), ("tiny-qwen3-g4", 4096, 4),
    ("tiny-qwen3-g5", 3072, 3), ("tiny-qwen3-embedding", 2048, 4), ("tiny-llama", 2048, None),
    ("tiny-llama", 1500, None)])
def test_tiny_models_go_to_four_times_their_window(name, window, yarn):
    base = MS.get_spec(name)
    spec = MS.with_window(base, window)
    assert spec.max_position == window
    want = base.rope_scaling if yarn is None else _yarn(yarn, base.max_position)
    assert spec.rope_scaling == want


@pytest.mark.parametrize("window,want", [(512, 8192), (8192, 8192), (16384, 16384),
                                         (32768, 32768), (65536, 32768), (98304, 32768),
                                         (131072, 32768)])
def test_default_prefill_budget(window, want):
    spec = MS.with_window(MS.get_spec("qwen-3-4b"), window)
    assert default_max_prefill_tokens(spec) == want


# --------------------------------------------------------------------------- config loader
def _qwen_cfg(**extra):
    cfg = {"model_type": "qwen3", "hidden_size": 2560, "num_attention_heads": 32,
           "num_key_value_heads": 8, "head_dim": 128, "num_hidden_layers": 36,
           "intermediate_size": 9728, "vocab_size": 151936, "tie_word_embeddings": True,
           "rms_norm_eps": 1e-6, "rope_theta": 1e6, "max_position_embeddings": 40960}
    cfg.update(extra)
    return cfg


PUBLISHED_YARN = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}


def test_loader_accepts_qwens_published_yarn_entry():
    cfg = _qwen_cfg(rope_scaling=dict(PUBLISHED_YARN))
    spec = PT.spec_from_hf_config(cfg, "qwen-3-4b", max_position=131072)
    assert spec.max_position == 131072 and spec.rope_scaling == _yarn(4, 32768)
    # the registered spec at the same window is the same model
    assert spec == MS.with_window(MS.get_spec("qwen-3-4b"), 131072)
    # without the option the window stays 32,768, with the config's YaRN
    spec = PT.spec_from_hf_config(cfg, "qwen-3-4b")
    assert spec.max_position == 32768 and spec.rope_scaling == _yarn(4, 32768)


@pytest.mark.parametrize("scaling,window", [
    ({"rope_type": "yarn", "factor": 4}, 32768),
    ({"rope_type": "yarn", "original_max_position_embeddings": 32768}, 32768),
    ({**PUBLISHED_YARN, "mscale": 0.707}, 32768),
    ({**PUBLISHED_YARN, "attention_factor": 1.2}, 32768),
    ({**PUBLISHED_YARN, "beta_fast": 16}, 32768),
    ({**PUBLISHED_YARN, "factor": 2.0}, 131072),
    (dict(PUBLISHED_YARN), 131073),
    ({"rope_type": "dynamic", "factor": 4.0}, 32768)])
def test_loader_refuses_incomplete_unknown_or_too_small_yarn(scaling, window):
    with pytest.raises(ValueError):
        PT.spec_from_hf_config(_qwen_cfg(rope_scaling=scaling), "m", max_position=window)


# --------------------------------------------------------------------------- YaRN tables
def _hf_rotary(spec):
    import transformers
    rp = {"rope_theta": spec.rope_theta, **spec.rope_scaling}
    cfg = transformers.Qwen3Config(
        vocab_size=spec.vocab_size, hidden_size=spec.d_model, intermediate_size=spec.d_ff,
        num_hidden_layers=spec.n_layers, num_attention_heads=spec.n_q_heads,
        num_key_value_heads=spec.n_kv_heads, head_dim=spec.head_dim,
        max_position_embeddings=spec.max_position, rms_norm_eps=spec.rms_eps,
        tie_word_embeddings=spec.tied_embeddings, attention_bias=False,
        attn_implementation="eager", rope_parameters=rp)
    return cfg


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("name", ["qwen-3-4b", "qwen-3-14b"])
def test_yarn_tables_match_transformers_at_every_position(name, k):
    """bf16 cos/sin at every position below 131,072 equal those of transformers'
    Qwen3RotaryEmbedding with a yarn rope type.  Only an element whose fp32 value lies within one
    fp32 ulp of a bf16 rounding midpoint may differ; such elements are counted."""
    import transformers
    spec = MS.with_window(MS.get_spec(name), k * 32768)
    rot = transformers.models.qwen3.modeling_qwen3.Qwen3RotaryEmbedding(_hf_rotary(spec))
    assert torch.equal(rot.inv_freq.float(), MS.rope_inv_freq(spec))
    assert rot.attention_scaling == pytest.approx(MS.rope_attention_factor(spec), abs=0)
    n, half = 131072, spec.head_dim // 2
    pos = torch.arange(n)[None]
    with torch.no_grad():
        hf32 = rot(torch.zeros(1, dtype=torch.float32), pos)
        hf16 = rot(torch.zeros(1, dtype=torch.bfloat16), pos)
    cos, sin = MS.rope_tables(spec, n)
    assert cos.shape == sin.shape == (n, half) and cos.dtype == torch.bfloat16
    near_mid = 0
    for what, mine, h32, h16 in (("cos", cos, hf32[0][0], hf16[0][0]),
                                 ("sin", sin, hf32[1][0], hf16[1][0])):
        assert torch.equal(h16[:, :half], h16[:, half:])
        diff = mine.view(torch.int16) != h16[:, :half].view(torch.int16)
        low = h32[:, :half].contiguous().view(torch.int32) & 0xFFFF
        mid = (low - 0x8000).abs() <= 1
        assert not (diff & ~mid).any(), (what, diff.nonzero()[:5].tolist())
        near_mid += int(diff.sum())
    print("YARN_TABLES", name, f"factor={k}", f"positions={n}",
          f"near_midpoint_differences={near_mid}")


def test_yarn_changes_short_rows_too():
    """YaRN rescales every position (and the attention factor scales cos/sin at position 0), so
    a window past 32,768 changes the tables from position 0 on: the reason it is opt-in."""
    base = MS.get_spec("qwen-3-4b")
    c0, _ = MS.rope_tables(base, 16)
    c1, _ = MS.rope_tables(MS.with_window(base, 131072), 16)
    assert not torch.equal(c0, c1)
    llama = MS.get_spec("llama-3.1-8b")
    assert torch.equal(MS.rope_tables(llama, 4096)[0],
                       MS.rope_tables(MS.with_window(llama, 131072), 4096)[0])


def test_oracle_matches_transformers_on_a_tiny_yarn_model():
    """RefModel on tiny-qwen3 at 2,048 positions (YaRN x4 over 512) against Qwen3ForCausalLM
    with the same yarn rope_parameters, on a 2,000-token row, in fp32 and bf16.  transformers'
    bf16 model drifts from its own fp32 model at this length (about 1.6 sigma at worst, with or
    without YaRN), so in bf16 the oracle must be no farther from it than its fp32 model is."""
    import transformers
    spec = MS.with_window(MS.get_spec("tiny-qwen3"), 2048)
    w = MS.make_weights(spec, seed=3, std=0.05)
    ids = torch.randint(0, spec.vocab_size, (2000,), generator=torch.Generator().manual_seed(7))
    ref = RefModel(spec, w).logits(ids.tolist())
    m = transformers.Qwen3ForCausalLM(_hf_rotary(spec)).eval()
    sd = {k: v.float() for k, v in w.items()}
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), missing
    with torch.no_grad():
        hf32 = m(ids[None]).logits[0].float()
        hf16 = m.to(torch.bfloat16)(ids[None]).logits[0].float()
    scale = hf32.std().item()
    assert (ref - hf32).abs().max().item() < 0.12 * scale
    assert (ref - hf32).abs().mean().item() < 0.015 * scale
    top2 = hf32.topk(2, dim=-1).values
    decided = (top2[:, 0] - top2[:, 1]) > 0.05 * scale
    assert decided.float().mean() > 0.5
    assert torch.equal(ref.argmax(-1)[decided], hf32.argmax(-1)[decided])
    assert (ref - hf16).abs().max() <= 1.05 * (hf32 - hf16).abs().max()
    assert (ref - hf16).abs().mean() <= 1.05 * (hf32 - hf16).abs().mean()


# --------------------------------------------------------------------------- load_pretrained
@pytest.mark.parametrize("name", ["qwen-3-4b", "qwen-3-14b-thinking"])
def test_loader_applies_the_window_rules_to_a_stock_qwen3_config(name):
    """Qwen3's stock config.json has no rope_scaling and max_position_embeddings 40960: asking
    for 131,072 switches it to YaRN x4 over 32,768, as for the registered model."""
    base = MS.get_spec(name)
    cfg = _qwen_cfg(hidden_size=base.d_model, num_attention_heads=base.n_q_heads,
                    num_hidden_layers=base.n_layers, intermediate_size=base.d_ff,
                    tie_word_embeddings=base.tied_embeddings)
    spec = PT.spec_from_hf_config(cfg, name, max_position=131072)
    assert spec.max_position == 131072 and spec.rope_scaling == _yarn(4, 32768)
    assert spec.name == name
    assert PT.spec_from_hf_config(cfg, name).max_position == 32768     # no option: unchanged
    with pytest.raises(ValueError, match="32768"):
        PT.spec_from_hf_config(cfg, name, max_position=40000)


def test_loader_refuses_a_long_window_for_an_unregistered_model():
    with pytest.raises(ValueError, match="40960"):
        PT.spec_from_hf_config(_qwen_cfg(), "my-finetune", max_position=131072)
    # a window up to 32,768 keeps being capped by the config, as before
    assert PT.spec_from_hf_config(_qwen_cfg(max_position_embeddings=2048), "m",
                                  max_position=4096).max_position == 2048


def test_loader_llama_131072_keeps_its_rope():
    cfg = {"model_type": "llama", "hidden_size": 4096, "num_attention_heads": 32,
           "num_key_value_heads": 8, "num_hidden_layers": 32, "intermediate_size": 14336,
           "vocab_size": 128256, "rms_norm_eps": 1e-5, "rope_theta": 5e5,
           "max_position_embeddings": 131072,
           "rope_scaling": {"rope_type": "llama3", **MS.LLAMA31_8B.rope_scaling}}
    spec = PT.spec_from_hf_config(cfg, "llama-3.1-8b", max_position=131072)
    assert spec == MS.with_window(MS.get_spec("llama-3.1-8b"), 131072)
