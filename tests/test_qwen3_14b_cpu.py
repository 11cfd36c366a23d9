"""qwen-3-14b and the GQA group of 5 on the host side: the spec, the config loader, the launchers'
group check and the tiny G = 5 test architecture against transformers (no GPU needed)."""
import ctypes
import os

import pytest

from sutro_b200 import modelspec as MS
from sutro_b200 import pretrained as PT
import test_abi_cpu as ABI
import test_golden as GOLD
import test_oracle_vs_hf as HF
import test_pretrained_cpu as PTC


def test_qwen3_14b_spec_fields():
    s = MS.get_spec("qwen-3-14b")
    assert (s.family, s.n_layers, s.d_model, s.n_q_heads, s.n_kv_heads, s.d_ff, s.vocab_size) == \
        ("qwen3", 40, 5120, 40, 8, 17408, 151936)
    assert s.tied_embeddings is False
    assert (s.rms_eps, s.rope_theta, s.qk_norm, s.max_position) == (1e-6, 1e6, True, 32768)
    assert s.rope_scaling is None and not s.embedding_model and s.head_dim == 128
    assert s.n_params() == 14_768_307_200                     # 14.77 B
    assert s.kv_bytes_per_token == 163_840
    assert MS.get_spec("qwen-3-14b-thinking") is s


def test_tiny_g5_spec():
    s = MS.get_spec("tiny-qwen3-g5")
    assert (s.n_q_heads, s.n_kv_heads, s.family, s.max_position) == (10, 2, "qwen3", 1024)
    assert s.n_q_heads // s.n_kv_heads == 5


def test_spec_from_hf_config_accepts_group_5():
    spec = MS.get_spec("qwen-3-14b")
    assert PT.spec_from_hf_config(PTC.hf_config(spec), spec.name) == spec
    from transformers import Qwen3Config
    c = Qwen3Config(hidden_size=5120, num_attention_heads=40, num_key_value_heads=8,
                    num_hidden_layers=40, intermediate_size=17408, vocab_size=151936,
                    tie_word_embeddings=False, rope_theta=1e6, head_dim=128,
                    max_position_embeddings=40960)
    assert PT.spec_from_hf_config(c.to_dict(), spec.name).n_params() == spec.n_params()
    tiny = MS.get_spec("tiny-qwen3-g5")
    assert PT.spec_from_hf_config(PTC.hf_config(tiny), tiny.name,
                                  max_position=tiny.max_position) == tiny


@pytest.mark.parametrize("hq,hkv", [(9, 3), (12, 2), (14, 2)])
def test_spec_from_hf_config_still_rejects_groups_3_6_7(hq, hkv):
    cfg = dict(PTC.hf_config(MS.get_spec("tiny-qwen3")), num_attention_heads=hq,
               num_key_value_heads=hkv)
    with pytest.raises(ValueError, match=f"GQA group {hq}/{hkv} is not supported"):
        PT.spec_from_hf_config(cfg, "x")


@pytest.mark.skipif(not os.path.exists(ABI.LIB), reason="library not built")
@pytest.mark.parametrize("hq,hkv,G", [(12, 4, 3), (12, 2, 6), (14, 2, 7), (48, 8, 6)])
def test_attention_launchers_reject_groups_3_6_7(hq, hkv, G):
    ABI.test_attention_launchers_reject_unsupported_gqa_groups(
        hq, hkv, f"unsupported GQA group size {G}")


@pytest.mark.skipif(not os.path.exists(ABI.LIB), reason="library not built")
def test_q_tile_of_group_5():
    lib = ctypes.CDLL(ABI.LIB)
    assert lib.sb200_attn_prefill_q_tile(40, 8) == 25
    assert lib.sb200_attn_prefill_q_tile(10, 2) == 25


def test_tiny_g5_oracle_matches_transformers():
    HF.test_oracle_logits_match_transformers("tiny-qwen3-g5")


def test_tiny_g5_oracle_matches_golden_transformers_logits():
    GOLD.test_oracle_logits_match_golden_transformers_logits("tiny-qwen3-g5")
