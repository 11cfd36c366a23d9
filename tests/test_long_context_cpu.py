"""Context windows and the defaults that must not move with them."""
import dataclasses

import pytest

from sutro_b200 import modelspec as MS
from sutro_b200 import pretrained as PT
from sutro_b200.engine import default_max_prefill_tokens
from sutro_b200.sdk import Sutro


@pytest.mark.parametrize("name", ["qwen-3-0.6b", "qwen-3-0.6B", "qwen-3-embedding-0.6b",
                                  "qwen-3-4b", "llama-3.1-8b", "llama-3-8b"])
def test_real_models_serve_32k_windows(name):
    assert MS.get_spec(name).max_position == 32768


@pytest.mark.parametrize("name,window", [("tiny-qwen3", 512), ("tiny-qwen3-g4", 1024),
                                         ("tiny-llama", 512), ("tiny-qwen3-embedding", 512)])
def test_tiny_specs_keep_their_windows(name, window):
    assert MS.get_spec(name).max_position == window


def _hf_config(max_pos=None):
    cfg = {"model_type": "qwen3", "hidden_size": 2560, "num_attention_heads": 32,
           "num_key_value_heads": 8, "head_dim": 128, "num_hidden_layers": 36,
           "intermediate_size": 9728, "vocab_size": 151936, "tie_word_embeddings": True,
           "rms_norm_eps": 1e-6, "rope_theta": 1e6}
    if max_pos is not None:
        cfg["max_position_embeddings"] = max_pos
    return cfg


@pytest.mark.parametrize("hf,cap,want", [(40960, None, 32768), (131072, None, 32768),
                                         (None, None, 32768), (2048, None, 2048),
                                         (32768, None, 32768), (40960, 4096, 4096),
                                         (1024, 4096, 1024)])
def test_spec_from_hf_config_caps_the_window(hf, cap, want):
    kw = {} if cap is None else {"max_position": cap}
    assert PT.spec_from_hf_config(_hf_config(hf), "m", **kw).max_position == want


def test_load_pretrained_default_cap_is_32k():
    import inspect
    assert inspect.signature(PT.load_pretrained).parameters["max_position"].default == 32768


class _Eng:
    def __init__(self, spec):
        self.spec = spec


@pytest.mark.parametrize("name", ["qwen-3-4b", "llama-3.1-8b", "qwen-3-0.6b"])
def test_default_output_budget_unchanged(name, monkeypatch):
    """2,048 for a schema whose longest path is longer, 512 for free text, as with 4k windows."""
    eng = _Eng(MS.get_spec(name))

    class _Dfa:
        def longest_path(self):
            return 100000

    eng.compile_schema = lambda schema, limits=None, *a: _Dfa()
    assert Sutro._default_max_new_tokens(eng, {"type": "object"}) == 2048
    assert Sutro._default_max_new_tokens(eng, None) == 512
    small = _Eng(MS.get_spec("tiny-qwen3"))
    small.compile_schema = eng.compile_schema
    assert Sutro._default_max_new_tokens(small, {"type": "object"}) == 256


@pytest.mark.parametrize("name,want", [("qwen-3-4b", 32768), ("llama-3.1-8b", 32768),
                                       ("tiny-qwen3", 8192), ("tiny-qwen3-g4", 8192)])
def test_default_max_prefill_tokens(name, want):
    assert default_max_prefill_tokens(MS.get_spec(name)) == want
    wide = dataclasses.replace(MS.get_spec(name), max_position=16384)
    assert default_max_prefill_tokens(wide) == 16384
