"""Loading real checkpoints (sutro_b200/pretrained.py), checked on CPU with files written by
the Hugging Face libraries themselves: `tokenizers` saves a tokenizer.json whose byte tokens
sit in GPT-2 order (not byte order), `safetensors` saves the weights, and the loader's output is
compared with what those libraries read back."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.bpe_ref import RefTokenizer
from sutro_b200 import modelspec as MS, pretrained as PT, vocab as VB

TEXTS = ["Hello, world!", "  leading spaces and 12345 numbers", "naïve café — “quotes”…",
         "日本語のテキスト 🙂", "tabs\tand\nnewlines\r\n", "it's the model's 1st re-run", ""]


ROWS_TXT = ["Great camera and build quality, would buy again!", "don't DON'T we'LL 1234567 3.14",
            "unicode: café naïve Straße 東京 ½ 🙂 end", "   ", "\n\n a"]


def gpt2_ordered_tokenizer(v: VB.Vocab):
    """A `tokenizers.Tokenizer` over the same merges whose ids follow the GPT-2 convention:
    byte tokens 0..255 in bytes_to_unicode order, merge results in rank order after them."""
    from tokenizers import AddedToken, Regex, Tokenizer, decoders, models, pre_tokenizers
    b2u = VB._bytes_to_unicode()
    order = list(b2u.keys())                                   # GPT-2's byte order

    def s(b: bytes) -> str:
        return "".join(b2u[x] for x in b)

    vocab = {b2u[b]: i for i, b in enumerate(order)}
    merges = []
    for a, b in v.merges:
        sa, sb = s(v.token_bytes[a]), s(v.token_bytes[b])
        if sa + sb not in vocab:
            vocab[sa + sb] = len(vocab)
        merges.append((sa, sb))
    tok = Tokenizer(models.BPE(vocab=vocab, merges=merges, fuse_unk=False, byte_fallback=False))
    tok.pre_tokenizer = pre_tokenizers.Sequence([
        pre_tokenizers.Split(Regex(VB.PRETOK_PATTERN % v.digits), behavior="isolated", invert=False),
        pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    names = [n for n, _ in sorted(v.specials.items(), key=lambda kv: kv[1])][:5]
    tok.add_special_tokens([AddedToken(n, special=True, normalized=False) for n in names])
    return tok


@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_tokenizer_json_round_trip_in_gpt2_byte_order(tmp_path, family):
    v = VB.build_vocab(family, 2048, seed=0, n_trained=600)
    hf = gpt2_ordered_tokenizer(v)
    path = str(tmp_path / "tokenizer.json")
    hf.save(path)
    loaded = PT.load_tokenizer_json(path, family, vocab_size=hf.get_vocab_size() + 11)
    assert loaded.vocab_size == hf.get_vocab_size() + 11
    assert [loaded.token_bytes[b] for b in range(256)] == [bytes([b]) for b in range(256)]
    assert sorted(loaded.id_map[:256].tolist()) == list(range(256))
    assert not np.array_equal(loaded.id_map[:256], np.arange(256))      # GPT-2 order != byte order
    assert np.array_equal(loaded.id_map[256:], np.arange(256, loaded.vocab_size))
    assert len(loaded.merges) == len(loaded.merged_ids) > 500
    ref = RefTokenizer(loaded)                       # the oracle the GPU tokenizer is tested against
    for text in TEXTS:
        engine_ids = ref.encode(text)
        assert loaded.to_real_ids(engine_ids) == hf.encode(text, add_special_tokens=False).ids
        assert loaded.decode(engine_ids).decode("utf-8") == text
    eos = "<|im_end|>" if family == "qwen3" else "<|eot_id|>"
    assert loaded.to_real_ids([loaded.eos_id]) == [hf.token_to_id(eos)]


def test_tokenizer_json_rejects_other_layouts(tmp_path):
    p = tmp_path / "t.json"
    p.write_text(json.dumps({"model": {"type": "Unigram", "vocab": []}}))
    with pytest.raises(ValueError):
        PT.load_tokenizer_json(str(p), "qwen3")
    p.write_text(json.dumps({"model": {"type": "BPE", "vocab": {"a": 0, "b": 1}, "merges": []},
                             "added_tokens": []}))
    with pytest.raises(ValueError):
        PT.load_tokenizer_json(str(p), "qwen3")      # the 256 byte tokens are not there


def hf_config(spec: MS.ModelSpec):
    cfg = {"model_type": "qwen3" if spec.family == "qwen3" else "llama",
           "hidden_size": spec.d_model, "num_attention_heads": spec.n_q_heads,
           "num_key_value_heads": spec.n_kv_heads, "head_dim": spec.head_dim,
           "num_hidden_layers": spec.n_layers, "intermediate_size": spec.d_ff,
           "vocab_size": spec.vocab_size, "tie_word_embeddings": spec.tied_embeddings,
           "rms_norm_eps": spec.rms_eps, "rope_theta": spec.rope_theta,
           "max_position_embeddings": 40960}
    if spec.rope_scaling:
        cfg["rope_scaling"] = dict(spec.rope_scaling, rope_type="llama3")
    return cfg


@pytest.mark.parametrize("name", ["tiny-qwen3", "tiny-llama", "qwen-3-4b", "llama-3.1-8b"])
def test_spec_from_hf_config(name):
    spec = MS.get_spec(name)
    got = PT.spec_from_hf_config(hf_config(spec), name, max_position=spec.max_position)
    assert got == spec
    # the same numbers transformers' config classes carry for the real models
    if name == "qwen-3-4b":
        from transformers import Qwen3Config
        c = Qwen3Config(hidden_size=2560, num_attention_heads=32, num_key_value_heads=8,
                        num_hidden_layers=36, intermediate_size=9728, vocab_size=151936,
                        tie_word_embeddings=True, rope_theta=1e6, head_dim=128)
        assert PT.spec_from_hf_config(c.to_dict(), name).n_params() == spec.n_params()


@pytest.mark.parametrize("bad", [{"model_type": "gemma3"}, {"head_dim": 64},
                                 {"num_key_value_heads": 3, "num_attention_heads": 9},
                                 {"attention_bias": True},
                                 {"rope_scaling": {"rope_type": "yarn", "factor": 4}}])
def test_unsupported_architectures_are_refused(bad):
    cfg = dict(hf_config(MS.get_spec("tiny-qwen3")), **bad)
    with pytest.raises(ValueError):
        PT.spec_from_hf_config(cfg, "x")


def test_safetensors_checkpoint_and_row_permutation(tmp_path):
    from safetensors.torch import save_file
    spec = MS.get_spec("tiny-llama")
    w = MS.make_weights(spec, seed=5)
    names = sorted(w)
    half = len(names) // 2
    save_file({k: w[k] for k in names[:half]}, str(tmp_path / "model-00001-of-00002.safetensors"))
    save_file({k: w[k] for k in names[half:]}, str(tmp_path / "model-00002-of-00002.safetensors"))
    (tmp_path / "model.safetensors.index.json").write_text(json.dumps({"weight_map": {
        k: ("model-00001-of-00002.safetensors" if i < half else "model-00002-of-00002.safetensors")
        for i, k in enumerate(names)}}))
    got = PT.load_hf_weights(str(tmp_path))
    assert sorted(got) == names and all(torch.equal(got[k], w[k]) for k in names)
    perm = np.arange(spec.vocab_size, dtype=np.int32)
    perm[:256] = np.random.RandomState(0).permutation(256)
    ew = MS.pack_for_engine(spec, got, "cpu", row_map=perm)
    assert torch.equal(ew.embed[7], w["model.embed_tokens.weight"][perm[7]])
    assert torch.equal(ew.lm_head[300], w["lm_head.weight"][300])
    plain = MS.pack_for_engine(spec, got, "cpu")
    assert torch.equal(plain.embed, w["model.embed_tokens.weight"])
    with pytest.raises(FileNotFoundError):
        PT.load_hf_weights(str(tmp_path / "nowhere"))


def test_real_pretokenizer_patterns_and_normalizers(tmp_path):
    """The Split regex as Qwen2/3 and Llama-3 files spell it, NFC normalizer, and refusals."""
    v = VB.build_vocab("qwen3", 2048, seed=0, n_trained=600)
    hf = gpt2_ordered_tokenizer(v)
    path = str(tmp_path / "tokenizer.json")
    hf.save(path)
    tj = json.load(open(path))
    qwen_rx = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*"
               r"|\s*[\r\n]+|\s+(?!\S)|\s+")
    tj["pre_tokenizer"]["pretokenizers"][0]["pattern"] = {"Regex": qwen_rx}
    tj["normalizer"] = {"type": "NFC"}
    json.dump(tj, open(path, "w"))
    loaded = PT.load_tokenizer_json(path, "qwen3")
    assert loaded.digits == 1 and loaded.normalize_nfc
    tj["pre_tokenizer"]["pretokenizers"][0]["pattern"] = {"Regex": qwen_rx.replace(r"\p{N}|", r"\p{N}{1,3}|")}
    tj["normalizer"] = None
    json.dump(tj, open(path, "w"))
    assert PT.load_tokenizer_json(path, "qwen3").digits == 3
    tj["pre_tokenizer"]["pretokenizers"][0]["pattern"] = {"Regex": r"\w+|\s+"}
    json.dump(tj, open(path, "w"))
    with pytest.raises(ValueError):
        PT.load_tokenizer_json(path, "qwen3")
    tj["pre_tokenizer"] = None
    tj["normalizer"] = {"type": "Lowercase"}
    json.dump(tj, open(path, "w"))
    with pytest.raises(ValueError):
        PT.load_tokenizer_json(path, "qwen3")
    from sutro_b200.engine import _nfc_rows
    assert _nfc_rows(["é", None, "plain", 3]) == ["é", None, "plain", 3]
    import pandas as pd
    import pyarrow as pa
    from sutro_b200.engine import normalize_rows
    # every input form the entry points accept comes out composed; without the flag, untouched
    rows = ["e\u0301", None, "A\u030a", "\u1100\u1161\u11a8"]
    want = ["\u00e9", None, "\u00c5", "\uac01"]
    assert normalize_rows(rows, loaded) == want
    assert normalize_rows(tuple(rows), loaded) == want
    assert normalize_rows(pd.Series(rows[2:]), loaded) == want[2:]
    assert normalize_rows(pa.array(rows), loaded).to_pylist() == want
    assert normalize_rows(pa.chunked_array([rows[:1], rows[1:]]), loaded).to_pylist() == want
    assert normalize_rows(pa.array(rows, type=pa.large_string()).slice(2),
                          loaded).to_pylist() == want[2:]
    ascii_col = pa.array(["plain", None])
    assert normalize_rows(ascii_col, loaded) is ascii_col
    import dataclasses
    assert normalize_rows(rows, dataclasses.replace(loaded, normalize_nfc=False)) is rows
    assert normalize_rows(rows, None) is rows


def test_duplicate_merges_rank_at_their_last_entry(tmp_path):
    """A merge listed twice takes the rank of its last entry in `tokenizers` (the merge map is
    filled in list order); the loader and the oracle do the same."""
    from tokenizers import Tokenizer
    v = VB.build_vocab("qwen3", 2048, seed=0, n_trained=600)
    path = str(tmp_path / "tokenizer.json")
    gpt2_ordered_tokenizer(v).save(path)
    tj = json.load(open(path))
    tj["model"]["ignore_merges"] = True
    json.dump(tj, open(path, "w"))
    plain = Tokenizer.from_file(path)
    tj["model"]["merges"] = tj["model"]["merges"] + tj["model"]["merges"][:60]
    json.dump(tj, open(path, "w"))
    hf = Tokenizer.from_file(path)
    loaded = PT.load_tokenizer_json(path, "qwen3")
    ref = RefTokenizer(loaded)
    changed = 0
    for text in TEXTS + ROWS_TXT + override_texts(loaded):
        want = hf.encode(text, add_special_tokens=False).ids
        assert loaded.to_real_ids(ref.encode(text)) == want, repr(text)
        changed += want != plain.encode(text, add_special_tokens=False).ids
    assert changed >= 3       # the demoted merges do change the tokenization


def ignore_merges_vocab(tmp_path, family="llama"):
    """A tokenizer.json with model.ignore_merges = true over the synthetic vocabulary (which has
    entries that their own merges do not rebuild), the `tokenizers` object for it and the loaded
    Vocab.  Shared with the GPU test."""
    from tokenizers import Tokenizer
    v = VB.build_vocab(family, 2048, seed=0, n_trained=600)
    path = str(tmp_path / "tokenizer.json")
    gpt2_ordered_tokenizer(v).save(path)
    tj = json.load(open(path))
    tj["model"]["ignore_merges"] = True
    json.dump(tj, open(path, "w"))
    return path, Tokenizer.from_file(path), PT.load_tokenizer_json(path, family)


def override_texts(loaded):
    """Texts that exercise the whole-word rule: every overridden entry alone, glued to a
    letter, and inside a sentence."""
    texts = []
    for _, e in loaded.word_overrides:
        try:
            w = loaded.token_bytes[e].decode("utf-8")
        except UnicodeDecodeError:
            continue
        texts += [w, "x" + w, "so " + w.strip() + " and" + w + w + "."]
    return texts


def test_ignore_merges_whole_words_match_tokenizers(tmp_path):
    """Llama-3 tokenizer files set model.ignore_merges: a pre-token that is itself a vocabulary
    entry is emitted as that token without merging.  The loader lists the entries for which that
    differs from plain BPE (Vocab.word_overrides); the oracle restates the rule; both are pinned
    against `tokenizers` reading the same file."""
    import dataclasses
    path, hf, loaded = ignore_merges_vocab(tmp_path)
    assert loaded.word_overrides, "the synthetic vocabulary has entries its merges do not rebuild"
    ref = RefTokenizer(loaded)
    plain = RefTokenizer(dataclasses.replace(loaded, word_overrides=None))
    hits = 0
    for text in override_texts(loaded) + ROWS_TXT:
        want = hf.encode(text, add_special_tokens=False).ids
        assert loaded.to_real_ids(ref.encode(text)) == want, repr(text)
    for seq, e in loaded.word_overrides:
        try:
            w = loaded.token_bytes[e].decode("utf-8")
        except UnicodeDecodeError:
            continue
        if ref.pretokenize(w) == [w]:
            hits += 1
            assert ref.encode(w) == [e] and plain.encode(w) == list(seq) and len(seq) >= 2
    assert hits >= 3
    # flag absent: nothing to override, plain BPE everywhere
    tj = json.load(open(path))
    del tj["model"]["ignore_merges"]
    json.dump(tj, open(path, "w"))
    assert PT.load_tokenizer_json(path, "llama").word_overrides is None
