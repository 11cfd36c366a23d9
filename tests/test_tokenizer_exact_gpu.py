"""The GPU tokenizer (csrc/tokenizer.cu: pre-tokeniser, BPE merge loop, scan + compaction,
detokeniser) checked for exact equality of token ids and bytes against `tokenizers` itself —
the library that defines the algorithm — and against the CPU oracle (oracle/bpe_ref.py).

  1  pre-tokeniser branches: a "boundary" vocabulary in which every character and every ordered
     pair of characters of an ~85-character alphabet is a token, so that a pre-token boundary
     placed anywhere else than where the library places it changes the ids; a seeded fuzz
     corpus plus hand-written cases for every alternative of the pattern
  2  the full-size vocabularies (151,936 and 128,256 entries): ~20,000 rows in one call
  3  a real tokenizer-file layout at full size (GPT-2 byte order, permuted ids), ignore_merges
     off and on
  4  layout edges of the C-ABI encode call: empty rows, an empty batch, a sliced Arrow column,
     truncated UTF-8 across rows, bytes that are not UTF-8, pre-tokens of 2,000-5,000 bytes
  5  the detokeniser's two passes against the vocabulary's byte strings
  6  decoding past 2^31 output bytes in one call
  7  NFC-normalising tokenizer files, end to end, for every input form of the entry points

Regex and `tokenizers` disagree on U+001C-U+001F (`regex` counts them as \\s); the GPU follows
`tokenizers` (tests/test_tokenizer_oracle.py), so texts containing them are compared with
`tokenizers` only."""
import functools
import json
import unicodedata

import numpy as np
import pytest
import torch

from oracle.bpe_ref import RefTokenizer
from sutro_b200 import _lib as L
from sutro_b200 import synth, vocab as VB

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
FULL = {"qwen3": 151936, "llama": 128256}

# the fuzz alphabet: each contraction letter in both cases and the long s (U+017F, which case-
# folds onto 's'); every kind of whitespace the pattern treats differently, and the separators
# that are not \s; letters (Latin, sharp s, CJK, Cyrillic, titlecase, an astral letter), numbers
# (ASCII, Arabic-Indic, a fraction, a Roman numeral), combining marks, emoji and punctuation
ALPHABET = ("sStTrReEvVmMlLdD\u017f'"
            " \r\n\t\x0b\x0c\x85\xa0\u3000\x1c\x1d\x1e\x1f"
            "azx\u00df\u00e9\u4e2d\u65e5\u0416\u044f\u01c5\U0001d4b3"
            "0159\u0661\u0662\u00bd\u216b"
            "\u0301\u0308"
            "\U0001f642\U0001f44d"
            ".,!?-\"()/:;_#@&*+=<>[]{}|~`$%^\\")
SEPARATORS = "\x1c\x1d\x1e\x1f"

# one or more cases for every alternative of the pattern
#   (?i:'s|'t|'re|'ve|'m|'ll|'d) | [^\r\n\p{L}\p{N}]?\p{L}+ | \p{N}{1,3} |
#    ?[^\s\p{L}\p{N}]+[\r\n]* | \s*[\r\n]+ | \s+(?!\S) | \s+
_CONTRACTIONS = ["'s", "'t", "'re", "'ve", "'m", "'ll", "'d"]
HAND = (
    [f"{pre}{c}{post}" for c in _CONTRACTIONS
     for c in sorted({c, c.upper(), c[:2].upper() + c[2:], c[:2] + c[2:].upper()})
     for pre, post in [("", ""), ("it", ""), ("x ", "d"), ("", "x"), ("'", "'"), ("", "1")]]
    + ["'\u017f", "'\u017fd)", "'\u017f d", "x'\u017ft", "'\u017f\u017f", "''\u017f", "'\u017f1",
       "'S\u017f", "'r", "'v", "'l", "'rx", "'lL", "'lx", "'vE", "'", "''", "'1", "' s", "'\u00e9"]
    # [^\r\n\p{L}\p{N}]?\p{L}+ with one-, two-, three- and four-byte prefixes, and without one
    + ["\u3000abc", "\u00a0\u0416\u044f", " \u4e2d\u65e5", "\u0301abc", "\U0001f642abc",
       "\x85x", "\tab", "!abc", "'abc", "\rabc", "\nabc", "1abc", "..abc", "\u01c5a\U0001d4b3",
       "\u00e9t\u00e9", "a\u0301b", "\x1cabc", "\x0bz"]
    # \p{N}{1,3}: runs of 1-7 digits
    + ["1234567"[:k] for k in range(1, 8)]
    + ["\u0661\u0662\u0661\u0662\u0661", "\u00bd\u216b12", "a123b", " 12345", "x1234567y",
       "9 99 999 9999"]
    #  ?[^\s\p{L}\p{N}]+[\r\n]*
    + [" ?!", "!!!\n\n", " ...\r\n\r\nx", "\U0001f642\U0001f44d\n", " \u0301\u0308", "x !?\r",
       "((a))", " \\/\r\r\n \n"]
    # \s*[\r\n]+
    + ["\n", "  \n", " \t\r\n\n", "\u3000\n x", "a \n\n b", "\x0b\x0c\n", "\r", "\n\n\n a",
       "\x85\n", " \n \n "]
    # \s+(?!\S) at the end and before a non-space, and a lone \s+
    + ["a   ", "a   b", "\u3000\u3000x", "\xa0\xa0\xa0!", "  \x85 z", "   ", " ", "a\t\t1",
       " 1", "a\t1", "\u3000\u00bd", "x \u0301", "\t\t\U0001f642"]
    # separators that are not \s
    + ["\x1c", "a\x1cb", " \x1f ", "\x1d\x1e1", "\x1c\n", " \x1c"]
)


def fuzz_corpus(n: int, seed: int):
    """n strings of 0-16 characters over ALPHABET (apostrophe, space and long s drawn more
    often, so contractions and their near misses are frequent)."""
    rng = np.random.RandomState(seed)
    w = np.ones(len(ALPHABET))
    for ch, weight in (("'", 8), (" ", 6), ("\u017f", 3)):
        w[ALPHABET.index(ch)] = weight
    chars = np.array(list(ALPHABET))
    return ["".join(rng.choice(chars, size=k, p=w / w.sum())) for k in rng.randint(0, 17, size=n)]


def boundary_vocab(seed: int, digits: int) -> VB.Vocab:
    """256 byte tokens; the merges that build every multi-byte character of ALPHABET (ranked
    first); then every ordered pair of characters, ranked in a seeded random order."""
    tok2id = {bytes([i]): i for i in range(256)}
    token_bytes = [bytes([i]) for i in range(256)]
    merges = []

    def add(a: bytes, b: bytes):
        if a + b not in tok2id:
            merges.append((tok2id[a], tok2id[b]))
            tok2id[a + b] = len(token_bytes)
            token_bytes.append(a + b)
    for ch in ALPHABET:
        enc = ch.encode("utf-8")
        for k in range(1, len(enc)):
            add(enc[:k], enc[k:k + 1])
    pairs = [(a.encode("utf-8"), b.encode("utf-8")) for a in ALPHABET for b in ALPHABET]
    for i in np.random.RandomState(seed).permutation(len(pairs)):
        add(*pairs[i])
    family = "qwen3" if digits == 1 else "llama"
    names = (["<|endoftext|>", "<|im_start|>", "<|im_end|>"] if family == "qwen3"
             else ["<|begin_of_text|>", "<|end_of_text|>", "<|eot_id|>"])
    specials = {n: len(token_bytes) + i for i, n in enumerate(names)}
    token_bytes += [b""] * len(names)
    return VB.Vocab(family, len(token_bytes), token_bytes, merges, specials, digits)


@functools.lru_cache(maxsize=None)
def full_vocab(family: str) -> VB.Vocab:
    return VB.build_vocab(family, FULL[family])


@functools.lru_cache(maxsize=None)
def full_hf(family: str):
    return VB.to_hf_tokenizer(full_vocab(family))


@functools.lru_cache(maxsize=None)
def full_gpu(family: str):
    from sutro_b200.engine import GpuTokenizer
    return GpuTokenizer(full_vocab(family), DEV)


def hf_ids(hf, texts):
    return [e.ids for e in hf.encode_batch(list(texts), add_special_tokens=False)]


def vocab_join_rows(v: VB.Vocab, n: int, seed: int):
    """Texts made of the byte strings of 1-8 random regular entries (invalid UTF-8 replaced):
    long merge chains and the <= 12-byte filler merges of the synthetic vocabulary."""
    rng = np.random.RandomState(seed)
    return [b"".join(v.token_bytes[i] for i in rng.randint(256, v.n_regular, size=k))
            .decode("utf-8", errors="replace") for k in rng.randint(1, 9, size=n)]


# --------------------------------------------------------------------------- the C-ABI, directly
def blob(rows_bytes):
    off = np.zeros(len(rows_bytes) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(b) for b in rows_bytes])
    return np.frombuffer(b"".join(rows_bytes), dtype=np.uint8), off


def encode_raw(tok, data: np.ndarray, off: np.ndarray):
    """sb200_tokenizer_encode over the column exactly as given: `data` is indexed by `off`, which
    may start past 0 (a sliced Arrow column); n_bytes = off[-1]."""
    off = np.ascontiguousarray(off, dtype=np.int64)
    n_rows, n_bytes = len(off) - 1, int(off[-1])
    d_text = (torch.from_numpy(np.array(data[:n_bytes], dtype=np.uint8)).to(DEV) if n_bytes
              else torch.zeros(1, dtype=torch.uint8, device=DEV))
    d_off = torch.from_numpy(off).to(DEV)
    d_tok = torch.full((max(n_bytes, 1),), -1, dtype=torch.int32, device=DEV)
    d_toff = torch.full((n_rows + 1,), -7, dtype=torch.int64, device=DEV)
    L.check(L.lib().sb200_tokenizer_encode(tok._h, d_text.data_ptr(), n_bytes, d_off.data_ptr(),
                                           n_rows, d_tok.data_ptr(), d_toff.data_ptr(),
                                           L.current_stream()))
    toff, toks = d_toff.cpu().numpy(), d_tok.cpu().numpy()
    assert toff[0] == 0 and (np.diff(toff) >= 0).all() and toff[-1] <= n_bytes, toff
    return [toks[toff[i]:toff[i + 1]].tolist() for i in range(n_rows)]


def decode_raw(tok, rows_ids):
    """Both passes of sb200_tokenizer_decode; pass 1 (no output buffer) must report exactly the
    offsets pass 2 writes by.  -> (bytes per row, int64 row byte offsets)."""
    toff = np.zeros(len(rows_ids) + 1, dtype=np.int64)
    toff[1:] = np.cumsum([len(r) for r in rows_ids])
    flat = np.asarray([t for r in rows_ids for t in r], dtype=np.int32)
    n_tok, n_rows = len(flat), len(rows_ids)
    d_tok = (torch.from_numpy(flat).to(DEV) if n_tok
             else torch.zeros(1, dtype=torch.int32, device=DEV))
    d_toff = torch.from_numpy(toff).to(DEV)
    lib = L.lib()
    b1 = torch.full((n_rows + 1,), -7, dtype=torch.int64, device=DEV)
    L.check(lib.sb200_tokenizer_decode(tok._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(), n_rows,
                                       None, b1.data_ptr(), L.current_stream()))
    total = int(b1[-1].item())
    out = torch.full((max(total, 1),), 0xA5, dtype=torch.uint8, device=DEV)
    b2 = torch.full((n_rows + 1,), -7, dtype=torch.int64, device=DEV)
    L.check(lib.sb200_tokenizer_decode(tok._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(), n_rows,
                                       out.data_ptr(), b2.data_ptr(), L.current_stream()))
    assert torch.equal(b1, b2)
    boff = b2.cpu().numpy()
    raw = out[:total].cpu().numpy().tobytes()
    return [raw[boff[i]:boff[i + 1]] for i in range(n_rows)], boff


def check_rows(tok, rows_bytes, hf=None, v=None):
    """(a) ids in the batch == ids of the row encoded alone, (b) decode(encode(b)) == b,
    (c) ids == `tokenizers`' where the row is valid UTF-8."""
    data, off = blob(rows_bytes)
    got = encode_raw(tok, data, off)
    for b, g in zip(rows_bytes, got):
        assert g == encode_raw(tok, *blob([b]))[0], b[:64]
    dec, _ = decode_raw(tok, got)
    for b, d in zip(rows_bytes, dec):
        assert d == b, (b[:64], d[:64])
    if hf is not None:
        valid = []
        for i, b in enumerate(rows_bytes):
            try:
                valid.append((i, b.decode("utf-8")))
            except UnicodeDecodeError:
                pass
        want = hf_ids(hf, [t for _, t in valid])
        for (i, t), w in zip(valid, want):
            assert v.to_real_ids(got[i]) == w, repr(t[:64])
    return got


# --------------------------------------------------------------------------- 1. pre-tokeniser
@pytest.mark.parametrize("digits", [1, 3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_pretokenizer_branches_on_a_boundary_vocabulary(seed, digits):
    from sutro_b200.engine import GpuTokenizer
    v = boundary_vocab(seed, digits)
    assert v.vocab_size > len(ALPHABET) ** 2 + 256
    hf = VB.to_hf_tokenizer(v)
    tok = GpuTokenizer(v, DEV)
    texts = HAND + fuzz_corpus(20000, seed=100 + 10 * seed + digits)
    got = tok.encode(texts)
    want = hf_ids(hf, texts)
    bad = [t for t, g, w in zip(texts, got, want) if g != w]
    assert not bad, (len(bad), [repr(t) for t in bad[:10]])
    # the CPU oracle agrees on the hand-written cases (its regex reads U+001C-U+001F as \s)
    ref = RefTokenizer(v)
    for t, g in zip(HAND, got):
        if not any(c in t for c in SEPARATORS):
            assert g == ref.encode(t), repr(t)
    # the vocabulary does pin boundaries: most strings of 3+ characters end in pair tokens
    pairs = sum(any(len(v.token_bytes[i].decode("utf-8", "replace")) == 2 for i in g)
                for t, g in zip(texts, got) if len(t) >= 3)
    assert pairs > 0.5 * sum(len(t) >= 3 for t in texts)


# --------------------------------------------------------------------------- 2. full-size vocabularies
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_full_size_vocabulary_matches_tokenizers(family):
    v, hf, tok = full_vocab(family), full_hf(family), full_gpu(family)
    texts = (synth.product_reviews(3000, seed=11) + synth.extraction_documents(2000, seed=12)
             + fuzz_corpus(10000, seed=13) + vocab_join_rows(v, 5000, seed=14))
    assert len(texts) == 20000
    got = tok.encode(texts)                       # one encode call for all rows
    want = hf_ids(hf, texts)
    bad = [t for t, g, w in zip(texts, got, want) if g != w]
    assert not bad, (len(bad), [repr(t[:80]) for t in bad[:5]])
    # the trained and filler merges were exercised: long tokens, ids near the top
    flat = np.concatenate([np.asarray(g, dtype=np.int64) for g in got if g])
    assert flat.max() > 0.9 * v.n_regular
    assert max(len(v.token_bytes[i]) for i in np.unique(flat)) >= 10
    dec, _ = decode_raw(tok, got)
    for t, d in zip(texts, dec):
        assert d == t.encode("utf-8")


# --------------------------------------------------------------------------- 3. tokenizer-file layout
@pytest.mark.parametrize("ignore_merges", [False, True])
def test_tokenizer_file_layout_at_full_size(tmp_path, ignore_merges):
    """A tokenizer.json in GPT-2 byte order with the regular ids permuted: the byte permutation
    (id_map) and the merge result ids (merged_ids) are not the identity."""
    from test_pretrained_cpu import gpt2_ordered_tokenizer, override_texts
    from tokenizers import Tokenizer

    from sutro_b200 import pretrained as PT
    from sutro_b200.engine import GpuTokenizer
    v = full_vocab("qwen3")
    path = str(tmp_path / "tokenizer.json")
    gpt2_ordered_tokenizer(v).save(path)
    tj = json.load(open(path, encoding="utf-8"))
    voc = tj["model"]["vocab"]
    regular = sorted(i for i in voc.values() if i >= 256)
    perm = dict(zip(regular, np.random.RandomState(3).permutation(regular).tolist()))
    tj["model"]["vocab"] = {s: perm.get(i, i) for s, i in voc.items()}
    # 300 trained merges listed a second time at the end: a duplicate ranks at its last entry
    merges = tj["model"]["merges"]
    tj["model"]["merges"] = merges + [merges[i] for i in
                                      np.random.RandomState(4).randint(0, 3000, size=300)]
    if ignore_merges:
        tj["model"]["ignore_merges"] = True
    json.dump(tj, open(path, "w", encoding="utf-8"), ensure_ascii=False)
    hf = Tokenizer.from_file(path)
    loaded = PT.load_tokenizer_json(path, "qwen3", vocab_size=FULL["qwen3"])
    assert not np.array_equal(loaded.id_map[:256], np.arange(256))
    assert loaded.merged_ids is not None and \
        loaded.merged_ids != list(range(256, 256 + len(loaded.merges)))
    assert (loaded.word_overrides is not None) == ignore_merges
    tok = GpuTokenizer(loaded, DEV)
    texts = (synth.product_reviews(1000, seed=21) + fuzz_corpus(3000, seed=22)
             + vocab_join_rows(v, 3000, seed=23) + HAND)
    if ignore_merges:
        assert len(loaded.word_overrides) > 100
        texts += override_texts(dataclass_head(loaded, 2000))
    got = tok.encode(texts)
    want = hf_ids(hf, texts)
    bad = [t for t, g, w in zip(texts, got, want) if loaded.to_real_ids(g) != w]
    assert not bad, (len(bad), [repr(t[:80]) for t in bad[:5]])
    if ignore_merges:     # whole-word overrides fired
        over = {e for _, e in loaded.word_overrides}
        assert sum(len(g) == 1 and g[0] in over for g in got) >= 20


def dataclass_head(v: VB.Vocab, n: int) -> VB.Vocab:
    import dataclasses
    return dataclasses.replace(v, word_overrides=v.word_overrides[:n])


# --------------------------------------------------------------------------- 4. layout edges
def test_encode_layout_edges():
    import pyarrow as pa
    v, hf, tok = full_vocab("qwen3"), full_hf("qwen3"), full_gpu("qwen3")
    # empty rows first, in the middle and last
    check_rows(tok, [b"", b"hello there", b"", b"", b"it's 12 o'clock\n", b""], hf, v)
    # a batch of empty rows only: n_bytes == 0
    assert encode_raw(tok, np.zeros(0, np.uint8), np.zeros(4, np.int64)) == [[], [], []]
    assert decode_raw(tok, [[], [], []])[0] == [b"", b"", b""]
    # a sliced Arrow column: row_off[0] > 0, n_bytes = row_off[n_rows]
    rows = synth.product_reviews(12, seed=31) + ["caf\u00e9 \u4e2d\u6587", "", "x"]
    col = pa.array(rows, type=pa.large_string())
    for lo, n in ((3, 9), (5, 1), (14, 1)):
        sl = col.slice(lo, n)
        bufs = sl.buffers()
        off = np.frombuffer(bufs[1], dtype=np.int64, count=n + 1, offset=sl.offset * 8).copy()
        data = np.frombuffer(bufs[2], dtype=np.uint8)
        assert off[0] > 0
        got = encode_raw(tok, data, off)
        assert got == [encode_raw(tok, *blob([r.encode("utf-8")]))[0] for r in rows[lo:lo + n]]
        assert [v.to_real_ids(g) for g in got] == hf_ids(hf, rows[lo:lo + n])
    # a row ending in a truncated lead byte, the next starting with continuation bytes
    check_rows(tok, [b"abc\xe4", b"\xb8\x80def", b"x \xf0\x9f", b"\x99\x82 y", b"\xc5",
                     b"\xbf'd", b"'\xc5", b"\xbfd"], hf, v)
    # arbitrary bytes that are not UTF-8
    rng = np.random.RandomState(32)
    junk = [rng.randint(0, 256, size=k).astype(np.uint8).tobytes()
            for k in rng.randint(0, 200, size=300)]
    junk += [bytes(range(256)), bytes(range(255, -1, -1)), b"\xff" * 40, b"\x80" * 40,
             b"\xf4\x90\x80\x80", b"\xed\xa0\x80", b"\xc0\xaf"]
    check_rows(tok, junk, hf, v)
    # long pre-tokens: a 5,000-byte word of letters, 3,000 spaces, 2,000 digits, a 4,000-byte
    # word of two-byte letters
    letters = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz"), size=5000))
    check_rows(tok, [letters.encode(), b" " * 3000 + b"x", b"7" * 2000,
                     ("\u0416\u044f" * 1000).encode(), b"ok"], hf, v)


# --------------------------------------------------------------------------- 5. detokeniser
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_detokenizer_matches_vocabulary_bytes(family):
    v, tok = full_vocab(family), full_gpu(family)
    rng = np.random.RandomState(41)
    special = np.asarray(sorted(v.specials.values()))
    rows = []
    for k in rng.randint(0, 65, size=3000):
        ids = rng.randint(0, v.vocab_size, size=k)
        pick = rng.rand(k)
        ids[pick < 0.1] = rng.choice(special, size=int((pick < 0.1).sum()))
        ids[(pick >= 0.1) & (pick < 0.15)] = v.vocab_size - 1
        rows.append(ids.tolist())
    rows[:3] = [[], [v.vocab_size - 1], [int(special[0])] * 5]
    rows += [[]] * 5
    got, boff = decode_raw(tok, rows)
    want = [b"".join(v.token_bytes[i] for i in r) for r in rows]
    assert got == want
    lens = np.asarray([len(w) for w in want], dtype=np.int64)
    assert boff.tolist() == [0] + np.cumsum(lens).tolist()
    assert all(v.token_bytes[i] == b"" for i in special) and v.token_bytes[-1] == b""


# --------------------------------------------------------------------------- 6. past 2^31 bytes
def test_decode_past_2_31_output_bytes():
    """~1.8e8 copies of one 12-byte token in one decode call, rows ending on both sides of
    byte 2^31.  Pass 1 is checked first against an int64 cumsum on the device, so a scan that
    wraps fails there, before pass 2 would write at the wrapped offsets."""
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < 16 * 2 ** 30:
        pytest.skip(f"needs 16 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    from sutro_b200.engine import GpuTokenizer
    v = full_vocab("qwen3")
    tid = next(i for i in range(v.n_regular - 1, 255, -1) if len(v.token_bytes[i]) == 12)
    tb = v.token_bytes[tid]
    tok = GpuTokenizer(v, DEV)
    B = 2 ** 31
    k = B // 12                        # token k starts 8 bytes before 2^31
    n_tok = 180_000_000
    row_tok = [0, 60_000_000, k - 1, k, k + 1, k + 2, n_tok]
    assert (k - 1) * 12 < B < (k + 2) * 12 < n_tok * 12
    d_tok = torch.full((n_tok,), tid, dtype=torch.int32, device=DEV)
    d_toff = torch.tensor(row_tok, dtype=torch.int64, device=DEV)
    n_rows = len(row_tok) - 1
    lib = L.lib()
    b1 = torch.full((n_rows + 1,), -7, dtype=torch.int64, device=DEV)
    L.check(lib.sb200_tokenizer_decode(tok._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(), n_rows,
                                       None, b1.data_ptr(), L.current_stream()))
    _, off = v.byte_blob()
    lens_tab = torch.from_numpy(np.diff(off).astype(np.int64)).to(DEV)
    cs = torch.cumsum(lens_tab[d_tok.long()], 0)
    want = torch.where(d_toff > 0, cs[(d_toff - 1).clamp(min=0)], torch.zeros_like(d_toff))
    del cs
    torch.cuda.empty_cache()
    assert torch.equal(b1, want), (b1.tolist(), want.tolist())
    total = int(b1[-1].item())
    assert total == 12 * n_tok > B
    out = torch.zeros(total, dtype=torch.uint8, device=DEV)
    b2 = torch.full((n_rows + 1,), -7, dtype=torch.int64, device=DEV)
    L.check(lib.sb200_tokenizer_decode(tok._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(), n_rows,
                                       out.data_ptr(), b2.data_ptr(), L.current_stream()))
    assert torch.equal(b2, b1)
    pattern = torch.tensor(list(tb), dtype=torch.uint8, device=DEV)
    for lo in ((k - 2) * 12, (n_tok - 4) * 12, 0):     # both sides of 2^31, the end, the start
        assert torch.equal(out[lo:lo + 48], pattern.repeat(4)), lo
    assert int(out.sum(dtype=torch.int64).item()) == n_tok * sum(tb)
    grid = out.view(n_tok, 12)
    step = 1 << 24
    for s in range(0, n_tok, step):
        blk = grid[s:s + step]
        assert torch.equal(blk, pattern.expand_as(blk)), s
    del tok, out, grid, d_tok
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------- 7. NFC end to end
DECOMPOSED = ["cafe\u0301 au lait, tre\u0300s bien", "\u1100\u1161\u11a8 \u1112\u1161\u11ab",
              "A\u030angstro\u0308m is a unit of length", "plain ascii row"]
COMPOSED = [unicodedata.normalize("NFC", r) for r in DECOMPOSED]
GEN = dict(max_new_tokens=8, ignore_eos=True, return_logprobs=True)


@pytest.fixture(scope="module")
def nfc_engine(tmp_path_factory):
    """A tiny Qwen3 engine whose vocabulary comes from a tokenizer.json declaring an NFC
    normalizer, the `tokenizers` object reading the same file, and the reference results of
    the precomposed rows."""
    from test_pretrained_cpu import gpt2_ordered_tokenizer
    from tokenizers import Tokenizer

    from sutro_b200 import modelspec as MS, pretrained as PT
    from sutro_b200.engine import LocalEngine
    spec = MS.get_spec("tiny-qwen3")
    v = VB.build_vocab("qwen3", spec.vocab_size, seed=0, n_trained=600)
    path = str(tmp_path_factory.mktemp("nfc") / "tokenizer.json")
    gpt2_ordered_tokenizer(v).save(path)
    tj = json.load(open(path, encoding="utf-8"))
    tj["normalizer"] = {"type": "NFC"}
    json.dump(tj, open(path, "w", encoding="utf-8"))
    loaded = PT.load_tokenizer_json(path, "qwen3", vocab_size=spec.vocab_size)
    assert loaded.normalize_nfc
    w = MS.make_weights(spec, seed=0, std=0.05)
    eng = LocalEngine(spec, MS.pack_for_engine(spec, w, "cuda:0", row_map=loaded.id_map), loaded,
                      device=0, kv_pages=256, max_slots=8, max_prefill_tokens=512)
    want = eng.generate(list(COMPOSED), return_tokens=True, return_first_logits=True, **GEN)
    want1 = eng.infer_one_call(list(COMPOSED), **GEN)
    return eng, loaded, Tokenizer.from_file(path), want, want1


def test_nfc_gpu_ids_match_tokenizers(nfc_engine):
    """The GPU ids of the normalised rows are `tokenizers`' ids of the raw rows; the raw bytes
    give other ids, so a path that skips NFC is visible in the ids."""
    from sutro_b200.engine import normalize_rows
    eng, loaded, hf, _, _ = nfc_engine
    assert all(d != c for d, c in zip(DECOMPOSED[:3], COMPOSED[:3]))
    gpu = eng.tokenizer.encode(normalize_rows(DECOMPOSED, loaded))
    assert [loaded.to_real_ids(g) for g in gpu] == hf_ids(hf, DECOMPOSED)
    raw = eng.tokenizer.encode(DECOMPOSED)
    assert all(r != g for r, g in zip(raw[:3], gpu[:3]))


def _nfc_form(name):
    import pandas as pd
    import pyarrow as pa
    return {"list": lambda: list(DECOMPOSED), "series": lambda: pd.Series(DECOMPOSED),
            "arrow": lambda: pa.array(DECOMPOSED),
            "chunked": lambda: pa.chunked_array([DECOMPOSED[:1], DECOMPOSED[1:]])}[name]()


@pytest.mark.parametrize("form", ["list", "series", "arrow", "chunked"])
def test_nfc_generate_and_infer_one_call(nfc_engine, form):
    """Decomposed rows in every input form give the outputs, tokens, first logits and
    log-probabilities of the same rows precomposed, bit for bit."""
    eng, _, _, want, want1 = nfc_engine
    got = eng.generate(_nfc_form(form), return_tokens=True, return_first_logits=True, **GEN)
    assert got.outputs == want.outputs and got.out_tokens == want.out_tokens
    assert torch.equal(got.first_logits, want.first_logits)
    assert np.array_equal(got.cum_logprobs, want.cum_logprobs)
    got1 = eng.infer_one_call(_nfc_form(form), **GEN)
    assert got1.outputs == want1.outputs and got1.out_tokens == want1.out_tokens
    assert np.array_equal(got1.cum_logprobs, want1.cum_logprobs)


@pytest.mark.parametrize("form", ["list", "frame", "csv"])
def test_nfc_through_sutro_infer(nfc_engine, tmp_path, form):
    """Sutro.infer on a list, a DataFrame column and a csv file (the last two travel as Arrow)
    returns the outputs and log-probabilities of the precomposed rows."""
    import pandas as pd

    from sutro_b200.sdk import Sutro
    eng, _, _, _, want1 = nfc_engine
    so = Sutro(verbose=False, cache_dir=str(tmp_path / "jobs"))
    so.register_engine("tiny-qwen3", eng)

    def run(data, column=None):
        jid = so.infer(data, model="tiny-qwen3", column=column, stay_attached=False,
                       sampling_params={"max_tokens": 8, "ignore_eos": True})
        job = so._job(jid)
        return job.outputs, np.asarray(job.cum_logprobs)
    ref_out, ref_lp = run(list(COMPOSED))
    assert ref_out == want1.outputs
    if form == "list":
        out, lp = run(list(DECOMPOSED))
    elif form == "frame":
        out, lp = run(pd.DataFrame({"text": DECOMPOSED}), "text")
    else:
        csv = tmp_path / "rows.csv"
        pd.DataFrame({"text": DECOMPOSED}).to_csv(csv, index=False)
        out, lp = run(str(csv), "text")
    assert out == ref_out and np.array_equal(lp, ref_lp)
