"""CPU oracle for the byte-level BPE tokenizer.  TEST INFRASTRUCTURE (see
oracle/model_ref.py header for who may import oracle/).

PARITY UNPINNED by the reference (tokenisation happens on Sutro's servers; the repo has
no tokenizer, SURVEY.md §0).  Algorithm restated: byte-level BPE as implemented by the
`tokenizers` 0.22.2 library (third-party, pinned by this image) — pre-tokenise with the
published GPT-4-style pattern (sutro_b200/vocab.py PRETOK_PATTERN), then inside each
pre-token repeatedly merge the adjacent pair with the lowest merge rank, leftmost first
(tokenizers/src/models/bpe/word.rs `merge_all`); with the model's `ignore_merges` flag a
pre-token that is itself a vocabulary entry is emitted as that token without merging
(tokenizers/src/models/bpe/model.rs `tokenize_with_cache`).  tests/test_tokenizer_oracle.py
pins this restatement against `tokenizers` itself on the same vocabulary, flag off and on.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import regex

from sutro_b200.vocab import PRETOK_PATTERN, Template, Vocab


class RefTokenizer:
    def __init__(self, v: Vocab):
        self.v = v
        self.pat = regex.compile(PRETOK_PATTERN % v.digits)
        self.rank: Dict[Tuple[int, int], Tuple[int, int]] = {}
        # a pair listed twice ranks at its last occurrence, as in `tokenizers` (its merge map is
        # filled in list order, later entries replacing earlier ones)
        for i, (a, b) in enumerate(v.merges):
            self.rank[(a, b)] = (i, 256 + i if v.merged_ids is None else v.merged_ids[i])
        # ignore_merges: whole pre-token -> id, over the model vocabulary (not the added tokens)
        self.whole: Dict[bytes, int] = {}
        if v.word_overrides is not None:
            special_ids = set(v.specials.values())
            for i, tb in enumerate(v.token_bytes):
                if tb and i not in special_ids:
                    self.whole.setdefault(tb, i)

    def _bpe(self, word: bytes) -> List[int]:
        if word in self.whole:
            return [self.whole[word]]
        s = list(word)
        while len(s) > 1:
            best, bi = None, -1
            for i in range(len(s) - 1):
                r = self.rank.get((s[i], s[i + 1]))
                if r is not None and (best is None or r[0] < best[0]):
                    best, bi = r, i
            if best is None:
                break
            s[bi:bi + 2] = [best[1]]
        return s

    def pretokenize(self, text: str) -> List[str]:
        return [m.group(0) for m in self.pat.finditer(text)]

    def encode(self, text: str) -> List[int]:
        out: List[int] = []
        for w in self.pretokenize(text):
            out += self._bpe(w.encode("utf-8"))
        return out

    def encode_pieces(self, pieces: List[str]) -> List[int]:
        out: List[int] = []
        for p in pieces:
            if p in self.v.specials:
                out.append(self.v.specials[p])
            else:
                out += self.encode(p)
        return out

    def render(self, tpl: Template, row: str, max_prompt: int | None = None) -> List[int]:
        """prefix | row | suffix; when `max_prompt` is given the row's tokens are cut so the
        whole prompt fits (the engine's truncate_rows=True behaviour)."""
        pre, suf = self.encode_pieces(tpl.prefix), self.encode_pieces(tpl.suffix)
        body = self.encode(row)
        if max_prompt is not None:
            body = body[:max(0, max_prompt - len(pre) - len(suf))]
        return pre + body + suf

    def decode(self, tokens) -> str:
        """Token ids -> text: the tokens' byte strings concatenated, UTF-8 with errors replaced
        (the detokenizer's contract, sutro_b200/engine.py blob_to_rows)."""
        if not hasattr(self, "_blob"):
            self._blob, self._off = self.v.byte_blob()
        raw = b"".join(bytes(self._blob[self._off[t]:self._off[t + 1]]) for t in tokens)
        return raw.decode("utf-8", errors="replace")
