"""Independent CPU reference of the constrained-decoding token masks (`fsm_build_mask_kernel`).

mask[s, t] is 1 iff
  * t is the end-of-sequence id: state s is accepting;
  * t has no bytes (special and unused ids): never;
  * otherwise: walking t's bytes from s never leaves the automaton.
Bits at and past `vocab` in the last word are 0.  Masks are packed as the kernel stores them:
uint32 words, token t at bit t & 31 of word t >> 5.

Unlike the kernel (one thread per (state, token) walking the token's bytes) and TokenFSM (one
state at a time over a padded token matrix), this walks a trie of the vocabulary's byte strings
once per block of states: every distinct token prefix is one trie node, the automaton's state
at a node is the parent's state stepped by the node's byte, and a token's verdict is read at the
node its last byte reaches.  The trie is built from the lexicographically sorted byte strings,
so tokens that share a prefix share the steps.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch


class VocabTrie:
    def __init__(self, token_bytes: Sequence[bytes]):
        V = len(token_bytes)
        lens = np.fromiter((len(b) for b in token_bytes), dtype=np.int64, count=V)
        order = np.asarray(sorted(range(V), key=lambda i: token_bytes[i]), dtype=np.int64)
        maxlen = int(lens.max()) if V else 0
        pad = np.zeros((V, max(maxlen, 1)), dtype=np.int64)
        for r, i in enumerate(order):
            b = token_bytes[i]
            if b:
                pad[r, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        slen = lens[order]
        self.vocab = V
        self.lens = lens
        # per depth d >= 1: (parent node at depth d-1, byte, node of every token of length d,
        # those tokens).  Depth 0 is the root, node 0.
        self.levels: List[tuple] = []
        node = np.zeros(V, dtype=np.int64)         # node of each sorted token at the last depth
        for d in range(1, maxlen + 1):
            el = np.nonzero(slen >= d)[0]
            byte = pad[el, d - 1]
            new = np.ones(len(el), dtype=bool)     # a new node where prefix[:d] changes
            new[1:] = (node[el[1:]] != node[el[:-1]]) | (byte[1:] != byte[:-1])
            ids = np.cumsum(new) - 1
            parent, nbyte = node[el][new], byte[new]
            node[el] = ids
            ends = slen[el] == d
            self.levels.append((torch.from_numpy(parent), torch.from_numpy(nbyte[:, None]),
                                torch.from_numpy(ids[ends]), torch.from_numpy(order[el[ends]])))
        self.n_nodes = sum(len(p) for p, _, _, _ in self.levels)


def allowed(trans: np.ndarray, accept: np.ndarray, trie: VocabTrie, eos_id: int,
            states: Sequence[int], block: int = 64) -> np.ndarray:
    """bool [len(states), vocab]: the mask rows of `states`.  (torch on the CPU only for its
    multi-threaded gathers.)"""
    n = trans.shape[0]
    # state n is a dead sink: every byte from it stays there
    tr = np.concatenate([np.where(trans >= 0, trans, n), np.full((1, 256), n)])
    tr = torch.from_numpy(tr.astype(np.int64).reshape(-1))
    states = np.asarray(states, dtype=np.int64)
    out = torch.zeros((len(states), trie.vocab), dtype=torch.bool)
    for c0 in range(0, len(states), block):
        cur = torch.from_numpy(states[None, c0:c0 + block])    # [nodes at this depth, block]
        rows = out[c0:c0 + block]
        for parent, byte, end_nodes, end_tokens in trie.levels:
            cur = tr.take(cur.index_select(0, parent).mul_(256).add_(byte))
            rows[:, end_tokens] = (cur.index_select(0, end_nodes) != n).T
    out = out.numpy()
    out[:, trie.lens == 0] = False
    if 0 <= eos_id < trie.vocab:
        out[:, eos_id] = accept[states].astype(bool)
    return out


def pack(rows: np.ndarray, words: int) -> np.ndarray:
    """bool [n, vocab] -> uint32 [n, words] (bits past vocab are 0)."""
    n, V = rows.shape
    assert words * 32 >= V
    pad = np.zeros((n, words * 32), dtype=bool)
    pad[:, :V] = rows
    return np.packbits(pad, axis=-1, bitorder="little").view("<u4")


def covered_states(dfa, walks: Sequence[int] = (), limit: int = 700, seed: int = 0) -> np.ndarray:
    """Every state when there are at most `limit`; otherwise a deterministic subset: the start
    state, the states the given walks visit, state 0, state n-1 and 512 seeded random states."""
    n = dfa.n_states
    if n <= limit:
        return np.arange(n)
    rng = np.random.default_rng(seed)
    pick = {dfa.start, 0, n - 1, *map(int, walks)} | set(rng.choice(n, 512, replace=False).tolist())
    return np.asarray(sorted(pick), dtype=np.int64)


def walk_states(dfa, seed: int, steps: int = 400) -> List[int]:
    """States of one seeded random byte walk from the start (to a final state, or `steps`)."""
    rng = np.random.default_rng(seed)
    s, seen = dfa.start, [dfa.start]
    for _ in range(steps):
        live = np.nonzero(dfa.trans[s] >= 0)[0]
        if len(live) == 0 or (dfa.accept[s] and rng.random() < 0.05):
            break
        s = int(dfa.trans[s, rng.choice(live)])
        seen.append(s)
    return seen
