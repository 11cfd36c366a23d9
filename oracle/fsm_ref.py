"""CPU oracle for constrained decoding.  TEST INFRASTRUCTURE (see oracle/model_ref.py).

PARITY UNPINNED by the reference (schema enforcement is server-side; the repo only
forwards `json_schema`, sutro/sdk.py:199).  What "correct" means is therefore defined by
the JSON-Schema semantics themselves: every string the automaton accepts must parse as
JSON and validate against the schema (checked with pydantic / a small validator below),
and every compact serialisation of a valid instance within the documented caps must be
accepted.  The token masks are additionally pinned against xgrammar (tests/
test_fsm_vs_xgrammar.py): identical allowed-token sets on finite-language schemas, a subset
on open ones (documented caps).  TokenFSM is the numpy restatement of the GPU mask kernel
(csrc/sampler_fsm.cu: fsm_build_mask_kernel, sample_greedy_kernel's state advance).
"""
from __future__ import annotations

from typing import Any, Dict, List

import numpy as np
import torch

from sutro_b200.schema_fsm import ByteDFA
from sutro_b200.vocab import Vocab


class TokenFSM:
    def __init__(self, dfa: ByteDFA, v: Vocab):
        self.dfa, self.v = dfa, v
        self.start = dfa.start
        lens = np.array([len(b) for b in v.token_bytes], dtype=np.int64)
        self.maxlen = int(lens.max())
        self.lens = lens
        pad = np.zeros((v.vocab_size, self.maxlen), dtype=np.int64)
        for i, b in enumerate(v.token_bytes):
            if b:
                pad[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        self.pad = pad
        self._cache: Dict[int, torch.Tensor] = {}
        self.forced_prefix: List[int] = []
        self.tails: Dict[int, List[int]] = {}

    def allowed(self, state: int) -> torch.Tensor:
        if state not in self._cache:
            s = np.full(self.v.vocab_size, state, dtype=np.int64)
            for j in range(self.maxlen):
                active = (self.lens > j) & (s >= 0)
                nxt = self.dfa.trans[np.clip(s, 0, None), self.pad[:, j]]
                s = np.where(active, nxt, s)
            ok = (s >= 0) & (self.lens > 0)
            ok[self.v.eos_id] = bool(self.dfa.accept[state])
            self._cache[state] = torch.from_numpy(ok)
        return self._cache[state]

    def step(self, state: int, tok: int) -> int:
        s = state
        for b in self.v.token_bytes[tok]:
            s = int(self.dfa.trans[s, b])
            if s < 0:
                break
        return s

    def is_final(self, state: int) -> bool:
        return state < 0 or bool(self.dfa.final[state])

    # ---- jump-forward decoding (restated independently of sutro_b200.schema_fsm) ----
    def _forced(self, state: int):
        out, s = bytearray(), state
        while not self.dfa.accept[s]:
            nxt = np.nonzero(self.dfa.trans[s] >= 0)[0]
            if len(nxt) != 1:
                break
            out.append(int(nxt[0]))
            s = int(self.dfa.trans[s, nxt[0]])
        return bytes(out), s

    def enable_jump_forward(self, tokenizer) -> bool:
        """tokenizer: oracle RefTokenizer.  Sets `forced_prefix` (token ids every output starts
        with), moves `start` past it, and fills `tails[state]` (token ids of a continuation
        that is forced up to a final state).  Returns False when the whole output is forced, or
        when a forced string is not valid UTF-8 (a tail that starts inside a multi-byte
        character has no text to encode); then nothing is enabled, like the engine."""
        prefix, after = self._forced(self.dfa.start)
        tails = {}
        for s in range(self.dfa.n_states):
            run, end = self._forced(s)
            if run and self.dfa.final[end]:
                tails[s] = run
        if self.dfa.final[after] or after in tails:
            return False
        try:
            texts = {s: b.decode("utf-8") for s, b in tails.items()}
            prefix_text = prefix.decode("utf-8")
        except UnicodeDecodeError:
            return False
        self.forced_prefix = tokenizer.encode(prefix_text)
        self.start = after
        self.tails = {s: tokenizer.encode(t) for s, t in texts.items()}
        return True


# ---- a deliberately small, independent JSON-Schema validator (subset used by tests) ----
def _resolve(root, sch):
    while isinstance(sch, dict) and "$ref" in sch:
        node = root
        for part in sch["$ref"][2:].split("/"):
            node = node[part]
        sch = node
    return sch


def validates(instance: Any, schema: Dict[str, Any], root=None) -> bool:
    root = root or schema
    sch = _resolve(root, schema)
    if sch is True or sch == {}:
        return True
    if sch is False:
        return False
    if "const" in sch:
        return instance == sch["const"]
    if "enum" in sch:
        return instance in sch["enum"]
    for k in ("anyOf", "oneOf"):
        if k in sch:
            return any(validates(instance, s, root) for s in sch[k])
    t = sch.get("type")
    if isinstance(t, list):
        return any(validates(instance, {**sch, "type": x}, root) for x in t)
    if t == "object" or (t is None and "properties" in sch):
        if not isinstance(instance, dict):
            return False
        props = sch.get("properties", {})
        if any(r not in instance for r in sch.get("required", [])):
            return False
        return all(validates(v, props[k], root) for k, v in instance.items() if k in props)
    if t == "string":
        return (isinstance(instance, str) and len(instance) >= sch.get("minLength", 0)
                and len(instance) <= sch.get("maxLength", 1 << 30))
    if t == "integer":
        return (isinstance(instance, int) and not isinstance(instance, bool)
                and instance >= sch.get("minimum", -1 << 62) and instance <= sch.get("maximum", 1 << 62))
    if t == "number":
        return isinstance(instance, (int, float)) and not isinstance(instance, bool)
    if t == "boolean":
        return isinstance(instance, bool)
    if t == "null":
        return instance is None
    if t == "array":
        pre = sch.get("prefixItems", [])
        return (isinstance(instance, list) and len(instance) >= sch.get("minItems", 0)
                and len(instance) <= sch.get("maxItems", 1 << 30)
                and all(validates(x, pre[i] if i < len(pre) else sch.get("items", {}), root)
                        for i, x in enumerate(instance)))
    return False


def random_accepted(dfa: ByteDFA, rng: np.random.RandomState, max_len: int = 4000) -> bytes:
    """Random walk through the automaton until a final/accepting state."""
    s, out = dfa.start, bytearray()
    while len(out) < max_len:
        if dfa.final[s] or (dfa.accept[s] and rng.rand() < 0.3):
            return bytes(out)
        nxt = np.nonzero(dfa.trans[s] >= 0)[0]
        b = int(nxt[rng.randint(len(nxt))])
        out.append(b)
        s = int(dfa.trans[s, b])
    raise AssertionError("walk did not terminate")
