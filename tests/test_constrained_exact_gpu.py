"""Constrained decoding at full vocabulary size, exact, over the schema corpus
(tests/schema_corpus.py), for the automata of both compilers.

* Masks: `sb200_fsm_build_mask` equals tests/mask_ref.py (itself pinned to xgrammar by
  test_masks_vs_xgrammar_cpu.py) bit for bit, as uint32 words including the padding bits of the
  last word, on the qwen3 (151,936) and llama (128,256) vocabularies and on a 151,939-token one
  (not a multiple of 32; its EOS id sits at bit 0 of a word, llama's at bit 31).
* Kernel edges: 65,535 states (the grid.y limit), spare and too few mask words, EOS at bit 0
  and 31, tokens that die at their last byte or pass through a final state before it.
* Jump-forward plans: LocalEngine._jump_plan against a reference that counts each state's
  completions (capped at 2) instead of following forced runs.
* End to end on tiny-qwen3 / tiny-llama with full-size vocabularies: every emitted sequence
  walks the automaton; rows that stop early stop in an accepting state and validate; two
  schemas replayed bit for bit (tests/engine_replay.py); the C host (`sb200_model_infer` on an
  exported bundle, native compiler and C jump-forward plan) identical to LocalEngine.generate.

Each case prints one PARITY line and fails when the path it is about did not run.
"""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import mask_ref as M
from engine_replay import Replay
from oracle.bpe_ref import RefTokenizer
from oracle.fsm_ref import TokenFSM, validates
from schema_corpus import BY_NAME, ENTRIES
from sutro_b200 import _lib as L
from sutro_b200 import modelspec as MS
from sutro_b200 import synth, vocab as VB
from sutro_b200.schema_fsm import ByteDFA, split_thinking

pytestmark = pytest.mark.gpu

DEV = "cuda"
VOCABS = {"qwen3": ("qwen3", 151936), "llama": ("llama", 128256),
          "qwen3_odd": ("qwen3", 151939)}
SENTINEL = 0x5A5A5A5A
SYS = synth.README_SYSTEM_PROMPT
ROWS = [synth.README_REVIEWS[0], "café naïve 東京", ""]

_WORLDS = {}


def world(key):
    """(vocab, trie, device token bytes, device token offsets) of a full-size vocabulary."""
    if key not in _WORLDS:
        fam, size = VOCABS[key]
        v = VB.build_vocab(fam, size, seed=0)
        blob, off = v.byte_blob()
        _WORLDS[key] = (v, M.VocabTrie(v.token_bytes), torch.from_numpy(blob).to(DEV),
                        torch.from_numpy(off).to(DEV))
    return _WORLDS[key]


def gpu_masks(trans, accept, d_tb, d_to, vocab, eos_id, words):
    """(return code, uint32 [n_states, words]) of sb200_fsm_build_mask on a sentinel-filled
    buffer."""
    n = trans.shape[0]
    d_tr = torch.from_numpy(np.ascontiguousarray(trans, dtype=np.int32)).to(DEV)
    d_ac = torch.from_numpy(np.ascontiguousarray(accept, dtype=np.uint8)).to(DEV)
    out = torch.full((n, words), SENTINEL, dtype=torch.int32, device=DEV)
    rc = L.lib().sb200_fsm_build_mask(L.ptr(d_tr), L.ptr(d_ac), n, L.ptr(d_tb), L.ptr(d_to),
                                      vocab, eos_id, L.ptr(out), words, L.current_stream())
    torch.cuda.synchronize()
    return rc, out.cpu().numpy().view(np.uint32)


def relabelling(a, b):
    """perm with b.trans[perm[p]] == perm[a.trans[p]] and b.accept[perm[p]] == a.accept[p] for
    every state p (b is a renumbered a), or None."""
    n = a.n_states
    if b.n_states != n:
        return None
    perm = np.full(n, -1, dtype=np.int64)
    perm[a.start] = b.start
    frontier = np.array([a.start])
    while len(frontier):
        ta, tb = a.trans[frontier], b.trans[perm[frontier]]
        if ((ta >= 0) != (tb >= 0)).any():
            return None
        pa, pb = ta[ta >= 0], tb[ta >= 0]
        new = np.unique(pa[perm[pa] < 0])
        first = {int(x): int(y) for x, y in zip(pa[::-1], pb[::-1])}
        perm[new] = [first[int(x)] for x in new]
        if (perm[pa] != pb).any():
            return None
        frontier = new
    if (perm < 0).any() or len(np.unique(perm)) != n or \
            not np.array_equal(a.accept, b.accept[perm]):
        return None
    return perm


def check_final_flags(dfa, label):
    """`final` is what the sampler stops on and what jump-forward tails end in: accepting with
    no outgoing byte."""
    want = dfa.accept.astype(bool) & (dfa.trans < 0).all(axis=1)
    assert np.array_equal(dfa.final.astype(bool), want), (label, np.nonzero(dfa.final != want))


def automata(e):
    out = [("python", e.compile())]
    if e.native:
        out.append(("native", e.compile_native()))
    return out


# ---------------------------------------------------------------------------------- masks
@pytest.mark.parametrize("name", [e.name for e in ENTRIES])
@pytest.mark.parametrize("vkey", list(VOCABS))
def test_masks_equal_the_reference(vkey, name):
    e = BY_NAME[name]
    v, trie, d_tb, d_to = world(vkey)
    V = v.vocab_size
    words = (V + 31) // 32
    first = None
    for comp, dfa in automata(e):
        check_final_flags(dfa, (name, comp))
        perm = None if first is None else relabelling(first[0], dfa)
        if perm is None:
            walks = [s for seed in range(3) for s in M.walk_states(dfa, seed)]
            states = M.covered_states(dfa, walks)
            want = M.pack(M.allowed(dfa.trans, dfa.accept, trie, v.eos_id, states), words)
            first = first or (dfa, states, want, walks)
        else:                           # the same automaton numbered differently: same rows
            _, states, want, walks = first
            states = perm[states]
        rc, got = gpu_masks(dfa.trans, dfa.accept, d_tb, d_to, V, v.eos_id, words)
        assert rc == 0
        bad = np.nonzero((got[states] != want).any(axis=1))[0]
        assert len(bad) == 0, (name, comp, [int(states[i]) for i in bad[:8]])
        cover = "all" if len(states) == dfa.n_states else "sampled"
        print("PARITY", f"masks[{vkey},{name},{comp}]", f"states={cover}:{len(states)}/{dfa.n_states}",
              f"tokens={V}", f"words={words}", f"walk_states={len(set(walks))}",
              f"eos_bit={v.eos_id & 31}", "relabelled" if perm is not None else "")


# ---------------------------------------------------------------------------- kernel edges
def test_mask_kernel_at_65535_states():
    v, trie, d_tb, d_to = world("qwen3")
    n = 65535                                        # grid.y limit, the compilers' cap
    s = np.arange(n, dtype=np.int64)[:, None]
    b = np.arange(256, dtype=np.int64)[None, :]
    trans = np.where((s * 31 + b * 7) % 5 != 0, (s * 131 + b * 17 + 1) % n, -1).astype(np.int32)
    accept = (np.arange(n) % 3 == 0).astype(np.uint8)
    words = (v.vocab_size + 31) // 32
    rc, got = gpu_masks(trans, accept, d_tb, d_to, v.vocab_size, v.eos_id, words)
    assert rc == 0
    rows = [0, 1, 2, n - 3, n - 2, n - 1]
    want = M.pack(M.allowed(trans, accept, trie, v.eos_id, rows), words)
    np.testing.assert_array_equal(got[rows], want)
    assert want.any() and not (want == want[0]).all()
    print("PARITY", "masks[65535_states]", f"states=sampled:{len(rows)}/{n}",
          f"tokens={v.vocab_size}")


def test_mask_words_spare_and_too_few():
    v, trie, d_tb, d_to = world("qwen3_odd")
    V = v.vocab_size
    assert V % 32 != 0
    words = (V + 31) // 32
    dfa = BY_NAME["bench.SCHEMA"].compile()
    want = M.pack(M.allowed(dfa.trans, dfa.accept, trie, v.eos_id, range(dfa.n_states)), words)
    # spare words: written as zero, the real ones unchanged, padding bits of the last word 0
    rc, got = gpu_masks(dfa.trans, dfa.accept, d_tb, d_to, V, v.eos_id, words + 3)
    assert rc == 0
    np.testing.assert_array_equal(got[:, :words], want)
    assert (got[:, words:] == 0).all()
    assert (got[:, words - 1] >> np.uint32(V & 31) == 0).all()
    # too few: refused, nothing written
    rc, got = gpu_masks(dfa.trans, dfa.accept, d_tb, d_to, V, v.eos_id, words - 1)
    assert rc != 0 and b"too small" in L.lib().sb200_last_error()
    assert (got == SENTINEL).all()
    print("PARITY", "masks[mask_words]", f"states=all:{dfa.n_states}", f"tokens={V}",
          f"words={words}+3,{words}-1")


def _edge_automaton():
    """a -> 1, 1 b -> 2 (accepting, not final), 2 c -> 3 (final); x -> 4 (final).
    Language {"ab", "abc", "x"}."""
    trans = np.full((5, 256), -1, dtype=np.int32)
    trans[0, ord("a")], trans[1, ord("b")], trans[2, ord("c")] = 1, 2, 3
    trans[0, ord("x")] = 4
    accept = np.array([0, 0, 1, 1, 1], dtype=np.uint8)
    final = np.array([0, 0, 0, 1, 1], dtype=np.uint8)
    return ByteDFA(trans, accept, final, 0)


@pytest.mark.parametrize("eos_id", [0, 31, 64])
def test_mask_kernel_edges(eos_id):
    """EOS at bit 0 / 31 of a word; tokens that die at their last byte ("abcd", "ad"), pass
    through a final state before their last byte ("xa", "abca"), or have no bytes."""
    dfa = _edge_automaton()
    rng = np.random.default_rng(eos_id)
    named = [b"a", b"ab", b"abc", b"abcd", b"ad", b"x", b"xa", b"abca", b"b", b"bc", b"c", b""]
    toks = list(named) + [bytes(rng.choice(list(b"abcdx"), rng.integers(1, 6)).tolist())
                         for _ in range(58)]
    toks.insert(eos_id, b"")                        # EOS: a special, no bytes
    V = len(toks)                                    # 71: three words, 7 used in the last
    words = (V + 31) // 32
    blob, off = np.frombuffer(b"".join(toks), np.uint8).copy(), np.zeros(V + 1, np.int32)
    off[1:] = np.cumsum([len(t) for t in toks])
    d_tb = torch.from_numpy(blob if len(blob) else np.zeros(1, np.uint8)).to(DEV)
    d_to = torch.from_numpy(off).to(DEV)
    rc, got = gpu_masks(dfa.trans, dfa.accept, d_tb, d_to, V, eos_id, words)
    assert rc == 0
    ref = M.allowed(dfa.trans, dfa.accept, M.VocabTrie(toks), eos_id, range(dfa.n_states))
    np.testing.assert_array_equal(got, M.pack(ref, words))
    idx = {t: i for i, t in reversed(list(enumerate(toks))) if i != eos_id}
    at0 = {t for t in named if t and ref[0, idx[t]]}
    assert at0 == {b"a", b"ab", b"abc", b"x"}, at0
    assert ref[1, idx[b"bc"]] and ref[1, idx[b"b"]] and not ref[1, idx[b"ad"]]
    assert [bool(ref[s, eos_id]) for s in range(5)] == [False, False, True, True, True]
    assert not ref[:, idx[b""]].any()
    print("PARITY", f"masks[edges,eos={eos_id}]", "states=all:5", f"tokens={V}",
          f"eos_word={eos_id >> 5}", f"eos_bit={eos_id & 31}")


# ---------------------------------------------------------------------------- engines
_ENGINES = {}
MODELS = {"tiny-qwen3": "qwen3", "tiny-llama": "llama"}


def engine(model):
    """tiny-qwen3 / tiny-llama over the full-size vocabulary of their family."""
    if model not in _ENGINES:
        from sutro_b200.engine import LocalEngine
        v, _, _, _ = world(MODELS[model])
        spec = MS.with_vocab(MS.get_spec(model), v.vocab_size)
        w = MS.make_weights(spec, seed=0, std=0.05)
        eng = LocalEngine(spec, MS.pack_for_engine(spec, w, DEV), v, device=0, kv_pages=512,
                          max_slots=8, max_prefill_tokens=512)
        _ENGINES[model] = (eng, RefTokenizer(v))
    return _ENGINES[model]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for eng, _ in _ENGINES.values():
        eng.close()
    _ENGINES.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------- jump-forward
def completions(dfa):
    """Number of strings each state accepts, capped at 2 (least fixed point of
    c(s) = min(2, accept(s) + sum of c over successors); a cycle drives it to 2)."""
    live = dfa.trans >= 0
    nxt = np.clip(dfa.trans, 0, None)
    acc = dfa.accept.astype(np.int64)
    c = np.zeros(dfa.n_states, dtype=np.int64)
    while True:
        new = np.minimum(2, acc + np.where(live, c[nxt], 0).sum(axis=1))
        if np.array_equal(new, c):
            return c
        c = new


def only_string(dfa, c, s):
    """The one string state s accepts (c[s] == 1)."""
    out = bytearray()
    while not dfa.accept[s]:
        nxt = [b for b in np.nonzero(dfa.trans[s] >= 0)[0] if c[dfa.trans[s, b]] > 0]
        assert len(nxt) == 1, (s, nxt)
        out.append(int(nxt[0]))
        s = int(dfa.trans[s, nxt[0]])
    return bytes(out)


def reference_plan(dfa, ref):
    """(plan, None) — the jump-forward plan the engine must make — or (None, why not)."""
    c = completions(dfa)
    tails = {s: only_string(dfa, c, s) for s in range(dfa.n_states)
             if c[s] == 1 and not dfa.accept[s]}
    prefix, s = bytearray(), dfa.start               # longest common prefix of the language
    while not dfa.accept[s] and (dfa.trans[s] >= 0).sum() == 1:
        b = int(np.nonzero(dfa.trans[s] >= 0)[0][0])
        prefix.append(b)
        s = int(dfa.trans[s, b])
    try:
        texts = {k: t.decode("utf-8") for k, t in tails.items()}
        prefix_text = bytes(prefix).decode("utf-8")
    except UnicodeDecodeError:
        return None, "utf8"
    if c[dfa.start] == 1:
        return None, "forced"
    if not (prefix or tails):
        return None, "nothing"
    return {"prefix": ref.encode(prefix_text), "start": s,
            "tails": {k: ref.encode(t) for k, t in texts.items()}}, None


@pytest.mark.parametrize("model", list(MODELS))
def test_jump_plans_equal_the_reference(model):
    eng, ref = engine(model)
    n_tails = n_none = n_plans = 0
    for e in ENTRIES:
        for comp, dfa in automata(e):
            want, why = reference_plan(dfa, ref)
            got = eng._jump_plan(dfa, ("corpus", e.name, comp))
            assert (got is None) == (want is None), (e.name, comp)
            # the oracle's restatement refuses the same automata (a non-ASCII tail included);
            # with nothing forced it enables an empty plan, which changes nothing
            assert TokenFSM(dfa, eng.vocab).enable_jump_forward(ref) == \
                (why not in ("forced", "utf8")), (e.name, comp)
            if e.non_ascii:
                assert got is None, e.name
            if got is None:
                n_none += 1
                continue
            n_plans += 1
            assert got["prefix_tokens"].tolist() == want["prefix"], (e.name, comp)
            assert got["start"] == want["start"], (e.name, comp)
            off, tok = got["tail_off"], got["tail_tok"]
            for s in range(dfa.n_states):
                assert tok[off[s]:off[s + 1]].tolist() == want["tails"].get(s, []), (e.name, comp, s)
            n_tails += len(want["tails"])
    assert n_tails > 0 and n_none > 0 and n_plans > 0
    print("PARITY", f"plans[{model}]", f"tokens={eng.vocab.vocab_size}", f"plans={n_plans}",
          f"tails={n_tails}", f"no_plan={n_none}")


# ---------------------------------------------------------------------------- end to end
def walk_row(dfa, v, toks):
    s = dfa.start
    for t in toks:
        assert t != v.eos_id and v.token_bytes[t], t
        for b in v.token_bytes[t]:
            s = int(dfa.trans[s, b])
            assert s >= 0, toks
    return s


def check_rows(e, dfa, v, res, max_new):
    stops = 0
    for toks, text in zip(res.out_tokens, res.outputs):
        s = walk_row(dfa, v, toks)
        if len(toks) < max_new:
            stops += 1
            assert dfa.accept[s], (e.name, text)
            content = split_thinking(text)[1] if e.thinking_chars is not None else text
            assert validates(json.loads(content), e.schema), (e.name, text)
    return stops


MODES = {"greedy": {}, "sampled": dict(temperature=0.8, top_k=40, top_p=0.95, seed=11,
                                       seed_per_row=True)}


@pytest.mark.parametrize("model", list(MODELS))
def test_rows_walk_the_automaton(model):
    eng, _ = engine(model)
    v = eng.vocab
    rows = steps = stops = forced = 0
    for e in ENTRIES:
        dfa = eng.compile_schema(e.schema, e.limits, e.thinking_chars)
        for mode, kw in MODES.items():
            for jump in (True, False):
                res = eng.generate(ROWS, system_prompt=SYS, json_schema=e.schema,
                                   fsm_limits=e.limits, max_new_tokens=e.max_new,
                                   thinking_chars=e.thinking_chars, jump_forward=jump,
                                   return_tokens=True, **kw)
                stops += check_rows(e, dfa, v, res, e.max_new)
                rows += len(ROWS)
                steps += res.stats["decode_steps"]
                forced += res.stats["forced_prefix_tokens"]
                assert jump or res.stats["forced_prefix_tokens"] == 0
    assert forced > 0 and stops > 0
    print("PARITY", f"e2e[{model}]", f"tokens={v.vocab_size}", f"rows={rows}", f"steps={steps}",
          f"early_stops={stops}", f"forced={forced}")


@pytest.mark.parametrize("name", ["bench.ORDER_SCHEMA", "non_ascii.enum"])
def test_rows_equal_the_replay(name):
    eng, _ = engine("tiny-qwen3")
    e = BY_NAME[name]
    rep = Replay(eng)
    steps = forced = 0
    for kw in ({}, dict(temperature=0.8, top_k=40, seed=3, seed_per_row=True)):
        job = dict(system_prompt=SYS, json_schema=e.schema, fsm_limits=e.limits,
                   max_new_tokens=e.max_new, **kw)
        res = eng.generate(ROWS, return_tokens=True, return_logprobs=True, **job)
        reps = rep.job(ROWS, **job)
        for i, r in enumerate(reps):
            assert res.out_tokens[i] == r.tokens, (name, i)
            assert np.float32(res.cum_logprobs[i]).view(np.int32) == \
                np.float32(r.cum_logprob).view(np.int32), (name, i)
        steps += sum(r.decode_steps for r in reps)
        forced += res.stats["forced_prefix_tokens"]
    assert steps > 0
    assert (forced > 0) == (not e.non_ascii)
    print("PARITY", f"replay[{name}]", f"tokens={eng.vocab.vocab_size}", f"rows={2 * len(ROWS)}",
          f"steps={steps}", f"forced={forced}")


# ---------------------------------------------------------------------------- the C host
def c_infer(model_h, e, rows, kw):
    from sutro_b200.engine import FsmLimitsC, JobC, JobStatsC, ResultC
    text = json.dumps(e.schema, ensure_ascii=False).encode("utf-8")
    lim = e.limits
    lc = FsmLimitsC(lim.max_string_chars, lim.max_array_items, lim.max_int_digits,
                    lim.max_frac_digits, lim.small_int_range, lim.max_recursion)
    job = JobC()
    job.truncate_rows = 1
    job.temperature, job.top_k = kw.get("temperature", 0.0), kw.get("top_k", 0)
    job.top_p, job.seed = kw.get("top_p", 1.0), kw.get("seed", 0)
    job.seed_per_row = int(kw.get("seed_per_row", False))
    blob = b"".join(r.encode("utf-8") for r in rows)
    off = np.zeros(len(rows) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(r.encode("utf-8")) for r in rows])
    buf = np.frombuffer(blob, np.uint8).copy() if blob else np.zeros(1, np.uint8)
    res, st = C.POINTER(ResultC)(), JobStatsC()
    L.check(L.lib().sb200_model_infer(model_h, SYS.encode("utf-8"), text, len(text), C.byref(lc),
                                      e.max_new, C.byref(job), buf.ctypes.data, off.ctypes.data,
                                      len(rows), 1, C.byref(res), C.byref(st)))
    try:
        r = res.contents
        n = len(rows)
        toff = np.ctypeslib.as_array(r.token_offsets, shape=(n + 1,)).copy()
        toks = (np.ctypeslib.as_array(r.tokens, shape=(int(toff[-1]),)).copy()
                if toff[-1] else np.zeros(0, np.int32))
        boff = np.ctypeslib.as_array(r.offsets, shape=(n + 1,)).copy()
        data = (bytes(np.ctypeslib.as_array(r.bytes, shape=(int(boff[-1]),)))
                if boff[-1] else b"")
        lp = np.ctypeslib.as_array(r.cum_logprob, shape=(n,)).copy()
    finally:
        L.lib().sb200_result_free(res)
    return ([toks[toff[i]:toff[i + 1]].tolist() for i in range(n)],
            [data[boff[i]:boff[i + 1]].decode("utf-8", "replace") for i in range(n)], lp,
            {k: int(getattr(st, k)) for k in ("input_tokens", "prefill_tokens", "decode_tokens")})


@pytest.mark.parametrize("model", list(MODELS))
def test_c_host_equals_the_python_host(model, tmp_path):
    from sutro_b200.bundle import export_bundle
    eng, _ = engine(model)
    bundle = export_bundle(eng, str(tmp_path / "bundle"))
    h = C.c_void_p()
    L.check(L.lib().sb200_model_open(bundle.encode(), 0, 8, 512, 512, C.byref(h)))
    cases = rows = forced = steps = no_plan = 0
    try:
        for e in ENTRIES:
            if not e.native:
                continue
            for mode, kw in MODES.items():
                want = eng.generate(ROWS, system_prompt=SYS, json_schema=e.schema,
                                    fsm_limits=e.limits, max_new_tokens=e.max_new,
                                    return_tokens=True, return_logprobs=True, **kw)
                toks, texts, lp, st = c_infer(h, e, ROWS, kw)
                label = (e.name, mode)
                assert toks == want.out_tokens, label
                assert texts == want.outputs, label
                assert np.array_equal(lp.view(np.int32),
                                      np.asarray(want.cum_logprobs, np.float32).view(np.int32)), label
                # the same forced prefix in the prompt and the same tails: same token counts
                for k in st:
                    assert st[k] == want.stats[k], (label, k, st[k], want.stats[k])
                cases += 1
                rows += len(ROWS)
                steps += st["decode_tokens"]
                forced += want.stats["forced_prefix_tokens"]
                no_plan += not want.stats["jump_forward"]
    finally:
        L.lib().sb200_model_close(h)
    assert forced > 0 and no_plan > 0
    print("PARITY", f"c_host[{model}]", f"tokens={eng.vocab.vocab_size}", f"cases={cases}",
          f"rows={rows}", f"decode_tokens={steps}", f"forced={forced}",
          f"cases_without_plan={no_plan}")
