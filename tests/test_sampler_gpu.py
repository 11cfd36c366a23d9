"""The sampler kernels (sampler_fsm.cu) against the numpy oracle, one step at a time through the
`sb200_sample` test hook, at vocabulary sizes from 7 to 151,936.

- Greedy: the token is the lowest index among the allowed maxima, bit for bit.
- Top-k / top-p: the kernel reports the key of its smallest kept z (`out_tau`); it must equal the
  oracle's key exactly for top-k, and for top-p whenever the oracle's boundary is further than
  TOP_P_MARGIN from being decided the other way.
- Draws: the Philox counter layout (seed, row id, step) is checked through tokens that expose u
  directly, and through counters found on the CPU that give the extreme draws.
- Log-probabilities against fp64 within the bound of `logprob_bound`.
- Row bookkeeping: every output buffer is filled with sentinels and compared, as integers, with a
  numpy restatement of `finish_row`.
"""
import math

import numpy as np
import pytest
import torch

from oracle import sampler_ref as S
from sutro_b200 import _lib as L
from sutro_b200 import engine as E

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -777                    # sentinel of every int32 output buffer
SENT_F = -1234.5
SENT_TAU = 0xDEADBEEF
VOCABS = [7, 33, 511, 512, 513, 1000, 50257, 128256, 151936]
QWEN, LLAMA = 151936, 128256

# top-p: the kernel's masses differ from the exact ones by __expf (<= (2 + 1.173|x|) ulp, so
# <= 4.4e-6 relative for x = z - zmax >= -30; smaller weights are < 1e-13 of W), by the fp32
# rounding of z - zmax when the compiler fuses it with the product (<= |z| 2^-24 <= 1.5e-5 for
# |z| <= 256, the range used here) and by the 2^-40 fixed point (< V 2^-41 <= 7e-8 of W).  Any
# partial mass is therefore within 2e-5 W of the exact one; 1e-4 leaves a factor of 2.5.
TOP_P_MARGIN = 1e-4
# draws: the kernel sums the kept weights in fp32 over chunks of up to ~300 terms per lane
# (relative error <= 300 * 2^-24 = 1.8e-5) on top of the weight errors above.
DRAW_SLACK = 1e-4

PHILOX_SEED, PHILOX_ROW = (1 << 33) + 12345, (1 << 32) + 7
STEP_U0, STEP_U1 = 20278614, 7548611     # u = 0 and u = 1 - 2^-24 for (PHILOX_SEED, PHILOX_ROW)


def i32(x):
    return torch.as_tensor(np.asarray(x, dtype=np.int32)).to(DEV)


def pack_masks(allowed):
    """bool [n_states, V] -> uint32 [n_states, ceil(V/32)], bit i & 31 of word i >> 5."""
    allowed = np.atleast_2d(allowed)
    n, V = allowed.shape
    words = (V + 31) // 32
    pad = np.zeros((n, words * 32), dtype=bool)
    pad[:, :V] = allowed
    return np.ascontiguousarray(np.packbits(pad, axis=-1, bitorder="little")).view(np.uint32)


def one_byte_vocab(V):
    """tok_bytes / tok_off for a vocabulary of one-byte tokens (token i = byte i % 256)."""
    return (np.arange(V) % 256).astype(np.uint8), np.arange(V + 1, dtype=np.int32)


def self_loop_dfa(n_states):
    """A DFA whose every byte keeps the state: masks given per state, no advance effects."""
    trans = np.tile(np.arange(n_states, dtype=np.int32)[:, None], (1, 256))
    return trans, np.zeros(n_states, np.uint8)


class Step:
    """One call of sb200_sample with every buffer sentinel-filled and read back."""

    def __init__(self, logits, *, T=0.0, k=0, p=1.0, seed=0, seed_per_row=0, row_ids=None,
                 masks=None, state=None, trans=None, final=None, tails=None, tok=None,
                 ngen=None, maxnew=None, done=None, eos=None, ignore_eos=0, cum=None,
                 row_slot=None, slot_row=None, n_slots=None, stride=None, ldl=None, B=None,
                 out_shift=0):
        self.lg = logits if torch.is_tensor(logits) else torch.as_tensor(np.asarray(logits, np.float32))
        self.lg = self.lg.to(DEV, torch.float32).contiguous()
        if self.lg.dim() == 1:
            self.lg = self.lg[None]
        V = self.lg.shape[1]
        B = self.lg.shape[0] if B is None else B
        n_slots = n_slots or B
        self.V, self.B = V, B
        self.row_slot = np.arange(B) if row_slot is None else np.asarray(row_slot)
        self.slot_row = np.arange(n_slots) if slot_row is None else np.asarray(slot_row)
        n_rows = int(self.slot_row.max()) + 1
        self.stride = stride or 8
        self.eos = V - 1 if eos is None else eos
        self.tb, self.to = one_byte_vocab(V) if tok is None else tok
        if masks is not None and trans is None:
            trans, final = self_loop_dfa(len(masks))
        self.trans, self.final, self.tails = trans, final, tails
        full = lambda v, d: np.full(n_slots, d, np.int32) if v is None else np.asarray(v, np.int32)
        self.in_state = full(state, 0 if masks is not None else -1)
        self.in_ngen = full(ngen, 0)
        self.in_maxnew = full(maxnew, self.stride)
        self.in_done = full(done, 0)
        self.in_cum = None if cum is None else np.asarray(cum, np.float32)
        d = lambda a, t=torch.int32: torch.as_tensor(np.array(a)).to(DEV, t).contiguous()
        self.d = {"state": d(self.in_state), "ngen": d(self.in_ngen), "done": d(self.in_done),
                  "next": d(np.full(n_slots, SENT)), "pos": d(np.arange(n_slots) * 10),
                  "out": d(np.full((n_rows, self.stride), SENT)), "len": d(np.full(n_rows, SENT)),
                  "tau": d(np.full(B, SENT_TAU, np.uint32).view(np.int32)),
                  "row_slot": d(self.row_slot), "slot_row": d(self.slot_row),
                  "maxnew": d(self.in_maxnew), "tb": d(self.tb, torch.uint8), "to": d(self.to)}
        self.in_pos = np.arange(n_slots) * 10
        if cum is not None:
            self.d["cum"] = d(self.in_cum, torch.float32)
            self.d["ocum"] = torch.full((n_rows,), SENT_F, device=DEV)
        if masks is not None:
            self.masks = np.atleast_2d(masks)
            self.d["mask"] = torch.as_tensor(pack_masks(self.masks).view(np.int32)).to(DEV)
        if trans is not None:
            self.d["trans"] = d(trans)
            self.d["final"] = d(final, torch.uint8)
        if tails is not None:
            self.d["toff"], self.d["ttok"] = d(tails[0]), d(tails[1])
        if row_ids is not None:
            self.row_ids = np.asarray(row_ids, np.int64)
            self.d["rid"] = d(self.row_ids, torch.int64)
        else:
            self.row_ids = None
        g = lambda n: L.ptr(self.d.get(n))
        a = E.SampleArgsC()
        a.logits, a.ldl, a.vocab, a.B = L.ptr(self.lg), V if ldl is None else ldl, V, B
        a.row_slot, a.slot_state, a.slot_ngen = g("row_slot"), g("state"), g("ngen")
        a.slot_next_tok, a.slot_pos, a.slot_done = g("next"), g("pos"), g("done")
        # out_shift: slots at step s write out_tokens[row * stride + s]; shifting the base lets
        # steps near 2^31 address a small buffer
        a.slot_row, a.slot_maxnew, a.out_len = g("slot_row"), g("maxnew"), g("len")
        a.out_tokens = g("out") - 4 * out_shift
        a.out_stride = self.stride
        a.mask_bits = g("mask")
        a.mask_words = (V + 31) // 32
        a.fsm_trans, a.fsm_final = g("trans"), g("final")
        a.fsm_tail_off, a.fsm_tail_tok = g("toff"), g("ttok")
        a.tok_bytes, a.tok_off = g("tb"), g("to")
        a.eos_id, a.ignore_eos = self.eos, ignore_eos
        a.temperature, a.top_k, a.top_p = T, k, p
        a.seed, a.seed_per_row, a.row_ids = seed, seed_per_row, g("rid")
        a.slot_cum_logprob, a.out_cum_logprob, a.out_tau = g("cum"), g("ocum"), g("tau")
        self.args = a
        self.T = T

    def run(self):
        L.check(L.lib().sb200_sample(E.C.byref(self.args), L.current_stream()))
        torch.cuda.synchronize()
        h = {n: t.cpu().numpy() for n, t in self.d.items()}
        h["tau"] = h["tau"].view(np.uint32)
        self.h = h
        return h

    def allowed(self, b):
        """bool [V]: the tokens row b may choose."""
        s = self.in_state[self.row_slot[b]]
        if s < 0 or not hasattr(self, "masks"):
            return np.ones(self.V, dtype=bool)
        return self.masks[s]

    def expect_rows(self, toks, stop=()):
        """Compare every int32 buffer with the numpy finish_row given the token of each row
        (None: the slot is done and must be untouched)."""
        state, ngen, done = self.in_state.copy(), self.in_ngen.copy(), self.in_done.copy()
        nxt, pos = np.full_like(state, SENT), self.in_pos.copy()
        out = np.full_like(self.h["out"], SENT)
        ln = np.full_like(self.h["len"], SENT)
        for b, tok in enumerate(toks):
            slot = self.row_slot[b]
            if self.in_done[slot]:
                continue
            row, n, fin, s = self.slot_row[slot], ngen[slot], False, state[slot]
            if b in stop or (tok == self.eos and not self.args.ignore_eos):
                fin = True
            else:
                out[row, n] = tok
                n += 1
                if s >= 0:
                    for byte in self.tb[self.to[tok]:self.to[tok + 1]]:
                        if s < 0:
                            break
                        s = self.trans[s, byte]
                    state[slot] = s
                    if s < 0 or self.final[s]:
                        fin = True
                    elif self.tails is not None and self.tails[0][s + 1] > self.tails[0][s]:
                        for t in self.tails[1][self.tails[0][s]:self.tails[0][s + 1]]:
                            if n >= self.in_maxnew[slot]:
                                break
                            out[row, n] = t
                            n += 1
                        fin = True
            if n >= self.in_maxnew[slot]:
                fin = True
            ngen[slot], ln[row] = n, n
            nxt[slot], pos[slot] = tok, pos[slot] + 1
            done[slot] |= int(fin)
        h = self.h
        np.testing.assert_array_equal(h["next"], nxt)
        np.testing.assert_array_equal(h["out"], out)
        np.testing.assert_array_equal(h["len"], ln)
        np.testing.assert_array_equal(h["ngen"], ngen)
        np.testing.assert_array_equal(h["pos"], pos)
        np.testing.assert_array_equal(h["done"], done)
        np.testing.assert_array_equal(h["state"], state)
        if self.in_cum is not None:           # done slots keep their sums bit for bit
            dn = self.in_done.astype(bool)
            np.testing.assert_array_equal(h["cum"][dn], self.in_cum[dn])


def logits_np(step, b):
    return step.lg[0 if step.args.ldl == 0 else b].cpu().numpy()


# --------------------------------------------------------------------------- log-prob bound
def logprob_bound(lg, allowed, T, tok):
    """Bound on |kernel log p(tok) - fp64 log p(tok)|.  The kernel sums se = sum_i __expf(x_i),
    x_i = z_i - zmax, in fp32 (a serial run of ceil(V/512) terms per thread, a 5-level warp
    tree, 16 warps in series) and returns (z_tok - zmax) - __logf(se).
    - __expf(x): <= 2 + floor(1.173|x|) ulp (CUDA C Programming Guide, intrinsic functions);
      x itself is rounded (|x| 2^-24) and may be fused with the product z = logit/T (|z| 2^-24).
    - the sum: first-order bound (n - 1) 2^-24 sum_i w_i with n the depth of the tree.
    - __logf(se): 2^-21.41 absolute for se in [0.5, 2], else 3 ulp.
    - the final subtraction: one fp32 rounding."""
    z = S.scaled(lg, T) if T > 0 else np.asarray(lg, np.float32)
    z = z[allowed & np.isfinite(z)].astype(np.float64)      # -inf terms are exactly 0
    zmax = z.max()
    x = z - zmax
    w = np.exp(x)
    se = w.sum()
    eps = (2 + 1.173 * np.abs(x)) * 2.0 ** -23 + (np.abs(x) + np.abs(z)) * 2.0 ** -24
    depth = math.ceil(len(lg) / 512) + 5 + 16
    rel = (eps * w).sum() / se + depth * 2.0 ** -24
    lse = math.log(se)
    log_err = 2.0 ** -21.41 if se <= 2 else 3 * float(np.spacing(np.float32(lse)))
    ztok = float(S.scaled(lg, T)[tok]) if T > 0 else float(lg[tok])
    lp = ztok - zmax - lse
    return 1.01 * (rel + log_err + (abs(ztok) + abs(ztok - zmax) + abs(lp)) * 2.0 ** -24) + 1e-12


RATIOS = {}


def note(group, ratio):
    RATIOS[group] = max(RATIOS.get(group, 0.0), float(ratio))
    print(f"[{group}] largest error/bound so far {RATIOS[group]:.3f}")


def check_logprob(step, toks, group):
    worst = 0.0
    for b, tok in enumerate(toks):
        if tok is None:
            continue
        allowed = step.allowed(b)
        lg = logits_np(step, b)
        ref = S.log_softmax(lg, allowed, step.T)[tok] + float(step.in_cum[step.row_slot[b]])
        got = float(step.h["cum"][step.row_slot[b]])
        bound = logprob_bound(lg, allowed, step.T, tok) + abs(ref) * 2.0 ** -24
        worst = max(worst, abs(got - ref) / bound)
        assert abs(got - ref) <= bound, (b, tok, got, ref, bound)
        assert step.h["ocum"][step.slot_row[step.row_slot[b]]] == got
    note(group, worst)


# --------------------------------------------------------------------------- greedy
def greedy_rows(V, rng):
    """Rows with planted exact ties and edge cases; -> (logits [B, V], masks [B, V])."""
    rows, masks = [], []
    full = np.ones(V, bool)

    def add(lg, m=full):
        rows.append(np.asarray(lg, np.float32))
        masks.append(m)

    base = lambda: rng.standard_normal(V).astype(np.float32) * 3
    chunk = ((V + 15) // 16 + 31) & ~31
    spots = sorted({0, V - 1, min(511, V - 1), min(512, V - 1), min(chunk - 1, V - 1),
                    min(chunk, V - 1), min(5 * chunk + 3, V - 1), V // 2})
    for a in spots:                       # ties at a and at every later spot: lowest index wins
        lg = base()
        lg[[s for s in spots if s >= a]] = 20.0
        add(lg)
    lg = base()
    lg[[0, V - 1]] = 9.0
    add(lg)
    add(-np.abs(base()) - 1)              # all negative
    lg = np.full(V, -np.inf, np.float32)  # all -inf but one
    lg[V // 3] = -5.0
    add(lg)
    m = rng.random(V) < 0.01              # random 1 % allowed
    m[rng.integers(V)] = True
    add(base(), m)
    m = np.zeros(V, bool)                 # a single allowed token, not the arg-max
    m[(V * 2) // 3] = True
    add(base(), m)
    m = np.zeros(V, bool)                 # only the last (partial) mask word
    m[(V - 1) // 32 * 32:] = True
    add(base(), m)
    lg = base()                           # tie between a masked and an allowed token
    lg[[1 % V, V - 1]] = 30.0
    m = full.copy()
    m[1 % V] = V == 1
    add(lg, m)
    return np.stack(rows), np.stack(masks)


def greedy_expect(lg, m):
    if not m.any():
        return None
    z = np.where(m, lg, -np.inf)
    return int(np.flatnonzero(z == z.max())[0])


@pytest.mark.parametrize("V", VOCABS)
def test_greedy_token_and_logprob(V):
    rng = np.random.default_rng(V)
    lg, masks = greedy_rows(V, rng)
    B = len(lg)
    cum = rng.standard_normal(B).astype(np.float32)
    st = Step(lg, masks=masks, state=np.arange(B), cum=cum, eos=V + 5, ignore_eos=0)
    st.run()
    toks = [greedy_expect(lg[b], masks[b]) for b in range(B)]
    st.expect_rows(toks)
    assert (st.h["tau"] == SENT_TAU).all()             # greedy leaves out_tau alone
    check_logprob(st, toks, "greedy log-prob")


def test_nothing_selectable_ends_the_row_without_output():
    """Greedy and stochastic, ignore_eos = 0 and 1: no allowed token -> done, EOS not appended,
    log-probability unchanged."""
    V = 1000
    for T in (0.0, 1.0):
        for ignore in (0, 1):
            masks = np.zeros((1, V), bool)
            st = Step(np.zeros((2, V)), T=T, masks=masks, state=[0, 0], ngen=[3, 0],
                      maxnew=[8, 8], eos=V - 2, ignore_eos=ignore, cum=[0.5, -1.0])
            st.run()
            st.expect_rows([V - 2, V - 2], stop=(0, 1))
            np.testing.assert_array_equal(st.h["cum"], np.float32([0.5, -1.0]))
            assert (st.h["tau"] == SENT_TAU).all()          # out_tau is not written


# --------------------------------------------------------------------------- top-k
def topk_cases(V, rng):
    """-> list of (logits, allowed, T, k)"""
    cases = []
    r = lambda: rng.standard_normal(V).astype(np.float32) * 2
    full = np.ones(V, bool)
    cases.append((r(), full, 1.0, 1))
    lg = r() - 10                                 # [5, 4, 4, 4, ...]: k = 3 keeps the three 4s
    lg[[0]] = 5
    idx = rng.choice(np.arange(1, V), size=min(3, V - 1), replace=False)
    lg[idx] = 4
    cases.append((lg, full, 1.0, 3))
    m = rng.random(V) < 0.3
    m[:2] = True
    cases.append((r(), m, 0.7, int(m.sum())))          # k = allowed count
    cases.append((r(), m, 0.7, int(m.sum()) + 1))      # k > allowed count
    cases.append((r(), full, 1.0, V + 10))             # k > V
    lg = r()
    lg[~m] = 50                                        # masked tokens would win without the mask
    cases.append((lg, m, 1.0, min(5, int(m.sum()))))
    cases.append((-np.abs(r()) - 3, full, 1.3, min(17, V)))   # negative range
    sub = (rng.standard_normal(V) * 1e-39).astype(np.float32)  # subnormal z
    cases.append((sub, full, 1.0, min(9, V)))
    zero = r() - 20                                   # signed zeros at the boundary
    zi = rng.choice(V, size=min(6, V), replace=False)
    zero[zi[:3]] = 0.0
    zero[zi[3:]] = -0.0
    zero[zi[0]] = 1.0
    cases.append((zero, full, 1.0, 2))
    return cases


@pytest.mark.parametrize("V", VOCABS)
def test_top_k_threshold_exact(V):
    rng = np.random.default_rng(1000 + V)
    for lg, m, T, k in topk_cases(V, rng):
        st = Step(lg, T=T, k=k, masks=m[None], seed=5)
        h = st.run()
        tau, _ = S.tau_expected(lg, m, T, k, 1.0)
        assert h["tau"][0] == tau, (T, k, hex(h["tau"][0]), hex(tau))
        keep = m & (S.fkey(S.scaled(lg, T)) >= tau)
        assert keep[h["next"][0]], (k, h["next"][0])


def test_signed_zero_ties_are_kept():
    """z = +0.0 is the k-th largest and another allowed token has z = -0.0: both are kept."""
    lg = np.array([3.0, 0.0, -1.0, -0.0, -2.0], np.float32)
    for k in (2, 3):
        st = Step(lg, T=1.0, k=k, seed=1)
        h = st.run()
        assert h["tau"][0] == S.fkey(np.float32(0.0)) == S.fkey(np.float32(-0.0))
    keep, _ = S.kept_set(lg, np.ones(5, bool), 1.0, 2, 1.0)
    assert keep.tolist() == [True, True, False, True, False]
    lg = np.array([0.0, -0.0, -0.0, -5.0], np.float32)        # top-p: the mode's ties
    st = Step(lg, T=1.0, p=1e-30, seed=1)
    assert st.run()["tau"][0] == S.fkey(np.float32(0.0))


def test_signed_zero_ties_are_drawn():
    """The kernel's own kept set, seen through its draws: when +0.0 is the threshold, the -0.0
    token (index 3) must be drawn wherever the oracle's u falls in its CDF interval."""
    B = 512
    rows = np.arange(B) + 2 ** 32
    us = S.uniform_np(5, rows.astype(np.uint64), 0, True)
    for lg, k, p in [([-1.0, 0.0, -3.0, -0.0, -2.0], 1, 1.0),     # top-1 keeps +0.0 and -0.0
                     ([-1.0, 0.0, -3.0, -0.0, -2.0], 0, 1e-30),   # top-p: the mode and its ties
                     ([3.0, 0.0, -1.0, -0.0, -2.0], 2, 1.0)]:     # +0.0 is the 2nd largest
        lg = np.array(lg, np.float32)
        st = Step(torch.as_tensor(lg)[None], T=1.0, k=k, p=p, seed=5, seed_per_row=1,
                  row_ids=rows, B=B, ldl=0, stride=1, eos=len(lg))
        h = st.run()
        want = [S.sample(lg, np.ones(len(lg), bool), 1.0, k, p, float(u)) for u in us]
        assert sum(t == 3 for t, _ in want) > 10
        for b, (tok, slack) in enumerate(want):
            assert h["next"][b] == tok or slack < DRAW_SLACK, (k, p, b, h["next"][b], tok)


# --------------------------------------------------------------------------- top-p
def topp_rows(V, rng, n):
    out = []
    for _ in range(n):
        # spread wide enough that the boundary token holds a fair share of the mass even at
        # V = 151,936; |z| stays below 256 (see TOP_P_MARGIN)
        lg = (rng.standard_normal(V) * rng.uniform(2, 6)).astype(np.float32)
        T = float(rng.choice([0.05, 0.7, 1.0, 1.7]))
        if T == 0.05:
            lg *= np.float32(min(1.0, 12.0 / np.abs(lg).max()))
        k = int(rng.choice([0, 0, 5, 40, 1000]))
        p = float(rng.choice([0.3, 0.8, 0.95, 0.99]))
        m = rng.random(V) < 0.5 if rng.random() < 0.3 else np.ones(V, bool)
        m[rng.integers(V)] = True
        out.append((lg, m, T, k, p))
    return out


@pytest.mark.parametrize("V", [33, 513, 50257, QWEN])
def test_top_p_threshold_matches_when_the_margin_allows(V):
    rng = np.random.default_rng(2000 + V)
    n = 48 if V <= LLAMA else 24
    cases = topp_rows(V, rng, n)
    checked = 0
    for T in sorted({c[2] for c in cases}):
        for k in sorted({c[3] for c in cases}):
            for p in sorted({c[4] for c in cases}):
                sel = [c for c in cases if c[2:] == (T, k, p)]
                if not sel:
                    continue
                lg = np.stack([c[0] for c in sel])
                ms = np.stack([c[1] for c in sel])
                st = Step(lg, T=T, k=k, p=p, masks=ms, state=np.arange(len(sel)), seed=11)
                h = st.run()
                for b, c in enumerate(sel):
                    tau, margin = S.tau_expected(c[0], c[1], T, k, p)
                    keep = c[1] & (S.fkey(S.scaled(c[0], T)) >= h["tau"][b])
                    assert keep[h["next"][b]]
                    if margin > TOP_P_MARGIN:
                        assert h["tau"][b] == tau, (V, T, k, p, hex(h["tau"][b]), hex(tau), margin)
                        checked += 1
    print(f"[top-p V={V}] {checked} of {n} margin-filtered cases checked")
    assert checked >= n // 2


@pytest.mark.parametrize("V", [7, 1000, QWEN])
def test_top_p_edges(V):
    rng = np.random.default_rng(3000 + V)
    full = np.ones(V, bool)
    cases = []
    lg = rng.standard_normal(V).astype(np.float32)
    ties = rng.choice(V, size=min(3, V), replace=False)
    lg[ties] = 6.0
    cases.append((lg, full, 1.0, 0, 1e-30))                # the mode and its ties
    m = np.zeros(V, bool)                                  # keeps all 7..20 allowed tokens
    m[rng.choice(V, size=min(20, V), replace=False)] = True
    cases.append((rng.uniform(-1, 1, V).astype(np.float32), m, 1.0, 0, 0.99999994))
    lg = rng.standard_normal(V).astype(np.float32)
    lg[rng.integers(V)] = 30.0                             # one token holds > p of the mass
    cases.append((lg, full, 1.0, 0, 0.9))
    cases.append((np.full(V, 0.25, np.float32), full, 1.0, 0, 0.5))   # flat: everything ties
    cases.append((rng.standard_normal(V).astype(np.float32), full, 0.7, min(20, V), 0.6))
    m = rng.random(V) < 0.2
    m[0] = True
    lg = rng.standard_normal(V).astype(np.float32)
    lg[m] *= 4
    lg[~m] += 20
    cases.append((lg, m, 1.0, 0, 0.7))
    checked = 0
    for lg, m, T, k, p in cases:
        st = Step(lg, T=T, k=k, p=p, masks=m[None], seed=3)
        h = st.run()
        tau, margin = S.tau_expected(lg, m, T, k, p)
        if margin > TOP_P_MARGIN:
            assert h["tau"][0] == tau, (T, k, p, hex(h["tau"][0]), hex(tau), margin)
            checked += 1
    print(f"[top-p edges V={V}] {checked} of {len(cases)} cases checked")
    assert checked >= len(cases) - 1


# --------------------------------------------------------------------------- draws
@pytest.mark.parametrize("V", [33, 1000, QWEN])
def test_uniform_rows_expose_the_philox_counter(V):
    """On flat rows every weight is 1: token = floor(fl(u * V)).  Seeds and row ids use both
    32-bit halves, steps reach 2^31 - 2 (the step is incremented after the draw)."""
    rng = np.random.default_rng(4000 + V)
    B = 64
    row_ids = (np.uint64(2 ** 32) * rng.integers(1, 2 ** 30, B).astype(np.uint64)
               + rng.integers(0, 2 ** 32, B).astype(np.uint64)).astype(np.int64)
    row_ids[0] = 0
    for seed in (0, (7 << 32) | 0x89ABCDEF, 2 ** 64 - 1):
        for spr in (0, 1):
            for step in (0, 1, int(rng.integers(2, 2 ** 31 - 2)), 2 ** 31 - 2):
                st = Step(torch.full((1, V), 0.5, device=DEV), T=0.8, seed=seed,
                          seed_per_row=spr, row_ids=row_ids, ngen=np.full(B, step),
                          maxnew=np.full(B, 2 ** 31 - 1), B=B, ldl=0, stride=1, out_shift=step,
                          eos=V)                      # no token is EOS: every draw is appended
                h = st.run()
                u = S.uniform_np(seed, row_ids.view(np.uint64), step, bool(spr))
                want = np.floor(u * np.float32(V)).astype(np.int64)
                np.testing.assert_array_equal(h["next"], want, err_msg=f"{seed} {spr} {step}")
                assert (h["tau"] == 0).all()
                np.testing.assert_array_equal(h["out"][:, 0], want)
                u = np.broadcast_to(u, B)
                assert u[1] == np.float32(S.uniform(seed, int(row_ids[1]), step, bool(spr)))


@pytest.mark.parametrize("V", [513, QWEN])
def test_extreme_draws_hit_the_first_and_last_kept_tokens(V):
    assert S.uniform(PHILOX_SEED, PHILOX_ROW, STEP_U0, True) == 0.0
    assert S.uniform(PHILOX_SEED, PHILOX_ROW, STEP_U1, True) == 1 - 2.0 ** -24
    chunk = ((V + 15) // 16 + 31) & ~31
    rng = np.random.default_rng(5000 + V)
    masks = []
    for lo, hi in [(0, V), (3 * chunk + 5, V), (0, V - 2 * chunk - 7), (chunk, chunk + 40)]:
        m = np.zeros(V, bool)
        m[lo:hi] = rng.random(hi - lo) < 0.5
        m[[lo, hi - 1]] = True
        masks.append(m)
    masks = np.stack(masks)
    nm = len(masks)
    lg = rng.standard_normal((nm, V)).astype(np.float32)
    for p in (1.0, 0.999):
        for step, pick in ((STEP_U0, 0), (STEP_U1, -1)):
            st = Step(lg, T=1.0, p=p, seed=PHILOX_SEED, seed_per_row=1,
                      row_ids=np.full(nm, PHILOX_ROW), masks=masks, state=np.arange(nm),
                      ngen=np.full(nm, step), maxnew=np.full(nm, 2 ** 31 - 1), stride=1,
                      out_shift=step)
            h = st.run()
            for b in range(nm):
                kept = np.flatnonzero(masks[b] & (S.fkey(S.scaled(lg[b], 1.0)) >= h["tau"][b]))
                assert h["next"][b] == kept[pick], (p, b, h["next"][b], kept[[0, -1]])


@pytest.mark.parametrize("V", [511, 50257, QWEN])
def test_random_draws_match_the_oracle(V):
    rng = np.random.default_rng(6000 + V)
    B = 64
    lg = (rng.standard_normal((B, V)) * 2).astype(np.float32)
    masks = rng.random((4, V)) < 0.6
    masks[:, 0] = True
    exceptions = 0
    for T, k, p in [(1.0, 0, 1.0), (0.7, 50, 0.9), (1.7, 0, 0.95)]:
        st = Step(lg, T=T, k=k, p=p, seed=99, seed_per_row=1, row_ids=np.arange(B) * 3 + 2 ** 40,
                  masks=masks, state=np.arange(B) % 4, ngen=np.arange(B) * 7, stride=512)
        h = st.run()
        for b in range(B):
            m = masks[b % 4]
            u = S.uniform(99, 3 * b + 2 ** 40, 7 * b, True)
            tau, margin = S.tau_expected(lg[b], m, T, k, p)
            if margin <= TOP_P_MARGIN:
                continue
            tok, slack = S.sample(lg[b], m, T, k, p, u)
            if h["next"][b] != tok:
                assert slack < DRAW_SLACK, (b, h["next"][b], tok, slack)
                exceptions += 1
    print(f"[draws V={V}] {exceptions} near-boundary exceptions of {3 * B}")
    assert exceptions <= 2


def test_small_kept_sets_hit_every_kept_token():
    """k <= 8 tokens of >= 5 % mass each: 2048 per-row draws hit all of them and nothing else."""
    V = QWEN
    rng = np.random.default_rng(7)
    for k in (2, 5, 8):
        lg = (rng.standard_normal(V) - 30).astype(np.float32)
        top = rng.choice(V, size=k, replace=False)
        lg[top] = np.log(rng.uniform(1.0, 2.0, k)).astype(np.float32)
        B = 2048
        st = Step(torch.as_tensor(lg)[None].to(DEV), T=1.0, k=k, seed=17, seed_per_row=1,
                  row_ids=np.arange(B) + 2 ** 33, B=B, ldl=0, stride=1)
        h = st.run()
        assert set(h["next"].tolist()) == set(top.tolist())
        us = S.uniform_np(17, np.arange(B, dtype=np.uint64) + np.uint64(2 ** 33), 0, True)
        want = [S.sample(lg, np.ones(V, bool), 1.0, k, 1.0, float(u)) for u in us[:64]]
        assert sum(h["next"][i] != t for i, (t, s) in enumerate(want) if s > DRAW_SLACK) == 0


# --------------------------------------------------------------------------- log-probabilities
@pytest.mark.parametrize("T", [0.05, 0.7, 1.0, 1.7, 10.0])
def test_logprob_against_fp64_over_three_steps(T):
    V, B = QWEN, 32
    rng = np.random.default_rng(int(T * 100))
    cum = np.zeros(B, np.float32)
    bound_sum = np.zeros(B)
    worst = 0.0
    ref_cum = np.zeros(B)
    masks = rng.random((2, V)) < 0.7
    masks[:, 5] = True
    ngen = np.zeros(B, np.int32)
    for step in range(3):
        lg = (rng.standard_normal((B, V)) * (2.0 if T >= 0.7 else 0.5)).astype(np.float32)
        st = Step(lg, T=T, k=0 if step != 1 else 100, p=1.0 if step != 2 else 0.9, seed=4,
                  seed_per_row=1, masks=masks, state=np.arange(B) % 2, cum=cum, ngen=ngen,
                  maxnew=np.full(B, 100), stride=100)
        h = st.run()
        for b in range(B):
            m = masks[b % 2]
            tok = int(h["next"][b])
            ref_cum[b] += S.log_softmax(lg[b], m, T)[tok]
            bound_sum[b] += logprob_bound(lg[b], m, T, tok) + abs(ref_cum[b]) * 2.0 ** -24
        err = np.abs(h["cum"].astype(np.float64) - ref_cum)
        worst = max(worst, float((err / bound_sum).max()))
        assert (err <= bound_sum).all(), (step, err.max(), bound_sum[err.argmax()])
        np.testing.assert_array_equal(h["ocum"], h["cum"])
        cum, ngen = h["cum"], h["ngen"]
    note(f"log-prob T={T}", worst)


# --------------------------------------------------------------------------- bookkeeping
def tiny_dfa():
    """Bytes a, b, c.  0 --c--> 0, 0 --a--> 1, 1 --b--> 2 (final), 1 --c--> 3, 3 --c--> 3,
    3 --b--> 4 (final).  Tokens: 0 a, 1 ab, 2 c, 3 b, 4 x (dead), 5 cc, 6 bc,
    7 <eos> (no bytes), 8 ca."""
    trans = np.full((5, 256), -1, np.int32)
    A, Bb, Cc = ord("a"), ord("b"), ord("c")
    trans[0, Cc], trans[0, A], trans[1, Bb], trans[1, Cc] = 0, 1, 2, 3
    trans[3, Cc], trans[3, Bb] = 3, 4
    accept = np.array([0, 0, 1, 0, 1], np.uint8)
    final = (accept.astype(bool) & (trans < 0).all(1)).astype(np.uint8)
    toks = [b"a", b"ab", b"c", b"b", b"x", b"cc", b"bc", b"", b"ca"]
    tb = np.frombuffer(b"".join(toks), np.uint8)
    to = np.concatenate([[0], np.cumsum([len(t) for t in toks])]).astype(np.int32)
    return trans, accept, final, tb, to


def test_row_bookkeeping_bit_exact():
    trans, accept, final, tb, to = tiny_dfa()
    V, eos = 9, 7
    # state 3 has the tail [3, 6, 3]; every other state none
    tails = (np.array([0, 0, 0, 0, 3, 3], np.int32), np.array([3, 6, 3], np.int32))
    cases = [  # (state, chosen token, ngen, maxnew, done)
        (0, 2, 0, 8, 0),     # c: stay in 0
        (0, 0, 1, 8, 0),     # a -> 1
        (1, 1, 0, 8, 0),     # a b from 1: dead -> done
        (1, 3, 2, 8, 0),     # b -> 2 final -> done
        (0, 4, 0, 8, 0),     # x: dead -> done
        (1, 2, 0, 8, 0),     # c -> 3: tail 3 6 3 appended, done
        (1, 2, 6, 8, 0),     # c -> 3: tail cut at maxnew
        (0, 5, 7, 8, 0),     # cc: maxnew reached
        (0, 7, 0, 8, 0),     # eos: done, not appended (ignore_eos = 0)
        (4, 2, 0, 8, 1),     # slot already done: untouched
        (0, 8, 0, 8, 0),     # ca -> 1
        (0, 2, 7, 7, 0),     # ngen already at maxnew
    ]
    n = len(cases)
    lg = np.full((n, V), -3.0, np.float32)
    for b, (_, t, *_r) in enumerate(cases):
        lg[b, t] = 5.0
    perm = np.random.default_rng(0).permutation(n)          # row b -> slot perm[b]
    slot_row = np.random.default_rng(1).permutation(n)      # slot -> output row
    st_ = np.zeros(n, np.int32)
    ng, mx, dn = (np.zeros(n, np.int32) for _ in range(3))
    for b, (s, t, g, m, d) in enumerate(cases):
        st_[perm[b]], ng[perm[b]], mx[perm[b]], dn[perm[b]] = s, g, m, d
    for T in (0.0, 0.5):
        for ignore in (0, 1):
            st = Step(lg, T=T, k=1 if T else 0, tok=(tb, to), trans=trans, final=final,
                      tails=tails, state=st_, ngen=ng, maxnew=mx, done=dn, eos=eos,
                      ignore_eos=ignore, row_slot=perm, slot_row=slot_row,
                      cum=np.arange(n, dtype=np.float32), stride=8)
            st.run()
            st.expect_rows([c[1] for c in cases])


def test_masks_at_full_size_from_a_compiled_schema():
    """sb200_fsm_build_mask over the qwen3 vocabulary against a numpy walk, then sampling
    under those masks."""
    from sutro_b200 import vocab as VB
    v = VB.build_vocab("qwen3", QWEN)
    schema = {"type": "object", "properties": {"label": {"enum": ["yes", "no", "maybe"]},
                                               "score": {"type": "integer", "minimum": 0,
                                                         "maximum": 99}},
              "required": ["label", "score"]}
    dfa = E.native_compile_schema(schema)
    n_st, V = len(dfa.accept), QWEN
    lens = np.array([len(t) for t in v.token_bytes])
    tb = np.frombuffer(b"".join(v.token_bytes), np.uint8)
    to = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    words = (V + 31) // 32
    d_mask = torch.zeros((n_st, words), dtype=torch.int32, device=DEV)
    d_tr, d_ac = i32(dfa.trans), torch.as_tensor(dfa.accept).to(DEV)
    d_tb, d_to = torch.as_tensor(tb).to(DEV), i32(to)
    L.check(L.lib().sb200_fsm_build_mask(L.ptr(d_tr), L.ptr(d_ac), n_st, L.ptr(d_tb), L.ptr(d_to),
                                         V, v.eos_id, L.ptr(d_mask), words, L.current_stream()))
    got = d_mask.cpu().numpy().view(np.uint32)
    pad = np.full((V, lens.max()), -1, np.int64)
    for i, t in enumerate(v.token_bytes):
        pad[i, :len(t)] = np.frombuffer(t, np.uint8)
    want = np.zeros((n_st, V), bool)
    for s in range(n_st):
        cur = np.full(V, s, np.int64)
        for j in range(pad.shape[1]):
            b = pad[:, j]
            go = (b >= 0) & (cur >= 0)
            cur[go] = dfa.trans[cur[go], b[go]]
        want[s] = (lens > 0) & (cur >= 0)
        want[s, v.eos_id] = bool(dfa.accept[s])
    np.testing.assert_array_equal(got, pack_masks(want))
    live = [s for s in range(n_st) if want[s].any()][:64]
    rng = np.random.default_rng(9)
    lg = rng.standard_normal((len(live), V)).astype(np.float32)
    for T, k, p in [(0.0, 0, 1.0), (1.0, 0, 0.9), (0.8, 3, 1.0)]:
        st = Step(lg, T=T, k=k, p=p, masks=want, state=live, tok=(tb, to), trans=dfa.trans,
                  final=dfa.final, eos=v.eos_id, seed=21, seed_per_row=1)
        st.d["mask"] = d_mask                       # sample under the kernel-built masks
        st.args.mask_bits = L.ptr(d_mask)
        h = st.run()
        for b, s in enumerate(live):
            if T == 0:
                assert h["next"][b] == greedy_expect(lg[b], want[s])
            else:
                tau, margin = S.tau_expected(lg[b], want[s], T, k, p)
                if margin > TOP_P_MARGIN:
                    assert h["tau"][b] == tau
                assert want[s][h["next"][b]]
        st.expect_rows(h["next"].tolist())


# --------------------------------------------------------------------------- determinism
def test_identical_launches_are_bit_identical():
    V, B = QWEN, 512
    g = torch.Generator(device=DEV).manual_seed(5)
    lg = torch.randn((B, V), generator=g, device=DEV) * 3
    for k in (0, 50):                       # top-p alone, and after top-k
        outs = []
        for _ in range(2):
            st = Step(lg, T=0.9, k=k, p=0.9, seed=8, seed_per_row=1, cum=np.zeros(B, np.float32))
            h = st.run()
            outs.append((h["next"].copy(), h["tau"].copy(), h["cum"].view(np.int32).copy()))
        for a, b in zip(*outs):
            np.testing.assert_array_equal(a, b)
        # every drawn token lies in the kept set the kernel reports
        z = lg[torch.arange(B, device=DEV), torch.as_tensor(outs[0][0]).to(DEV).long()].cpu().numpy()
        assert (S.fkey(S.scaled(z, 0.9)) >= outs[0][1]).all()
