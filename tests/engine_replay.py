"""Test helper: replay one row of an engine job through the verified kernels, with no scheduling.

The engine (csrc/engine.cu) batches rows, shares the system prompt's K/V between them, copies
the prefix's partial tail page into every row, recycles pages and slots, and chunks the LM head.
None of that may change a result: every kernel is batch-invariant (DESIGN.md §6).  So a row run
alone, here, through the same C-ABI kernels — its own freshly zeroed pages, one slot, one row per
launch — must give bit for bit the engine's tokens, first-decision logits and cumulative
log-probability.

The replay follows the engine's arithmetic contract, point by point:
  prompt     prefix | row | suffix (RefTokenizer.render, with the engine's truncation); under
             jump-forward the suffix also carries the forced output prefix (TokenFSM), which
             must equal the engine's own plan, as must its forced tails.
  split      share_prefix with n_prefix >= 16: the prefix runs first from position 0 (its
             post-RoPE K|V columns are kept in a dense buffer [layer][row][K|V]), then the rest
             runs from position n_prefix and reads that buffer.  Otherwise one pass from 0.
             Work items are (seq, t0) for t0 in steps of sb200_attn_prefill_q_tile.
  paged K/V  every position is written into the row's own pages, the prefix included (the
             engine shares the prefix's full pages and copies its partial tail page instead).
  decode     the first decode token sits at position P (prompt length), later ones follow;
             ctx_len = pos + 1.  The fused QKV GEMM of the C-ABI always stores the dense K/V
             columns, which the engine skips during decode: that changes neither the q columns
             nor the paged writes.
  sampling   sb200_sample with B = 1 on the replay's own slot, initialised as init_slots_kernel
             does (ngen = n_forced, pos = P - 1, state = fsm start, cum = 0); the Philox key is
             the row's id in the engine job.
  embedding  the last row, the final RMSNorm, then L2 normalisation.

The shared-prefix branch of the engine where the prompt ends inside the prefix is not replayed:
chat templates always end in a non-empty suffix, so no public call reaches it.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from oracle.bpe_ref import RefTokenizer
from oracle.fsm_ref import TokenFSM
from sutro_b200 import _lib as L
from sutro_b200 import engine as E
from sutro_b200 import vocab as VB

PAGE = 16
HD = 128
EPI_RESIDUAL_BF16, EPI_SWIGLU_BF16, EPI_STORE_F32 = 1, 2, 3
# switches that move the replay off the engine's path (SB200_QKV_DENSE=0: sb200_gemm_qkv_rope
# skips the dense K/V copy that the replayed prefill attention reads)
ENGINE_SWITCHES = ("SB200_QKV_DENSE",)


@dataclass
class RowReplay:
    tokens: List[int]
    first_logits: Optional[torch.Tensor]      # fp32 [vocab], cpu
    step_logits: List[torch.Tensor] = field(default_factory=list)
    cum_logprob: Optional[np.float32] = None
    embedding: Optional[np.ndarray] = None    # fp32 [d_model]
    prompt_len: int = 0
    decode_steps: int = 0


def _dev(a, dtype, device):
    return torch.as_tensor(np.ascontiguousarray(a)).to(device=device, dtype=dtype)


class Replay:
    """One-row replays for the jobs of one LocalEngine (same spec, weights and vocabulary)."""

    def __init__(self, eng):
        for k in ENGINE_SWITCHES:
            assert k not in os.environ, f"{k} changes the engine's path; unset it"
        self.eng, self.spec, self.w, self.v = eng, eng.spec, eng.weights, eng.vocab
        self.dev = eng.device
        self.lib = L.lib()
        s = self.spec
        self.q_tile = self.lib.sb200_attn_prefill_q_tile(s.n_q_heads, s.n_kv_heads)
        self.max_pages = (s.max_position + PAGE - 1) // PAGE + 1
        self.scale = float(np.float32(1.0) / np.sqrt(np.float32(HD)))
        self.ref = RefTokenizer(self.v)
        blob, off = self.v.byte_blob()
        self.tok_bytes = _dev(blob, torch.uint8, self.dev)
        self.tok_off = _dev(off, torch.int32, self.dev)

    # ---- prompt framing ------------------------------------------------------------------
    def template(self, system_prompt):
        s = self.spec
        if s.embedding_model:
            return VB.embedding_template(s.family)
        return VB.chat_template(s.family, system_prompt, getattr(self.eng, "empty_think_block",
                                                                 False))

    def framing(self, system_prompt):
        """(prefix ids, template suffix ids), checked against what the engine sends."""
        tpl = self.template(system_prompt)
        pre, suf = self.ref.encode_pieces(tpl.prefix), self.ref.encode_pieces(tpl.suffix)
        e_pre, e_suf = self.eng._template_tokens(system_prompt)
        assert list(e_pre) == pre and list(e_suf) == suf, "template ids differ from the engine's"
        return pre, suf

    def jump_plan(self, json_schema, fsm_limits, jump_forward, max_new):
        """(dfa, forced prefix ids, fsm start, tail_off, tail_tok) as the engine runs the job;
        the forced prefix and the tails come from the oracle's TokenFSM and must equal the
        engine's plan."""
        if json_schema is None:
            return None, [], -1, None, None
        dfa = self.eng.compile_schema(json_schema, fsm_limits)
        if not jump_forward:
            return dfa, [], dfa.start, None, None
        plan = self.eng._jump_plan(dfa, (id(dfa),))
        fsm = TokenFSM(dfa, self.v)
        if not fsm.enable_jump_forward(self.ref):
            assert plan is None
            return dfa, [], dfa.start, None, None
        assert plan is not None
        assert plan["prefix_tokens"].tolist() == fsm.forced_prefix
        assert plan["start"] == fsm.start
        off, tok = plan["tail_off"], plan["tail_tok"]
        for st in range(dfa.n_states):
            assert tok[off[st]:off[st + 1]].tolist() == fsm.tails.get(st, []), st
        if len(fsm.forced_prefix) >= max_new:        # the engine drops the plan then
            return dfa, [], dfa.start, None, None
        return dfa, list(fsm.forced_prefix), fsm.start, off, tok

    # ---- one forward pass of one sequence --------------------------------------------------
    def _forward(self, ids, past, pool, pt, prefix_kv=None, fill_prefix=False, ctx_len=None):
        """T = len(ids) tokens at positions past.. (prefill), or one token (ctx_len given:
        decode against the paged history).  Returns the residual stream x [T, d]."""
        s, w, lib, dev = self.spec, self.w, self.lib, self.dev
        st = L.current_stream()
        T, d = len(ids), s.d_model
        hq, hkv = s.n_q_heads, s.n_kv_heads
        q_dim, qkv_dim = hq * HD, (hq + 2 * hkv) * HD
        tok = _dev(ids, torch.int32, dev)
        pos = torch.arange(past, past + T, dtype=torch.int32, device=dev)
        slot = torch.zeros(T, dtype=torch.int32, device=dev)
        x = torch.empty(T, d, dtype=torch.bfloat16, device=dev)
        h = torch.empty_like(x)
        qkv = torch.zeros(T, qkv_dim, dtype=torch.bfloat16, device=dev)
        attn = torch.empty(T, q_dim, dtype=torch.bfloat16, device=dev)
        act = torch.empty(T, s.d_ff, dtype=torch.bfloat16, device=dev)
        if ctx_len is None:
            items = _dev([[0, t0] for t0 in range(0, T, self.q_tile)], torch.int32, dev)
            q_start = torch.zeros(1, dtype=torch.int32, device=dev)
            q_len = torch.full((1,), T, dtype=torch.int32, device=dev)
            seq_past = torch.full((1,), past, dtype=torch.int32, device=dev)
        else:
            row_slot = torch.zeros(1, dtype=torch.int32, device=dev)
            ctx = torch.full((1,), ctx_len, dtype=torch.int32, device=dev)
        L.check(lib.sb200_embed_gather(tok.data_ptr(), w.embed.data_ptr(), x.data_ptr(), T, d, st))
        for l in range(s.n_layers):
            kv_layer = pool[l].data_ptr()
            L.check(lib.sb200_rmsnorm(x.data_ptr(), w.ln1[l].data_ptr(), h.data_ptr(), T, d,
                                      s.rms_eps, st))
            L.check(lib.sb200_gemm_qkv_rope(
                h.data_ptr(), T, w.wqkv[l].data_ptr(), qkv.data_ptr(), T, d, 0,
                L.ptr(w.q_norm[l] if s.qk_norm else None),
                L.ptr(w.k_norm[l] if s.qk_norm else None),
                self.eng.cos.data_ptr(), self.eng.sin.data_ptr(), slot.data_ptr(), pos.data_ptr(),
                pt.data_ptr(), self.max_pages, kv_layer, hq, hkv, s.rms_eps, st))
            if ctx_len is None:
                if fill_prefix:
                    prefix_kv[l, :T].copy_(qkv[:, q_dim:])
                L.check(lib.sb200_attn_prefill_dense(
                    qkv.data_ptr(), T, attn.data_ptr(), L.ptr(prefix_kv),
                    0 if prefix_kv is None else prefix_kv.shape[1], s.n_layers, l,
                    items.data_ptr(), items.shape[0], q_start.data_ptr(), q_len.data_ptr(),
                    seq_past.data_ptr(), hq, hkv, self.scale, st))
            else:
                L.check(lib.sb200_attn_decode(qkv.data_ptr(), attn.data_ptr(), kv_layer,
                                              pt.data_ptr(), self.max_pages, row_slot.data_ptr(),
                                              ctx.data_ptr(), 1, hq, hkv, self.scale, st))
            L.check(lib.sb200_gemm_bf16_tn(attn.data_ptr(), T, w.wo[l].data_ptr(), x.data_ptr(),
                                           x.data_ptr(), T, d, q_dim, d, EPI_RESIDUAL_BF16, 0, st))
            L.check(lib.sb200_rmsnorm(x.data_ptr(), w.ln2[l].data_ptr(), h.data_ptr(), T, d,
                                      s.rms_eps, st))
            L.check(lib.sb200_gemm_bf16_tn(h.data_ptr(), T, w.wgu[l].data_ptr(), act.data_ptr(),
                                           None, T, 2 * s.d_ff, d, s.d_ff, EPI_SWIGLU_BF16, 0, st))
            L.check(lib.sb200_gemm_bf16_tn(act.data_ptr(), T, w.wd[l].data_ptr(), x.data_ptr(),
                                           x.data_ptr(), T, d, s.d_ff, d, EPI_RESIDUAL_BF16, 0, st))
        return x

    def _final_norm(self, x_last):
        s = self.spec
        hn = torch.empty(1, s.d_model, dtype=torch.bfloat16, device=self.dev)
        L.check(self.lib.sb200_rmsnorm(x_last.data_ptr(), self.w.final_norm.data_ptr(),
                                       hn.data_ptr(), 1, s.d_model, s.rms_eps,
                                       L.current_stream()))
        return hn

    def _logits(self, x_last, out):
        s = self.spec
        hn = self._final_norm(x_last)
        L.check(self.lib.sb200_gemm_bf16_tn(hn.data_ptr(), 1, self.w.lm_head.data_ptr(),
                                            out.data_ptr(), None, 1, s.vocab_size, s.d_model,
                                            s.vocab_size, EPI_STORE_F32, 0, L.current_stream()))

    # ---- one row ---------------------------------------------------------------------------
    def row(self, prompt: List[int], n_prefix: int, share_prefix: bool, max_new: int,
            row_id: int = 0, dfa=None, fsm_start: int = -1, forced=(), tail_off=None,
            tail_tok=None, mask=None, ignore_eos=False, temperature=0.0, top_k=0, top_p=1.0,
            seed=0, seed_per_row=False, keep_step_logits=False) -> RowReplay:
        s, dev = self.spec, self.dev
        P = len(prompt)
        emb_mode = s.embedding_model
        max_new = 0 if emb_mode else max_new
        prefix_cached = n_prefix if (share_prefix and n_prefix >= PAGE) else 0
        if prefix_cached:
            assert P - 1 >= prefix_cached, "prompt ends inside the shared prefix (not replayed)"
        n_pages = (P + max_new + PAGE - 1) // PAGE
        pool = torch.zeros(s.n_layers, n_pages, s.n_kv_heads, 2, PAGE, HD, dtype=torch.bfloat16,
                           device=dev)
        pt = torch.zeros(1, self.max_pages, dtype=torch.int32)
        pt[0, :n_pages] = torch.arange(n_pages - 1, -1, -1, dtype=torch.int32)  # non-trivial ids
        pt = pt.to(dev)
        if prefix_cached:
            prefix_kv = torch.zeros(s.n_layers, prefix_cached, 2 * s.n_kv_heads * HD,
                                    dtype=torch.bfloat16, device=dev)
            self._forward(prompt[:prefix_cached], 0, pool, pt, prefix_kv, fill_prefix=True)
            x = self._forward(prompt[prefix_cached:], prefix_cached, pool, pt, prefix_kv)
        else:
            x = self._forward(prompt, 0, pool, pt)
        x_last = x[-1:]
        if emb_mode:
            hn = self._final_norm(x_last)
            e = torch.empty(1, s.d_model, dtype=torch.float32, device=dev)
            L.check(self.lib.sb200_l2_normalize_rows(hn.data_ptr(), e.data_ptr(), 1, s.d_model,
                                                     L.current_stream()))
            return RowReplay([], None, embedding=e[0].cpu().numpy(), prompt_len=P)

        i32 = lambda v: torch.tensor([v], dtype=torch.int32, device=dev)  # noqa: E731
        n_forced = len(forced)
        st = dict(state=i32(fsm_start if dfa is not None else -1), ngen=i32(n_forced),
                  next=i32(0), pos=i32(P - 1), done=i32(0), row=i32(0), maxnew=i32(max_new),
                  slot=i32(0))
        out = torch.zeros(1, max_new, dtype=torch.int32, device=dev)
        if n_forced:
            out[0, :n_forced] = torch.as_tensor(list(forced), dtype=torch.int32)
        out_len = i32(n_forced)
        cum = torch.zeros(1, dtype=torch.float32, device=dev)
        out_cum = torch.zeros(1, dtype=torch.float32, device=dev)
        rid = torch.tensor([row_id], dtype=torch.int64, device=dev)
        logits = torch.empty(1, s.vocab_size, dtype=torch.float32, device=dev)
        keep = []
        a = E.SampleArgsC()
        a.logits, a.ldl, a.vocab, a.B = logits.data_ptr(), s.vocab_size, s.vocab_size, 1
        a.row_slot, a.slot_state, a.slot_ngen = (st["slot"].data_ptr(), st["state"].data_ptr(),
                                                 st["ngen"].data_ptr())
        a.slot_next_tok, a.slot_pos, a.slot_done = (st["next"].data_ptr(), st["pos"].data_ptr(),
                                                    st["done"].data_ptr())
        a.slot_row, a.slot_maxnew = st["row"].data_ptr(), st["maxnew"].data_ptr()
        a.out_tokens, a.out_len, a.out_stride = out.data_ptr(), out_len.data_ptr(), max_new
        if dfa is not None:
            trans = _dev(dfa.trans, torch.int32, dev)
            accept = _dev(dfa.accept, torch.uint8, dev)
            final = _dev(dfa.final, torch.uint8, dev)
            keep += [trans, accept, final]
            a.mask_bits, a.mask_words = mask.data_ptr(), mask.shape[1]
            a.fsm_trans, a.fsm_accept, a.fsm_final = (trans.data_ptr(), accept.data_ptr(),
                                                      final.data_ptr())
            if tail_off is not None:
                t_off, t_tok = _dev(tail_off, torch.int32, dev), _dev(tail_tok, torch.int32, dev)
                keep += [t_off, t_tok]
                a.fsm_tail_off, a.fsm_tail_tok = t_off.data_ptr(), t_tok.data_ptr()
        a.tok_bytes, a.tok_off = self.tok_bytes.data_ptr(), self.tok_off.data_ptr()
        a.eos_id, a.ignore_eos = self.v.eos_id, int(ignore_eos)
        # the engine's reading of the sampling fields (Engine::head_and_sample)
        a.temperature = temperature if temperature > 0 else 0.0
        a.top_k = top_k
        a.top_p = top_p if 0.0 < top_p < 1.0 else 1.0
        a.seed, a.seed_per_row = int(seed) & (2 ** 64 - 1), int(seed_per_row)
        a.row_ids = rid.data_ptr()
        a.slot_cum_logprob, a.out_cum_logprob = cum.data_ptr(), out_cum.data_ptr()

        res = RowReplay([], None, prompt_len=P)

        def head_and_sample(x_last):
            self._logits(x_last, logits)
            if res.first_logits is None:
                res.first_logits = logits[0].cpu()
            if keep_step_logits:
                res.step_logits.append(logits[0].cpu())
            L.check(self.lib.sb200_sample(C.byref(a), L.current_stream()))

        head_and_sample(x_last)
        pos = P                                   # position of the first decode token
        while not int(st["done"].item()):
            x = self._forward([int(st["next"].item())], pos, pool, pt, ctx_len=pos + 1)
            head_and_sample(x)
            pos += 1
            res.decode_steps += 1
            assert res.decode_steps <= max_new, "replay did not stop"
        n = int(out_len.item())
        res.tokens = out[0, :n].cpu().tolist()
        res.cum_logprob = np.float32(out_cum.item())
        return res

    # ---- one job ---------------------------------------------------------------------------
    def job(self, rows, system_prompt=None, json_schema=None, fsm_limits=None, max_new_tokens=64,
            ignore_eos=False, truncate_rows=True, share_prefix=True, jump_forward=True,
            temperature=0.0, top_k=0, top_p=1.0, seed=0, seed_per_row=False, row_ids=None,
            keep_step_logits=False) -> List[RowReplay]:
        """Replay every row of `eng.generate(rows, **same arguments)`."""
        assert truncate_rows, "only the truncating framing is replayed"
        s = self.spec
        max_new = 0 if s.embedding_model else max_new_tokens
        pre, suf = self.framing(system_prompt)
        dfa, forced, fsm_start, tail_off, tail_tok = (None, [], -1, None, None)
        mask = None
        if not s.embedding_model:
            dfa, forced, fsm_start, tail_off, tail_tok = self.jump_plan(
                json_schema, fsm_limits, jump_forward, max_new)
        if dfa is not None:
            words = (s.vocab_size + 31) // 32
            mask = torch.empty(dfa.n_states, words, dtype=torch.int32, device=self.dev)
            trans = _dev(dfa.trans, torch.int32, self.dev)
            accept = _dev(dfa.accept, torch.uint8, self.dev)
            L.check(self.lib.sb200_fsm_build_mask(trans.data_ptr(), accept.data_ptr(), dfa.n_states,
                                                  self.tok_bytes.data_ptr(),
                                                  self.tok_off.data_ptr(), s.vocab_size,
                                                  self.v.eos_id, mask.data_ptr(), words,
                                                  L.current_stream()))
        tpl = self.template(system_prompt)
        out = []
        for i, r in enumerate(rows):
            prompt = self.ref.render(tpl, "" if r is None else r,
                                     s.max_position - max_new - len(forced))
            prompt = prompt + forced
            rid = i if (row_ids is None or not seed_per_row) else int(row_ids[i])
            out.append(self.row(prompt, len(pre), share_prefix, max_new, rid, dfa, fsm_start,
                                forced, tail_off, tail_tok, mask, ignore_eos, temperature, top_k,
                                top_p, seed, seed_per_row, keep_step_logits))
        return out
