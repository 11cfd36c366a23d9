"""Python host for the engine-level C-ABI (include/sutro_b200.h).

`LocalEngine` is one model replica on one GPU: weights (PyTorch tensors, only as
storage), the GPU tokenizer, and the C++ scheduler.  `LocalEngine.generate()` is the
whole hot path for a list of rows: encode -> H2D -> tokenize -> prefill/decode with
optional schema mask -> detokenize -> D2H.  No step runs on the CPU; if the shared
library or a CUDA device is missing this module raises.
"""
from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import modelspec as MS
from . import vocab as VB
from .common import check_penalties
from .schema_fsm import ByteDFA, FsmLimits, compile_schema, compile_thinking
from .unicode_tables import class_table

c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_u8p = C.POINTER(C.c_uint8)
c_vpp = C.POINTER(C.c_void_p)


class EngineConfigC(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("n_layers", "d_model", "n_q_heads", "n_kv_heads", "d_ff",
                                       "vocab", "max_position")] + \
               [("rms_eps", C.c_float), ("qk_norm", C.c_int), ("embedding_model", C.c_int),
                ("eos_id", C.c_int), ("max_slots", C.c_int), ("max_prefill_tokens", C.c_int),
                ("logit_chunk_rows", C.c_int), ("min_admit_rows", C.c_int),
                ("num_pages", C.c_int64)]


class EngineWeightsC(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("embed", "lm_head", "final_norm", "rope_cos",
                                          "rope_sin")] + \
               [(n, c_vpp) for n in ("ln1", "ln2", "wqkv", "wo", "wgu", "wd", "q_norm", "k_norm")]


PROGRESS_FN = C.CFUNCTYPE(None, C.c_int64, C.c_int64, C.c_int64, C.c_void_p)


class JobC(C.Structure):
    _fields_ = [("row_tokens_dev", C.c_void_p), ("row_tok_off_dev", C.c_void_p),
                ("row_tok_off", c_i64p), ("n_rows", C.c_int64),
                ("prefix_tokens", c_i32p), ("n_prefix", C.c_int),
                ("suffix_tokens", c_i32p), ("n_suffix", C.c_int),
                ("share_prefix", C.c_int), ("max_new_tokens", C.c_int), ("ignore_eos", C.c_int),
                ("truncate_rows", C.c_int),
                ("fsm_trans", c_i32p), ("fsm_accept", c_u8p), ("fsm_final", c_u8p),
                ("fsm_states", C.c_int), ("fsm_start", C.c_int),
                ("n_forced_prefix", C.c_int), ("fsm_tail_off", c_i32p), ("fsm_tail_tok", c_i32p),
                ("out_tokens_dev", C.c_void_p), ("out_len_dev", C.c_void_p),
                ("out_embed_dev", C.c_void_p),
                ("progress", PROGRESS_FN), ("progress_user", C.c_void_p), ("profile", C.c_int),
                ("out_first_logits_dev", C.c_void_p),
                ("temperature", C.c_float), ("top_k", C.c_int), ("top_p", C.c_float),
                ("seed", C.c_uint64), ("seed_per_row", C.c_int),
                ("out_cum_logprob_dev", C.c_void_p), ("row_ids_dev", C.c_void_p),
                ("presence_penalty", C.c_float), ("frequency_penalty", C.c_float),
                ("repetition_penalty", C.c_float), ("min_p", C.c_float)]


# indexed by SB200_KC_*; "rope" stays in the stats layout but counts 0: RoPE and the K/V write
# run in the QKV GEMM's epilogue, counted under "gemm"
KERNEL_CLASSES = ["gemm", "attn_decode", "attn_prefill", "norm", "rope", "sample", "embed",
                  "other"]
_STAT_INTS = ("rows_done", "input_tokens", "prefill_tokens", "decode_tokens", "prefill_steps",
              "decode_steps", "rows_truncated", "prefix_cached_tokens")


class JobStatsC(C.Structure):
    _fields_ = [(n, C.c_int64) for n in _STAT_INTS] + \
               [("kernel_launches", C.c_int64 * 8), ("kernel_ms", C.c_double * 8),
                ("gemm_flops", C.c_double), ("attn_decode_bytes", C.c_double),
                ("t_h2d_ms", C.c_double), ("t_device_ms", C.c_double), ("t_d2h_ms", C.c_double)]

    def counters(self) -> Dict[str, Any]:
        """The job's counters as every entry point's stats dict reports them."""
        stats: Dict[str, Any] = {k: int(getattr(self, k)) for k in _STAT_INTS}
        stats["kernel_launches"] = dict(zip(KERNEL_CLASSES, list(self.kernel_launches)))
        stats["kernel_ms"] = dict(zip(KERNEL_CLASSES, list(self.kernel_ms)))
        stats["gemm_flops"], stats["attn_decode_bytes"] = self.gemm_flops, self.attn_decode_bytes
        return stats


L.register("sb200_engine_create", C.c_int, [C.POINTER(EngineConfigC), C.POINTER(EngineWeightsC),
                                            C.POINTER(C.c_void_p)])
L.register("sb200_engine_destroy", None, [C.c_void_p])
L.register("sb200_engine_set_vocab", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p])
L.register("sb200_engine_run", C.c_int, [C.c_void_p, C.POINTER(JobC), C.POINTER(JobStatsC)])
L.register("sb200_engine_stream", C.c_void_p, [C.c_void_p])
L.register("sb200_tokenizer_create", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                               C.POINTER(C.c_void_p)])
L.register("sb200_tokenizer_set_word_overrides", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p,
                                                           C.c_void_p, C.c_int])
L.register("sb200_tokenizer_destroy", None, [C.c_void_p])
L.register("sb200_tokenizer_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                               C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p])
L.register("sb200_tokenizer_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                               C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p])


def word_override_arrays(v: VB.Vocab):
    """Vocab.word_overrides -> (flat tokens, offsets[n+1], ids), int32, as the C-ABI takes them."""
    seqs = v.word_overrides or []
    off = np.zeros(len(seqs) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(s) for s, _ in seqs])
    toks = np.asarray([t for s, _ in seqs for t in s], dtype=np.int32)
    ids = np.asarray([e for _, e in seqs], dtype=np.int32)
    return np.ascontiguousarray(toks), off, np.ascontiguousarray(ids)


class ResultC(C.Structure):          # sb200_result (include/sutro_b200.h)
    _fields_ = [("n_rows", C.c_int64), ("bytes", c_u8p), ("offsets", c_i64p),
                ("tokens", c_i32p), ("token_offsets", c_i64p), ("cum_logprob", C.POINTER(C.c_float)),
                ("embeddings", C.POINTER(C.c_float)), ("d_model", C.c_int)]


class SampleArgsC(C.Structure):     # sb200_sample_args (test hook: one sampling step)
    _fields_ = [("logits", C.c_void_p), ("ldl", C.c_int), ("vocab", C.c_int), ("B", C.c_int)] + \
               [(n, C.c_void_p) for n in ("row_slot", "slot_state", "slot_ngen", "slot_next_tok",
                                          "slot_pos", "slot_done", "slot_row", "slot_maxnew",
                                          "out_tokens", "out_len")] + \
               [("out_stride", C.c_int), ("mask_bits", C.c_void_p), ("mask_words", C.c_int)] + \
               [(n, C.c_void_p) for n in ("fsm_trans", "fsm_accept", "fsm_final", "fsm_tail_off",
                                          "fsm_tail_tok", "tok_bytes", "tok_off")] + \
               [("eos_id", C.c_int), ("ignore_eos", C.c_int), ("temperature", C.c_float),
                ("top_k", C.c_int), ("top_p", C.c_float), ("seed", C.c_uint64),
                ("seed_per_row", C.c_int)] + \
               [(n, C.c_void_p) for n in ("row_ids", "slot_cum_logprob", "out_cum_logprob",
                                          "out_tau")] + \
               [(n, C.c_float) for n in ("presence_penalty", "frequency_penalty",
                                         "repetition_penalty", "min_p")] + \
               [("prompt_prefix", C.c_void_p), ("n_prompt_prefix", C.c_int),
                ("prompt_suffix", C.c_void_p), ("n_prompt_suffix", C.c_int)] + \
               [(n, C.c_void_p) for n in ("row_tokens", "row_tok_off", "slot_n_row_tok")]


L.register("sb200_sample", C.c_int, [C.POINTER(SampleArgsC), C.c_void_p])
L.register("sb200_engine_info", C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 4)
L.register("sb200_infer_text", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                         C.POINTER(JobC), C.c_int, C.c_int,
                                         C.POINTER(C.POINTER(ResultC)), C.POINTER(JobStatsC)])
L.register("sb200_result_free", None, [C.POINTER(ResultC)])
L.register("sb200_compact_rows", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p])
L.register("sb200_rows_select", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p])


class FsmLimitsC(C.Structure):       # sb200_fsm_limits
    _fields_ = [(n, C.c_int) for n in ("max_string_chars", "max_array_items", "max_int_digits",
                                       "max_frac_digits", "small_int_range", "max_recursion")]


L.register("sb200_fsm_limits_default", None, [C.POINTER(FsmLimitsC)])
L.register("sb200_schema_compile", C.c_int, [C.c_char_p, C.c_int64, C.POINTER(FsmLimitsC),
                                             C.POINTER(C.c_void_p)])
L.register("sb200_schema_destroy", None, [C.c_void_p])
L.register("sb200_schema_tables", C.c_int, [C.c_void_p, C.POINTER(c_i32p), C.POINTER(c_u8p),
                                            C.POINTER(c_u8p), C.POINTER(C.c_int),
                                            C.POINTER(C.c_int)])
L.register("sb200_schema_longest_path", C.c_int64, [C.c_void_p])
L.register("sb200_model_open", C.c_int, [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int64,
                                         C.POINTER(C.c_void_p)])
L.register("sb200_model_close", None, [C.c_void_p])
L.register("sb200_model_engine", C.c_void_p, [C.c_void_p])
L.register("sb200_model_tokenizer", C.c_void_p, [C.c_void_p])
L.register("sb200_model_infer", C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int64,
                                          C.POINTER(FsmLimitsC), C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p])


def native_compile_schema(schema: Dict[str, Any], limits: Optional[FsmLimits] = None) -> ByteDFA:
    """JSON schema -> ByteDFA through the C-ABI compiler (csrc/schema_compile.cu): what a
    non-Python host calls.  Raises SchemaError (a ValueError) for argument errors, exactly
    like schema_fsm.compile_schema; the Python compiler covers a larger keyword set."""
    import json

    from .schema_fsm import SchemaError
    text = json.dumps(schema, ensure_ascii=False).encode("utf-8")
    lim = None
    if limits is not None:
        lim = FsmLimitsC(limits.max_string_chars, limits.max_array_items, limits.max_int_digits,
                         limits.max_frac_digits, limits.small_int_range, limits.max_recursion)
    h = C.c_void_p()
    rc = L.lib().sb200_schema_compile(text, len(text), None if lim is None else C.byref(lim),
                                      C.byref(h))
    if rc != 0:
        msg = L.lib().sb200_last_error().decode("utf-8", "replace")
        raise SchemaError(msg) if rc == -2 else L.Sb200Error(msg)
    try:
        tr, ac, fi = c_i32p(), c_u8p(), c_u8p()
        n, start = C.c_int(), C.c_int()
        L.check(L.lib().sb200_schema_tables(h, C.byref(tr), C.byref(ac), C.byref(fi), C.byref(n),
                                            C.byref(start)))
        ns = n.value
        return ByteDFA(np.ctypeslib.as_array(tr, shape=(ns, 256)).copy(),
                       np.ctypeslib.as_array(ac, shape=(ns,)).copy(),
                       np.ctypeslib.as_array(fi, shape=(ns,)).copy(), int(start.value))
    finally:
        L.lib().sb200_schema_destroy(h)


def _np_ptr(a: np.ndarray, typ):
    return a.ctypes.data_as(typ)


# --------------------------------------------------------------------------- Arrow-style text
def rows_to_blob(rows) -> Tuple[np.ndarray, np.ndarray]:
    """list[str] / pyarrow array / pandas Series -> (uint8 blob, int64 offsets[n+1]).
    None becomes the empty string (the reference maps nulls to "" when concatenating
    columns, sutro/common.py:83,97)."""
    import pyarrow as pa
    if isinstance(rows, (pa.Array, pa.ChunkedArray)):
        arr = rows
    else:
        arr = pa.array(["" if r is None else (r if isinstance(r, str) else str(r)) for r in rows]
                       if not _all_str(rows) else rows, type=pa.large_string())
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    if arr.type != pa.large_string():
        arr = arr.cast(pa.large_string())
    if arr.null_count:
        arr = arr.fill_null("")
    bufs = arr.buffers()
    n = len(arr)
    off = np.frombuffer(bufs[1], dtype=np.int64, count=n + 1, offset=arr.offset * 8)
    data = (np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None
            else np.zeros(0, dtype=np.uint8))
    if off[0] != 0:
        data = data[off[0]:off[-1]]
        off = off - off[0]
    else:
        data = data[:off[-1]]
    return data, off


def _nfc_rows(rows):
    """NFC-normalised rows.  Arrow input stays Arrow: an all-ASCII column is already NFC and is
    returned as is, any other is normalised row by row (`pyarrow.compute.utf8_normalize` is not
    used: pyarrow 24.0 returns decomposed text for form "NFC").  Lists, pandas Series and other
    iterables become lists with every string normalised (None and non-strings kept as they are,
    rows_to_blob converts them)."""
    import unicodedata

    import pyarrow as pa

    def nfc(rs):
        return [r if r is None or not isinstance(r, str) or unicodedata.is_normalized("NFC", r)
                else unicodedata.normalize("NFC", r) for r in rs]
    if isinstance(rows, (pa.Array, pa.ChunkedArray)):
        data, _ = rows_to_blob(rows)
        if not (data >= 0x80).any():
            return rows
        return pa.array(nfc(rows.cast(pa.large_string()).to_pylist()), type=pa.large_string())
    return nfc(rows)


def normalize_rows(rows, vocab: Optional[VB.Vocab]):
    """The rows as the vocabulary's tokenizer file wants them before pre-tokenisation: NFC when
    it declares an NFC normalizer (Vocab.normalize_nfc, real Qwen files), unchanged otherwise.
    Every entry point that tokenises host rows calls this, whatever the input form."""
    if vocab is None or not vocab.normalize_nfc:
        return rows
    return _nfc_rows(rows)


def _all_str(rows) -> bool:
    return isinstance(rows, list) and all(isinstance(r, str) for r in rows)


def blob_to_rows(data: np.ndarray, off: np.ndarray) -> List[str]:
    """Decode with errors='replace': an unconstrained model may emit bytes that are not
    UTF-8 (same policy as HF byte-level decoders)."""
    raw = data.tobytes()
    return [raw[off[i]:off[i + 1]].decode("utf-8", errors="replace") for i in range(len(off) - 1)]


# --------------------------------------------------------------------------- tokenizer
class GpuTokenizer:
    """Byte-level BPE on the GPU (csrc/tokenizer.cu)."""

    def __init__(self, v: VB.Vocab, device: torch.device):
        self.v, self.device = v, device
        blob, off = v.byte_blob()
        self._blob, self._off = blob, off
        merges = np.ascontiguousarray(v.merge_array())
        cls = np.ascontiguousarray(class_table())
        # real tokenizer files give every merge its own result id; synthetic ones use 256 + rank
        mids = None if v.merged_ids is None else np.ascontiguousarray(v.merged_ids, dtype=np.int32)
        h = C.c_void_p()
        with torch.cuda.device(device):
            L.check(L.lib().sb200_tokenizer_create(
                merges.ctypes.data, len(v.merges), None if mids is None else mids.ctypes.data,
                cls.ctypes.data, v.digits,
                blob.ctypes.data, off.ctypes.data, v.vocab_size, C.byref(h)))
        self._h = h
        if v.word_overrides:      # the tokenizer file sets ignore_merges (vocab.Vocab)
            toks, off, ids = word_override_arrays(v)
            L.check(L.lib().sb200_tokenizer_set_word_overrides(
                h, toks.ctypes.data, off.ctypes.data, ids.ctypes.data, len(ids)))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                L.lib().sb200_tokenizer_destroy(self._h)
        except Exception:  # interpreter shutdown
            pass

    def encode_blob_dev(self, data: np.ndarray, off: np.ndarray):
        """-> (tokens[int32, device], row_tok_off[int64, device]); includes the H2D copy."""
        dev = self.device
        n_bytes, n_rows = int(off[-1]), len(off) - 1
        d_text = torch.from_numpy(np.ascontiguousarray(data)).to(dev, non_blocking=False) \
            if n_bytes else torch.zeros(1, dtype=torch.uint8, device=dev)
        d_off = torch.from_numpy(np.ascontiguousarray(off)).to(dev)
        d_tok = torch.empty(max(n_bytes, 1), dtype=torch.int32, device=dev)
        d_toff = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            L.check(L.lib().sb200_tokenizer_encode(self._h, d_text.data_ptr(), n_bytes,
                                                   d_off.data_ptr(), n_rows, d_tok.data_ptr(),
                                                   d_toff.data_ptr(), L.current_stream()))
        return d_tok, d_toff

    def encode(self, texts: Sequence[str]) -> List[List[int]]:
        data, off = rows_to_blob(list(texts))
        d_tok, d_toff = self.encode_blob_dev(data, off)
        toff = d_toff.cpu().numpy()
        tok = d_tok[:int(toff[-1])].cpu().numpy()
        return [tok[toff[i]:toff[i + 1]].tolist() for i in range(len(texts))]

    def encode_pieces(self, pieces: Sequence[str]) -> List[int]:
        """Template pieces: special-token names map to their ids, text is tokenised."""
        text_idx = [i for i, p in enumerate(pieces) if p not in self.v.specials]
        enc = self.encode([pieces[i] for i in text_idx]) if text_idx else []
        out: List[int] = []
        it = iter(enc)
        for p in pieces:
            out += [self.v.specials[p]] if p in self.v.specials else next(it)
        return out

    def decode_dev(self, d_tok: torch.Tensor, d_toff: torch.Tensor) -> Tuple[np.ndarray, np.ndarray]:
        """compact tokens + row offsets (device) -> (uint8 blob, int64 offsets) on the host."""
        dev = self.device
        n_tok, n_rows = int(d_tok.numel()), int(d_toff.numel()) - 1
        d_boff = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
        lib = L.lib()
        with torch.cuda.device(dev):
            L.check(lib.sb200_tokenizer_decode(self._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(),
                                               n_rows, None, d_boff.data_ptr(), L.current_stream()))
            total = int(d_boff[-1].item())
            d_bytes = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
            L.check(lib.sb200_tokenizer_decode(self._h, d_tok.data_ptr(), n_tok, d_toff.data_ptr(),
                                               n_rows, d_bytes.data_ptr(), d_boff.data_ptr(),
                                               L.current_stream()))
        return d_bytes[:total].cpu().numpy(), d_boff.cpu().numpy()


# --------------------------------------------------------------------------- engine
@dataclass
class GenerationResult:
    outputs: Optional[List[str]]
    out_tokens: Optional[List[List[int]]]
    embeddings: Optional[np.ndarray]
    stats: Dict[str, Any] = field(default_factory=dict)
    first_logits: Optional[Any] = None   # torch fp32 [n_rows, vocab] (debug/parity only)
    cum_logprobs: Optional[np.ndarray] = None  # fp32 [n_rows] when return_logprobs=True


@dataclass(frozen=True)
class JobOptions:
    """What a job asks for: prompt framing, output schema, output budget and sampling.
    `generate`, `run_blob_dev` and `infer_one_call` take these fields as keywords; the defaults
    here are theirs."""
    system_prompt: Optional[str] = None
    json_schema: Optional[Dict[str, Any]] = None
    max_new_tokens: int = 64
    ignore_eos: bool = False
    truncate_rows: bool = True
    share_prefix: bool = True
    fsm_limits: Optional[FsmLimits] = None
    jump_forward: bool = True
    temperature: float = 0.0
    top_k: int = 0
    top_p: float = 1.0
    seed: int = 0
    seed_per_row: bool = False
    thinking_chars: Optional[int] = None
    presence_penalty: float = 0.0
    frequency_penalty: float = 0.0
    repetition_penalty: float = 1.0
    min_p: float = 0.0


def default_max_prefill_tokens(spec: MS.ModelSpec) -> int:
    """The default step holds one row that fills a window of up to 32,768 tokens, and at least
    8,192 tokens.  Rows of longer windows are prefilled in chunks, so activation memory stays
    that of a 32,768-token step."""
    return max(8192, min(spec.max_position, 32768))


class LocalEngine:
    def __init__(self, spec: MS.ModelSpec, weights: MS.EngineWeights, vocab: VB.Vocab,
                 device: int | str | torch.device = 0, max_slots: int = 512,
                 max_prefill_tokens: Optional[int] = None, kv_pages: Optional[int] = None,
                 kv_fraction: float = 0.8, logit_chunk_rows: int = 1024,
                 min_admit_rows: Optional[int] = None):
        if not torch.cuda.is_available():
            raise L.Sb200Error("sutro_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.spec, self.weights, self.vocab = spec, weights, vocab
        if vocab.vocab_size != spec.vocab_size:
            raise ValueError("vocabulary size does not match the model")
        if max_prefill_tokens is None:
            max_prefill_tokens = default_max_prefill_tokens(spec)
        self.max_slots, self.max_prefill_tokens = max_slots, max_prefill_tokens
        with torch.cuda.device(self.device):
            self.cos, self.sin = (t.to(self.device).contiguous() for t in MS.rope_tables(spec))
            page_bytes = spec.kv_bytes_per_token * 16
            if kv_pages is None:
                free, _ = torch.cuda.mem_get_info(self.device)
                act = max(max_prefill_tokens, max_slots) * 2 * (
                    2 * spec.d_model + spec.qkv_dim + spec.q_dim + spec.d_ff)
                act += min(logit_chunk_rows, max_slots) * spec.vocab_size * 4
                kv_pages = int(max(0, (free - act) * kv_fraction) // page_bytes)
                # never more than every slot at full context
                kv_pages = min(kv_pages, max_slots * (spec.max_position // 16 + 1) + 64)
            if kv_pages < 8:
                raise L.Sb200Error("not enough device memory for a KV pool")
            self.kv_pages = kv_pages
            cfg = EngineConfigC(spec.n_layers, spec.d_model, spec.n_q_heads, spec.n_kv_heads,
                                spec.d_ff, spec.vocab_size, spec.max_position, spec.rms_eps,
                                int(spec.qk_norm), int(spec.embedding_model), vocab.eos_id,
                                max_slots, max_prefill_tokens, logit_chunk_rows,
                                min_admit_rows if min_admit_rows is not None
                                else max(1, max_slots // 4), kv_pages)
            self._keep: List[Any] = []

            def arr(ts):
                a = (C.c_void_p * spec.n_layers)(*[L.ptr(t) for t in ts])
                self._keep.append(a)
                return C.cast(a, c_vpp)

            w = weights
            wc = EngineWeightsC(L.ptr(w.embed), L.ptr(w.lm_head), L.ptr(w.final_norm),
                                L.ptr(self.cos), L.ptr(self.sin), arr(w.ln1), arr(w.ln2),
                                arr(w.wqkv), arr(w.wo), arr(w.wgu), arr(w.wd),
                                arr(w.q_norm) if spec.qk_norm else None,
                                arr(w.k_norm) if spec.qk_norm else None)
            torch.cuda.synchronize(self.device)
            h = C.c_void_p()
            L.check(L.lib().sb200_engine_create(C.byref(cfg), C.byref(wc), C.byref(h)))
            self._h = h
            self.tokenizer = GpuTokenizer(vocab, self.device)
            L.check(L.lib().sb200_engine_set_vocab(self._h, self.tokenizer._blob.ctypes.data,
                                                   self.tokenizer._off.ctypes.data))
        self._fsm_cache: Dict[str, ByteDFA] = {}
        self._jump_cache: Dict[Any, Any] = {}
        self._tpl_cache: Dict[Any, Tuple[np.ndarray, np.ndarray]] = {}

    # ---- construction helpers -------------------------------------------
    @classmethod
    def from_seed(cls, model: str, seed: int = 0, device=0, vocab_seed: int = 0,
                  max_position: Optional[int] = None, **kw):
        """Random-init replica of a named architecture (no checkpoints exist offline), serving
        a `max_position`-token window (None: the registered one; see `modelspec.with_window`)."""
        spec = MS.with_window(MS.get_spec(model), max_position)
        dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if spec.n_params() > 50_000_000:
            weights = MS.make_engine_weights_on_device(spec, seed, dev)
        else:
            weights = MS.pack_for_engine(spec, MS.make_weights(spec, seed), dev)
        v = VB.build_vocab(spec.family, spec.vocab_size, seed=vocab_seed)
        return cls(spec, weights, v, device=dev, **kw)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                L.lib().sb200_engine_destroy(self._h)
        except Exception:
            pass

    def close(self):
        if getattr(self, "_h", None):
            L.lib().sb200_engine_destroy(self._h)
            self._h = None

    # ---- the hot path -----------------------------------------------------
    def _template_tokens(self, system_prompt: Optional[str], thinking: bool = False):
        key = (system_prompt, self.spec.embedding_model, bool(thinking))
        if key not in self._tpl_cache:
            tpl = (VB.embedding_template(self.spec.family) if self.spec.embedding_model
                   else VB.chat_template(self.spec.family, system_prompt,
                                         getattr(self, "empty_think_block", False)
                                         and not thinking))
            suffix = list(tpl.suffix)
            if thinking and not self.spec.embedding_model:
                suffix += ["<think>", "\n"]     # a thinking turn opens its reasoning block
            pre = np.asarray(self.tokenizer.encode_pieces(tpl.prefix), dtype=np.int32)
            suf = np.asarray(self.tokenizer.encode_pieces(suffix), dtype=np.int32)
            self._tpl_cache[key] = (pre, suf)
        return self._tpl_cache[key]

    def _jump_plan(self, dfa: ByteDFA, key) -> Optional[Dict[str, Any]]:
        """Jump-forward plan for a compiled schema (cached): canonical tokenisation of the
        forced output prefix and of every forced terminal tail (GPU tokenizer)."""
        if key in self._jump_cache:
            return self._jump_cache[key]
        plan = None
        prefix, start_after, tails = dfa.forced_plan()
        fully_forced = bool(dfa.final[start_after]) or start_after in tails
        try:
            texts = [prefix.decode("utf-8")] + [t.decode("utf-8") for t in tails.values()]
        except UnicodeDecodeError:
            texts = None
        if texts is not None and not fully_forced and (prefix or tails):
            enc = self.tokenizer.encode(texts)
            off = np.zeros(dfa.n_states + 1, dtype=np.int32)
            toks: List[int] = []
            by_state = dict(zip(tails.keys(), enc[1:]))
            for st in range(dfa.n_states):
                toks += by_state.get(st, [])
                off[st + 1] = len(toks)
            plan = {"prefix_tokens": np.asarray(enc[0], dtype=np.int32), "start": int(start_after),
                    "tail_off": off, "tail_tok": np.asarray(toks or [0], dtype=np.int32)}
        self._jump_cache[key] = plan
        return plan

    def compile_schema(self, schema: Optional[Dict[str, Any]], limits: Optional[FsmLimits] = None,
                       thinking_chars: Optional[int] = None) -> ByteDFA:
        """output_schema -> byte automaton (cached).  `thinking_chars`: the automaton of a
        thinking model's turn instead — free reasoning of at most that many characters, the
        closing `</think>` line, then the schema instance (or free text when schema is None)."""
        import json
        key = json.dumps(schema, sort_keys=True) + repr(limits) + repr(thinking_chars)
        if key not in self._fsm_cache:
            self._fsm_cache[key] = (compile_schema(schema, limits) if thinking_chars is None
                                    else compile_thinking(schema, limits, thinking_chars))
        return self._fsm_cache[key]

    def _job_options(self, job: "JobC", opts: JobOptions):
        """Fill the host-side fields of an sb200_job (prompt framing, schema automaton, jump-forward
        plan, sampling).  Returns (dfa, plan, keep) — `keep` holds the arrays the job points at."""
        emb_mode = self.spec.embedding_model
        thinking = opts.thinking_chars is not None and not emb_mode
        pre, suf = self._template_tokens(opts.system_prompt, thinking)
        dfa = None
        if thinking:
            dfa = self.compile_schema(opts.json_schema, opts.fsm_limits, int(opts.thinking_chars))
        elif opts.json_schema is not None:
            dfa = self.compile_schema(opts.json_schema, opts.fsm_limits)
        plan = None
        if dfa is not None and opts.jump_forward and not emb_mode:
            # jump-forward decoding: bytes the automaton forces are not the model's choice —
            # the forced output prefix rides with the prompt, forced terminal tails are
            # appended by the sampler without another forward pass
            plan = self._jump_plan(dfa, (id(dfa),))
            if plan is not None and len(plan["prefix_tokens"]) >= opts.max_new_tokens:
                plan = None
        if plan is not None:
            suf = np.concatenate([suf, plan["prefix_tokens"]]).astype(np.int32)
        job.prefix_tokens, job.n_prefix = _np_ptr(pre, c_i32p), len(pre)
        job.suffix_tokens, job.n_suffix = _np_ptr(suf, c_i32p), len(suf)
        job.share_prefix, job.max_new_tokens = int(opts.share_prefix), opts.max_new_tokens
        job.ignore_eos, job.truncate_rows = int(opts.ignore_eos), int(opts.truncate_rows)
        if dfa is not None:
            job.fsm_trans = _np_ptr(dfa.trans, c_i32p)
            job.fsm_accept = _np_ptr(dfa.accept, c_u8p)
            job.fsm_final = _np_ptr(dfa.final, c_u8p)
            job.fsm_states, job.fsm_start = dfa.n_states, dfa.start
            if plan is not None:
                job.fsm_start = plan["start"]
                job.n_forced_prefix = len(plan["prefix_tokens"])
                job.fsm_tail_off = _np_ptr(plan["tail_off"], c_i32p)
                job.fsm_tail_tok = _np_ptr(plan["tail_tok"], c_i32p)
        job.temperature, job.top_k = float(opts.temperature), int(opts.top_k)
        job.top_p = float(opts.top_p)
        job.seed, job.seed_per_row = int(opts.seed) & (2 ** 64 - 1), int(opts.seed_per_row)
        job.presence_penalty, job.frequency_penalty, job.repetition_penalty, job.min_p = \
            check_penalties(opts.presence_penalty, opts.frequency_penalty,
                            opts.repetition_penalty, opts.min_p)
        return dfa, plan, (pre, suf)

    def run_blob_dev(self, d_text: torch.Tensor, d_off: torch.Tensor, n_rows: int, n_bytes: int,
                     *, progress: Optional[Callable[[int, int, int], None]] = None,
                     return_text: bool = True, profile: bool = False,
                     return_first_logits: bool = False, return_logprobs: bool = False,
                     row_ids: Optional[Sequence[int]] = None, **options) -> Dict[str, Any]:
        """Phase B of the hot path, HBM to HBM: a device-resident Arrow column (uint8 bytes +
        int64 offsets[n_rows+1]) -> tokenise -> prefill/decode (+mask) -> detokenise ->
        device-resident results (`d_bytes`/`d_boff`, `flat`/`ooff` tokens, `d_emb`, ...).
        Used by generate() and by the row-sharded multi-GPU path (sharding.py), which moves
        these buffers between ranks over NCCL.  `options`: the fields of JobOptions."""
        return self._run_blob_dev(d_text, d_off, n_rows, n_bytes, JobOptions(**options),
                                  progress=progress, return_text=return_text, profile=profile,
                                  return_first_logits=return_first_logits,
                                  return_logprobs=return_logprobs, row_ids=row_ids)

    def _run_blob_dev(self, d_text, d_off, n_rows, n_bytes, opts: JobOptions, *, progress,
                      return_text, profile, return_first_logits, return_logprobs, row_ids):
        max_new_tokens = opts.max_new_tokens
        dev = self.device
        emb_mode = self.spec.embedding_model
        lib = L.lib()
        with torch.cuda.device(dev):
            d_tok = torch.empty(max(n_bytes, 1), dtype=torch.int32, device=dev)
            d_toff = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
            L.check(lib.sb200_tokenizer_encode(self.tokenizer._h, d_text.data_ptr(), n_bytes,
                                               d_off.data_ptr(), n_rows, d_tok.data_ptr(),
                                               d_toff.data_ptr(), L.current_stream()))
            toff = d_toff.cpu().numpy()          # the scheduler needs row lengths on the host
            d_out = d_len = d_emb = None
            if emb_mode:
                d_emb = torch.empty(n_rows, self.spec.d_model, dtype=torch.float32, device=dev)
            else:
                d_out = torch.empty(n_rows, max_new_tokens, dtype=torch.int32, device=dev)
                d_len = torch.zeros(n_rows, dtype=torch.int32, device=dev)
            cb = PROGRESS_FN(lambda r, i, o, u: progress(r, i, o)) if progress else PROGRESS_FN()
            job = JobC()
            dfa, plan, keep = self._job_options(job, opts)
            job.row_tokens_dev, job.row_tok_off_dev = d_tok.data_ptr(), d_toff.data_ptr()
            job.row_tok_off, job.n_rows = _np_ptr(toff, c_i64p), n_rows
            job.out_tokens_dev = L.ptr(d_out)
            job.out_len_dev = L.ptr(d_len)
            job.out_embed_dev = L.ptr(d_emb)
            job.progress = cb
            job.profile = int(profile)
            d_first = None
            if return_first_logits and not emb_mode:
                d_first = torch.zeros(n_rows, self.spec.vocab_size, dtype=torch.float32, device=dev)
                job.out_first_logits_dev = d_first.data_ptr()
            d_ids = None
            if row_ids is not None and opts.seed_per_row:
                # rows of a sharded job keep the Philox stream of their index in the whole job
                ids = np.ascontiguousarray(row_ids, dtype=np.int64)
                if ids.shape != (n_rows,):
                    raise ValueError("row_ids must hold one id per row")
                d_ids = torch.from_numpy(ids).to(dev)
                job.row_ids_dev = d_ids.data_ptr()
            d_lp = None
            if return_logprobs and not emb_mode:
                d_lp = torch.zeros(n_rows, dtype=torch.float32, device=dev)
                job.out_cum_logprob_dev = d_lp.data_ptr()
            st = JobStatsC()
            torch.cuda.synchronize(dev)
            t_tok = time.perf_counter()
            L.check(lib.sb200_engine_run(self._h, C.byref(job), C.byref(st)))
            t_run = time.perf_counter()
            n_out = 0
            d_bytes = d_boff = flat = ooff = None
            if not emb_mode:
                # compaction of the [n_rows, max_new] token matrix: native kernels, no tensor ops
                ooff = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
                flat = torch.empty(max(n_rows * max_new_tokens, 1), dtype=torch.int32, device=dev)
                L.check(lib.sb200_compact_rows(d_out.data_ptr(), d_len.data_ptr(), n_rows,
                                               max_new_tokens, ooff.data_ptr(), flat.data_ptr(),
                                               L.current_stream()))
                n_out = int(ooff[-1].item())
                flat = flat[:n_out]
                if return_text:
                    d_boff = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
                    L.check(lib.sb200_tokenizer_decode(self.tokenizer._h, flat.data_ptr(), n_out,
                                                       ooff.data_ptr(), n_rows, None,
                                                       d_boff.data_ptr(), L.current_stream()))
                    total = int(d_boff[-1].item())
                    d_bytes = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
                    L.check(lib.sb200_tokenizer_decode(self.tokenizer._h, flat.data_ptr(), n_out,
                                                       ooff.data_ptr(), n_rows,
                                                       d_bytes.data_ptr(), d_boff.data_ptr(),
                                                       L.current_stream()))
                    d_bytes = d_bytes[:total]
            torch.cuda.synchronize(dev)
        stats = st.counters()
        # my kernels outside the engine: tokenizer encode (4), compaction (widen + scan + compact)
        # and decode (2 passes: 2 + 3)
        stats["tokenizer_launches"] = 4 + (0 if emb_mode else 3) + \
            (5 if (return_text and not emb_mode) else 0)
        stats.update(output_tokens=n_out, n_rows=n_rows, t_engine_s=t_run - t_tok,
                     fsm_states=0 if dfa is None else dfa.n_states, jump_forward=plan is not None,
                     forced_prefix_tokens=0 if plan is None else int(len(plan["prefix_tokens"])))
        return dict(d_bytes=d_bytes, d_boff=d_boff, flat=flat, ooff=ooff, d_emb=d_emb,
                    d_first=d_first, d_lp=d_lp, stats=stats, t_tok=t_tok, t_run=t_run)

    def rows_select(self, d_bytes: torch.Tensor, d_off: torch.Tensor, part_rows: int,
                    part_bytes: int, d_idx: torch.Tensor, capacity: int):
        """Device-side Arrow row selection (sb200_rows_select): rows `d_idx` of the resident
        column (or batch of equally strided columns) -> (offsets[m+1], bytes[capacity])."""
        m = int(d_idx.numel())
        dev = self.device
        with torch.cuda.device(dev):
            out_off = torch.empty(m + 1, dtype=torch.int64, device=dev)
            out_bytes = torch.empty(max(int(capacity), 1), dtype=torch.uint8, device=dev)
            L.check(L.lib().sb200_rows_select(d_bytes.data_ptr(), d_off.data_ptr(), int(part_rows),
                                              int(part_bytes), d_idx.data_ptr(), m,
                                              out_off.data_ptr(), out_bytes.data_ptr(),
                                              L.current_stream()))
        return out_off, out_bytes

    def generate(self, rows, *, progress: Optional[Callable[[int, int, int], None]] = None,
                 return_tokens: bool = False, return_text: bool = True, profile: bool = False,
                 return_first_logits: bool = False, return_logprobs: bool = False,
                 row_ids: Optional[Sequence[int]] = None, **options) -> GenerationResult:
        """The whole hot path for one frame column.  Three phases, timed separately:
          A  host -> HBM   : rows -> Arrow blob, template/schema compile (cached), H2D copy
          B  device        : tokenize, prefill/decode (+mask), detokenize — HBM to HBM
          C  HBM -> host   : D2H of bytes/offsets, Python strings
        stats["t_device_s"] is phase B alone (inputs resident in HBM), stats["t_total_s"]
        is A+B+C.  `options`: the fields of JobOptions."""
        opts = JobOptions(**options)
        dev = self.device
        emb_mode = self.spec.embedding_model
        t0 = time.perf_counter()
        # ---- phase A -------------------------------------------------------------
        rows = normalize_rows(rows, self.vocab)
        data, off = rows_to_blob(rows)
        n_rows, n_bytes = len(off) - 1, int(off[-1])
        if n_rows == 0:
            return GenerationResult([] if not emb_mode else None, [] if return_tokens else None,
                                    np.zeros((0, self.spec.d_model), np.float32) if emb_mode
                                    else None, {"n_rows": 0, "input_tokens": 0,
                                                "output_tokens": 0, "rows_done": 0})
        # template / schema compilation (cached) belongs to the host phase
        self._template_tokens(opts.system_prompt, opts.thinking_chars is not None)
        if opts.json_schema is not None or opts.thinking_chars is not None:
            self.compile_schema(opts.json_schema, opts.fsm_limits, opts.thinking_chars)
        with torch.cuda.device(dev):
            d_text = (torch.from_numpy(np.ascontiguousarray(data)).to(dev) if n_bytes
                      else torch.zeros(1, dtype=torch.uint8, device=dev))
            d_off = torch.from_numpy(np.ascontiguousarray(off)).to(dev)
            torch.cuda.synchronize(dev)
            t_a = time.perf_counter()
            # ---- phase B ---------------------------------------------------------
            r = self._run_blob_dev(d_text, d_off, n_rows, n_bytes, opts, progress=progress,
                                   return_text=return_text, profile=profile,
                                   return_first_logits=return_first_logits,
                                   return_logprobs=return_logprobs, row_ids=row_ids)
            t_b = time.perf_counter()
            # ---- phase C ---------------------------------------------------------
            outputs = out_tokens = emb = None
            d2h = 0
            if emb_mode:
                emb = r["d_emb"].cpu().numpy()
                d2h = emb.nbytes
            else:
                if return_text:
                    b, boff = r["d_bytes"].cpu().numpy(), r["d_boff"].cpu().numpy()
                    d2h += b.nbytes + boff.nbytes
                    outputs = blob_to_rows(b, boff)
                if return_tokens:
                    fl, oo = r["flat"].cpu().numpy(), r["ooff"].cpu().numpy()
                    d2h += fl.nbytes + oo.nbytes
                    out_tokens = [fl[oo[i]:oo[i + 1]].tolist() for i in range(n_rows)]
            t_end = time.perf_counter()
        stats = r["stats"]
        stats.update(h2d_bytes=int(data.nbytes + off.nbytes), d2h_bytes=int(d2h),
                     t_h2d_s=t_a - t0, t_tokenize_s=r["t_tok"] - t_a,
                     t_detok_s=t_b - r["t_run"], t_device_s=t_b - t_a, t_d2h_s=t_end - t_b,
                     t_total_s=t_end - t0)
        return GenerationResult(outputs, out_tokens, emb, stats,
                                None if r["d_first"] is None else r["d_first"].cpu(),
                                None if r["d_lp"] is None else r["d_lp"].cpu().numpy())

    def infer_one_call(self, rows, *, return_logprobs: bool = False, return_tokens: bool = True,
                       progress: Optional[Callable[[int, int, int], None]] = None,
                       profile: bool = False, **options) -> GenerationResult:
        """The same job through `sb200_infer_text`: ONE C-ABI call with host buffers in and out
        (what a non-Python host would bind; the SDK's infer() and bench.py's `e2e` use it).
        `generate` is the phased form of the same work; the results are identical.  The call times
        its three phases with CUDA events on the engine's stream: stats["t_h2d_ms"] (rows -> HBM),
        stats["t_device_ms"] (tokenise -> prefill/decode -> detokenise, HBM to HBM) and
        stats["t_d2h_ms"].  `options`: the fields of JobOptions."""
        opts = JobOptions(**options)
        rows = normalize_rows(rows, self.vocab)
        t0 = time.perf_counter()
        data, off = rows_to_blob(rows)
        n_rows = len(off) - 1
        emb_mode = self.spec.embedding_model
        data, off = np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64)
        job = JobC()
        dfa, plan, keep = self._job_options(job, opts)
        cb = PROGRESS_FN(lambda r, i, o, u: progress(r, i, o)) if progress else PROGRESS_FN()
        job.progress = cb
        job.profile = int(profile)
        st, res = JobStatsC(), C.POINTER(ResultC)()
        t1 = time.perf_counter()
        L.check(L.lib().sb200_infer_text(self._h, self.tokenizer._h, data.ctypes.data,
                                         off.ctypes.data, n_rows, C.byref(job), 1,
                                         int(return_logprobs), C.byref(res), C.byref(st)))
        t2 = time.perf_counter()
        n_out = d2h = 0
        try:
            r = res.contents
            outputs = out_tokens = emb = lp = None
            if emb_mode:
                emb = np.ctypeslib.as_array(r.embeddings, shape=(n_rows, r.d_model)).copy() \
                    if n_rows else np.zeros((0, self.spec.d_model), np.float32)
                d2h = emb.nbytes
            else:
                toff = np.ctypeslib.as_array(r.token_offsets, shape=(n_rows + 1,)).copy()
                n_out = int(toff[-1])
                if return_tokens:
                    toks = (np.ctypeslib.as_array(r.tokens, shape=(n_out,)).copy()
                            if n_out else np.zeros(0, np.int32))
                    out_tokens = [toks[toff[i]:toff[i + 1]].tolist() for i in range(n_rows)]
                boff = np.ctypeslib.as_array(r.offsets, shape=(n_rows + 1,)).copy()
                blob = (np.ctypeslib.as_array(r.bytes, shape=(int(boff[-1]),)).copy()
                        if boff[-1] else np.zeros(0, np.uint8))
                outputs = blob_to_rows(blob, boff)
                d2h = int(blob.nbytes + boff.nbytes + toff.nbytes + 4 * n_out)
                if return_logprobs and n_rows:
                    lp = np.ctypeslib.as_array(r.cum_logprob, shape=(n_rows,)).copy()
        finally:
            L.lib().sb200_result_free(res)
        stats = st.counters()
        stats["tokenizer_launches"] = 4 + (0 if emb_mode else 3 + 5)
        stats.update(n_rows=n_rows, output_tokens=n_out, t_total_s=time.perf_counter() - t0,
                     t_call_s=t2 - t1, t_h2d_ms=st.t_h2d_ms, t_device_ms=st.t_device_ms,
                     t_d2h_ms=st.t_d2h_ms, t_device_s=st.t_device_ms * 1e-3,
                     h2d_bytes=int(data.nbytes + off.nbytes), d2h_bytes=int(d2h),
                     fsm_states=0 if dfa is None else dfa.n_states, jump_forward=plan is not None,
                     forced_prefix_tokens=0 if plan is None else int(len(plan["prefix_tokens"])))
        return GenerationResult(outputs, out_tokens, emb, stats, None, lp)


# --------------------------------------------------------------------------- several GPUs, one process
class MultiGpuEngine:
    """Row-sharded replicas inside one process: one LocalEngine per device, each driven from
    its own host thread (the C-ABI calls release the GIL).  Rows are split into contiguous
    blocks, results are concatenated in order — the path has no exchange step, so there is no
    data-path collective.  Weights are drawn once on the first device and broadcast to the
    others (`torch.cuda.comm.broadcast`: NCCL over NVLink when available)."""

    def __init__(self, engines: List[LocalEngine]):
        if not engines:
            raise ValueError("MultiGpuEngine needs at least one engine")
        self.engines = engines
        self.spec, self.vocab = engines[0].spec, engines[0].vocab
        self.tokenizer = engines[0].tokenizer

    @classmethod
    def from_seed(cls, model: str, devices: Sequence[int], seed: int = 0, vocab_seed: int = 0,
                  max_position: Optional[int] = None, **kw):
        spec = MS.with_window(MS.get_spec(model), max_position)
        devs = [torch.device("cuda", d) for d in devices]
        if spec.n_params() > 50_000_000:
            w0 = MS.make_engine_weights_on_device(spec, seed, devs[0])
        else:
            w0 = MS.pack_for_engine(spec, MS.make_weights(spec, seed), devs[0])
        v = VB.build_vocab(spec.family, spec.vocab_size, seed=vocab_seed)
        replicas = [w0] + [cls._replicate(spec, w0, d) for d in devs[1:]]
        return cls([LocalEngine(spec, w, v, device=d, **kw) for w, d in zip(replicas, devs)])

    @staticmethod
    def _replicate(spec, w0: MS.EngineWeights, dev) -> MS.EngineWeights:
        import torch.cuda.comm as comm

        def cp(t):
            return None if t is None else comm.broadcast(t, [t.device.index, dev.index])[1]
        embed = cp(w0.embed)
        lm = embed if spec.tied_embeddings else cp(w0.lm_head)
        out = MS.EngineWeights(embed=embed, lm_head=lm, final_norm=cp(w0.final_norm))
        for name in ("ln1", "ln2", "wqkv", "wo", "wgu", "wd", "q_norm", "k_norm"):
            setattr(out, name, [cp(t) for t in getattr(w0, name)])
        return out

    def close(self):
        for e in self.engines:
            e.close()

    def generate(self, rows, balance: str = "bytes", **kw) -> GenerationResult:
        """Same arguments as `LocalEngine.generate`.  `balance="bytes"` deals rows to the GPUs
        longest-first (`sharding.balanced_shards`, byte length as the proxy for tokens);
        `"rows"` uses contiguous blocks.  Either way row i of the result belongs to row i of
        the input, and per-row random streams are keyed by the row's index in the whole job,
        so the outputs do not depend on how many GPUs shared the work."""
        from concurrent.futures import ThreadPoolExecutor

        from .sharding import balanced_shards, shard_bounds
        progress = kw.pop("progress", None)
        if not isinstance(rows, list):
            rows = rows.to_pylist() if hasattr(rows, "to_pylist") else list(rows)
        n, g = len(rows), len(self.engines)
        if balance == "rows":
            shards = [list(range(*shard_bounds(n, g, r))) for r in range(g)]
        elif balance == "bytes":
            shards = balanced_shards([0 if r is None else len(str(r).encode("utf-8"))
                                      for r in rows], g)
        else:
            raise ValueError("balance must be 'rows' or 'bytes'")
        work = [(e, idx) for e, idx in zip(self.engines, shards) if idx]
        if not work:
            return self.engines[0].generate(rows, progress=progress, **kw)

        def shard_progress(k):
            # every shard reports its own running totals; the caller sees their sum
            if progress is None:
                return None

            def cb(rows_done, in_tok, out_tok):
                with lock:
                    seen[k] = (rows_done, in_tok, out_tok)
                    progress(*(sum(s[j] for s in seen) for j in range(3)))
            return cb
        import threading
        lock, seen = threading.Lock(), [(0, 0, 0)] * len(work)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=len(work)) as pool:
            parts = list(pool.map(
                lambda a: a[1][0].generate([rows[i] for i in a[1][1]], row_ids=a[1][1],
                                           progress=shard_progress(a[0]), **kw),
                list(enumerate(work))))
        return self._merge(parts, [idx for _, idx in work], n, time.perf_counter() - t0)

    @staticmethod
    def _merge(parts: List[GenerationResult], shards: List[List[int]], n_rows: int,
               wall_s: float) -> GenerationResult:
        def scatter(name):
            vals = [getattr(p, name) for p in parts]
            if any(v is None for v in vals):
                return None
            if isinstance(vals[0], np.ndarray):
                out = np.empty((n_rows,) + vals[0].shape[1:], dtype=vals[0].dtype)
                for idx, v in zip(shards, vals):
                    out[idx] = v
                return out
            if torch.is_tensor(vals[0]):
                out = torch.empty((n_rows,) + tuple(vals[0].shape[1:]), dtype=vals[0].dtype)
                for idx, v in zip(shards, vals):
                    out[torch.as_tensor(idx, dtype=torch.long)] = v
                return out
            out = [None] * n_rows
            for idx, v in zip(shards, vals):
                for i, x in zip(idx, v):
                    out[i] = x
            return out
        stats: Dict[str, Any] = {"n_gpus": len(parts), "t_total_s": wall_s,
                                 "per_gpu": [p.stats for p in parts]}
        for k in ("n_rows", "input_tokens", "output_tokens", "decode_tokens", "prefill_tokens",
                  "rows_done", "rows_truncated", "h2d_bytes", "d2h_bytes"):
            stats[k] = sum(int(p.stats.get(k, 0)) for p in parts)
        return GenerationResult(scatter("outputs"), scatter("out_tokens"), scatter("embeddings"),
                                stats, scatter("first_logits"), scatter("cum_logprobs"))
