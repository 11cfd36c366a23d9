// sutro_b200 — K7: batched byte-level BPE tokenizer / detokenizer on the GPU.
//
// Input is Arrow-style: one UTF-8 byte blob + int64 row offsets.  Three passes,
// all indexed by byte position so no per-row host work exists:
//   1. pretok_kernel   one thread per row runs the GPT-4-style pre-tokenisation
//      pattern (ordered alternation, restated as a hand-written scanner over
//      Unicode classes from a 1.1 MB code-point table that lives in L2) and
//      flags the first byte of every pre-token.
//   2. bpe_kernel      one thread per flagged byte: seeds one symbol per byte,
//      then repeatedly merges the lowest-rank adjacent pair (leftmost on ties)
//      using an open-addressing hash of (left,right)->(rank,id) (8 MB, L2
//      resident), in place in a scratch array; records the token count.
//      Optional whole-word overrides (`ignore_merges` of Llama-3 tokenizer files: a pre-token
//      that is itself a vocabulary entry is emitted as that token even when its merges would
//      build something else): the host lists, for every such entry, the sequence its merges DO
//      build; a pre-token whose merge result equals one of those sequences is replaced by the
//      entry's id (two byte strings never merge to the same tokens, so the match is exact).
//   3. exclusive scan (CUB, 64-bit counts) of the counts + compaction into the output.
// HBM traffic: text bytes in, 4 B per token out, plus scratch at 21 B per byte (flag, symbol,
// count, output position).
#include <cub/device/device_scan.cuh>

#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace sb {

namespace {

enum : uint8_t { CLS_OTHER = 0, CLS_LETTER = 1, CLS_NUMBER = 2, CLS_SPACE = 3 };

struct TokTables {
  const uint8_t* cls;        // [0x110000]
  const uint64_t* hkeys;     // [cap]
  const uint64_t* hvals;     // [cap]  rank<<32 | id
  uint32_t hmask;
  const int32_t* byte_to_id; // [256]
  int digits;
  // whole-word overrides (fmask == 0: none): open-addressing table keyed by seq_hash
  const uint64_t* fkeys;     // [fmask + 1]
  const int4* fslots;        // {id, arena offset, length, 0}
  const int32_t* farena;     // the sequences, back to back
  uint32_t fmask;
};

constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr int kOverrideMaxLen = 32;

__host__ __device__ inline uint64_t seq_hash(const int32_t* s, int n) {   // FNV-1a over the ids
  uint64_t h = 0xCBF29CE484222325ull ^ static_cast<uint64_t>(n);
  for (int i = 0; i < n; ++i) {
    h ^= static_cast<uint32_t>(s[i]);
    h *= 0x100000001B3ull;
  }
  h ^= h >> 29;
  return h == kEmptyKey ? 0 : h;
}

__host__ __device__ inline uint32_t pair_hash(uint32_t a, uint32_t b) {
  uint32_t h = a * 0x9E3779B1u;
  h ^= (b + 0x7F4A7C15u) * 0x85EBCA77u;
  h ^= h >> 15;
  return h;
}

__device__ __forceinline__ uint32_t decode_utf8(const uint8_t* p, const uint8_t* end, int& n) {
  const uint32_t b0 = p[0];
  if (b0 < 0x80) {
    n = 1;
    return b0;
  }
  if ((b0 >> 5) == 0x6 && p + 1 < end) {
    n = 2;
    return ((b0 & 0x1F) << 6) | (p[1] & 0x3F);
  }
  if ((b0 >> 4) == 0xE && p + 2 < end) {
    n = 3;
    return ((b0 & 0x0F) << 12) | ((p[1] & 0x3F) << 6) | (p[2] & 0x3F);
  }
  if ((b0 >> 3) == 0x1E && p + 3 < end) {
    n = 4;
    const uint32_t cp =
        ((b0 & 0x07) << 18) | ((p[1] & 0x3F) << 12) | ((p[2] & 0x3F) << 6) | (p[3] & 0x3F);
    return cp < 0x110000 ? cp : 0xFFFD;
  }
  n = 1;  // malformed: treat the byte as an unclassified symbol
  return 0xFFFD;
}

__device__ __forceinline__ uint8_t lower_ascii(uint8_t c) {
  return (c >= 'A' && c <= 'Z') ? c + 32 : c;
}

__global__ void __launch_bounds__(128)
pretok_kernel(TokTables tb, const uint8_t* __restrict__ text, const int64_t* __restrict__ row_off,
              int64_t n_rows, uint8_t* __restrict__ flags) {
  const int64_t row = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (row >= n_rows) return;
  const uint8_t* p = text + row_off[row];
  const uint8_t* end = text + row_off[row + 1];
  uint8_t* fl = flags + row_off[row];
  const uint8_t* base = p;
  auto cls_at = [&](const uint8_t* q, int& n) -> uint8_t { return tb.cls[decode_utf8(q, end, n)]; };

  while (p < end) {
    fl[p - base] = 1;
    int n;
    const uint32_t c = decode_utf8(p, end, n);
    const uint8_t k = tb.cls[c];
    // (1) contractions, ASCII case-insensitive
    if (c == '\'' && p + 1 < end) {
      const uint8_t c1 = lower_ascii(p[1]);
      if (c1 == 's' || c1 == 't' || c1 == 'm' || c1 == 'd') {
        p += 2;
        continue;
      }
      // U+017F LATIN SMALL LETTER LONG S (C5 BF) case-folds onto 's', so the pattern's (?i:'s)
      // matches "'ſ"; it is the only non-ASCII code point that folds onto a contraction letter
      if (p[1] == 0xC5 && p + 2 < end && p[2] == 0xBF) {
        p += 3;
        continue;
      }
      if (p + 2 < end) {
        const uint8_t c2 = lower_ascii(p[2]);
        if ((c1 == 'r' && c2 == 'e') || (c1 == 'v' && c2 == 'e') || (c1 == 'l' && c2 == 'l')) {
          p += 3;
          continue;
        }
      }
    }
    // (2) [^\r\n\p{L}\p{N}]?\p{L}+
    {
      const uint8_t* q = nullptr;
      if (k == CLS_LETTER) {
        q = p;
      } else if (c != '\r' && c != '\n' && k != CLS_NUMBER && p + n < end) {
        int n2;
        if (cls_at(p + n, n2) == CLS_LETTER) q = p + n;
      }
      if (q) {
        while (q < end) {
          int n2;
          if (cls_at(q, n2) != CLS_LETTER) break;
          q += n2;
        }
        p = q;
        continue;
      }
    }
    // (3) \p{N}{1,digits}
    if (k == CLS_NUMBER) {
      const uint8_t* q = p + n;
      for (int d = 1; d < tb.digits && q < end; ++d) {
        int n2;
        if (cls_at(q, n2) != CLS_NUMBER) break;
        q += n2;
      }
      p = q;
      continue;
    }
    // (4)  ?[^\s\p{L}\p{N}]+[\r\n]*
    {
      const uint8_t* q = (c == ' ') ? p + 1 : p;
      int n2;
      if (q < end && cls_at(q, n2) == CLS_OTHER) {
        while (q < end) {
          if (cls_at(q, n2) != CLS_OTHER) break;
          q += n2;
        }
        while (q < end && (*q == '\r' || *q == '\n')) ++q;
        p = q;
        continue;
      }
    }
    // (5)-(7) whitespace runs
    {
      const uint8_t* q = p;
      const uint8_t* last_nl_end = nullptr;
      const uint8_t* last_char = p;
      int count = 0;
      while (q < end) {
        int n2;
        if (cls_at(q, n2) != CLS_SPACE) break;
        if (*q == '\r' || *q == '\n') last_nl_end = q + 1;
        last_char = q;
        q += n2;
        ++count;
      }
      if (count == 0) {  // unreachable for well-formed input; never stall
        p += n;
        continue;
      }
      if (last_nl_end) {
        p = last_nl_end;  // \s*[\r\n]+
      } else if (q == end) {
        p = q;  // \s+(?!\S) at end of text
      } else if (count >= 2) {
        p = last_char;  // \s+(?!\S): leave one whitespace char for the next match
      } else {
        p = q;  // \s+
      }
    }
  }
}

__device__ __forceinline__ bool merge_lookup(const TokTables& tb, uint32_t a, uint32_t b,
                                             uint32_t& rank, uint32_t& id) {
  const uint64_t key = (static_cast<uint64_t>(a) << 32) | b;
  uint32_t h = pair_hash(a, b) & tb.hmask;
  while (true) {
    const uint64_t k = tb.hkeys[h];
    if (k == key) {
      const uint64_t v = tb.hvals[h];
      rank = static_cast<uint32_t>(v >> 32);
      id = static_cast<uint32_t>(v);
      return true;
    }
    if (k == kEmptyKey) return false;
    h = (h + 1) & tb.hmask;
  }
}

__global__ void __launch_bounds__(256)
bpe_kernel(TokTables tb, const uint8_t* __restrict__ text, int64_t n_bytes,
           const uint8_t* __restrict__ flags, int32_t* __restrict__ sym, int64_t* __restrict__ cnt) {
  const int64_t pos = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (pos >= n_bytes || !flags[pos]) return;
  int64_t e = pos + 1;
  while (e < n_bytes && !flags[e]) ++e;
  int n = static_cast<int>(e - pos);
  int32_t* s = sym + pos;
  for (int i = 0; i < n; ++i) s[i] = tb.byte_to_id[text[pos + i]];
  while (n > 1) {
    uint32_t best_rank = 0xFFFFFFFFu, best_id = 0;
    int best_i = -1;
    for (int i = 0; i + 1 < n; ++i) {
      uint32_t r, id;
      if (merge_lookup(tb, s[i], s[i + 1], r, id) && r < best_rank) {
        best_rank = r;
        best_id = id;
        best_i = i;
      }
    }
    if (best_i < 0) break;
    s[best_i] = static_cast<int32_t>(best_id);
    for (int i = best_i + 1; i + 1 < n; ++i) s[i] = s[i + 1];
    --n;
  }
  if (tb.fmask != 0 && n >= 2 && n <= kOverrideMaxLen) {   // whole-word override?
    const uint64_t key = seq_hash(s, n);
    uint32_t h = static_cast<uint32_t>(key) & tb.fmask;
    while (true) {
      const uint64_t k = tb.fkeys[h];
      if (k == kEmptyKey) break;
      if (k == key) {
        const int4 sl = tb.fslots[h];
        bool same = sl.z == n;
        for (int i = 0; same && i < n; ++i) same = tb.farena[sl.y + i] == s[i];
        if (same) {
          s[0] = sl.x;
          n = 1;
          break;
        }
      }
      h = (h + 1) & tb.fmask;
    }
  }
  cnt[pos] = n;
}

__global__ void __launch_bounds__(256)
compact_kernel(int64_t n_bytes, const int32_t* __restrict__ sym, const int64_t* __restrict__ cnt,
               const int64_t* __restrict__ outpos, int32_t* __restrict__ out_tokens) {
  const int64_t pos = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (pos >= n_bytes) return;
  const int n = static_cast<int>(cnt[pos]);
  if (n == 0) return;
  int32_t* dst = out_tokens + outpos[pos];
  for (int i = 0; i < n; ++i) dst[i] = sym[pos + i];
}

__global__ void row_offsets_kernel(const int64_t* __restrict__ row_off, int64_t n_rows,
                                   const int64_t* __restrict__ outpos,
                                   int64_t* __restrict__ row_tok_off) {
  const int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (r > n_rows) return;
  row_tok_off[r] = outpos[row_off[r]];
}

// ---- detokeniser: token ids -> bytes --------------------------------------
__global__ void __launch_bounds__(256)
detok_len_kernel(const int32_t* __restrict__ toks, int64_t n, const int32_t* __restrict__ tok_off,
                 int64_t* __restrict__ lens) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i > n) return;
  lens[i] = (i < n) ? (tok_off[toks[i] + 1] - tok_off[toks[i]]) : 0;
}

__global__ void __launch_bounds__(256)
detok_copy_kernel(const int32_t* __restrict__ toks, int64_t n, const int32_t* __restrict__ tok_off,
                  const uint8_t* __restrict__ tok_bytes, const int64_t* __restrict__ bytepos,
                  uint8_t* __restrict__ out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int b0 = tok_off[toks[i]], b1 = tok_off[toks[i] + 1];
  uint8_t* dst = out + bytepos[i];
  for (int b = b0; b < b1; ++b) dst[b - b0] = tok_bytes[b];
}

__global__ void detok_rows_kernel(const int64_t* __restrict__ row_tok_off, int64_t n_rows,
                                  const int64_t* __restrict__ bytepos,
                                  int64_t* __restrict__ row_byte_off) {
  const int64_t r = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (r > n_rows) return;
  row_byte_off[r] = bytepos[row_tok_off[r]];
}

}  // namespace

struct Tokenizer {
  uint8_t* d_cls = nullptr;
  uint64_t* d_hkeys = nullptr;
  uint64_t* d_hvals = nullptr;
  uint32_t hmask = 0;
  int32_t* d_byte_to_id = nullptr;
  int digits = 1;
  // vocabulary bytes for the detokeniser
  uint8_t* d_tok_bytes = nullptr;
  int32_t* d_tok_off = nullptr;
  int vocab = 0;
  // whole-word overrides (tokenizer_set_word_overrides)
  uint64_t* d_fkeys = nullptr;
  int4* d_fslots = nullptr;
  int32_t* d_farena = nullptr;
  uint32_t fmask = 0;
  // growable scratch
  int64_t cap = 0;
  uint8_t* d_flags = nullptr;
  int32_t* d_sym = nullptr;
  // per-position counts (tokens, or bytes when decoding) are 64-bit so that CUB's scan, which
  // accumulates in its input type, does not wrap past 2^31 tokens or output bytes in one call
  int64_t* d_cnt = nullptr;
  int64_t* d_outpos = nullptr;
  void* d_cub = nullptr;
  size_t cub_bytes = 0;

  ~Tokenizer() {
    cudaFree(d_cls);
    cudaFree(d_hkeys);
    cudaFree(d_hvals);
    cudaFree(d_byte_to_id);
    cudaFree(d_tok_bytes);
    cudaFree(d_tok_off);
    cudaFree(d_fkeys);
    cudaFree(d_fslots);
    cudaFree(d_farena);
    cudaFree(d_flags);
    cudaFree(d_sym);
    cudaFree(d_cnt);
    cudaFree(d_outpos);
    cudaFree(d_cub);
  }

  int reserve(int64_t n) {
    if (n + 1 <= cap) return 0;
    cudaFree(d_flags);
    cudaFree(d_sym);
    cudaFree(d_cnt);
    cudaFree(d_outpos);
    cudaFree(d_cub);
    d_flags = nullptr, d_sym = nullptr, d_cnt = nullptr, d_outpos = nullptr, d_cub = nullptr;
    cap = n + 1 + n / 4;
    SB_CUDA_CHECK(cudaMalloc(&d_flags, cap));
    SB_CUDA_CHECK(cudaMalloc(&d_sym, cap * sizeof(int32_t)));
    SB_CUDA_CHECK(cudaMalloc(&d_cnt, cap * sizeof(int64_t)));
    SB_CUDA_CHECK(cudaMalloc(&d_outpos, cap * sizeof(int64_t)));
    cub_bytes = 0;
    SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, d_cnt, d_outpos, cap));
    SB_CUDA_CHECK(cudaMalloc(&d_cub, cub_bytes));
    return 0;
  }
};

int tokenizer_create(const int32_t* merges, int n_merges, const int32_t* merged_ids,
                     const uint8_t* cls_table, int digits, const uint8_t* tok_bytes,
                     const int32_t* tok_off, int vocab, Tokenizer** out) {
  auto* t = new Tokenizer();
  t->digits = digits;
  t->vocab = vocab;
  uint32_t capn = 1024;
  while (capn < static_cast<uint32_t>(n_merges) * 2u + 16u) capn <<= 1;
  t->hmask = capn - 1;
  std::vector<uint64_t> keys(capn, kEmptyKey), vals(capn, 0);
  for (int i = 0; i < n_merges; ++i) {
    const uint32_t a = merges[2 * i], b = merges[2 * i + 1];
    const uint64_t key = (static_cast<uint64_t>(a) << 32) | b;
    uint32_t h = pair_hash(a, b) & t->hmask;
    while (keys[h] != kEmptyKey && keys[h] != key) h = (h + 1) & t->hmask;
    // a pair listed twice takes the rank of its LAST occurrence: `tokenizers` builds its merge
    // map by inserting the list in order, so a later entry replaces an earlier one
    keys[h] = key;
    const uint32_t id = merged_ids ? static_cast<uint32_t>(merged_ids[i]) : 256u + i;
    vals[h] = (static_cast<uint64_t>(i) << 32) | id;
  }
  int32_t b2i[256];
  for (int i = 0; i < 256; ++i) b2i[i] = i;
  const int64_t nbytes = tok_off[vocab];
  if (cudaMalloc(&t->d_cls, 0x110000) != cudaSuccess ||
      cudaMalloc(&t->d_hkeys, capn * 8ull) != cudaSuccess ||
      cudaMalloc(&t->d_hvals, capn * 8ull) != cudaSuccess ||
      cudaMalloc(&t->d_byte_to_id, 256 * 4) != cudaSuccess ||
      cudaMalloc(&t->d_tok_bytes, nbytes > 0 ? nbytes : 1) != cudaSuccess ||
      cudaMalloc(&t->d_tok_off, (vocab + 1) * 4ull) != cudaSuccess) {
    set_last_error("tokenizer_create: cudaMalloc failed: %s",
                   cudaGetErrorString(cudaGetLastError()));
    delete t;
    return -1;
  }
  cudaMemcpy(t->d_cls, cls_table, 0x110000, cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_hkeys, keys.data(), capn * 8ull, cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_hvals, vals.data(), capn * 8ull, cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_byte_to_id, b2i, sizeof(b2i), cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_tok_bytes, tok_bytes, nbytes, cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_tok_off, tok_off, (vocab + 1) * 4ull, cudaMemcpyHostToDevice);
  if (cudaGetLastError() != cudaSuccess) {
    set_last_error("tokenizer_create: upload failed");
    delete t;
    return -1;
  }
  *out = t;
  return 0;
}

// n sequences (seq_off[n+1] into seq_tokens), each the merge result of the vocabulary entry
// ids[i]; n == 0 clears the table.  Replaces any previous table.
int tokenizer_set_word_overrides(Tokenizer* t, const int32_t* seq_tokens, const int32_t* seq_off,
                                 const int32_t* ids, int n) {
  cudaFree(t->d_fkeys);
  cudaFree(t->d_fslots);
  cudaFree(t->d_farena);
  t->d_fkeys = nullptr, t->d_fslots = nullptr, t->d_farena = nullptr, t->fmask = 0;
  if (n <= 0) return 0;
  uint32_t capn = 64;
  while (capn < static_cast<uint32_t>(n) * 2u + 16u) capn <<= 1;
  std::vector<uint64_t> keys(capn, kEmptyKey);
  std::vector<int4> slots(capn, make_int4(0, 0, 0, 0));
  for (int i = 0; i < n; ++i) {
    const int off = seq_off[i], len = seq_off[i + 1] - seq_off[i];
    if (len < 2 || len > kOverrideMaxLen || ids[i] < 0 || ids[i] >= t->vocab) {
      set_last_error("tokenizer: word override %d has length %d (2..%d supported) or a bad id", i,
                     len, kOverrideMaxLen);
      return -1;
    }
    const uint64_t key = seq_hash(seq_tokens + off, len);
    uint32_t h = static_cast<uint32_t>(key) & (capn - 1);
    while (keys[h] != kEmptyKey) h = (h + 1) & (capn - 1);
    keys[h] = key;
    slots[h] = make_int4(ids[i], off, len, 0);
  }
  const size_t arena = static_cast<size_t>(seq_off[n]) * sizeof(int32_t);
  if (cudaMalloc(&t->d_fkeys, capn * 8ull) != cudaSuccess ||
      cudaMalloc(&t->d_fslots, capn * sizeof(int4)) != cudaSuccess ||
      cudaMalloc(&t->d_farena, arena) != cudaSuccess) {
    set_last_error("tokenizer: cudaMalloc of the override table failed: %s",
                   cudaGetErrorString(cudaGetLastError()));
    return -1;
  }
  cudaMemcpy(t->d_fkeys, keys.data(), capn * 8ull, cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_fslots, slots.data(), capn * sizeof(int4), cudaMemcpyHostToDevice);
  cudaMemcpy(t->d_farena, seq_tokens, arena, cudaMemcpyHostToDevice);
  SB_CUDA_CHECK(cudaGetLastError());
  t->fmask = capn - 1;
  return 0;
}

void tokenizer_destroy(Tokenizer* t) { delete t; }

const uint8_t* tokenizer_tok_bytes(const Tokenizer* t) { return t->d_tok_bytes; }
const int32_t* tokenizer_tok_off(const Tokenizer* t) { return t->d_tok_off; }

// text_dev/row_off_dev/out_* are device pointers; out_tokens has capacity n_bytes.
int tokenizer_encode(Tokenizer* t, const uint8_t* text_dev, int64_t n_bytes,
                     const int64_t* row_off_dev, int64_t n_rows, int32_t* out_tokens_dev,
                     int64_t* row_tok_off_dev, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (t->reserve(n_bytes)) return -1;
  TokTables tb{t->d_cls,    t->d_hkeys,  t->d_hvals,  t->hmask, t->d_byte_to_id, t->digits,
               t->d_fkeys,  t->d_fslots, t->d_farena, t->fmask};
  const int64_t n1 = n_bytes + 1;
  SB_CUDA_CHECK(cudaMemsetAsync(t->d_flags, 0, n1, stream));
  SB_CUDA_CHECK(cudaMemsetAsync(t->d_cnt, 0, n1 * sizeof(int64_t), stream));
  if (n_bytes > 0) {
    pretok_kernel<<<static_cast<unsigned>((n_rows + 127) / 128), 128, 0, stream>>>(
        tb, text_dev, row_off_dev, n_rows, t->d_flags);
    bpe_kernel<<<static_cast<unsigned>((n_bytes + 255) / 256), 256, 0, stream>>>(
        tb, text_dev, n_bytes, t->d_flags, t->d_sym, t->d_cnt);
  }
  size_t tmp = t->cub_bytes;
  SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(t->d_cub, tmp, t->d_cnt, t->d_outpos, n1, stream));
  if (n_bytes > 0) {
    compact_kernel<<<static_cast<unsigned>((n_bytes + 255) / 256), 256, 0, stream>>>(
        n_bytes, t->d_sym, t->d_cnt, t->d_outpos, out_tokens_dev);
  }
  row_offsets_kernel<<<static_cast<unsigned>((n_rows + 1 + 255) / 256), 256, 0, stream>>>(
      row_off_dev, n_rows, t->d_outpos, row_tok_off_dev);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// tokens[n_tok] grouped by row_tok_off[n_rows+1] -> bytes (capacity out_cap) + row_byte_off.
// Pass 1 (out_bytes == nullptr) only computes row_byte_off so the caller can size the blob.
int tokenizer_decode(Tokenizer* t, const int32_t* toks_dev, int64_t n_tok,
                     const int64_t* row_tok_off_dev, int64_t n_rows, uint8_t* out_bytes_dev,
                     int64_t* row_byte_off_dev, cudaStream_t stream) {
  if (t->reserve(n_tok)) return -1;
  const int64_t n1 = n_tok + 1;
  detok_len_kernel<<<static_cast<unsigned>((n1 + 255) / 256), 256, 0, stream>>>(
      toks_dev, n_tok, t->d_tok_off, t->d_cnt);
  size_t tmp = t->cub_bytes;
  SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(t->d_cub, tmp, t->d_cnt, t->d_outpos, n1, stream));
  detok_rows_kernel<<<static_cast<unsigned>((n_rows + 1 + 255) / 256), 256, 0, stream>>>(
      row_tok_off_dev, n_rows, t->d_outpos, row_byte_off_dev);
  if (out_bytes_dev && n_tok > 0) {
    detok_copy_kernel<<<static_cast<unsigned>((n_tok + 255) / 256), 256, 0, stream>>>(
        toks_dev, n_tok, t->d_tok_off, t->d_tok_bytes, t->d_outpos, out_bytes_dev);
  }
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
