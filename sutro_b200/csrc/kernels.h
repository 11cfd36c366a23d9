// sutro_b200 — internal launcher declarations shared by the kernels, the engine
// and the C-ABI (capi.cu).  All launchers return 0 on success, -1 on error
// (message retrievable through sb::last_error()).  No launcher synchronises.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sutro_b200.h"

namespace sb {

const char* last_error();
void set_last_error(const char* fmt, ...);

// ---------------------------------------------------------------------------
// geometry of the paged KV cache (see DESIGN.md "data layout in HBM")
//   pool[layer][page][kv_head][K|V][kPageTokens][kHeadDim]  bf16
//   inside one [16][128] tile the 16-byte chunk c of token row r is stored at
//   chunk position c ^ (r & 7): a flat 4 KiB bulk copy then lands in shared
//   memory already bank-conflict-free for ldmatrix.
// ---------------------------------------------------------------------------
constexpr int kHeadDim = 128;
constexpr int kPageTokens = 16;
constexpr int kTileElems = kPageTokens * kHeadDim;   // one K (or V) tile of one head
constexpr int kTileBytes = kTileElems * 2;           // 4096

// The layout above in code: every kernel that reads or writes the pool, and every host-side
// size of it, goes through these.
// elements of one page of one layer: the K and V tiles of every kv head
__host__ __device__ inline size_t kv_page_elems(int hkv) {
  return static_cast<size_t>(hkv) * 2 * kTileElems;
}
// element offset, within one layer, of the K (is_k) or V tile of kv head kvh of a page; the
// V tile directly follows the K tile, so one copy of 2 * kTileBytes from the K tile fetches both
__host__ __device__ inline size_t kv_tile_offset(size_t page, int hkv, int kvh, bool is_k) {
  return (page * hkv + kvh) * (2 * kTileElems) + (is_k ? 0 : kTileElems);
}
// stored position of the 16-byte chunk c of token row r of a tile
__host__ __device__ inline int kv_chunk(int r, int c) { return c ^ (r & 7); }
// physical page that holds position pos of the sequence in slot `slot` (row pos % kPageTokens)
__host__ __device__ inline int kv_page(const int32_t* page_table, int max_pages, int slot, int pos) {
  return page_table[static_cast<size_t>(slot) * max_pages + pos / kPageTokens];
}

enum GemmEpilogue {
  EPI_STORE_BF16 = 0,
  EPI_RESIDUAL_BF16 = 1,
  EPI_SWIGLU_BF16 = 2,
  EPI_STORE_F32 = 3,
  EPI_QKV_ROPE = 4,  // QKV projection fused with q/k-norm + RoPE + paged K/V write (K1+K5)
};

// Extra operands of EPI_QKV_ROPE: everything rope_kv_write needs, applied to the
// accumulators in the GEMM epilogue so the [T, qkv_dim] tensor never round-trips HBM.
struct QkvEpiArgs {
  const int32_t* tok_pos;
  const int32_t* tok_slot;
  const int32_t* page_table;
  int max_pages;
  void* kv_layer;
  const void* cos_tab;
  const void* sin_tab;
  const void* q_norm_w;  // nullptr: no per-head norm
  const void* k_norm_w;
  int hq, hkv;
  float eps;
  int write_dense;  // also leave post-norm/RoPE K and V in their qkv columns (dense prefill attention)
};

// K1 — D = A · W^T (+ fused epilogue); A:[a_rows>=M, K] bf16, W:[N,K] bf16.
int gemm_bf16_tn(const void* a, int a_rows, const void* w, void* d, const void* resid, int M,
                 int N, int K, int ldd, int epilogue, int block_n, cudaStream_t stream,
                 const QkvEpiArgs* qkv_args = nullptr);
int gemm_pick_block_n(int M, int N);

// K4 — RMSNorm over rows: out = bf16(w * bf16(x * rsqrt(mean(x^2) + eps))).
int rmsnorm(const void* x, const void* w, void* out, int rows, int d, float eps,
            cudaStream_t stream);

// K9a — embedding gather: out[t,:] = table[ids[t],:].
int embed_gather(const int32_t* ids, const void* table, void* out, int rows, int d,
                 cudaStream_t stream);
// gather rows of x by index (last-token selection before the lm_head).
int gather_rows(const int32_t* idx, const void* x, void* out, int rows, int d,
                cudaStream_t stream);

// K5 — per-head q/k RMSNorm (optional) + RoPE on q and k, K/V scatter into the
// paged cache.  qkv:[T, (hq+2*hkv)*128] is updated in place for q.
int rope_kv_write(void* qkv, const void* q_norm_w, const void* k_norm_w, const void* cos_tab,
                  const void* sin_tab, const int32_t* tok_slot, const int32_t* tok_pos,
                  const int32_t* page_table, int max_pages, void* kv_layer, int T, int hq,
                  int hkv, float eps, cudaStream_t stream);

// K2 — paged-KV decode attention (one query token per sequence).
// A row of more than kDecodeSplitTokens tokens is attended in splits of kDecodeSplitTokens
// tokens at absolute positions, merged in split order (split-KV); a shorter row is one split.
// Rows split_rows[0 .. n_split_rows) (null: rows 0 .. n_split_rows) may be split, into at most
// max_splits splits each; ws holds attn_decode_ws_floats() floats.  Every row longer than
// kDecodeSplitTokens must be among them, unless max_splits <= 1 or n_split_rows == 0: then no
// row is split, and the launch is the single-split kernel alone.
constexpr int kDecodeSplitTokens = 4096;
inline int attn_decode_splits(int64_t ctx) {
  return static_cast<int>((ctx + kDecodeSplitTokens - 1) / kDecodeSplitTokens);
}
inline size_t attn_decode_ws_floats(int n_split_rows, int hq, int max_splits) {
  return static_cast<size_t>(n_split_rows) * hq * max_splits * (kHeadDim + 2);
}
int attn_decode(const void* qkv, void* out, const void* kv_layer, const int32_t* page_table,
                int max_pages, const int32_t* row_slot, const int32_t* ctx_len, int B, int hq,
                int hkv, float scale, const int32_t* split_rows, int n_split_rows, int max_splits,
                float* ws, cudaStream_t stream);

// K3 — causal prefill attention over DENSE K/V: new tokens' K/V are the k/v columns
// of the qkv buffer itself (post-norm/RoPE, written by the fused QKV epilogue), the shared
// prefix's K/V live in prefix_kv[n_layers][prefix_rows][2*hkv*128] (K heads | V heads).
// items: [n_items] {seq, q_tile_start} with q tile = attn_prefill_q_tile(); every sequence
// attends to prefix rows [0, seq_past) and its own rows causally.
int attn_prefill_dense(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                       int prefix_rows, int n_layers, int layer, const int32_t* items, int n_items,
                       const int32_t* seq_q_start, const int32_t* seq_q_len,
                       const int32_t* seq_past, int hq, int hkv, float scale, cudaStream_t stream);
int attn_prefill_q_tile(int hq, int hkv);  // query tokens per work item: 128 / G
// The same attention for rows prefilled in chunks: sequence i's own tokens [0, seq_hist[i]) come
// from the paged pool (kv_layer, page_table row seq_slot[i]); seq_hist[i] is a multiple of
// attn_prefill_hist_align(), which makes the result bit-identical to one unchunked call.
int attn_prefill_chunked(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                         int prefix_rows, int n_layers, int layer, const int32_t* items,
                         int n_items, const int32_t* seq_q_start, const int32_t* seq_q_len,
                         const int32_t* seq_past, int hq, int hkv, float scale,
                         const void* kv_layer, const int32_t* page_table, int max_pages,
                         const int32_t* seq_slot, const int32_t* seq_hist, cudaStream_t stream);
int attn_prefill_hist_align(int hq, int hkv);  // lcm(128, q tile); 0 for an unsupported group

// bf16 tensor map, 128-byte swizzle, rank 2..5 (gemm_wgmma.cu)
int encode_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box);

// K8 — FSM token-mask build, masked greedy sampling + FSM advance.  The sampler's arguments are
// the public sb200_sample_args, documented in the header.
using SampleArgs = sb200_sample_args;
// The row-history table of the penalty kernel is sized by out_stride; longer outputs are refused.
constexpr int kPenaltyMaxOutput = 8192;
bool penalties_active(const SampleArgs& a);  // sample_greedy() then launches the penalty kernel
// Penalties (when active), then the greedy or the stochastic kernel, dispatched on a.temperature.
int sample_greedy(const SampleArgs& a, cudaStream_t stream);
int prepare_decode(const int32_t* row_slot, const int32_t* slot_next_tok, const int32_t* slot_pos,
                   int32_t* tok_ids, int32_t* tok_pos, int32_t* tok_slot, int32_t* ctx_len, int B,
                   cudaStream_t stream);
int fsm_build_mask(const int32_t* fsm_trans, const uint8_t* fsm_accept, int n_states,
                   const uint8_t* tok_bytes, const int32_t* tok_off, int vocab, int eos_id,
                   uint32_t* mask_bits, int mask_words, cudaStream_t stream);

// K7 — GPU byte-level BPE tokenizer / detokenizer (tokenizer.cu).
struct Tokenizer;
int tokenizer_create(const int32_t* merges, int n_merges, const int32_t* merged_ids,
                     const uint8_t* cls_table, int digits, const uint8_t* tok_bytes,
                     const int32_t* tok_off, int vocab, Tokenizer** out);
int tokenizer_set_word_overrides(Tokenizer* t, const int32_t* seq_tokens, const int32_t* seq_off,
                                 const int32_t* ids, int n);
void tokenizer_destroy(Tokenizer* t);
const uint8_t* tokenizer_tok_bytes(const Tokenizer* t);
const int32_t* tokenizer_tok_off(const Tokenizer* t);
int tokenizer_encode(Tokenizer* t, const uint8_t* text_dev, int64_t n_bytes,
                     const int64_t* row_off_dev, int64_t n_rows, int32_t* out_tokens_dev,
                     int64_t* row_tok_off_dev, cudaStream_t stream);
int tokenizer_decode(Tokenizer* t, const int32_t* toks_dev, int64_t n_tok,
                     const int64_t* row_tok_off_dev, int64_t n_rows, uint8_t* out_bytes_dev,
                     int64_t* row_byte_off_dev, cudaStream_t stream);

// K9b — embedding head: last-token rows -> fp32 L2-normalised vectors.
int l2_normalize_rows(const void* x, float* out, int rows, int d, cudaStream_t stream);

}  // namespace sb
