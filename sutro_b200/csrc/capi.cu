// sutro_b200 — C-ABI (see include/sutro_b200.h).  Plain pointers and sizes,
// integer status codes, never throws across the boundary.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/sutro_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace sb {

static thread_local char g_err[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

}  // namespace sb

using namespace sb;

#define STREAM(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

const char* sb200_last_error(void) { return last_error(); }
int sb200_abi_version(void) { return SB200_ABI_VERSION; }

int sb200_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem) {
  int dev = 0;
  SB_CUDA_CHECK(cudaGetDevice(&dev));
  cudaDeviceProp p;
  SB_CUDA_CHECK(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  if (total_mem) *total_mem = p.totalGlobalMem;
  return 0;
}

int sb200_gemm_bf16_tn(const void* a, int a_rows, const void* w, void* d, const void* resid, int M,
                       int N, int K, int ldd, int epilogue, int block_n, void* stream) {
  return gemm_bf16_tn(a, a_rows, w, d, resid, M, N, K, ldd, epilogue, block_n, STREAM(stream));
}

int sb200_gemm_qkv_rope(const void* a, int a_rows, const void* w, void* qkv_out, int M, int K,
                        int block_n, const void* q_norm_w, const void* k_norm_w,
                        const void* cos_tab, const void* sin_tab, const int32_t* tok_slot,
                        const int32_t* tok_pos, const int32_t* page_table, int max_pages,
                        void* kv_layer, int hq, int hkv, float eps, void* stream) {
  // SB200_QKV_DENSE=0: skip the dense K/V copy (A/B timing of the epilogue only)
  static const int dense = [] {
    const char* e = getenv("SB200_QKV_DENSE");
    return (e != nullptr && e[0] == '0') ? 0 : 1;
  }();
  QkvEpiArgs ea{tok_pos, tok_slot, page_table, max_pages, kv_layer, cos_tab, sin_tab,
                q_norm_w, k_norm_w, hq, hkv, eps, dense};
  const int N = (hq + 2 * hkv) * kHeadDim;
  return gemm_bf16_tn(a, a_rows, w, qkv_out, nullptr, M, N, K, N, EPI_QKV_ROPE, block_n,
                      STREAM(stream), &ea);
}

int sb200_rmsnorm(const void* x, const void* w, void* out, int rows, int d, float eps,
                  void* stream) {
  return rmsnorm(x, w, out, rows, d, eps, STREAM(stream));
}

int sb200_embed_gather(const int32_t* ids, const void* table, void* out, int rows, int d,
                       void* stream) {
  return embed_gather(ids, table, out, rows, d, STREAM(stream));
}

int sb200_l2_normalize_rows(const void* x, float* out, int rows, int d, void* stream) {
  return l2_normalize_rows(x, out, rows, d, STREAM(stream));
}

int sb200_rope_kv_write(void* qkv, const void* q_norm_w, const void* k_norm_w, const void* cos_tab,
                        const void* sin_tab, const int32_t* tok_slot, const int32_t* tok_pos,
                        const int32_t* page_table, int max_pages, void* kv_layer, int T, int hq,
                        int hkv, float eps, void* stream) {
  return rope_kv_write(qkv, q_norm_w, k_norm_w, cos_tab, sin_tab, tok_slot, tok_pos, page_table,
                       max_pages, kv_layer, T, hq, hkv, eps, STREAM(stream));
}

int sb200_attn_decode(const void* qkv, void* out, const void* kv_layer, const int32_t* page_table,
                      int max_pages, const int32_t* row_slot, const int32_t* ctx_len, int B, int hq,
                      int hkv, float scale, void* stream) {
  // The contexts live on the device; max_pages bounds them without a synchronise.  A bound
  // past kDecodeSplitTokens lets every row split, in a workspace allocated stream-ordered.
  const int max_splits = attn_decode_splits(static_cast<int64_t>(max_pages) * kPageTokens);
  if (max_splits <= 1 || B <= 0)
    return attn_decode(qkv, out, kv_layer, page_table, max_pages, row_slot, ctx_len, B, hq, hkv,
                       scale, nullptr, 0, 1, nullptr, STREAM(stream));
  float* ws = nullptr;
  SB_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&ws),
                                attn_decode_ws_floats(B, hq, max_splits) * sizeof(float),
                                STREAM(stream)));
  const int rc = attn_decode(qkv, out, kv_layer, page_table, max_pages, row_slot, ctx_len, B, hq,
                             hkv, scale, nullptr, B, max_splits, ws, STREAM(stream));
  SB_CUDA_CHECK(cudaFreeAsync(ws, STREAM(stream)));
  return rc;
}

// Kept for callers of ABI version 1 (see the header).
void sb200_attn_decode_force_variant(int) {}

int sb200_attn_prefill(const void*, void*, const void*, const int32_t*, int, const int32_t*, int,
                       const int32_t*, const int32_t*, const int32_t*, const int32_t*, int hq,
                       int hkv, float, void*) {
  // the GQA group is still rejected as the other attention launchers reject it
  return dispatch_gqa("attn_prefill", hq, hkv, [](auto) {
    set_last_error("sb200_attn_prefill: the library has no paged prefill attention; use "
                   "sb200_attn_prefill_dense");
    return -1;
  });
}

int sb200_attn_prefill_q_tile(int hq, int hkv) { return attn_prefill_q_tile(hq, hkv); }

int sb200_attn_prefill_dense(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                             int prefix_rows, int n_layers, int layer, const int32_t* items,
                             int n_items, const int32_t* seq_q_start, const int32_t* seq_q_len,
                             const int32_t* seq_past, int hq, int hkv, float scale, void* stream) {
  return attn_prefill_dense(qkv, t_rows, out, prefix_kv, prefix_rows, n_layers, layer, items,
                            n_items, seq_q_start, seq_q_len, seq_past, hq, hkv, scale,
                            STREAM(stream));
}

int sb200_attn_prefill_chunked(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                               int prefix_rows, int n_layers, int layer, const int32_t* items,
                               int n_items, const int32_t* seq_q_start, const int32_t* seq_q_len,
                               const int32_t* seq_past, int hq, int hkv, float scale,
                               const void* kv_layer, const int32_t* page_table, int max_pages,
                               const int32_t* seq_slot, const int32_t* seq_hist, void* stream) {
  return attn_prefill_chunked(qkv, t_rows, out, prefix_kv, prefix_rows, n_layers, layer, items,
                              n_items, seq_q_start, seq_q_len, seq_past, hq, hkv, scale, kv_layer,
                              page_table, max_pages, seq_slot, seq_hist, STREAM(stream));
}

int sb200_attn_prefill_hist_align(int hq, int hkv) { return attn_prefill_hist_align(hq, hkv); }

int sb200_fsm_build_mask(const int32_t* fsm_trans, const uint8_t* fsm_accept, int n_states,
                         const uint8_t* tok_bytes, const int32_t* tok_off, int vocab, int eos_id,
                         uint32_t* mask_bits, int mask_words, void* stream) {
  return fsm_build_mask(fsm_trans, fsm_accept, n_states, tok_bytes, tok_off, vocab, eos_id,
                        mask_bits, mask_words, STREAM(stream));
}

int sb200_sample(const sb200_sample_args* p, void* stream) {
  return sample_greedy(*p, STREAM(stream));
}

int sb200_tokenizer_create(const int32_t* merges, int n_merges, const int32_t* merged_ids,
                           const uint8_t* cls_table, int digits, const uint8_t* tok_bytes,
                           const int32_t* tok_off, int vocab, void** out) {
  Tokenizer* t = nullptr;
  const int rc = tokenizer_create(merges, n_merges, merged_ids, cls_table, digits, tok_bytes,
                                  tok_off, vocab, &t);
  *out = t;
  return rc;
}
int sb200_tokenizer_set_word_overrides(void* tok, const int32_t* seq_tokens, const int32_t* seq_off,
                                       const int32_t* ids, int n) {
  return tokenizer_set_word_overrides(static_cast<Tokenizer*>(tok), seq_tokens, seq_off, ids, n);
}
void sb200_tokenizer_destroy(void* tok) { tokenizer_destroy(static_cast<Tokenizer*>(tok)); }
int sb200_tokenizer_encode(void* tok, const uint8_t* text_dev, int64_t n_bytes,
                           const int64_t* row_off_dev, int64_t n_rows, int32_t* out_tokens_dev,
                           int64_t* row_tok_off_dev, void* stream) {
  return tokenizer_encode(static_cast<Tokenizer*>(tok), text_dev, n_bytes, row_off_dev, n_rows,
                          out_tokens_dev, row_tok_off_dev, STREAM(stream));
}
int sb200_tokenizer_decode(void* tok, const int32_t* toks_dev, int64_t n_tok,
                           const int64_t* row_tok_off_dev, int64_t n_rows, uint8_t* out_bytes_dev,
                           int64_t* row_byte_off_dev, void* stream) {
  return tokenizer_decode(static_cast<Tokenizer*>(tok), toks_dev, n_tok, row_tok_off_dev, n_rows,
                          out_bytes_dev, row_byte_off_dev, STREAM(stream));
}

}  // extern "C"
