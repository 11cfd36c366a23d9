// sutro_b200 — the batch-inference engine: what the reference leaves to its
// hosted service after `POST batch-inference` (sutro/sdk.py:223): for N rows,
// prefill + greedy decode over one model replica, with continuous batching, a
// paged KV cache, shared-prefix reuse and constrained decoding.
//
// One engine == one GPU == one host thread.  All scheduling is host C++; every
// arithmetic step is one of the kernels in this directory.  There is no CPU
// compute path: if a launch fails the job fails.
//
// Memory plan (see DESIGN.md): weights are caller-owned device tensors; the
// engine owns the KV pool (num_pages x layers x hkv x 8 KiB), activation
// workspaces sized for max(max_prefill_tokens, max_slots) tokens, a logits
// chunk, the page table and the per-slot decode state.
#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "../../include/sutro_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace sb {

namespace {

using bf16 = __nv_bfloat16;

// ---- small device helpers owned by the engine -----------------------------
struct SeqInit {  // one admitted row
  int32_t slot, row, q_start, q_len, past, n_row_tok, max_new, fsm_start;
};

// Fill the flattened token batch of a prefill step from (prefix | row | suffix).
__global__ void __launch_bounds__(128)
prefill_prepare_kernel(const SeqInit* __restrict__ seqs, const int32_t* __restrict__ prefix,
                       int n_prefix, const int32_t* __restrict__ suffix, int n_suffix,
                       const int32_t* __restrict__ row_tokens,
                       const int64_t* __restrict__ row_tok_off, int32_t* __restrict__ tok_ids,
                       int32_t* __restrict__ tok_pos, int32_t* __restrict__ tok_slot,
                       int32_t* __restrict__ last_idx) {
  const SeqInit s = seqs[blockIdx.x];
  const int64_t roff = s.row >= 0 ? row_tok_off[s.row] : 0;
  for (int j = threadIdx.x; j < s.q_len; j += blockDim.x) {
    const int p = s.past + j;
    int tok;
    if (p < n_prefix) {
      tok = prefix[p];
    } else if (p < n_prefix + s.n_row_tok) {
      tok = row_tokens[roff + (p - n_prefix)];
    } else {
      tok = suffix[p - n_prefix - s.n_row_tok];
    }
    tok_ids[s.q_start + j] = tok;
    tok_pos[s.q_start + j] = p;
    tok_slot[s.q_start + j] = s.slot;
  }
  if (threadIdx.x == 0) last_idx[blockIdx.x] = s.q_start + s.q_len - 1;
}

// Install page-table rows and decode state for newly admitted rows.
__global__ void __launch_bounds__(128)
init_slots_kernel(const SeqInit* __restrict__ seqs, const int32_t* __restrict__ pt_rows,
                  int max_pages, int32_t* __restrict__ page_table, int32_t* slot_state,
                  int32_t* slot_ngen, int32_t* slot_pos, int32_t* slot_done, int32_t* slot_row,
                  int32_t* slot_maxnew, int32_t* slot_next_tok, const int32_t* __restrict__ forced,
                  int n_forced, int32_t* __restrict__ out_tokens, int32_t* __restrict__ out_len,
                  int out_stride, float* __restrict__ slot_cum_logprob) {
  const SeqInit s = seqs[blockIdx.x];
  for (int i = threadIdx.x; i < max_pages; i += blockDim.x)
    page_table[static_cast<size_t>(s.slot) * max_pages + i] =
        pt_rows[static_cast<size_t>(blockIdx.x) * max_pages + i];
  // jump-forward: the forced output prefix was fed with the prompt; it is output too
  if (s.row >= 0 && out_tokens != nullptr)
    for (int i = threadIdx.x; i < n_forced; i += blockDim.x)
      out_tokens[static_cast<size_t>(s.row) * out_stride + i] = forced[i];
  if (threadIdx.x == 0) {
    if (s.row >= 0 && out_len != nullptr) out_len[s.row] = n_forced;
    slot_state[s.slot] = s.fsm_start;
    slot_ngen[s.slot] = s.row >= 0 ? n_forced : 0;
    slot_pos[s.slot] = s.past + s.q_len - 1;  // sampler increments: next position = prompt length
    slot_done[s.slot] = 0;
    slot_row[s.slot] = s.row;
    slot_maxnew[s.slot] = s.max_new;
    slot_next_tok[s.slot] = 0;
    slot_cum_logprob[s.slot] = 0.f;
  }
}

// Seed the first own page of newly admitted rows with the partially filled last page of the
// shared prefix (all layers, all kv heads): sharing is page-granular, but the tail of the
// prefix need not be recomputed per row — a 2.3 MB copy replaces up to 15 tokens of prefill.
__global__ void __launch_bounds__(256)
copy_prefix_page_kernel(__nv_bfloat16* __restrict__ kv_pool, size_t layer_stride,
                        size_t page_elems, int src_page, const int32_t* __restrict__ dst_pages) {
  const int dst = dst_pages[blockIdx.x];
  if (dst < 0) return;
  __nv_bfloat16* base = kv_pool + static_cast<size_t>(blockIdx.y) * layer_stride;
  const uint4* s = reinterpret_cast<const uint4*>(base + static_cast<size_t>(src_page) * page_elems);
  uint4* d = reinterpret_cast<uint4*>(base + static_cast<size_t>(dst) * page_elems);
  for (size_t i = threadIdx.x; i < page_elems / 8; i += blockDim.x) d[i] = s[i];
}

__global__ void scatter_embed_kernel(const float* __restrict__ src, const SeqInit* __restrict__ seqs,
                                     float* __restrict__ dst, int d) {
  const int row = seqs[blockIdx.x].row;
  for (int i = threadIdx.x; i < d; i += blockDim.x)
    dst[static_cast<size_t>(row) * d + i] = src[static_cast<size_t>(blockIdx.x) * d + i];
}

// Per-kernel-class device timing (job.profile): CUDA events around every launch on the
// engine stream, resolved after the job.  Used by bench.py for the roofline numbers.
struct Profiler {
  bool on = false;
  cudaStream_t stream = nullptr;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  std::vector<std::pair<int, size_t>> spans;
  double ms[SB200_KC_COUNT] = {0};
  int64_t launches[SB200_KC_COUNT] = {0};
  void reset(bool enable, cudaStream_t s) {
    on = enable;
    stream = s;
    used = 0;
    spans.clear();
    for (int i = 0; i < SB200_KC_COUNT; ++i) ms[i] = 0, launches[i] = 0;
  }
  void begin(int cls) {
    ++launches[cls];
    if (!on) return;
    while (pool.size() < used + 2) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      pool.push_back(e);
    }
    cudaEventRecord(pool[used], stream);
    spans.emplace_back(cls, used);
  }
  void end() {
    if (!on) return;
    cudaEventRecord(pool[used + 1], stream);
    used += 2;
  }
  void resolve() {
    if (!on) return;
    cudaStreamSynchronize(stream);
    for (auto& sp : spans) {
      float t = 0.f;
      cudaEventElapsedTime(&t, pool[sp.second], pool[sp.second + 1]);
      ms[sp.first] += t;
    }
  }
  ~Profiler() {
    for (auto e : pool) cudaEventDestroy(e);
  }
};
#define SB_K(cls, call)        \
  do {                         \
    prof.begin(cls);           \
    const int _rc = (call);    \
    prof.end();                \
    if (_rc) return -1;        \
  } while (0)

__global__ void scatter_logits_kernel(const float* __restrict__ logits,
                                      const int32_t* __restrict__ row_slot,
                                      const int32_t* __restrict__ slot_row, float* __restrict__ dst,
                                      int vocab) {
  const int row = slot_row[row_slot[blockIdx.x]];
  const float4* src = reinterpret_cast<const float4*>(logits + static_cast<size_t>(blockIdx.x) * vocab);
  float4* d = reinterpret_cast<float4*>(dst + static_cast<size_t>(row) * vocab);
  for (int i = threadIdx.x; i < vocab / 4; i += blockDim.x) d[i] = src[i];
}

template <typename T>
int dmalloc(T** p, size_t n) {
  SB_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  return 0;
}

}  // namespace

struct Engine {
  sb200_engine_config cfg{};
  sb200_engine_weights w{};
  std::vector<const void*> ln1, ln2, wqkv, wo, wgu, wd, qn, kn;
  cudaStream_t stream = nullptr;
  int qkv_dim = 0, q_dim = 0, max_pages = 0, t_max = 0, logit_rows = 0, q_tile = 0;
  int64_t num_pages = 0;
  size_t layer_stride = 0;  // elements between consecutive layers in the KV pool

  bf16 *x = nullptr, *h = nullptr, *qkv = nullptr, *attn = nullptr, *act = nullptr, *hl = nullptr,
       *hn = nullptr, *kv_pool = nullptr;
  float *logits = nullptr, *embed_tmp = nullptr;
  int32_t *tok_ids = nullptr, *tok_pos = nullptr, *tok_slot = nullptr, *ctx_len = nullptr,
          *row_slot = nullptr, *last_idx = nullptr, *page_table = nullptr;
  int32_t *slot_state = nullptr, *slot_ngen = nullptr, *slot_next_tok = nullptr,
          *slot_pos = nullptr, *slot_done = nullptr, *slot_row = nullptr, *slot_maxnew = nullptr;
  float* slot_cum_logprob = nullptr;
  // staging
  int32_t *h_stage = nullptr, *d_stage = nullptr;
  size_t stage_cap = 0;  // int32 elements
  int32_t* h_done = nullptr;
  // vocabulary bytes + FSM tables
  uint8_t* d_tok_bytes = nullptr;
  int32_t* d_tok_off = nullptr;
  int32_t* d_fsm_trans = nullptr;
  uint8_t *d_fsm_accept = nullptr, *d_fsm_final = nullptr;
  uint32_t* d_mask_bits = nullptr;
  int32_t *d_tail_off = nullptr, *d_tail_tok = nullptr;  // jump-forward terminal tails
  int mask_words = 0;
  size_t fsm_cap_states = 0;
  // job-scoped prompt pieces
  int32_t *d_prefix = nullptr, *d_suffix = nullptr;
  int prefix_cap = 0, suffix_cap = 0;
  // host page allocator
  std::vector<int32_t> free_pages;
  Profiler prof;
  double gemm_flops = 0, attn_decode_bytes = 0;
  int device = 0;
  bf16* prefix_kv = nullptr;  // [n_layers][prefix_rows][2*hkv*128]: dense K|V of the shared prefix
  int prefix_rows = 0;
  bool fill_prefix = false;   // this forward pass is the prefix prefill: keep its K/V

  ~Engine() {
    for (void* p : {(void*)x, (void*)h, (void*)qkv, (void*)attn, (void*)act, (void*)hl, (void*)hn,
                    (void*)kv_pool, (void*)logits, (void*)embed_tmp, (void*)tok_ids,
                    (void*)tok_pos, (void*)tok_slot, (void*)ctx_len, (void*)row_slot,
                    (void*)last_idx, (void*)page_table, (void*)slot_state, (void*)slot_ngen,
                    (void*)slot_next_tok, (void*)slot_pos, (void*)slot_done, (void*)slot_row,
                    (void*)slot_maxnew, (void*)slot_cum_logprob, (void*)d_stage, (void*)d_tok_bytes, (void*)d_tok_off,
                    (void*)d_fsm_trans, (void*)d_fsm_accept, (void*)d_fsm_final,
                    (void*)d_mask_bits, (void*)d_prefix, (void*)d_suffix, (void*)d_tail_off,
                    (void*)d_tail_tok, (void*)prefix_kv})
      cudaFree(p);
    if (h_stage) cudaFreeHost(h_stage);
    if (h_done) cudaFreeHost(h_done);
    if (stream) cudaStreamDestroy(stream);
  }

  bf16* kv_layer(int l) const { return kv_pool + static_cast<size_t>(l) * layer_stride; }

  int init() {
    const auto& c = cfg;
    q_dim = c.n_q_heads * kHeadDim;
    qkv_dim = (c.n_q_heads + 2 * c.n_kv_heads) * kHeadDim;
    max_pages = (c.max_position + kPageTokens - 1) / kPageTokens + 1;
    t_max = std::max(c.max_prefill_tokens, c.max_slots);
    logit_rows = std::min(std::max(c.logit_chunk_rows, 1), std::max(c.max_slots, 1));
    q_tile = attn_prefill_q_tile(c.n_q_heads, c.n_kv_heads);
    num_pages = c.num_pages;
    layer_stride = num_pages * kv_page_elems(c.n_kv_heads);
    SB_CUDA_CHECK(cudaGetDevice(&device));
    SB_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    const size_t T = t_max, S = c.max_slots + 2;  // +prefix slot, +dummy slot
    if (dmalloc(&x, T * c.d_model) || dmalloc(&h, T * c.d_model) || dmalloc(&qkv, T * qkv_dim) ||
        dmalloc(&attn, T * q_dim) || dmalloc(&act, T * c.d_ff) ||
        dmalloc(&hl, static_cast<size_t>(c.max_slots) * c.d_model) ||
        dmalloc(&hn, static_cast<size_t>(c.max_slots) * c.d_model) ||
        dmalloc(&kv_pool, layer_stride * c.n_layers) ||
        dmalloc(&tok_ids, T) || dmalloc(&tok_pos, T) || dmalloc(&tok_slot, T) ||
        dmalloc(&ctx_len, S) || dmalloc(&row_slot, S) || dmalloc(&last_idx, S) ||
        dmalloc(&page_table, S * max_pages) || dmalloc(&slot_state, S) || dmalloc(&slot_ngen, S) ||
        dmalloc(&slot_next_tok, S) || dmalloc(&slot_pos, S) || dmalloc(&slot_done, S) ||
        dmalloc(&slot_row, S) || dmalloc(&slot_maxnew, S) || dmalloc(&slot_cum_logprob, S))
      return -1;
    if (c.embedding_model) {
      if (dmalloc(&embed_tmp, static_cast<size_t>(c.max_slots) * c.d_model)) return -1;
    } else {
      if (dmalloc(&logits, static_cast<size_t>(logit_rows) * c.vocab)) return -1;
    }
    // K/V tiles must hold finite values everywhere (masked P * V must stay 0); the same goes
    // for the k/v columns of the qkv buffer, which the dense prefill attention reads in
    // 32-row boxes that may run past the end of a sequence.
    SB_CUDA_CHECK(cudaMemsetAsync(kv_pool, 0, layer_stride * c.n_layers * sizeof(bf16), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(qkv, 0, T * qkv_dim * sizeof(bf16), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(page_table, 0, S * max_pages * sizeof(int32_t), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(slot_done, 0, S * sizeof(int32_t), stream));
    stage_cap = (sizeof(SeqInit) / 4) * S + static_cast<size_t>(S) * max_pages + 2 * (T / 16 + S) +
                5 * S + 64;
    SB_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&h_stage), stage_cap * 4));
    if (dmalloc(&d_stage, stage_cap)) return -1;
    SB_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&h_done), S * 4));
    free_pages.reserve(num_pages);
    for (int64_t p = num_pages - 1; p >= 0; --p) free_pages.push_back(static_cast<int32_t>(p));
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
    return 0;
  }

  // ---- one pass of the transformer stack over T flattened tokens -----------
  // prefill: attention over (cached prefix | new tokens) per sequence;
  // decode : one token per sequence against its paged history.
  int forward(int T, bool prefill, const int32_t* d_work, int n_work,
              const int32_t* d_seq_q_start, const int32_t* d_seq_q_len, const int32_t* d_seq_past) {
    const auto& c = cfg;
    const float scale = 1.0f / sqrtf(static_cast<float>(kHeadDim));
    auto gemm = [&](const void* a, const void* wt, void* d, const void* r, int M, int N, int K,
                    int ldd, int epi) {
      gemm_flops += 2.0 * M * N * K;
      return gemm_bf16_tn(a, t_max, wt, d, r, M, N, K, ldd, epi, 0, stream);
    };
    SB_K(SB200_KC_EMBED, embed_gather(tok_ids, w.embed, x, T, c.d_model, stream));
    for (int l = 0; l < c.n_layers; ++l) {
      SB_K(SB200_KC_NORM, rmsnorm(x, ln1[l], h, T, c.d_model, c.rms_eps, stream));
      // K1+K5 fused: q/k-norm, RoPE and the paged K/V write happen in the GEMM epilogue; in
      // prefill it also leaves K/V in their qkv columns for the dense prefill attention
      QkvEpiArgs qa{tok_pos, tok_slot, page_table, max_pages, kv_layer(l), w.rope_cos,
                    w.rope_sin, qn[l], kn[l], c.n_q_heads, c.n_kv_heads, c.rms_eps,
                    prefill ? 1 : 0};
      gemm_flops += 2.0 * T * qkv_dim * c.d_model;
      SB_K(SB200_KC_GEMM, gemm_bf16_tn(h, t_max, wqkv[l], qkv, nullptr, T, qkv_dim, c.d_model,
                                       qkv_dim, EPI_QKV_ROPE, 0, stream, &qa));
      if (prefill && fill_prefix && prefix_kv != nullptr) {
        // the shared prefix's K/V (k|v columns of its rows) go to the dense side buffer
        const size_t cols = 2ull * c.n_kv_heads * kHeadDim;
        SB_CUDA_CHECK(cudaMemcpy2DAsync(prefix_kv + static_cast<size_t>(l) * prefix_rows * cols,
                                        cols * sizeof(bf16), qkv + q_dim, qkv_dim * sizeof(bf16),
                                        cols * sizeof(bf16), T, cudaMemcpyDeviceToDevice, stream));
      }
      if (prefill) {
        SB_K(SB200_KC_ATTN_PREFILL,
             attn_prefill_dense(qkv, t_max, attn, prefix_kv, prefix_rows, c.n_layers, l, d_work,
                                n_work, d_seq_q_start, d_seq_q_len, d_seq_past, c.n_q_heads,
                                c.n_kv_heads, scale, stream));
      } else {
        SB_K(SB200_KC_ATTN_DECODE,
             attn_decode(qkv, attn, kv_layer(l), page_table, max_pages, row_slot, ctx_len, T,
                         c.n_q_heads, c.n_kv_heads, scale, stream));
      }
      SB_K(SB200_KC_GEMM, gemm(attn, wo[l], x, x, T, c.d_model, q_dim, c.d_model,
                               EPI_RESIDUAL_BF16));
      SB_K(SB200_KC_NORM, rmsnorm(x, ln2[l], h, T, c.d_model, c.rms_eps, stream));
      SB_K(SB200_KC_GEMM, gemm(h, wgu[l], act, nullptr, T, 2 * c.d_ff, c.d_model, c.d_ff,
                               EPI_SWIGLU_BF16));
      SB_K(SB200_KC_GEMM, gemm(act, wd[l], x, x, T, c.d_model, c.d_ff, c.d_model,
                               EPI_RESIDUAL_BF16));
    }
    return 0;
  }

  // final norm + lm_head + masked greedy sampling for `n` rows whose hidden
  // states are rows idx[0..n) of x (idx == nullptr: rows 0..n).
  int head_and_sample(int n, const int32_t* idx, const int32_t* d_row_slot,
                      const sb200_job& job, bool has_fsm, bool first_decision = false) {
    const auto& c = cfg;
    const bf16* src = x;
    if (idx) {
      SB_K(SB200_KC_EMBED, gather_rows(idx, x, hl, n, c.d_model, stream));
      src = hl;
    }
    SB_K(SB200_KC_NORM, rmsnorm(src, w.final_norm, hn, n, c.d_model, c.rms_eps, stream));
    for (int r0 = 0; r0 < n; r0 += logit_rows) {
      const int nr = std::min(logit_rows, n - r0);
      gemm_flops += 2.0 * nr * c.vocab * c.d_model;
      SB_K(SB200_KC_GEMM,
           gemm_bf16_tn(hn + static_cast<size_t>(r0) * c.d_model, c.max_slots - r0, w.lm_head,
                        logits, nullptr, nr, c.vocab, c.d_model, c.vocab, EPI_STORE_F32, 0,
                        stream));
      if (first_decision && job.out_first_logits_dev) {
        scatter_logits_kernel<<<nr, 256, 0, stream>>>(logits, d_row_slot + r0, slot_row,
                                                      job.out_first_logits_dev, c.vocab);
        SB_CUDA_CHECK(cudaGetLastError());
      }
      SampleArgs a{};
      a.logits = logits;
      a.ldl = c.vocab;
      a.vocab = c.vocab;
      a.B = nr;
      a.row_slot = d_row_slot + r0;
      a.slot_state = slot_state;
      a.slot_ngen = slot_ngen;
      a.slot_next_tok = slot_next_tok;
      a.slot_pos = slot_pos;
      a.slot_done = slot_done;
      a.slot_row = slot_row;
      a.slot_maxnew = slot_maxnew;
      a.out_tokens = job.out_tokens_dev;
      a.out_len = job.out_len_dev;
      a.out_stride = job.max_new_tokens;
      a.mask_bits = has_fsm ? d_mask_bits : nullptr;
      a.mask_words = mask_words;
      a.fsm_trans = d_fsm_trans;
      a.fsm_accept = d_fsm_accept;
      a.fsm_final = d_fsm_final;
      a.fsm_tail_off = has_fsm ? d_tail_off : nullptr;
      a.fsm_tail_tok = d_tail_tok;
      a.tok_bytes = d_tok_bytes;
      a.tok_off = d_tok_off;
      a.eos_id = c.eos_id;
      a.ignore_eos = job.ignore_eos;
      a.temperature = job.temperature > 0.f ? job.temperature : 0.f;
      a.top_k = job.top_k;
      a.top_p = (job.top_p > 0.f && job.top_p < 1.f) ? job.top_p : 1.f;
      a.seed = job.seed;
      a.seed_per_row = job.seed_per_row;
      a.row_ids = job.row_ids_dev;
      a.slot_cum_logprob = job.out_cum_logprob_dev ? slot_cum_logprob : nullptr;
      a.out_cum_logprob = job.out_cum_logprob_dev;
      SB_K(SB200_KC_SAMPLE, sample_greedy(a, stream));
    }
    return 0;
  }

  int upload_fsm(const sb200_job& job) {
    const size_t n = job.fsm_states;
    if (!d_tok_bytes) {
      set_last_error("engine: output_schema given but no vocabulary bytes were set");
      return -1;
    }
    mask_words = (cfg.vocab + 31) / 32;
    if (n > fsm_cap_states) {
      cudaFree(d_fsm_trans);
      cudaFree(d_fsm_accept);
      cudaFree(d_fsm_final);
      cudaFree(d_mask_bits);
      d_fsm_trans = nullptr, d_fsm_accept = nullptr, d_fsm_final = nullptr, d_mask_bits = nullptr;
      fsm_cap_states = 0;
      if (dmalloc(&d_fsm_trans, n * 256) || dmalloc(&d_fsm_accept, n) || dmalloc(&d_fsm_final, n) ||
          dmalloc(&d_mask_bits, n * mask_words))
        return -1;
      fsm_cap_states = n;
    }
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_trans, job.fsm_trans, n * 256 * 4, cudaMemcpyHostToDevice,
                                  stream));
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_accept, job.fsm_accept, n, cudaMemcpyHostToDevice, stream));
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_final, job.fsm_final, n, cudaMemcpyHostToDevice, stream));
    cudaFree(d_tail_off);
    cudaFree(d_tail_tok);
    d_tail_off = nullptr, d_tail_tok = nullptr;
    if (job.fsm_tail_off != nullptr) {
      const size_t nt = job.fsm_tail_off[n];
      if (dmalloc(&d_tail_off, n + 1) || dmalloc(&d_tail_tok, nt > 0 ? nt : 1)) return -1;
      SB_CUDA_CHECK(cudaMemcpyAsync(d_tail_off, job.fsm_tail_off, (n + 1) * 4, cudaMemcpyHostToDevice,
                                    stream));
      if (nt)
        SB_CUDA_CHECK(cudaMemcpyAsync(d_tail_tok, job.fsm_tail_tok, nt * 4, cudaMemcpyHostToDevice,
                                      stream));
    }
    return fsm_build_mask(d_fsm_trans, d_fsm_accept, static_cast<int>(n), d_tok_bytes, d_tok_off,
                          cfg.vocab, cfg.eos_id, d_mask_bits, mask_words, stream);
  }

  int run(const sb200_job& job, sb200_job_stats* stats);
};

// ---------------------------------------------------------------------------
// the scheduling loop
// ---------------------------------------------------------------------------
int Engine::run(const sb200_job& job, sb200_job_stats* stats) {
  const auto& c = cfg;
  const int64_t N = job.n_rows;
  SB_CUDA_CHECK(cudaSetDevice(device));
  prof.reset(job.profile != 0, stream);
  gemm_flops = 0;
  attn_decode_bytes = 0;
  const bool embed_mode = c.embedding_model != 0;
  const bool has_fsm = !embed_mode && job.fsm_states > 0;
  const int max_new = embed_mode ? 0 : job.max_new_tokens;
  if (N <= 0) return 0;
  if (!embed_mode && max_new <= 0) {
    set_last_error("engine: max_new_tokens must be positive");
    return -1;
  }
  if (embed_mode ? job.out_embed_dev == nullptr
                 : (job.out_tokens_dev == nullptr || job.out_len_dev == nullptr)) {
    set_last_error("engine: output buffers missing");
    return -1;
  }
  const int n_prefix = job.n_prefix, n_suffix = job.n_suffix;
  const int n_forced = (has_fsm && job.n_forced_prefix > 0) ? job.n_forced_prefix : 0;
  if (n_forced > n_suffix || (n_forced > 0 && n_forced >= max_new)) {
    set_last_error("engine: forced output prefix (%d tokens) does not fit suffix/max_new_tokens",
                   n_forced);
    return -1;
  }
  const int ctx_budget = c.max_position - max_new;  // prompt tokens that fit
  if (n_prefix + n_suffix + 1 > ctx_budget) {
    set_last_error("engine: system prompt + template (%d tokens) leave no room in the %d-token "
                   "context window", n_prefix + n_suffix, c.max_position);
    return -1;
  }
  // prompt pieces -> device
  if (n_prefix > prefix_cap) {
    cudaFree(d_prefix);
    d_prefix = nullptr;
    if (dmalloc(&d_prefix, static_cast<size_t>(n_prefix))) return -1;
    prefix_cap = n_prefix;
  }
  if (n_suffix > suffix_cap) {
    cudaFree(d_suffix);
    d_suffix = nullptr;
    if (dmalloc(&d_suffix, static_cast<size_t>(n_suffix))) return -1;
    suffix_cap = n_suffix;
  }
  if (n_prefix)
    SB_CUDA_CHECK(cudaMemcpyAsync(d_prefix, job.prefix_tokens, n_prefix * 4ull,
                                  cudaMemcpyHostToDevice, stream));
  if (n_suffix)
    SB_CUDA_CHECK(cudaMemcpyAsync(d_suffix, job.suffix_tokens, n_suffix * 4ull,
                                  cudaMemcpyHostToDevice, stream));
  if (has_fsm && upload_fsm(job)) return -1;
  if (!embed_mode)
    SB_CUDA_CHECK(cudaMemsetAsync(job.out_len_dev, 0, N * sizeof(int32_t), stream));

  // per-row prompt lengths (host)
  const int64_t* roff = job.row_tok_off;
  std::vector<int32_t> n_row_tok(N);
  int64_t n_truncated = 0;
  for (int64_t r = 0; r < N; ++r) {
    int64_t n = roff[r + 1] - roff[r];
    const int64_t room = ctx_budget - n_prefix - n_suffix;
    if (n > room) {
      if (!job.truncate_rows) {
        set_last_error("engine: row %lld has %lld tokens but only %lld fit the context window "
                       "(truncate_rows=False)", (long long)r, (long long)n, (long long)room);
        return -1;
      }
      n = room;
      ++n_truncated;
    }
    n_row_tok[r] = static_cast<int32_t>(n);
  }

  // staging layout (int32 units)
  const int S = c.max_slots;
  const int prefix_slot = S;  // page-table row S holds the shared prefix
  SeqInit* h_seqs = reinterpret_cast<SeqInit*>(h_stage);
  const size_t seq_words = (sizeof(SeqInit) / 4) * (S + 2);
  int32_t* h_pt = h_stage + seq_words;
  int32_t* h_work = h_pt + static_cast<size_t>(S + 2) * max_pages;
  int32_t* h_misc = h_work + 2 * (t_max / 16 + S + 2);  // seq_slot|q_start|q_len|past : 4*(S+2)
  int32_t* h_copy = h_misc + 4 * (S + 2);               // first own page to seed, or -1
  const SeqInit* d_seqs = reinterpret_cast<const SeqInit*>(d_stage);
  const int32_t* d_pt = d_stage + seq_words;
  const int32_t* d_work = d_pt + static_cast<size_t>(S + 2) * max_pages;
  const int32_t* d_misc = d_work + 2 * (t_max / 16 + S + 2);
  const int32_t* d_copy = d_misc + 4 * (S + 2);
  int prefix_tail_page = -1;  // physical page holding the partial tail of the shared prefix

  std::vector<int32_t> prefix_pages;
  std::vector<std::vector<int32_t>> slot_pages(S);
  std::vector<int32_t> free_slots;
  for (int s = S - 1; s >= 0; --s) free_slots.push_back(s);
  std::vector<int32_t> active;  // slots in the decode batch
  std::vector<int32_t> slot_ctx(S, 0);  // host mirror: position of the next fed token

  auto release_all = [&]() {
    for (auto& v : slot_pages) {
      for (int32_t p : v) free_pages.push_back(p);
      v.clear();
    }
    for (int32_t p : prefix_pages) free_pages.push_back(p);
    prefix_pages.clear();
  };

  // every exit path of run() (early error returns included) hands the pages back to the
  // engine-lifetime pool; release_all is idempotent
  struct ReleaseGuard {
    std::function<void()> f;
    ~ReleaseGuard() { f(); }
  } release_guard{release_all};

  // Launch one prefill step for seqs h_seqs[0..n) (page rows in h_pt), T tokens total.
  auto run_prefill = [&](int n, int T, bool sample) -> int {
    int n_work = 0;
    for (int i = 0; i < n; ++i) {
      h_misc[i] = h_seqs[i].slot;
      h_misc[(S + 2) + i] = h_seqs[i].q_start;
      h_misc[2 * (S + 2) + i] = h_seqs[i].q_len;
      h_misc[3 * (S + 2) + i] = h_seqs[i].past;
      for (int t0 = 0; t0 < h_seqs[i].q_len; t0 += q_tile) {
        h_work[2 * n_work] = i;
        h_work[2 * n_work + 1] = t0;
        ++n_work;
      }
    }
    SB_CUDA_CHECK(cudaMemcpyAsync(d_stage, h_stage, stage_cap * 4, cudaMemcpyHostToDevice, stream));
    prof.launches[SB200_KC_OTHER] += 2;
    init_slots_kernel<<<n, 128, 0, stream>>>(d_seqs, d_pt, max_pages, page_table, slot_state,
                                             slot_ngen, slot_pos, slot_done, slot_row, slot_maxnew,
                                             slot_next_tok, d_suffix + (n_suffix - n_forced),
                                             n_forced, embed_mode ? nullptr : job.out_tokens_dev,
                                             embed_mode ? nullptr : job.out_len_dev,
                                             job.max_new_tokens, slot_cum_logprob);
    prefill_prepare_kernel<<<n, 128, 0, stream>>>(d_seqs, d_prefix, n_prefix, d_suffix, n_suffix,
                                                  job.row_tokens_dev, job.row_tok_off_dev, tok_ids,
                                                  tok_pos, tok_slot, last_idx);
    if (prefix_tail_page >= 0 && sample) {
      ++prof.launches[SB200_KC_OTHER];
      copy_prefix_page_kernel<<<dim3(n, c.n_layers), 256, 0, stream>>>(
          kv_pool, layer_stride, kv_page_elems(c.n_kv_heads),
          prefix_tail_page, d_copy);
    }
    SB_CUDA_CHECK(cudaGetLastError());
    if (forward(T, true, d_work, n_work, d_misc + (S + 2), d_misc + 2 * (S + 2),
                d_misc + 3 * (S + 2)))
      return -1;
    if (!sample) return 0;
    if (embed_mode) {
      if (gather_rows(last_idx, x, hl, n, c.d_model, stream)) return -1;
      if (rmsnorm(hl, w.final_norm, hn, n, c.d_model, c.rms_eps, stream)) return -1;
      if (l2_normalize_rows(hn, embed_tmp, n, c.d_model, stream)) return -1;
      scatter_embed_kernel<<<n, 128, 0, stream>>>(embed_tmp, d_seqs, job.out_embed_dev, c.d_model);
      SB_CUDA_CHECK(cudaGetLastError());
      return 0;
    }
    return head_and_sample(n, last_idx, d_misc /* seq_slot */, job, has_fsm, true);
  };

  // ---- shared prefix: compute its KV once, every row's page table points at it ----
  // The whole prefix is computed once; full pages are shared through the page tables and
  // the partially filled last page is copied into each row's first own page.
  const int prefix_cached = (job.share_prefix && n_prefix >= kPageTokens) ? n_prefix : 0;
  if (prefix_cached > 0) {
    if (prefix_cached > c.max_prefill_tokens) {
      set_last_error("engine: shared prefix (%d tokens) exceeds max_prefill_tokens", prefix_cached);
      return -1;
    }
    const int np = (prefix_cached + kPageTokens - 1) / kPageTokens;
    if (static_cast<int64_t>(free_pages.size()) < np) {
      set_last_error("engine: KV pool too small for the shared prefix");
      return -1;
    }
    for (int i = 0; i < np; ++i) {
      prefix_pages.push_back(free_pages.back());
      free_pages.pop_back();
    }
    h_seqs[0] = SeqInit{prefix_slot, -1, 0, prefix_cached, 0, 0, 1, -1};
    std::fill(h_pt, h_pt + max_pages, 0);
    std::copy(prefix_pages.begin(), prefix_pages.end(), h_pt);
    if (prefix_cached > prefix_rows) {
      cudaFree(prefix_kv);
      prefix_kv = nullptr;
      prefix_rows = 0;
      const size_t n = static_cast<size_t>(c.n_layers) * prefix_cached * 2 * c.n_kv_heads * kHeadDim;
      if (dmalloc(&prefix_kv, n)) {
        release_all();
        return -1;
      }
      prefix_rows = prefix_cached;
      cudaMemsetAsync(prefix_kv, 0, n * sizeof(bf16), stream);
    }
    fill_prefix = true;
    const int prc = run_prefill(1, prefix_cached, false);
    fill_prefix = false;
    if (prc) {
      release_all();
      return -1;
    }
    if (prefix_cached % kPageTokens != 0) prefix_tail_page = prefix_pages.back();
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
  }

  int64_t next_row = 0, rows_done = 0, in_tokens = 0, steps_prefill = 0, steps_decode = 0;
  int64_t decode_tokens = 0, prefill_tokens = prefix_cached;
  int rc = 0;

  auto admit = [&]() -> int {  // returns number of rows admitted, <0 on error
    int n = 0, T = 0;
    while (next_row < N && !free_slots.empty() && n < S) {
      const int64_t r = next_row;
      const int P = n_prefix + n_row_tok[r] + n_suffix;
      if (P <= 0) {
        set_last_error("engine: row %lld renders to an empty prompt", (long long)r);
        return -1;
      }
      int past = std::min(prefix_cached, P - 1);
      if (past < prefix_cached) past = (past / kPageTokens) * kPageTokens;  // prompt ends inside the prefix
      const int q_len = P - past;
      if (T + q_len > c.max_prefill_tokens) {
        if (n == 0) {
          set_last_error("engine: row %lld needs %d prefill tokens > max_prefill_tokens=%d",
                         (long long)r, q_len, c.max_prefill_tokens);
          return -1;
        }
        break;
      }
      const int total_pages = (P + max_new + kPageTokens - 1) / kPageTokens;
      const int own = total_pages - past / kPageTokens;
      if (static_cast<int64_t>(free_pages.size()) < own) {
        if (n == 0 && active.empty()) {
          set_last_error("engine: KV pool (%lld pages) cannot hold one row of %d tokens",
                         (long long)num_pages, P + max_new);
          return -1;
        }
        break;
      }
      const int slot = free_slots.back();
      free_slots.pop_back();
      int32_t* pt = h_pt + static_cast<size_t>(n) * max_pages;
      std::fill(pt, pt + max_pages, 0);
      for (int i = 0; i < past / kPageTokens; ++i) pt[i] = prefix_pages[i];
      auto& mine = slot_pages[slot];
      h_copy[n] = -1;
      for (int i = 0; i < own; ++i) {
        mine.push_back(free_pages.back());
        pt[past / kPageTokens + i] = free_pages.back();
        free_pages.pop_back();
      }
      // positions [16*(past/16), past) of the first own page hold prefix tokens: seed them
      if (past % kPageTokens != 0) h_copy[n] = pt[past / kPageTokens];
      h_seqs[n] = SeqInit{slot, static_cast<int32_t>(r), T, q_len, past, n_row_tok[r], max_new,
                          has_fsm ? job.fsm_start : -1};
      slot_ctx[slot] = P;
      T += q_len;
      in_tokens += P;
      ++n;
      ++next_row;
    }
    if (n == 0) return 0;
    if (run_prefill(n, T, true)) return -1;
    prefill_tokens += T;
    ++steps_prefill;
    for (int i = 0; i < n; ++i) active.push_back(h_seqs[i].slot);
    return n;
  };

  auto retire = [&]() -> int {  // reads the done flags, frees finished slots
    SB_CUDA_CHECK(cudaMemcpyAsync(h_done, slot_done, (S + 2) * 4ull, cudaMemcpyDeviceToHost, stream));
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
    size_t k = 0;
    for (size_t i = 0; i < active.size(); ++i) {
      const int s = active[i];
      if (h_done[s]) {
        for (int32_t p : slot_pages[s]) free_pages.push_back(p);
        slot_pages[s].clear();
        free_slots.push_back(s);
        ++rows_done;
      } else {
        active[k++] = s;
      }
    }
    active.resize(k);
    return 0;
  };

  const int min_admit = std::max(1, c.min_admit_rows);
  while (rows_done < N) {
    // ---- admission: refill free slots with new rows (their prefill) ----
    const bool can_admit = next_row < N && !free_slots.empty();
    if (can_admit && (active.empty() || static_cast<int>(free_slots.size()) >= min_admit ||
                      N - next_row <= static_cast<int64_t>(free_slots.size()))) {
      const int n = admit();
      if (n < 0) {
        rc = -1;
        break;
      }
      if (embed_mode) {
        // prefill-only: rows are complete, recycle their slots right away
        SB_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (int s : active) {
          for (int32_t p : slot_pages[s]) free_pages.push_back(p);
          slot_pages[s].clear();
          free_slots.push_back(s);
          ++rows_done;
        }
        active.clear();
        if (job.progress) job.progress(rows_done, in_tokens, 0, job.progress_user);
        continue;
      }
      if (n > 0) {
        if (retire()) {
          rc = -1;
          break;
        }
        if (job.progress) job.progress(rows_done, in_tokens, decode_tokens, job.progress_user);
        continue;  // try to admit more before decoding
      }
    }
    if (active.empty()) {
      if (next_row >= N) break;
      set_last_error("engine: scheduler stalled (no active rows, none admissible)");
      rc = -1;
      break;
    }
    // ---- one decode step over all active rows ----
    const int B = static_cast<int>(active.size());
    std::copy(active.begin(), active.end(), h_misc);
    SB_CUDA_CHECK(cudaMemcpyAsync(row_slot, h_misc, B * 4ull, cudaMemcpyHostToDevice, stream));
    prof.begin(SB200_KC_OTHER);
    const int prc = prepare_decode(row_slot, slot_next_tok, slot_pos, tok_ids, tok_pos, tok_slot,
                                   ctx_len, B, stream);
    prof.end();
    if (prc || forward(B, false, nullptr, 0, nullptr, nullptr, nullptr) ||
        head_and_sample(B, nullptr, row_slot, job, has_fsm)) {
      rc = -1;
      break;
    }
    decode_tokens += B;
    ++steps_decode;
    {
      int64_t ctx_sum = 0;
      for (int s : active) ctx_sum += ++slot_ctx[s];
      attn_decode_bytes += static_cast<double>(ctx_sum) * c.n_layers * c.n_kv_heads * 2.0 *
                           kHeadDim * 2.0;
    }
    if (retire()) {
      rc = -1;
      break;
    }
    if (job.progress && (steps_decode % 8 == 0 || rows_done == N))
      job.progress(rows_done, in_tokens, decode_tokens, job.progress_user);
  }
  cudaStreamSynchronize(stream);
  release_all();
  prof.resolve();
  if (stats) {
    for (int i = 0; i < SB200_KC_COUNT; ++i) {
      stats->kernel_ms[i] = prof.ms[i];
      stats->kernel_launches[i] = prof.launches[i];
    }
    stats->gemm_flops = gemm_flops;
    stats->attn_decode_bytes = attn_decode_bytes;
    stats->rows_done = rows_done;
    stats->input_tokens = in_tokens;
    stats->prefill_tokens = prefill_tokens;
    stats->decode_tokens = decode_tokens;
    stats->prefill_steps = steps_prefill;
    stats->decode_steps = steps_decode;
    stats->rows_truncated = n_truncated;
    stats->prefix_cached_tokens = prefix_cached;
  }
  if (rc == 0) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      set_last_error("engine: CUDA error after run: %s", cudaGetErrorString(e));
      rc = -1;
    }
  }
  return rc;
}

}  // namespace sb

// ---------------------------------------------------------------------------
// C-ABI
// ---------------------------------------------------------------------------
using namespace sb;

extern "C" {

int sb200_engine_create(const sb200_engine_config* cfg, const sb200_engine_weights* w, void** out) {
  *out = nullptr;
  if (!cfg || !w) {
    set_last_error("engine_create: null config/weights");
    return -1;
  }
  if (cfg->n_q_heads % cfg->n_kv_heads != 0 || cfg->d_model % 64 != 0 || cfg->d_ff % 64 != 0 ||
      cfg->vocab % 32 != 0 || cfg->max_slots <= 0 || cfg->max_prefill_tokens < 16 ||
      cfg->num_pages <= 0) {
    set_last_error("engine_create: unsupported geometry (d_model/d_ff %% 64, vocab %% 32, ...)");
    return -1;
  }
  auto* e = new Engine();
  e->cfg = *cfg;
  e->w = *w;
  const int L = cfg->n_layers;
  auto cp = [&](std::vector<const void*>& v, const void* const* src) {
    v.assign(L, nullptr);
    if (src)
      for (int i = 0; i < L; ++i) v[i] = src[i];
  };
  cp(e->ln1, w->ln1);
  cp(e->ln2, w->ln2);
  cp(e->wqkv, w->wqkv);
  cp(e->wo, w->wo);
  cp(e->wgu, w->wgu);
  cp(e->wd, w->wd);
  cp(e->qn, cfg->qk_norm ? w->q_norm : nullptr);
  cp(e->kn, cfg->qk_norm ? w->k_norm : nullptr);
  for (int i = 0; i < L; ++i) {
    if (!e->ln1[i] || !e->ln2[i] || !e->wqkv[i] || !e->wo[i] || !e->wgu[i] || !e->wd[i] ||
        (cfg->qk_norm && (!e->qn[i] || !e->kn[i]))) {
      set_last_error("engine_create: missing weight pointer in layer %d", i);
      delete e;
      return -1;
    }
  }
  if (e->init()) {
    delete e;
    return -1;
  }
  *out = e;
  return 0;
}

void sb200_engine_destroy(void* engine) { delete static_cast<Engine*>(engine); }

int sb200_engine_set_vocab(void* engine, const uint8_t* tok_bytes, const int32_t* tok_off) {
  auto* e = static_cast<Engine*>(engine);
  SB_CUDA_CHECK(cudaSetDevice(e->device));
  const int V = e->cfg.vocab;
  cudaFree(e->d_tok_bytes);
  cudaFree(e->d_tok_off);
  e->d_tok_bytes = nullptr, e->d_tok_off = nullptr;
  const size_t nb = tok_off[V] > 0 ? tok_off[V] : 1;
  SB_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&e->d_tok_bytes), nb));
  SB_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&e->d_tok_off), (V + 1) * 4ull));
  SB_CUDA_CHECK(cudaMemcpy(e->d_tok_bytes, tok_bytes, tok_off[V], cudaMemcpyHostToDevice));
  SB_CUDA_CHECK(cudaMemcpy(e->d_tok_off, tok_off, (V + 1) * 4ull, cudaMemcpyHostToDevice));
  return 0;
}

int sb200_engine_run(void* engine, const sb200_job* job, sb200_job_stats* stats) {
  if (!engine || !job) {
    set_last_error("engine_run: null argument");
    return -1;
  }
  return static_cast<Engine*>(engine)->run(*job, stats);
}

void* sb200_engine_stream(void* engine) { return static_cast<Engine*>(engine)->stream; }

int sb200_engine_info(void* engine, int* device, int* embedding_model, int* d_model, int* vocab) {
  if (!engine) {
    set_last_error("engine_info: null engine");
    return -1;
  }
  const auto* e = static_cast<const Engine*>(engine);
  if (device) *device = e->device;
  if (embedding_model) *embedding_model = e->cfg.embedding_model;
  if (d_model) *d_model = e->cfg.d_model;
  if (vocab) *vocab = e->cfg.vocab;
  return 0;
}

}  // extern "C"
