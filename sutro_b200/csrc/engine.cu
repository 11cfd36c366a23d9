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
// chunk, the page table and the per-slot decode state; the split-KV decode
// workspace grows with the longest rows a decode step has seen.
#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "../../include/sutro_b200.h"
#include "common.cuh"
#include "dev_buf.h"
#include "kernels.h"

namespace sb {

namespace {

using bf16 = __nv_bfloat16;

// ---- small device helpers owned by the engine -----------------------------
struct SeqInit {  // one sequence of a prefill step: a row, or one chunk of a row
  int32_t slot, row, q_start, q_len, past, n_row_tok, max_new, fsm_start;
  int32_t hist;   // own tokens prefilled by earlier chunks: this step feeds [hist, hist + q_len)
  int32_t n_own;  // the row's own tokens in all (prompt - past); hist + q_len == n_own: last chunk
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
    const int p = s.past + s.hist + j;
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
                  int pt_cols, int max_pages, int32_t* __restrict__ page_table,
                  int32_t* slot_state, int32_t* slot_ngen, int32_t* slot_pos, int32_t* slot_done,
                  int32_t* slot_row, int32_t* slot_maxnew, int32_t* slot_next_tok, const int32_t* __restrict__ forced,
                  int n_forced, int32_t* __restrict__ out_tokens, int32_t* __restrict__ out_len,
                  int out_stride, float* __restrict__ slot_cum_logprob,
                  int32_t* __restrict__ slot_n_row_tok) {
  const SeqInit s = seqs[blockIdx.x];
  if (s.hist > 0) return;  // a later chunk: its row was installed with its first chunk
  // the first pt_cols entries: every page the row reserved; nothing reads the entries past them
  for (int i = threadIdx.x; i < pt_cols; i += blockDim.x)
    page_table[static_cast<size_t>(s.slot) * max_pages + i] =
        pt_rows[static_cast<size_t>(blockIdx.x) * pt_cols + i];
  // jump-forward: the forced output prefix was fed with the prompt; it is output too
  if (s.row >= 0 && out_tokens != nullptr)
    for (int i = threadIdx.x; i < n_forced; i += blockDim.x)
      out_tokens[static_cast<size_t>(s.row) * out_stride + i] = forced[i];
  if (threadIdx.x == 0) {
    if (s.row >= 0 && out_len != nullptr) out_len[s.row] = n_forced;
    slot_state[s.slot] = s.fsm_start;
    slot_ngen[s.slot] = s.row >= 0 ? n_forced : 0;
    slot_pos[s.slot] = s.past + s.n_own - 1;  // sampler increments: next position = prompt length
    slot_done[s.slot] = 0;
    slot_row[s.slot] = s.row;
    slot_maxnew[s.slot] = s.max_new;
    slot_next_tok[s.slot] = 0;
    slot_cum_logprob[s.slot] = 0.f;
    slot_n_row_tok[s.slot] = s.n_row_tok;  // the row's share of the prompt (penalties)
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

// The prefill staging buffer: what one prefill step builds on the host, uploaded in one copy.
// Its sections follow each other in the order of View's fields; offsets count int32 words.
struct StageLayout {
  struct View {     // the sections of one buffer, host or device
    SeqInit* seqs;  // [n_seqs]
    int32_t* pt;    // [n_seqs][pt_cols] page-table rows: the pages the rows reserved
    int32_t* work;  // [n_work][2] {sequence, first query token}: dense prefill attention items
    int32_t *slot, *q_start, *q_len, *past, *hist;  // [n_seqs] each: that attention's arrays
    int32_t* copy;  // [n_seqs] page to seed with the shared prefix's partial last page, or -1
  };
  size_t pt, work, slot, q_start, q_len, past, hist, copy, words;  // offsets, and the total

  StageLayout(size_t n_seqs, size_t n_work, size_t pt_cols)
      : pt(n_seqs * (sizeof(SeqInit) / 4)),
        work(pt + n_seqs * pt_cols),
        slot(work + 2 * n_work),
        q_start(slot + n_seqs),
        q_len(q_start + n_seqs),
        past(q_len + n_seqs),
        hist(past + n_seqs),
        copy(hist + n_seqs),
        words(copy + n_seqs) {}
  View at(int32_t* base) const {
    return {reinterpret_cast<SeqInit*>(base), base + pt,   base + work,
            base + slot,                      base + q_start, base + q_len,
            base + past,                      base + hist, base + copy};
  }
};
static_assert(sizeof(SeqInit) % 4 == 0, "SeqInit records are staged as int32 words");

// What forward() needs of a prefill step (device pointers into the staging buffer).  The first
// n_final sequences end their prompt in this step, and their work items come first; a sequence
// after them is a row's non-final chunk, which needs no last-layer attention or O/MLP.
struct PrefillStep {
  const int32_t* work;  // work items of the prefill attention
  int n_work, n_work_final;
  int n_seqs, n_final;
  const int32_t *slot, *q_start, *q_len, *past;  // per sequence
  const int32_t* hist;  // per sequence, or nullptr when no sequence has history in the pool
  bool keep_prefix;  // this pass is the shared prefix's: keep its K/V in prefix_kv
};

// What forward() needs of a decode step whose rows may exceed kDecodeSplitTokens: the batch rows
// that may (device), and the most splits any of them has.  n_rows == 0: no row is split.
struct DecodeSplit {
  const int32_t* rows;
  int n_rows, max_splits;
};

}  // namespace

struct Engine {
  sb200_engine_config cfg{};
  sb200_engine_weights w{};
  std::vector<const void*> ln1, ln2, wqkv, wo, wgu, wd, qn, kn;
  cudaStream_t stream = nullptr;
  int qkv_dim = 0, q_dim = 0, max_pages = 0, t_max = 0, logit_rows = 0, q_tile = 0;
  int chunk_tokens = 0;  // prefill chunk of a row longer than max_prefill_tokens (0: none fits)
  int64_t num_pages = 0;
  size_t layer_stride = 0;  // elements between consecutive layers in the KV pool

  DevArray<bf16> x, h, qkv, attn, act, hl, hn, kv_pool;
  DevArray<float> logits, embed_tmp;
  DevArray<int32_t> tok_ids, tok_pos, tok_slot, ctx_len, row_slot, last_idx, page_table;
  DevArray<int32_t> slot_state, slot_ngen, slot_next_tok, slot_pos, slot_done, slot_row,
      slot_maxnew, slot_n_row_tok;
  DevArray<float> slot_cum_logprob;
  DevArray<int32_t> split_rows;  // a decode step's rows longer than kDecodeSplitTokens
  DevArray<float> split_ws;      // their split-KV partials (attn_decode_ws_floats), grow-only
  // Staging: a prefill step's StageLayout, or a decode step's row_slot.  The host buffer is
  // written only after the stream has been synchronised since its previous copy was enqueued:
  // every step that copies it is followed by a synchronise (JobRun::retire, or the one after
  // the shared prefix's pass) before the next step writes it.
  int32_t* h_stage = nullptr;  // pinned
  DevArray<int32_t> d_stage;
  int32_t* h_done = nullptr;  // pinned
  // vocabulary bytes + FSM tables
  DevArray<uint8_t> d_tok_bytes;
  DevArray<int32_t> d_tok_off, d_fsm_trans;
  DevArray<uint8_t> d_fsm_accept, d_fsm_final;
  DevArray<uint32_t> d_mask_bits;
  DevArray<int32_t> d_tail_off, d_tail_tok;  // jump-forward terminal tails
  int mask_words = 0;
  // job-scoped prompt pieces
  DevArray<int32_t> d_prefix, d_suffix;
  // host page allocator
  std::vector<int32_t> free_pages;
  Profiler prof;
  double gemm_flops = 0;
  int device = 0;
  DevArray<bf16> prefix_kv;  // [n_layers][prefix_rows][2*hkv*128]: dense K|V of the shared prefix
  int prefix_rows = 0;

  ~Engine() {
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
    if (q_tile <= 0) {
      set_last_error("engine_create: GQA group %d is too large", c.n_q_heads / c.n_kv_heads);
      return -1;
    }
    const int align = attn_prefill_hist_align(c.n_q_heads, c.n_kv_heads);
    chunk_tokens = align > 0 ? c.max_prefill_tokens / align * align : 0;
    num_pages = c.num_pages;
    layer_stride = num_pages * kv_page_elems(c.n_kv_heads);
    SB_CUDA_CHECK(cudaGetDevice(&device));
    SB_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    const size_t T = t_max, S = c.max_slots + 2;  // +prefix slot, +dummy slot
    if (x.alloc(T * c.d_model) || h.alloc(T * c.d_model) || qkv.alloc(T * qkv_dim) ||
        attn.alloc(T * q_dim) || act.alloc(T * c.d_ff) ||
        hl.alloc(static_cast<size_t>(c.max_slots) * c.d_model) ||
        hn.alloc(static_cast<size_t>(c.max_slots) * c.d_model) ||
        kv_pool.alloc(layer_stride * c.n_layers) ||
        tok_ids.alloc(T) || tok_pos.alloc(T) || tok_slot.alloc(T) ||
        ctx_len.alloc(S) || row_slot.alloc(S) || last_idx.alloc(S) ||
        page_table.alloc(S * max_pages) || slot_state.alloc(S) || slot_ngen.alloc(S) ||
        slot_next_tok.alloc(S) || slot_pos.alloc(S) || slot_done.alloc(S) ||
        slot_row.alloc(S) || slot_maxnew.alloc(S) || slot_cum_logprob.alloc(S) ||
        slot_n_row_tok.alloc(S) || split_rows.alloc(S))
      return -1;
    if (c.embedding_model) {
      if (embed_tmp.alloc(static_cast<size_t>(c.max_slots) * c.d_model)) return -1;
    } else {
      if (logits.alloc(static_cast<size_t>(logit_rows) * c.vocab)) return -1;
    }
    // K/V tiles must hold finite values everywhere (masked P * V must stay 0); the same goes
    // for the k/v columns of the qkv buffer, which the dense prefill attention reads in
    // 32-row boxes that may run past the end of a sequence.
    SB_CUDA_CHECK(cudaMemsetAsync(kv_pool, 0, layer_stride * c.n_layers * sizeof(bf16), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(qkv, 0, T * qkv_dim * sizeof(bf16), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(page_table, 0, S * max_pages * sizeof(int32_t), stream));
    SB_CUDA_CHECK(cudaMemsetAsync(slot_done, 0, S * sizeof(int32_t), stream));
    // A prefill step has at most max_slots sequences and t_max tokens; a sequence of q_len
    // tokens has ceil(q_len / q_tile) work items, so the step has at most t_max / q_tile +
    // max_slots of them.
    const size_t stage_words =
        StageLayout(c.max_slots, t_max / q_tile + c.max_slots, max_pages).words;
    SB_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&h_stage), stage_words * 4));
    if (d_stage.alloc(stage_words)) return -1;
    SB_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void**>(&h_done), S * 4));
    free_pages.reserve(num_pages);
    for (int64_t p = num_pages - 1; p >= 0; --p) free_pages.push_back(static_cast<int32_t>(p));
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
    return 0;
  }

  // Every GEMM of the stack and of the LM head: adds its FLOPs to the job's count and launches.
  int gemm(const void* a, int a_rows, const void* wt, void* d, const void* r, int M, int N, int K,
           int ldd, int epi, const QkvEpiArgs* qa = nullptr) {
    gemm_flops += 2.0 * M * N * K;
    return gemm_bf16_tn(a, a_rows, wt, d, r, M, N, K, ldd, epi, 0, stream, qa);
  }

  // O (+ residual), RMSNorm, gate/up (SwiGLU) and down (+ residual) of layer l over M rows:
  // a [M, q_dim] and the residual stream in [M, d_model] rows of x_in -> x_out (may alias).
  int layer_tail(int l, const bf16* a, int a_rows, bf16* x_in, bf16* x_out, int M) {
    const auto& c = cfg;
    SB_K(SB200_KC_GEMM, gemm(a, a_rows, wo[l], x_in, x_in, M, c.d_model, q_dim, c.d_model,
                             EPI_RESIDUAL_BF16));
    SB_K(SB200_KC_NORM, rmsnorm(x_in, ln2[l], h, M, c.d_model, c.rms_eps, stream));
    SB_K(SB200_KC_GEMM, gemm(h, t_max, wgu[l], act, nullptr, M, 2 * c.d_ff, c.d_model, c.d_ff,
                             EPI_SWIGLU_BF16));
    SB_K(SB200_KC_GEMM, gemm(act, t_max, wd[l], x_out, x_in, M, c.d_model, c.d_ff, c.d_model,
                             EPI_RESIDUAL_BF16));
    return 0;
  }

  // ---- one pass of the transformer stack over T flattened tokens -----------
  // prefill (pf != nullptr): attention over (cached prefix | new tokens) per sequence;
  // decode (pf == nullptr): one token per sequence against its paged history.
  // Leaves the hidden state of the rows the head reads in rows [0, n) of x: decode's T rows,
  // or each prefill sequence's last token.  Every layer's K/V covers all T tokens, but nothing
  // reads the last layer's O/MLP output of a prefill token that is not its sequence's last, so
  // that layer's tail runs on the last tokens only (rows do not depend on M: exact), and not
  // at all in the shared prefix's pass, which has no head.
  int forward(int T, const PrefillStep* pf, const DecodeSplit& ds = DecodeSplit{nullptr, 0, 1}) {
    const auto& c = cfg;
    const float scale = 1.0f / sqrtf(static_cast<float>(kHeadDim));
    SB_K(SB200_KC_EMBED, embed_gather(tok_ids, w.embed, x, T, c.d_model, stream));
    for (int l = 0; l < c.n_layers; ++l) {
      SB_K(SB200_KC_NORM, rmsnorm(x, ln1[l], h, T, c.d_model, c.rms_eps, stream));
      // K1+K5 fused: q/k-norm, RoPE and the paged K/V write happen in the GEMM epilogue; in
      // prefill it also leaves K/V in their qkv columns for the dense prefill attention
      QkvEpiArgs qa{tok_pos, tok_slot, page_table, max_pages, kv_layer(l), w.rope_cos,
                    w.rope_sin, qn[l], kn[l], c.n_q_heads, c.n_kv_heads, c.rms_eps,
                    pf ? 1 : 0};
      SB_K(SB200_KC_GEMM, gemm(h, t_max, wqkv[l], qkv, nullptr, T, qkv_dim, c.d_model, qkv_dim,
                               EPI_QKV_ROPE, &qa));
      if (pf && pf->keep_prefix) {
        // the shared prefix's K/V (k|v columns of its rows) go to the dense side buffer
        const size_t cols = 2ull * c.n_kv_heads * kHeadDim;
        SB_CUDA_CHECK(cudaMemcpy2DAsync(prefix_kv + static_cast<size_t>(l) * prefix_rows * cols,
                                        cols * sizeof(bf16), qkv + q_dim, qkv_dim * sizeof(bf16),
                                        cols * sizeof(bf16), T, cudaMemcpyDeviceToDevice, stream));
      }
      if (pf) {
        const int nw = l + 1 < c.n_layers ? pf->n_work : pf->n_work_final;
        if (nw > 0 && !pf->hist)
          SB_K(SB200_KC_ATTN_PREFILL,
               attn_prefill_dense(qkv, t_max, attn, prefix_kv, prefix_rows, c.n_layers, l,
                                  pf->work, nw, pf->q_start, pf->q_len, pf->past, c.n_q_heads,
                                  c.n_kv_heads, scale, stream));
        else if (nw > 0)
          SB_K(SB200_KC_ATTN_PREFILL,
               attn_prefill_chunked(qkv, t_max, attn, prefix_kv, prefix_rows, c.n_layers, l,
                                    pf->work, nw, pf->q_start, pf->q_len, pf->past, c.n_q_heads,
                                    c.n_kv_heads, scale, kv_layer(l), page_table, max_pages,
                                    pf->slot, pf->hist, stream));
      } else {
        SB_K(SB200_KC_ATTN_DECODE,
             attn_decode(qkv, attn, kv_layer(l), page_table, max_pages, row_slot, ctx_len, T,
                         c.n_q_heads, c.n_kv_heads, scale, ds.rows, ds.n_rows, ds.max_splits,
                         split_ws, stream));
        if (ds.n_rows > 0) ++prof.launches[SB200_KC_ATTN_DECODE];  // the split merge
      }
      if (!pf || l + 1 < c.n_layers) {
        if (layer_tail(l, attn, t_max, x, x, T)) return -1;
      } else if (!pf->keep_prefix && pf->n_final > 0) {
        // last tokens: attention rows -> the dead qkv buffer (wider than attn: they fit),
        // residual rows -> hl; the down GEMM writes the result to rows [0, n) of x
        const int n = pf->n_final;
        SB_K(SB200_KC_EMBED, gather_rows(last_idx, attn, qkv, n, q_dim, stream));
        SB_K(SB200_KC_EMBED, gather_rows(last_idx, x, hl, n, c.d_model, stream));
        if (layer_tail(l, qkv, n, hl, x, n)) return -1;
      }
    }
    return 0;
  }

  // final norm + lm_head + masked greedy sampling for the `n` rows [0, n) of x
  int head_and_sample(int n, const int32_t* d_row_slot, const sb200_job& job, bool has_fsm,
                      bool first_decision = false) {
    const auto& c = cfg;
    SB_K(SB200_KC_NORM, rmsnorm(x, w.final_norm, hn, n, c.d_model, c.rms_eps, stream));
    const bool has_tails = has_fsm && job.fsm_tail_off != nullptr;
    for (int r0 = 0; r0 < n; r0 += logit_rows) {
      const int nr = std::min(logit_rows, n - r0);
      SB_K(SB200_KC_GEMM, gemm(hn + static_cast<size_t>(r0) * c.d_model, c.max_slots - r0,
                               w.lm_head, logits, nullptr, nr, c.vocab, c.d_model, c.vocab,
                               EPI_STORE_F32));
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
      a.mask_bits = has_fsm ? d_mask_bits.get() : nullptr;
      a.mask_words = mask_words;
      a.fsm_trans = d_fsm_trans;
      a.fsm_accept = d_fsm_accept;
      a.fsm_final = d_fsm_final;
      // the tail buffers outlive the job that uploaded them: only this job's are passed
      a.fsm_tail_off = has_tails ? d_tail_off.get() : nullptr;
      a.fsm_tail_tok = has_tails ? d_tail_tok.get() : nullptr;
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
      a.slot_cum_logprob = job.out_cum_logprob_dev ? slot_cum_logprob.get() : nullptr;
      a.out_cum_logprob = job.out_cum_logprob_dev;
      // penalties over prefix | row tokens after truncation | suffix and the row's output
      a.prompt_prefix = d_prefix;
      a.n_prompt_prefix = job.n_prefix;
      a.prompt_suffix = d_suffix;
      a.n_prompt_suffix = job.n_suffix;
      a.row_tokens = job.row_tokens_dev;
      a.row_tok_off = job.row_tok_off_dev;
      a.slot_n_row_tok = slot_n_row_tok;
      a.presence_penalty = job.presence_penalty;
      a.frequency_penalty = job.frequency_penalty;
      a.repetition_penalty = job.repetition_penalty;
      a.min_p = job.min_p;
      if (penalties_active(a)) ++prof.launches[SB200_KC_SAMPLE];  // the penalty kernel
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
    if (d_fsm_trans.reserve(n * 256) || d_fsm_accept.reserve(n) || d_fsm_final.reserve(n) ||
        d_mask_bits.reserve(n * mask_words))
      return -1;
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_trans, job.fsm_trans, n * 256 * 4, cudaMemcpyHostToDevice,
                                  stream));
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_accept, job.fsm_accept, n, cudaMemcpyHostToDevice, stream));
    SB_CUDA_CHECK(cudaMemcpyAsync(d_fsm_final, job.fsm_final, n, cudaMemcpyHostToDevice, stream));
    if (job.fsm_tail_off != nullptr) {
      const size_t nt = job.fsm_tail_off[n];
      if (d_tail_off.reserve(n + 1) || d_tail_tok.reserve(nt > 0 ? nt : 1)) return -1;
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

namespace {

// The parameters of one job, checked before anything is uploaded.
struct JobSpec {
  bool embed_mode = false, has_fsm = false;
  int max_new = 0, n_prefix = 0, n_suffix = 0, n_forced = 0;
  int prefix_cached = 0;           // prefix tokens whose K/V are computed once for every row
  std::vector<int32_t> n_row_tok;  // prompt tokens of each row, after truncation
  int64_t n_truncated = 0;
};

int validate_job(const sb200_engine_config& c, const sb200_job& job, JobSpec& s) {
  s.embed_mode = c.embedding_model != 0;
  s.has_fsm = !s.embed_mode && job.fsm_states > 0;
  s.max_new = s.embed_mode ? 0 : job.max_new_tokens;
  if (!s.embed_mode && s.max_new <= 0) {
    set_last_error("engine: max_new_tokens must be positive");
    return -1;
  }
  if (s.embed_mode ? job.out_embed_dev == nullptr
                   : (job.out_tokens_dev == nullptr || job.out_len_dev == nullptr)) {
    set_last_error("engine: output buffers missing");
    return -1;
  }
  if (!s.embed_mode) {
    const bool penalised = job.presence_penalty != 0.f || job.frequency_penalty != 0.f ||
                           (job.repetition_penalty > 0.f && job.repetition_penalty != 1.f);
    if (penalised && s.max_new > kPenaltyMaxOutput) {
      set_last_error("engine: presence/frequency/repetition penalties support max_new_tokens <= "
                     "%d (got %d)", kPenaltyMaxOutput, s.max_new);
      return -1;
    }
    if (!(job.min_p <= 1.f) || !(job.presence_penalty == job.presence_penalty) ||
        !(job.frequency_penalty == job.frequency_penalty) ||
        !(job.repetition_penalty == job.repetition_penalty)) {
      set_last_error("engine: min_p must be in [0, 1] and the penalties must be numbers");
      return -1;
    }
  }
  s.n_prefix = job.n_prefix;
  s.n_suffix = job.n_suffix;
  s.n_forced = (s.has_fsm && job.n_forced_prefix > 0) ? job.n_forced_prefix : 0;
  if (s.n_forced > s.n_suffix || (s.n_forced > 0 && s.n_forced >= s.max_new)) {
    set_last_error("engine: forced output prefix (%d tokens) does not fit suffix/max_new_tokens",
                   s.n_forced);
    return -1;
  }
  const int ctx_budget = c.max_position - s.max_new;  // prompt tokens that fit
  if (s.n_prefix + s.n_suffix + 1 > ctx_budget) {
    set_last_error("engine: system prompt + template (%d tokens) leave no room in the %d-token "
                   "context window", s.n_prefix + s.n_suffix, c.max_position);
    return -1;
  }
  const int64_t room = ctx_budget - s.n_prefix - s.n_suffix;
  s.n_row_tok.resize(job.n_rows);
  for (int64_t r = 0; r < job.n_rows; ++r) {
    int64_t n = job.row_tok_off[r + 1] - job.row_tok_off[r];
    if (n > room) {
      if (!job.truncate_rows) {
        set_last_error("engine: row %lld has %lld tokens but only %lld fit the context window "
                       "(truncate_rows=False)", (long long)r, (long long)n, (long long)room);
        return -1;
      }
      n = room;
      ++s.n_truncated;
    }
    s.n_row_tok[r] = static_cast<int32_t>(n);
  }
  s.prefix_cached = (job.share_prefix && s.n_prefix >= kPageTokens) ? s.n_prefix : 0;
  if (s.prefix_cached > c.max_prefill_tokens) {
    set_last_error("engine: shared prefix (%d tokens) exceeds max_prefill_tokens", s.prefix_cached);
    return -1;
  }
  return 0;
}

// One sb200_engine_run call: the checked job, the host bookkeeping of its slots and pages, its
// counters, and one method per scheduling step.  Destroying it hands the job's pages back to the
// engine's pool, however the run ends.
struct JobRun {
  Engine& e;
  const sb200_job& job;
  const JobSpec p;
  const int S;  // decode slots; slot S (page-table row S) holds the shared prefix
  std::vector<std::vector<int32_t>> slot_pages;  // [S + 1] pages owned by each slot
  std::vector<int32_t> free_slots;
  std::vector<int32_t> active;    // slots in the decode batch
  std::vector<int32_t> slot_ctx;  // host mirror: position of the next fed token
  std::vector<SeqInit> batch;     // the sequences of the next prefill step
  SeqInit chunked{};              // the row being prefilled in chunks (slot -1: none); its hist
                                  // is the first own token of its next chunk
  int prefix_tail_page = -1;      // physical page holding the partial tail of the shared prefix
  int64_t next_row = 0, rows_done = 0, in_tokens = 0, prefill_tokens = 0, decode_tokens = 0;
  int64_t steps_prefill = 0, steps_decode = 0;
  double attn_decode_bytes = 0;

  JobRun(Engine& engine, const sb200_job& j, JobSpec spec)
      : e(engine), job(j), p(std::move(spec)), S(engine.cfg.max_slots), slot_pages(S + 1),
        slot_ctx(S, 0) {
    for (int s = S - 1; s >= 0; --s) free_slots.push_back(s);
    chunked.slot = -1;
  }
  ~JobRun() {
    for (const auto& v : slot_pages) e.free_pages.insert(e.free_pages.end(), v.begin(), v.end());
  }

  // The shared prefix is prefilled once: its full pages are shared through the page tables,
  // its partially filled last page is copied into each row's first own page.
  int cache_prefix() {
    const int n = p.prefix_cached;
    if (n == 0) return 0;
    const int np = (n + kPageTokens - 1) / kPageTokens;
    if (static_cast<int64_t>(e.free_pages.size()) < np) {
      set_last_error("engine: KV pool too small for the shared prefix");
      return -1;
    }
    std::vector<int32_t>& pages = slot_pages[S];
    for (int i = 0; i < np; ++i) {
      pages.push_back(e.free_pages.back());
      e.free_pages.pop_back();
    }
    if (n > e.prefix_rows) {
      const size_t elems =
          static_cast<size_t>(e.cfg.n_layers) * n * 2 * e.cfg.n_kv_heads * kHeadDim;
      e.prefix_rows = 0;
      if (e.prefix_kv.alloc(elems)) return -1;
      e.prefix_rows = n;
      cudaMemsetAsync(e.prefix_kv, 0, elems * sizeof(bf16), e.stream);
    }
    batch.assign(1, SeqInit{S, -1, 0, n, 0, 0, 1, -1, 0, n});
    if (prefill(n, true)) return -1;
    if (n % kPageTokens != 0) prefix_tail_page = pages.back();
    prefill_tokens = n;
    SB_CUDA_CHECK(cudaStreamSynchronize(e.stream));
    return 0;
  }

  // Takes rows in order while a slot, the prefill budget and the KV pool allow, reserves each
  // row's pages up front and runs their prefill step.  A row whose new tokens exceed the budget is
  // prefilled in chunks of e.chunk_tokens, one row at a time: each step carries its next chunk
  // first, and new rows fill the rest of the budget.  Returns the sequences prefilled, or -1.
  int admit() {
    const auto& c = e.cfg;
    batch.clear();
    int T = 0;
    SeqInit held{};  // the in-flight row's next chunk, when it is not its last
    held.slot = -1;
    if (chunked.slot >= 0) {
      SeqInit x = chunked;
      x.q_start = 0;
      x.q_len = std::min(e.chunk_tokens, x.n_own - x.hist);
      T = x.q_len;
      if (x.hist + x.q_len == x.n_own) {
        batch.push_back(x);
        chunked.slot = -1;
      } else {
        held = x;
        chunked.hist += x.q_len;
      }
    }
    while (next_row < job.n_rows && !free_slots.empty() &&
           static_cast<int>(batch.size()) + (held.slot >= 0) < S) {
      const int64_t r = next_row;
      const int P = p.n_prefix + p.n_row_tok[r] + p.n_suffix;
      if (P <= 0) {
        set_last_error("engine: row %lld renders to an empty prompt", (long long)r);
        return -1;
      }
      int past = std::min(p.prefix_cached, P - 1);
      // the prompt ends inside the prefix
      if (past < p.prefix_cached) past = (past / kPageTokens) * kPageTokens;
      const int q_len = P - past;
      const bool chunks = q_len > c.max_prefill_tokens;
      if (chunks && e.chunk_tokens <= 0) {
        set_last_error("engine: row %lld needs %d prefill tokens > max_prefill_tokens=%d, and "
                       "longer rows are prefilled in chunks of a multiple of %d tokens",
                       (long long)r, q_len, c.max_prefill_tokens,
                       attn_prefill_hist_align(c.n_q_heads, c.n_kv_heads));
        return -1;
      }
      const int first = chunks ? e.chunk_tokens : q_len;
      if (T + first > c.max_prefill_tokens || (chunks && (held.slot >= 0 || chunked.slot >= 0)))
        break;
      const int total_pages = (P + p.max_new + kPageTokens - 1) / kPageTokens;
      const int own = total_pages - past / kPageTokens;
      if (static_cast<int64_t>(e.free_pages.size()) < own) {
        if (batch.empty() && active.empty() && held.slot < 0) {
          set_last_error("engine: KV pool (%lld pages) cannot hold one row of %d tokens",
                         (long long)e.num_pages, P + p.max_new);
          return -1;
        }
        break;
      }
      const int slot = free_slots.back();
      free_slots.pop_back();
      for (int i = 0; i < own; ++i) {
        slot_pages[slot].push_back(e.free_pages.back());
        e.free_pages.pop_back();
      }
      const SeqInit x{slot, static_cast<int32_t>(r), T, first, past, p.n_row_tok[r],
                      p.max_new, p.has_fsm ? job.fsm_start : -1, 0, q_len};
      slot_ctx[slot] = P;
      T += first;
      in_tokens += P;
      ++next_row;
      if (chunks) {
        held = x;
        chunked = x;
        chunked.hist = first;
        break;  // the non-final chunk is the step's last sequence
      }
      batch.push_back(x);
    }
    if (held.slot >= 0) batch.push_back(held);
    if (batch.empty()) return 0;
    if (prefill(T, false)) return -1;
    prefill_tokens += T;
    ++steps_prefill;
    for (const SeqInit& s : batch)
      if (s.hist + s.q_len == s.n_own) active.push_back(s.slot);
    return static_cast<int>(batch.size());
  }

  bool chunking() const { return chunked.slot >= 0; }

  // One prefill step over the sequences in `batch`, T new tokens in all: stages and uploads
  // them, installs their page-table rows and decode state, and runs the stack; then, except in
  // the shared prefix's own pass, the head: each row's first token, or its embedding.
  int prefill(int T, bool prefix_pass) {
    const auto& c = e.cfg;
    const int n = static_cast<int>(batch.size());
    int n_work = 0, n_work_final = 0, n_final = 0, pt_cols = 1;
    bool any_hist = false;
    for (const SeqInit& s : batch) {
      n_work += (s.q_len + e.q_tile - 1) / e.q_tile;
      if (s.hist + s.q_len == s.n_own) {  // only a step's last sequence may be a non-final chunk
        n_work_final = n_work;
        ++n_final;
      }
      any_hist |= s.hist > 0;
      const int reserved = s.past / kPageTokens + static_cast<int>(slot_pages[s.slot].size());
      pt_cols = std::max(pt_cols, reserved);
    }
    const StageLayout L(n, n_work, pt_cols);
    const StageLayout::View h = L.at(e.h_stage), d = L.at(e.d_stage);
    for (int i = 0, wi = 0; i < n; ++i) {
      const SeqInit& s = batch[i];
      const std::vector<int32_t>& own = slot_pages[s.slot];
      const int shared = s.past / kPageTokens;  // full prefix pages before the first own page
      int32_t* pt = h.pt + static_cast<size_t>(i) * pt_cols;
      std::fill(pt, pt + pt_cols, 0);
      std::copy(slot_pages[S].begin(), slot_pages[S].begin() + shared, pt);
      std::copy(own.begin(), own.end(), pt + shared);
      h.seqs[i] = s;
      h.slot[i] = s.slot;
      h.q_start[i] = s.q_start;
      h.q_len[i] = s.q_len;
      h.past[i] = s.past;
      h.hist[i] = s.hist;
      // positions [16*(past/16), past) of the first own page hold prefix tokens: seed them, with
      // the row's first chunk (later chunks' own tokens are in that page by then)
      h.copy[i] = s.past % kPageTokens != 0 && s.hist == 0 ? own[0] : -1;
      for (int t0 = 0; t0 < s.q_len; t0 += e.q_tile, ++wi) {
        h.work[2 * wi] = i;
        h.work[2 * wi + 1] = t0;
      }
    }
    SB_CUDA_CHECK(cudaMemcpyAsync(e.d_stage, e.h_stage, L.words * 4, cudaMemcpyHostToDevice,
                                  e.stream));
    e.prof.launches[SB200_KC_OTHER] += 2;
    init_slots_kernel<<<n, 128, 0, e.stream>>>(
        d.seqs, d.pt, pt_cols, e.max_pages, e.page_table, e.slot_state, e.slot_ngen, e.slot_pos,
        e.slot_done, e.slot_row, e.slot_maxnew, e.slot_next_tok,
        e.d_suffix + (p.n_suffix - p.n_forced), p.n_forced,
        p.embed_mode ? nullptr : job.out_tokens_dev, p.embed_mode ? nullptr : job.out_len_dev,
        job.max_new_tokens, e.slot_cum_logprob, e.slot_n_row_tok);
    prefill_prepare_kernel<<<n, 128, 0, e.stream>>>(d.seqs, e.d_prefix, p.n_prefix, e.d_suffix,
                                                    p.n_suffix, job.row_tokens_dev,
                                                    job.row_tok_off_dev, e.tok_ids, e.tok_pos,
                                                    e.tok_slot, e.last_idx);
    if (prefix_tail_page >= 0) {
      ++e.prof.launches[SB200_KC_OTHER];
      copy_prefix_page_kernel<<<dim3(n, c.n_layers), 256, 0, e.stream>>>(
          e.kv_pool, e.layer_stride, kv_page_elems(c.n_kv_heads), prefix_tail_page, d.copy);
    }
    SB_CUDA_CHECK(cudaGetLastError());
    const PrefillStep step{d.work,    n_work, n_work_final, n,
                           n_final,   d.slot, d.q_start,    d.q_len,
                           d.past,    any_hist ? d.hist : nullptr, prefix_pass};
    if (e.forward(T, &step)) return -1;
    if (prefix_pass || n_final == 0) return 0;
    const int n_head = n_final;
    if (p.embed_mode) {
      if (rmsnorm(e.x, e.w.final_norm, e.hn, n_head, c.d_model, c.rms_eps, e.stream)) return -1;
      if (l2_normalize_rows(e.hn, e.embed_tmp, n_head, c.d_model, e.stream)) return -1;
      scatter_embed_kernel<<<n_head, 128, 0, e.stream>>>(e.embed_tmp, d.seqs, job.out_embed_dev,
                                                         c.d_model);
      SB_CUDA_CHECK(cudaGetLastError());
      return 0;
    }
    return e.head_and_sample(n_head, d.slot, job, p.has_fsm, true);
  }

  // One decode step: one token for every slot in the decode batch.
  int decode_step() {
    const auto& c = e.cfg;
    const int B = static_cast<int>(active.size());
    std::copy(active.begin(), active.end(), e.h_stage);
    SB_CUDA_CHECK(cudaMemcpyAsync(e.row_slot, e.h_stage, B * 4ull, cudaMemcpyHostToDevice,
                                  e.stream));
    e.prof.begin(SB200_KC_OTHER);
    const int prc = prepare_decode(e.row_slot, e.slot_next_tok, e.slot_pos, e.tok_ids, e.tok_pos,
                                   e.tok_slot, e.ctx_len, B, e.stream);
    e.prof.end();
    // slot_ctx + 1 is each row's context in this step (prepare_decode: ctx = pos + 1)
    int32_t* h_split = e.h_stage + B;
    DecodeSplit ds{e.split_rows, 0, 1};
    for (int b = 0; b < B; ++b) {
      const int splits = attn_decode_splits(slot_ctx[active[b]] + 1);
      if (splits > 1) {
        h_split[ds.n_rows++] = b;
        ds.max_splits = std::max(ds.max_splits, splits);
      }
    }
    if (ds.n_rows > 0) {
      if (e.split_ws.reserve(attn_decode_ws_floats(ds.n_rows, c.n_q_heads, ds.max_splits)))
        return -1;
      SB_CUDA_CHECK(cudaMemcpyAsync(e.split_rows, h_split, ds.n_rows * 4ull,
                                    cudaMemcpyHostToDevice, e.stream));
    }
    if (prc || e.forward(B, nullptr, ds) || e.head_and_sample(B, e.row_slot, job, p.has_fsm))
      return -1;
    decode_tokens += B;
    ++steps_decode;
    int64_t ctx_sum = 0;
    for (int s : active) ctx_sum += ++slot_ctx[s];
    attn_decode_bytes +=
        static_cast<double>(ctx_sum) * c.n_layers * c.n_kv_heads * 2.0 * kHeadDim * 2.0;
    return 0;
  }

  // Waits for the stream, then frees the slots and pages of finished rows: those whose done
  // flag is set, or every admitted row of an embedding model (its prefill finished it).
  int retire() {
    if (!p.embed_mode)
      SB_CUDA_CHECK(cudaMemcpyAsync(e.h_done, e.slot_done, (S + 2) * 4ull, cudaMemcpyDeviceToHost,
                                    e.stream));
    SB_CUDA_CHECK(cudaStreamSynchronize(e.stream));
    size_t k = 0;
    for (size_t i = 0; i < active.size(); ++i) {
      const int s = active[i];
      if (p.embed_mode || e.h_done[s]) {
        e.free_pages.insert(e.free_pages.end(), slot_pages[s].begin(), slot_pages[s].end());
        slot_pages[s].clear();
        free_slots.push_back(s);
        ++rows_done;
      } else {
        active[k++] = s;
      }
    }
    active.resize(k);
    return 0;
  }

  void fill_stats(sb200_job_stats* st) const {
    for (int i = 0; i < SB200_KC_COUNT; ++i) {
      st->kernel_ms[i] = e.prof.ms[i];
      st->kernel_launches[i] = e.prof.launches[i];
    }
    st->gemm_flops = e.gemm_flops;
    st->attn_decode_bytes = attn_decode_bytes;
    st->rows_done = rows_done;
    st->input_tokens = in_tokens;
    st->prefill_tokens = prefill_tokens;
    st->decode_tokens = decode_tokens;
    st->prefill_steps = steps_prefill;
    st->decode_steps = steps_decode;
    st->rows_truncated = p.n_truncated;
    st->prefix_cached_tokens = p.prefix_cached;
  }
};

}  // namespace

// ---------------------------------------------------------------------------
// the scheduling loop
// ---------------------------------------------------------------------------
int Engine::run(const sb200_job& job, sb200_job_stats* stats) {
  const int64_t N = job.n_rows;
  SB_CUDA_CHECK(cudaSetDevice(device));
  prof.reset(job.profile != 0, stream);
  gemm_flops = 0;
  if (N <= 0) return 0;
  JobSpec spec;
  if (validate_job(cfg, job, spec)) return -1;
  // prompt pieces and FSM -> device
  if (d_prefix.reserve(spec.n_prefix) || d_suffix.reserve(spec.n_suffix)) return -1;
  if (spec.n_prefix)
    SB_CUDA_CHECK(cudaMemcpyAsync(d_prefix, job.prefix_tokens, spec.n_prefix * 4ull,
                                  cudaMemcpyHostToDevice, stream));
  if (spec.n_suffix)
    SB_CUDA_CHECK(cudaMemcpyAsync(d_suffix, job.suffix_tokens, spec.n_suffix * 4ull,
                                  cudaMemcpyHostToDevice, stream));
  if (spec.has_fsm && upload_fsm(job)) return -1;
  if (!spec.embed_mode)
    SB_CUDA_CHECK(cudaMemsetAsync(job.out_len_dev, 0, N * sizeof(int32_t), stream));

  JobRun j(*this, job, std::move(spec));
  if (j.cache_prefix()) return -1;
  const int min_admit = std::max(1, cfg.min_admit_rows);
  int rc = 0;
  while (rc == 0 && j.rows_done < N) {
    // ---- admission: refill free slots with new rows (their prefill) ----
    // (a row being prefilled in chunks takes its next chunk after every decode step)
    const int64_t n_free = static_cast<int64_t>(j.free_slots.size());
    if (j.chunking() || (j.next_row < N && n_free > 0 &&
                         (j.active.empty() || n_free >= min_admit || N - j.next_row <= n_free))) {
      const int n = j.admit();
      if (n < 0) {
        rc = -1;
        break;
      }
      if (n > 0) {
        rc = j.retire();
        if (rc == 0 && job.progress)
          job.progress(j.rows_done, j.in_tokens, j.decode_tokens, job.progress_user);
        if (rc != 0 || !j.chunking() || j.active.empty())
          continue;  // try to admit more before decoding
      }
    }
    if (j.active.empty()) {
      if (j.next_row >= N) break;
      set_last_error("engine: scheduler stalled (no active rows, none admissible)");
      rc = -1;
      break;
    }
    // ---- one decode step over all active rows ----
    rc = (j.decode_step() || j.retire()) ? -1 : 0;
    if (rc == 0 && job.progress && (j.steps_decode % 8 == 0 || j.rows_done == N))
      job.progress(j.rows_done, j.in_tokens, j.decode_tokens, job.progress_user);
  }
  cudaStreamSynchronize(stream);
  prof.resolve();
  if (stats) j.fill_stats(stats);
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
  const size_t nb = tok_off[V] > 0 ? tok_off[V] : 1;
  if (e->d_tok_bytes.alloc(nb) || e->d_tok_off.alloc(V + 1ull)) return -1;
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
