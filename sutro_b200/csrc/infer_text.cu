// sutro_b200 — one-call entry point with HOST buffers: rows in, strings (or vectors) out.
//
// sb200_infer_text is what a non-Python host binds in place of the reference's
// `POST batch-inference` + `POST job-results` round trip (sutro/sdk.py:223, :384): it owns the
// host->device copy of the row bytes, tokenisation, the engine run, compaction of the
// generated tokens, detokenisation and the device->host copy of the results.  Everything on
// the device goes through the same entry points the Python host uses (sb200_tokenizer_encode,
// sb200_engine_run, sb200_tokenizer_decode); nothing here computes on the CPU.
#include <cub/device/device_scan.cuh>

#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/sutro_b200.h"
#include "common.cuh"
#include "dev_buf.h"
#include "kernels.h"

namespace sb {
namespace {

// three phases of the one-call path, timed with CUDA events on the engine's stream
struct PhaseEvents {
  cudaEvent_t e[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaStream_t stream = nullptr;
  bool ok = false;
  explicit PhaseEvents(cudaStream_t s) : stream(s) {
    ok = true;
    for (auto& x : e) ok = ok && cudaEventCreate(&x) == cudaSuccess;
  }
  ~PhaseEvents() {
    for (auto x : e)
      if (x) cudaEventDestroy(x);
  }
  void mark(int i) {
    if (ok) cudaEventRecord(e[i], stream);
  }
  void store(sb200_job_stats* st) {  // call after the final stream synchronisation
    if (!st) return;
    st->t_h2d_ms = st->t_device_ms = st->t_d2h_ms = 0.0;
    if (!ok) return;
    float a = 0.f, b = 0.f, c = 0.f;
    if (cudaEventElapsedTime(&a, e[0], e[1]) == cudaSuccess) st->t_h2d_ms = a;
    if (cudaEventElapsedTime(&b, e[1], e[2]) == cudaSuccess) st->t_device_ms = b;
    if (cudaEventElapsedTime(&c, e[2], e[3]) == cudaSuccess) st->t_d2h_ms = c;
  }
};

__global__ void widen_lengths_kernel(const int32_t* __restrict__ len, int64_t* __restrict__ out,
                                     int64_t n) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = len[i];
  if (i == n) out[i] = 0;  // slot n of the exclusive scan input
}

// out_tokens[n_rows, stride] (row i holds len[i] tokens) -> flat[off[i] .. off[i+1])
__global__ void compact_rows_kernel(const int32_t* __restrict__ out_tokens, int stride,
                                    const int64_t* __restrict__ off, int32_t* __restrict__ flat,
                                    int64_t n_rows) {
  const int64_t row = blockIdx.x;
  if (row >= n_rows) return;
  const int64_t lo = off[row], n = off[row + 1] - lo;
  const int32_t* src = out_tokens + row * stride;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) flat[lo + i] = src[i];
}

// ---- Arrow-style row selection (row sharding across GPUs and the ordered gather) ----------
// Source row j lives in part j / part_rows (parts are equally strided blobs: what an NCCL
// gather of padded per-rank results looks like; one part == a plain column).
SB_DEVICE void select_src(const int64_t* __restrict__ off, int64_t part_rows, int64_t part_bytes,
                          int64_t j, int64_t& start, int64_t& len) {
  const int64_t part = j / part_rows, local = j - part * part_rows;
  const int64_t* o = off + part * (part_rows + 1) + local;
  start = part * part_bytes + o[0];
  len = o[1] - o[0];
}

__global__ void select_lens_kernel(const int64_t* __restrict__ off, int64_t part_rows,
                                   int64_t part_bytes, const int64_t* __restrict__ idx, int64_t m,
                                   int64_t* __restrict__ lens) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < m) {
    int64_t start, len;
    select_src(off, part_rows, part_bytes, idx[i], start, len);
    lens[i] = len;
  }
  if (i == m) lens[i] = 0;
}

__global__ void select_copy_kernel(const uint8_t* __restrict__ bytes,
                                   const int64_t* __restrict__ off, int64_t part_rows,
                                   int64_t part_bytes, const int64_t* __restrict__ idx,
                                   const int64_t* __restrict__ out_off,
                                   uint8_t* __restrict__ out_bytes, int64_t m) {
  const int64_t i = blockIdx.x;
  if (i >= m) return;
  int64_t start, len;
  select_src(off, part_rows, part_bytes, idx[i], start, len);
  const uint8_t* src = bytes + start;
  uint8_t* dst = out_bytes + out_off[i];
  for (int64_t b = threadIdx.x; b < len; b += blockDim.x) dst[b] = src[b];
}

// exclusive scan of n int64 values with stream-ordered scratch
int exclusive_scan_i64(const int64_t* in, int64_t* out, int64_t n, cudaStream_t stream) {
  size_t cub_bytes = 0;
  SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, in, out, n, stream));
  void* tmp = nullptr;
  SB_CUDA_CHECK(cudaMallocAsync(&tmp, cub_bytes ? cub_bytes : 1, stream));
  const cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, cub_bytes, in, out, n, stream);
  cudaFreeAsync(tmp, stream);
  SB_CUDA_CHECK(e);
  return 0;
}

// len[n_rows] (int32) -> off[n_rows+1], the exclusive scan of the lengths widened to int64
int row_offsets(const int32_t* len, int64_t n_rows, int64_t* off, cudaStream_t stream) {
  const int64_t n1 = n_rows + 1;
  int64_t* len64 = nullptr;
  SB_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&len64), n1 * 8, stream));
  widen_lengths_kernel<<<static_cast<unsigned>((n1 + 255) / 256), 256, 0, stream>>>(len, len64,
                                                                                   n_rows);
  const int rc = exclusive_scan_i64(len64, off, n1, stream);
  cudaFreeAsync(len64, stream);
  return rc;
}

// out_tokens[n_rows, stride] -> flat[off[i] .. off[i+1]), off from row_offsets()
int compact_rows(const int32_t* out_tokens, int stride, const int64_t* off, int32_t* flat,
                 int64_t n_rows, cudaStream_t stream) {
  if (n_rows > 0)
    compact_rows_kernel<<<static_cast<unsigned>(n_rows), 64, 0, stream>>>(out_tokens, stride, off,
                                                                           flat, n_rows);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <class T>
T* host_alloc(size_t n) {
  return static_cast<T*>(std::malloc((n ? n : 1) * sizeof(T)));
}

}  // namespace
}  // namespace sb

using namespace sb;

extern "C" {

void sb200_result_free(sb200_result* r) {
  if (!r) return;
  std::free(r->bytes);
  std::free(r->offsets);
  std::free(r->tokens);
  std::free(r->token_offsets);
  std::free(r->cum_logprob);
  std::free(r->embeddings);
  std::free(r);
}

// out_tokens[n_rows, stride] (row i holds len[i] tokens) -> off[n_rows+1] + flat tokens, all on
// the device (what LocalEngine.generate hands to the detokenizer).
int sb200_compact_rows(const int32_t* out_tokens_dev, const int32_t* out_len_dev, int64_t n_rows,
                       int stride, int64_t* off_dev, int32_t* flat_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n_rows < 0 || !off_dev || (n_rows > 0 && (!out_tokens_dev || !out_len_dev || !flat_dev))) {
    set_last_error("compact_rows: null argument");
    return -1;
  }
  if (row_offsets(out_len_dev, n_rows, off_dev, stream)) return -1;
  return compact_rows(out_tokens_dev, stride, off_dev, flat_dev, n_rows, stream);
}

// Select m rows (idx, any order, no repeats needed) of a device-resident string column:
// out_off[m+1] and out_bytes (capacity: the selected rows' bytes; the source size is always
// enough).  part_rows/part_bytes describe a batch of equally strided columns (see above);
// pass part_rows = the row count and part_bytes = 0 for a plain column.
int sb200_rows_select(const uint8_t* bytes_dev, const int64_t* off_dev, int64_t part_rows,
                      int64_t part_bytes, const int64_t* idx_dev, int64_t m, int64_t* out_off_dev,
                      uint8_t* out_bytes_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (m < 0 || part_rows <= 0 || !off_dev || !out_off_dev || (m > 0 && !idx_dev)) {
    set_last_error("rows_select: bad argument");
    return -1;
  }
  const int64_t m1 = m + 1;
  int64_t* lens = nullptr;
  SB_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&lens), m1 * 8, stream));
  select_lens_kernel<<<static_cast<unsigned>((m1 + 255) / 256), 256, 0, stream>>>(
      off_dev, part_rows, part_bytes, idx_dev, m, lens);
  const int rc = exclusive_scan_i64(lens, out_off_dev, m1, stream);
  cudaFreeAsync(lens, stream);
  if (rc) return -1;
  if (m > 0 && out_bytes_dev != nullptr)
    select_copy_kernel<<<static_cast<unsigned>(m), 128, 0, stream>>>(
        bytes_dev, off_dev, part_rows, part_bytes, idx_dev, out_off_dev, out_bytes_dev, m);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int sb200_infer_text(void* engine, void* tokenizer, const uint8_t* rows_bytes,
                     const int64_t* rows_offsets, int64_t n_rows, const sb200_job* options,
                     int want_text, int want_logprobs, sb200_result** out,
                     sb200_job_stats* stats) {
  if (out) *out = nullptr;
  if (!engine || !tokenizer || !rows_offsets || !options || !out || n_rows < 0) {
    set_last_error("infer_text: null argument");
    return -1;
  }
  int device = 0, embedding = 0, d_model = 0, vocab = 0;
  if (sb200_engine_info(engine, &device, &embedding, &d_model, &vocab)) return -1;
  SB_CUDA_CHECK(cudaSetDevice(device));
  cudaStream_t stream = static_cast<cudaStream_t>(sb200_engine_stream(engine));
  const int64_t n_bytes = rows_offsets[n_rows];
  if (rows_offsets[0] != 0 || n_bytes < 0 || (n_bytes > 0 && !rows_bytes)) {
    set_last_error("infer_text: offsets must start at 0 and rows_bytes must hold %lld bytes",
                   static_cast<long long>(n_bytes));
    return -1;
  }
  if (n_rows == 0) {  // nothing to run: an empty, well-formed result
    auto* r0 = static_cast<sb200_result*>(std::calloc(1, sizeof(sb200_result)));
    if (!r0) {
      set_last_error("infer_text: out of host memory");
      return -1;
    }
    r0->offsets = host_alloc<int64_t>(1);
    r0->token_offsets = host_alloc<int64_t>(1);
    if (r0->offsets) r0->offsets[0] = 0;
    if (r0->token_offsets) r0->token_offsets[0] = 0;
    r0->d_model = d_model;
    if (stats) std::memset(stats, 0, sizeof(*stats));
    *out = r0;
    return 0;
  }
  const int max_new = embedding ? 0 : options->max_new_tokens;
  if (!embedding && max_new <= 0) {
    set_last_error("infer_text: max_new_tokens must be positive");
    return -1;
  }

  // ---- host -> HBM, tokenise ------------------------------------------------------------
  DevBuf d_text, d_off, d_tok, d_toff;
  if (d_text.alloc(n_bytes) || d_off.alloc((n_rows + 1) * 8) || d_tok.alloc(n_bytes * 4) ||
      d_toff.alloc((n_rows + 1) * 8))
    return -1;
  PhaseEvents ev(stream);
  ev.mark(0);
  if (n_bytes)
    SB_CUDA_CHECK(cudaMemcpyAsync(d_text.p, rows_bytes, n_bytes, cudaMemcpyHostToDevice, stream));
  SB_CUDA_CHECK(cudaMemcpyAsync(d_off.p, rows_offsets, (n_rows + 1) * 8, cudaMemcpyHostToDevice,
                                stream));
  ev.mark(1);  // inputs resident in HBM
  if (sb200_tokenizer_encode(tokenizer, d_text.as<uint8_t>(), n_bytes, d_off.as<int64_t>(),
                             n_rows, d_tok.as<int32_t>(), d_toff.as<int64_t>(), stream))
    return -1;
  std::vector<int64_t> h_toff(n_rows + 1);
  SB_CUDA_CHECK(cudaMemcpyAsync(h_toff.data(), d_toff.p, (n_rows + 1) * 8,
                                cudaMemcpyDeviceToHost, stream));
  SB_CUDA_CHECK(cudaStreamSynchronize(stream));  // the scheduler reads row lengths on the host

  // ---- the engine -------------------------------------------------------------------------
  DevBuf d_out, d_len, d_emb, d_lp;
  sb200_job job = *options;
  job.row_tokens_dev = d_tok.as<int32_t>();
  job.row_tok_off_dev = d_toff.as<int64_t>();
  job.row_tok_off = h_toff.data();
  job.n_rows = n_rows;
  job.out_tokens_dev = nullptr, job.out_len_dev = nullptr, job.out_embed_dev = nullptr;
  job.out_first_logits_dev = nullptr, job.out_cum_logprob_dev = nullptr;
  if (embedding) {
    if (d_emb.alloc(static_cast<size_t>(n_rows) * d_model * 4)) return -1;
    job.out_embed_dev = d_emb.as<float>();
  } else {
    if (d_out.alloc(static_cast<size_t>(n_rows) * max_new * 4) || d_len.alloc(n_rows * 4))
      return -1;
    SB_CUDA_CHECK(cudaMemsetAsync(d_len.p, 0, static_cast<size_t>(n_rows) * 4, stream));
    job.out_tokens_dev = d_out.as<int32_t>();
    job.out_len_dev = d_len.as<int32_t>();
    if (want_logprobs) {
      if (d_lp.alloc(n_rows * 4)) return -1;
      SB_CUDA_CHECK(cudaMemsetAsync(d_lp.p, 0, static_cast<size_t>(n_rows) * 4, stream));
      job.out_cum_logprob_dev = d_lp.as<float>();
    }
  }
  if (sb200_engine_run(engine, &job, stats)) return -1;

  // ---- results: compact, detokenise, HBM -> host ---------------------------------------------
  auto* r = static_cast<sb200_result*>(std::calloc(1, sizeof(sb200_result)));
  if (!r) {
    set_last_error("infer_text: out of host memory");
    return -1;
  }
  r->n_rows = n_rows;
  struct Guard {  // frees a half-built result on failure
    sb200_result* r;
    ~Guard() {
      if (r) sb200_result_free(r);
    }
  } guard{r};

  if (embedding) {
    r->d_model = d_model;
    r->embeddings = host_alloc<float>(static_cast<size_t>(n_rows) * d_model);
    if (!r->embeddings) {
      set_last_error("infer_text: out of host memory");
      return -1;
    }
    ev.mark(2);
    SB_CUDA_CHECK(cudaMemcpyAsync(r->embeddings, d_emb.p,
                                  static_cast<size_t>(n_rows) * d_model * 4,
                                  cudaMemcpyDeviceToHost, stream));
    ev.mark(3);
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
    ev.store(stats);
    guard.r = nullptr;
    *out = r;
    return 0;
  }

  DevBuf d_ooff, d_flat, d_boff, d_bytes;
  const int64_t n1 = n_rows + 1;
  if (d_ooff.alloc(n1 * 8) ||
      row_offsets(d_len.as<int32_t>(), n_rows, d_ooff.as<int64_t>(), stream))
    return -1;
  r->token_offsets = host_alloc<int64_t>(n1);
  if (!r->token_offsets) {
    set_last_error("infer_text: out of host memory");
    return -1;
  }
  SB_CUDA_CHECK(cudaMemcpyAsync(r->token_offsets, d_ooff.p, n1 * 8, cudaMemcpyDeviceToHost,
                                stream));
  SB_CUDA_CHECK(cudaStreamSynchronize(stream));
  const int64_t n_out = r->token_offsets[n_rows];
  if (d_flat.alloc(n_out * 4) || compact_rows(d_out.as<int32_t>(), max_new, d_ooff.as<int64_t>(),
                                              d_flat.as<int32_t>(), n_rows, stream))
    return -1;
  r->tokens = host_alloc<int32_t>(n_out);
  if (!r->tokens) {
    set_last_error("infer_text: out of host memory");
    return -1;
  }
  if (want_logprobs) {
    r->cum_logprob = host_alloc<float>(n_rows);
    if (!r->cum_logprob) {
      set_last_error("infer_text: out of host memory");
      return -1;
    }
  }
  int64_t total = 0;
  if (want_text) {
    if (d_boff.alloc(n1 * 8)) return -1;
    if (sb200_tokenizer_decode(tokenizer, d_flat.as<int32_t>(), n_out, d_ooff.as<int64_t>(),
                               n_rows, nullptr, d_boff.as<int64_t>(), stream))  // sizing pass
      return -1;
    r->offsets = host_alloc<int64_t>(n1);
    if (!r->offsets) {
      set_last_error("infer_text: out of host memory");
      return -1;
    }
    SB_CUDA_CHECK(cudaMemcpyAsync(r->offsets, d_boff.p, n1 * 8, cudaMemcpyDeviceToHost, stream));
    SB_CUDA_CHECK(cudaStreamSynchronize(stream));
    total = r->offsets[n_rows];
    if (d_bytes.alloc(total)) return -1;
    if (sb200_tokenizer_decode(tokenizer, d_flat.as<int32_t>(), n_out, d_ooff.as<int64_t>(),
                               n_rows, d_bytes.as<uint8_t>(), d_boff.as<int64_t>(), stream))
      return -1;
    r->bytes = host_alloc<uint8_t>(total);
    if (!r->bytes) {
      set_last_error("infer_text: out of host memory");
      return -1;
    }
  }
  // results resident in HBM -> host (the two offset arrays above are sizing reads the host needs
  // to allocate; they are part of the device phase)
  ev.mark(2);
  if (n_out)
    SB_CUDA_CHECK(cudaMemcpyAsync(r->tokens, d_flat.p, n_out * 4, cudaMemcpyDeviceToHost, stream));
  if (want_logprobs && n_rows)
    SB_CUDA_CHECK(cudaMemcpyAsync(r->cum_logprob, d_lp.p, n_rows * 4, cudaMemcpyDeviceToHost,
                                  stream));
  if (want_text && total)
    SB_CUDA_CHECK(cudaMemcpyAsync(r->bytes, d_bytes.p, total, cudaMemcpyDeviceToHost, stream));
  ev.mark(3);
  SB_CUDA_CHECK(cudaStreamSynchronize(stream));
  ev.store(stats);
  guard.r = nullptr;
  *out = r;
  return 0;
}

}  // extern "C"
