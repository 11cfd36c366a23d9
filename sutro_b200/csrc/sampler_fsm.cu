// sutro_b200 — K8: constrained decoding.
//   fsm_build_mask   for every (DFA state, token) walk the token's bytes through
//                    the byte-level DFA compiled from output_schema and pack the
//                    "token keeps the automaton alive" bits, 32 tokens per word
//                    (warp ballot).  Runs once per schema.
//   sample_greedy    per logits row: masked arg-max over the vocabulary (lowest
//                    index wins ties), append to the row's output, advance the
//                    row's DFA state by the chosen token's bytes, raise the done
//                    flag on EOS / final state / max_new_tokens.
//   sample_random    temperature / min-p / top-k / top-p sampling under the same mask
//                    (exact radix-select thresholds, Philox4x32-10 draws).
//   apply_penalties  presence / frequency / repetition penalties on the logits, in place,
//                    before either sampler (vLLM's semantics).
//   prepare_decode   gathers next-step inputs (token, position, context length)
//                    from the per-slot decode state, entirely on device.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace sb {

namespace {

__global__ void __launch_bounds__(256)
fsm_build_mask_kernel(const int32_t* __restrict__ trans, const uint8_t* __restrict__ accept,
                      const uint8_t* __restrict__ tok_bytes, const int32_t* __restrict__ tok_off,
                      int vocab, int eos_id, uint32_t* __restrict__ mask_bits, int mask_words) {
  const int state = blockIdx.y;
  const int tok = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  if (tok < vocab) {
    if (tok == eos_id) {
      ok = accept[state] != 0;
    } else {
      const int b0 = tok_off[tok], b1 = tok_off[tok + 1];
      int s = state;
      for (int i = b0; i < b1 && s >= 0; ++i) s = trans[s * 256 + tok_bytes[i]];
      ok = (b1 > b0) && (s >= 0);
    }
  }
  const uint32_t word = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && (tok >> 5) < mask_words)
    mask_bits[static_cast<size_t>(state) * mask_words + (tok >> 5)] = word;
}

constexpr int kSampleThreads = 512;
constexpr int kSampleWarps = kSampleThreads / 32;

// Row bookkeeping shared by the greedy and the stochastic sampler (thread 0 of the CTA):
// append the token, advance the DFA by its bytes, apply jump-forward tails, raise `done`.
// `stop`: nothing was selectable; the row ends without output whatever ignore_eos says.
__device__ void finish_row(const SampleArgs& a, int slot, int state, int tok, float logprob,
                           bool stop = false) {
  const int row = a.slot_row[slot];
  int ngen = a.slot_ngen[slot];
  bool done = false;
  if (stop || (tok == a.eos_id && !a.ignore_eos)) {
    done = true;
  } else {
    a.out_tokens[static_cast<size_t>(row) * a.out_stride + ngen] = tok;
    ++ngen;
    if (state >= 0) {
      int s = state;
      const int b0 = a.tok_off[tok], b1 = a.tok_off[tok + 1];
      for (int i = b0; i < b1 && s >= 0; ++i) s = a.fsm_trans[s * 256 + a.tok_bytes[i]];
      a.slot_state[slot] = s;
      if (s < 0 || a.fsm_final[s]) {
        done = true;
      } else if (a.fsm_tail_off != nullptr) {
        // jump-forward: everything from here to a final state is forced -> emit it now
        const int t0 = a.fsm_tail_off[s], t1 = a.fsm_tail_off[s + 1];
        if (t1 > t0) {
          const int maxnew = a.slot_maxnew[slot];
          for (int i = t0; i < t1 && ngen < maxnew; ++i)
            a.out_tokens[static_cast<size_t>(row) * a.out_stride + ngen++] = a.fsm_tail_tok[i];
          done = true;
        }
      }
    }
  }
  if (ngen >= a.slot_maxnew[slot]) done = true;
  a.slot_ngen[slot] = ngen;
  a.out_len[row] = ngen;
  if (a.slot_cum_logprob != nullptr) {
    const float c = a.slot_cum_logprob[slot] + logprob;
    a.slot_cum_logprob[slot] = c;
    if (a.out_cum_logprob != nullptr) a.out_cum_logprob[row] = c;
  }
  a.slot_next_tok[slot] = tok;
  a.slot_pos[slot] += 1;
  if (done) a.slot_done[slot] = 1;
}

struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ ArgMax better(ArgMax x, ArgMax y) {
  return (y.v > x.v || (y.v == x.v && y.i < x.i)) ? y : x;  // NaN never wins
}
__device__ ArgMax block_argmax(ArgMax m, float* sv, int* si) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    m = better(m, ArgMax{__shfl_xor_sync(0xffffffffu, m.v, o), __shfl_xor_sync(0xffffffffu, m.i, o)});
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = m.v;
    si[threadIdx.x >> 5] = m.i;
  }
  __syncthreads();
  ArgMax r{sv[0], si[0]};
  for (int w = 1; w < kSampleWarps; ++w) r = better(r, ArgMax{sv[w], si[w]});
  __syncthreads();
  return r;  // same value in every thread
}
__device__ float block_sum(float v, float* sv) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int w = 0; w < kSampleWarps; ++w) r += sv[w];
  __syncthreads();
  return r;
}

// ---------------------------------------------------------------------------
// presence / frequency / repetition penalties, in place on the fp32 logits, in vLLM's order
// (vllm.model_executor.layers.utils.apply_penalties):
//   l *= (l > 0 ? 1/r : r)       for every token of prompt ∪ output
//   l -= f * count               count = occurrences in the output
//   l -= p * (count > 0)
// One CTA per row rebuilds the row's history table from its prompt pieces and out_tokens: a
// bitmap of the prompt's tokens and a hash of the output's token counts, both in shared memory.
// Every logit is then rewritten at most once, by the thread that owns its token, from the raw
// logit, the count and the in-prompt bit alone, so the result does not depend on the order of
// the atomics or on the batch.  The roundings are spelled out: l - f*c must not become an FMA.
// ---------------------------------------------------------------------------
constexpr int kPenaltyThreads = 256;

struct PenaltyParams {
  float rep, rep_inv, freq, pres;
  int hash_size;   // power of two >= 2 * out_stride: the hash never fills
  int zero_pass;   // f or p has its sign bit set: vLLM's l - (f*0) turns -0.0 into +0.0
};

__device__ __forceinline__ float penalize(float l, int count, bool seen, const PenaltyParams& q) {
  if (seen) l = __fmul_rn(l, l > 0.f ? q.rep_inv : q.rep);
  l = __fsub_rn(l, __fmul_rn(q.freq, static_cast<float>(count)));
  return __fsub_rn(l, __fmul_rn(q.pres, count > 0 ? 1.f : 0.f));
}

__global__ void __launch_bounds__(kPenaltyThreads) apply_penalties_kernel(SampleArgs a,
                                                                          PenaltyParams q) {
  extern __shared__ uint32_t pen_smem[];
  const int b = blockIdx.x;
  const int slot = a.row_slot[b];
  if (a.slot_done[slot]) return;
  const int row = a.slot_row[slot];
  const int V = a.vocab;
  const int words = (V + 31) >> 5;
  uint32_t* in_prompt = pen_smem;                                      // [words]
  int32_t* hkey = reinterpret_cast<int32_t*>(pen_smem + words);        // [hash_size], -1 empty
  int32_t* hcnt = hkey + q.hash_size;                                  // [hash_size]
  const uint32_t hmask = static_cast<uint32_t>(q.hash_size - 1);
  float* lg = a.logits + static_cast<size_t>(b) * a.ldl;
  for (int i = threadIdx.x; i < words; i += kPenaltyThreads) in_prompt[i] = 0u;
  for (int i = threadIdx.x; i < q.hash_size; i += kPenaltyThreads) hkey[i] = -1, hcnt[i] = 0;
  __syncthreads();

  // 1. the table: prompt bitmap, output counts
  const int n_pre = a.n_prompt_prefix, n_row = a.slot_n_row_tok[slot], n_suf = a.n_prompt_suffix;
  const int n_prompt = n_pre + n_row + n_suf;
  const int32_t* row_toks = a.row_tokens + a.row_tok_off[row];
  auto prompt_tok = [&](int j) {
    return j < n_pre ? a.prompt_prefix[j]
                     : (j < n_pre + n_row ? row_toks[j - n_pre] : a.prompt_suffix[j - n_pre - n_row]);
  };
  for (int j = threadIdx.x; j < n_prompt; j += kPenaltyThreads) {
    const int t = prompt_tok(j);
    if (t >= 0 && t < V) atomicOr(&in_prompt[t >> 5], 1u << (t & 31));
  }
  const int n_out = a.slot_ngen[slot];
  const int32_t* out = a.out_tokens + static_cast<size_t>(row) * a.out_stride;
  for (int j = threadIdx.x; j < n_out; j += kPenaltyThreads) {
    const int t = out[j];
    if (t < 0 || t >= V) continue;
    for (uint32_t h = (static_cast<uint32_t>(t) * 2654435761u) & hmask;; h = (h + 1) & hmask) {
      const int k = atomicCAS(&hkey[h], -1, t);
      if (k == -1 || k == t) {
        atomicAdd(&hcnt[h], 1);
        break;
      }
    }
  }
  __syncthreads();

  // 2. every output token, once (its hash entry); its prompt bit is taken so step 3 skips it
  for (int h = threadIdx.x; h < q.hash_size; h += kPenaltyThreads) {
    const int t = hkey[h];
    if (t < 0) continue;
    atomicAnd(&in_prompt[t >> 5], ~(1u << (t & 31)));
    lg[t] = penalize(lg[t], hcnt[h], true, q);
  }
  __syncthreads();

  // 3. every prompt token that is not in the output, once: the thread that clears its bit
  for (int j = threadIdx.x; j < n_prompt; j += kPenaltyThreads) {
    const int t = prompt_tok(j);
    if (t < 0 || t >= V) continue;
    const uint32_t bit = 1u << (t & 31);
    if (atomicAnd(&in_prompt[t >> 5], ~bit) & bit) lg[t] = penalize(lg[t], 0, true, q);
  }

  // 4. the tokens outside the history: l - (f*0) - (p*0) is l, except that a negative f or p
  //    (whose product with 0 is -0.0) turns -0.0 into +0.0.  A token steps 2-3 rewrote never
  //    ends at -0.0 then, so this still rewrites every logit at most once.
  if (q.zero_pass) {
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += kPenaltyThreads)
      if (__float_as_uint(lg[i]) == 0x80000000u) lg[i] = 0.f;
  }
}

__global__ void __launch_bounds__(kSampleThreads) sample_greedy_kernel(SampleArgs a) {
  const int b = blockIdx.x;
  const int slot = a.row_slot[b];
  if (a.slot_done[slot]) return;
  const int state = a.slot_state ? a.slot_state[slot] : -1;
  const float* lg = a.logits + static_cast<size_t>(b) * a.ldl;
  const uint32_t* mask =
      (state >= 0 && a.mask_bits) ? a.mask_bits + static_cast<size_t>(state) * a.mask_words
                                  : nullptr;
  __shared__ float sv[kSampleWarps];
  __shared__ int si[kSampleWarps];
  ArgMax m{-INFINITY, 0x7fffffff};
  for (int i = threadIdx.x; i < a.vocab; i += kSampleThreads) {
    if (mask && !((mask[i >> 5] >> (i & 31)) & 1u)) continue;
    m = better(m, ArgMax{lg[i], i});
  }
  m = block_argmax(m, sv, si);
  const bool none = m.i < 0 || m.i >= a.vocab;  // nothing selectable: terminate the row
  const int tok = none ? a.eos_id : m.i;
  float logprob = 0.f;
  if (a.slot_cum_logprob != nullptr && !none) {  // log-softmax of the masked logits at the arg-max
    float se = 0.f;
    for (int i = threadIdx.x; i < a.vocab; i += kSampleThreads) {
      if (mask && !((mask[i >> 5] >> (i & 31)) & 1u)) continue;
      se += __expf(lg[i] - m.v);
    }
    se = block_sum(se, sv);
    logprob = -__logf(se);
  }
  if (threadIdx.x == 0) finish_row(a, slot, state, tok, logprob, none);
}

// ---------------------------------------------------------------------------
// temperature / top-k / top-p sampling.  One CTA per row, everything exact on the
// fp32 logits: radix-select on the order-preserving integer image of z = logit / T gives
// the k-th largest value (ties kept); the same descent weighted by exp(z - max) gives the
// smallest value whose upper tail holds top_p of the mass; the token is then drawn by
// inverse CDF over the kept set in vocabulary order with one Philox4x32-10 draw per
// (seed, row, step).
// ---------------------------------------------------------------------------
// Order-preserving key of a float.  -0.0 is mapped to +0.0 first: they compare equal, so a
// tie at zero must give one key or a threshold at +0.0 would drop the -0.0 tokens.
__device__ __forceinline__ uint32_t fkey(float f) {
  const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ uint4 philox4x32_10(uint2 key, uint4 c) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ key.x, lo1, hi0 ^ c.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return c;
}

// 4 CTAs per SM (32 registers): a 512-row chunk then runs in one wave on 132 SMs.
// log_min_p = fp32(ln min_p), computed on the host; read only when a.min_p > 0.
__global__ void __launch_bounds__(kSampleThreads, 4) sample_random_kernel(SampleArgs a,
                                                                          float log_min_p) {
  const int b = blockIdx.x;
  const int slot = a.row_slot[b];
  if (a.slot_done[slot]) return;
  const int state = a.slot_state ? a.slot_state[slot] : -1;
  const float* lg = a.logits + static_cast<size_t>(b) * a.ldl;
  const uint32_t* mask =
      (state >= 0 && a.mask_bits) ? a.mask_bits + static_cast<size_t>(state) * a.mask_words
                                  : nullptr;
  const float inv_t = 1.0f / a.temperature;
  const int V = a.vocab;
  auto allowed = [&](int i) { return !mask || ((mask[i >> 5] >> (i & 31)) & 1u); };

  __shared__ float sv[kSampleWarps];
  __shared__ int si[kSampleWarps];
  __shared__ uint32_t hist_u[256];
  __shared__ unsigned long long hist_m[256];
  __shared__ uint32_t sh_prefix, sh_pmask;
  __shared__ int sh_k;
  __shared__ unsigned long long sh_above, sh_target;
  __shared__ float wsum[kSampleWarps + 1];
  __shared__ int sh_tok;
  __shared__ uint32_t sh_tau;

  // 1. max of z over the allowed tokens
  ArgMax m{-INFINITY, 0x7fffffff};
  for (int i = threadIdx.x; i < V; i += kSampleThreads)
    if (allowed(i)) m = better(m, ArgMax{lg[i] * inv_t, i});
  m = block_argmax(m, sv, si);
  if (m.i < 0 || m.i >= V) {  // nothing selectable
    if (threadIdx.x == 0) finish_row(a, slot, state, a.eos_id, 0.f, true);
    return;
  }
  const float zmax = m.v;

  // 2. min_p (vLLM v1: before top-k / top-p) keeps z >= zmax + ln(min_p); top-k keeps the z
  //    >= the k-th largest (ties kept).  Every filter keeps an upper set of z, so their
  //    intersection is the one with the largest threshold.
  if (threadIdx.x == 0) sh_tau = a.min_p > 0.f ? fkey(__fadd_rn(zmax, log_min_p)) : 0u;
  __syncthreads();
  uint32_t tau = sh_tau;
  if (a.top_k > 0) {
    if (threadIdx.x == 0) sh_prefix = 0, sh_pmask = 0, sh_k = a.top_k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = threadIdx.x; i < 256; i += kSampleThreads) hist_u[i] = 0;
      __syncthreads();
      const uint32_t prefix = sh_prefix, pmask = sh_pmask;
      for (int i = threadIdx.x; i < V; i += kSampleThreads) {
        if (!allowed(i)) continue;
        const uint32_t key = fkey(lg[i] * inv_t);
        if ((key & pmask) == prefix) atomicAdd(&hist_u[(key >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int cum = 0, sel = 0;
        for (int bin = 255; bin >= 0; --bin) {
          const int c = static_cast<int>(hist_u[bin]);
          if (cum + c >= sh_k) {
            sel = bin;
            break;
          }
          cum += c;
        }
        sh_k -= cum;
        sh_prefix = prefix | (static_cast<uint32_t>(sel) << shift);
        sh_pmask = pmask | (255u << shift);
      }
      __syncthreads();
    }
    tau = max(tau, sh_prefix);
    __syncthreads();  // every thread holds tau before the top-p descent reuses sh_prefix
  }

  // 3. top-p threshold on the same ordering, weighted by the softmax mass exp(z - zmax) of the
  //    (top-k filtered) set.  The masses are summed in 24.40 fixed point (the largest weight is
  //    1, so V < 2^24 terms cannot overflow 64 bits): integer sums do not depend on the order of
  //    the atomics, so the kept set is a function of the logits alone.  Rounding each weight to
  //    2^-40 moves the mass of the whole row by less than V * 2^-41 <= 2e-7 (W >= 1).
  if (a.top_p < 1.0f) {
    if (threadIdx.x == 0) sh_prefix = 0, sh_pmask = 0, sh_above = 0ull;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int i = threadIdx.x; i < 256; i += kSampleThreads) hist_m[i] = 0ull;
      __syncthreads();
      const uint32_t prefix = sh_prefix, pmask = sh_pmask;
      const int lane = threadIdx.x & 31;
      for (int base = threadIdx.x & ~31; base < V; base += kSampleThreads) {  // warp-uniform
        const int i = base + lane;
        uint32_t bin = 0u;
        unsigned long long w = 0ull;
        bool in = false;
        if (i < V && allowed(i)) {
          const float z = lg[i] * inv_t;
          const uint32_t key = fkey(z);
          in = key >= tau && (key & pmask) == prefix;
          bin = (key >> shift) & 255u;
          if (in) w = __float2ull_rn(__expf(z - zmax) * 1099511627776.0f);  // * 2^40
        }
        // one shared atomic per distinct bin of the warp; w <= 2^40 is summed as two 20-bit
        // halves so that 32 lanes cannot overflow the 32-bit warp reduction
        for (unsigned todo = __ballot_sync(~0u, in); todo != 0u;) {
          const int lead = __ffs(todo) - 1;
          const uint32_t b0 = __shfl_sync(~0u, bin, lead);
          const bool mine = in && bin == b0;
          todo &= ~__ballot_sync(~0u, mine);
          const uint32_t lo = __reduce_add_sync(~0u, mine ? static_cast<uint32_t>(w) & 0xFFFFFu : 0u);
          const uint32_t hi = __reduce_add_sync(~0u, mine ? static_cast<uint32_t>(w >> 20) : 0u);
          if (lane == lead) atomicAdd(&hist_m[b0], (static_cast<unsigned long long>(hi) << 20) + lo);
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        if (shift == 24) {  // the first pass sees the whole set: target = ceil(top_p * W)
          unsigned long long w = 0ull;
          for (int bin = 0; bin < 256; ++bin) w += hist_m[bin];
          sh_target =
              static_cast<unsigned long long>(ceil(fmax(0.0, static_cast<double>(a.top_p)) * w));
        }
        // The bin chosen by the previous pass holds exactly the mass of this pass's bins, so
        // some non-empty bin reaches the target (top_p < 1 puts it at or below W).
        const unsigned long long target = sh_target;
        unsigned long long cum = sh_above;
        int sel = 0;
        for (int bin = 255; bin >= 0; --bin) {
          const unsigned long long c = hist_m[bin];
          if (c > 0ull && cum + c >= target) {
            sel = bin;
            break;
          }
          cum += c;
        }
        sh_above = cum;
        sh_prefix = prefix | (static_cast<uint32_t>(sel) << shift);
        sh_pmask = pmask | (255u << shift);
      }
      __syncthreads();
    }
    if (sh_prefix > tau) tau = sh_prefix;
    __syncthreads();
  }

  // 4. inverse-CDF draw over the kept set in vocabulary order.  Warp w owns a contiguous
  //    chunk; inside it, (iteration, lane) order == index order.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int chunk = ((V + kSampleWarps - 1) / kSampleWarps + 31) & ~31;
  const int c0 = warp * chunk, c1 = min(V, c0 + chunk);
  auto weight = [&](int i) -> float {
    if (i >= c1 || !allowed(i)) return 0.f;
    const float z = lg[i] * inv_t;
    return fkey(z) >= tau ? __expf(z - zmax) : 0.f;
  };
  float part = 0.f;
  for (int i = c0 + lane; i < c1; i += 32) part += weight(i);
  part = warp_sum(part);
  if (lane == 0) wsum[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float run = 0.f;
    for (int w = 0; w < kSampleWarps; ++w) {
      const float t = wsum[w];
      wsum[w] = run;  // exclusive prefix
      run += t;
    }
    wsum[kSampleWarps] = run;
    sh_tok = -1;
  }
  __syncthreads();
  const float total = wsum[kSampleWarps];
  const int row = a.slot_row[slot];
  const uint64_t row_id =
      a.row_ids != nullptr ? static_cast<uint64_t>(a.row_ids[row]) : static_cast<uint64_t>(row);
  const uint64_t ctr_row = a.seed_per_row ? row_id : 0ull;
  const uint4 rnd = philox4x32_10(
      make_uint2(static_cast<uint32_t>(a.seed), static_cast<uint32_t>(a.seed >> 32)),
      make_uint4(static_cast<uint32_t>(ctr_row), static_cast<uint32_t>(ctr_row >> 32),
                 static_cast<uint32_t>(a.slot_ngen[slot]), 0u));
  const float u = static_cast<float>(rnd.x >> 8) * (1.0f / 16777216.0f);
  const float target = u * total;
  const float wlo = wsum[warp];
  const float whi = (warp + 1 < kSampleWarps) ? wsum[warp + 1] : total;
  if (target >= wlo && (target < whi || warp == kSampleWarps - 1) && whi > wlo) {
    // this warp's chunk contains the target (the last warp also catches target == total)
    float run = wlo;
    int found = -1, last_kept = -1;
    for (int base = c0; base < c1 && found < 0; base += 32) {
      const float w = weight(base + lane);
      float incl = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, w > 0.f && run + incl > target);
      const unsigned kept = __ballot_sync(0xffffffffu, w > 0.f);
      if (kept) last_kept = base + 31 - __clz(kept);
      if (hit) found = base + __ffs(hit) - 1;
      run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (found < 0) found = last_kept;  // fp rounding at the very end of the chunk
    if (lane == 0 && found >= 0) sh_tok = found;
  }
  __syncthreads();
  int tok = sh_tok;
  if (tok < 0) tok = m.i;  // degenerate rounding: fall back to the mode
  float logprob = 0.f;
  if (a.slot_cum_logprob != nullptr) {
    float se = 0.f;  // log-softmax over all allowed tokens at temperature T
    for (int i = threadIdx.x; i < V; i += kSampleThreads)
      if (allowed(i)) se += __expf(lg[i] * inv_t - zmax);
    se = block_sum(se, sv);
    logprob = (lg[tok] * inv_t - zmax) - __logf(se);
  }
  if (threadIdx.x == 0) {
    if (a.out_tau != nullptr) a.out_tau[b] = tau;
    finish_row(a, slot, state, tok, logprob);
  }
}

__global__ void prepare_decode_kernel(const int32_t* __restrict__ row_slot,
                                      const int32_t* __restrict__ slot_next_tok,
                                      const int32_t* __restrict__ slot_pos,
                                      int32_t* __restrict__ tok_ids, int32_t* __restrict__ tok_pos,
                                      int32_t* __restrict__ tok_slot, int32_t* __restrict__ ctx_len,
                                      int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int slot = row_slot[b];
  const int pos = slot_pos[slot];
  tok_ids[b] = slot_next_tok[slot];
  tok_pos[b] = pos;
  tok_slot[b] = slot;
  ctx_len[b] = pos + 1;
}

}  // namespace

int fsm_build_mask(const int32_t* fsm_trans, const uint8_t* fsm_accept, int n_states,
                   const uint8_t* tok_bytes, const int32_t* tok_off, int vocab, int eos_id,
                   uint32_t* mask_bits, int mask_words, cudaStream_t stream) {
  if (n_states <= 0) return 0;
  if (mask_words * 32 < vocab) {
    set_last_error("fsm_build_mask: mask_words=%d too small for vocab=%d", mask_words, vocab);
    return -1;
  }
  dim3 grid((mask_words * 32 + 255) / 256, n_states);
  fsm_build_mask_kernel<<<grid, 256, 0, stream>>>(fsm_trans, fsm_accept, tok_bytes, tok_off, vocab,
                                                  eos_id, mask_bits, mask_words);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static float repetition_of(const SampleArgs& a) {
  return a.repetition_penalty > 0.f ? a.repetition_penalty : 1.f;  // a zeroed struct: off
}

bool penalties_active(const SampleArgs& a) {
  return a.presence_penalty != 0.f || a.frequency_penalty != 0.f || repetition_of(a) != 1.f;
}

int sample_greedy(const SampleArgs& a, cudaStream_t stream) {
  if (a.B <= 0) return 0;
  if (penalties_active(a)) {
    if (a.out_stride > kPenaltyMaxOutput) {
      set_last_error("sample: penalties support at most %d output tokens per row (max_new_tokens "
                     "= %d)", kPenaltyMaxOutput, a.out_stride);
      return -1;
    }
    if (a.slot_n_row_tok == nullptr || a.row_tokens == nullptr || a.row_tok_off == nullptr ||
        (a.n_prompt_prefix > 0 && a.prompt_prefix == nullptr) ||
        (a.n_prompt_suffix > 0 && a.prompt_suffix == nullptr)) {
      set_last_error("sample: penalties need the rows' prompt tokens");
      return -1;
    }
    PenaltyParams q;
    q.rep = repetition_of(a);
    q.rep_inv = 1.f / q.rep;
    q.freq = a.frequency_penalty;
    q.pres = a.presence_penalty;
    q.hash_size = 32;
    while (q.hash_size < 2 * a.out_stride) q.hash_size *= 2;
    q.zero_pass = std::signbit(a.frequency_penalty) || std::signbit(a.presence_penalty);
    const size_t smem = ((a.vocab + 31) / 32) * 4ull + q.hash_size * 8ull;
    if (smem > 48 * 1024)
      SB_CUDA_CHECK(cudaFuncSetAttribute(apply_penalties_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem)));
    apply_penalties_kernel<<<a.B, kPenaltyThreads, smem, stream>>>(a, q);
    SB_CUDA_CHECK(cudaGetLastError());
  }
  if (a.temperature > 0.f) {
    // ln(min_p) on the host, in double, rounded once to fp32
    const double min_p = std::min(a.min_p, 1.f);
    const float log_min_p = a.min_p > 0.f ? static_cast<float>(std::log(min_p)) : 0.f;
    sample_random_kernel<<<a.B, kSampleThreads, 0, stream>>>(a, log_min_p);
  } else
    sample_greedy_kernel<<<a.B, kSampleThreads, 0, stream>>>(a);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int prepare_decode(const int32_t* row_slot, const int32_t* slot_next_tok, const int32_t* slot_pos,
                   int32_t* tok_ids, int32_t* tok_pos, int32_t* tok_slot, int32_t* ctx_len, int B,
                   cudaStream_t stream) {
  if (B <= 0) return 0;
  prepare_decode_kernel<<<(B + 127) / 128, 128, 0, stream>>>(row_slot, slot_next_tok, slot_pos,
                                                             tok_ids, tok_pos, tok_slot, ctx_len, B);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
