// sutro_b200 — K2: paged-KV decode attention (one query token per sequence).
//
// HBM-bound: per generated token each sequence streams its whole K/V history
// once (ctx_len x 2 x hkv x 256 B per layer).  Design:
//   * one WARP per (sequence, kv head) pair, 4 pairs per CTA; the G = hq/hkv
//     query heads that share a KV head are processed together so K/V are read
//     from HBM exactly once (GQA).
//   * each warp streams its pair's pages through a private kDecStages-deep ring
//     of 8 KiB stages filled by cp.async.bulk (UBLKCP): one lane issues a single
//     flat 8 KiB copy per page (K tile + V tile of one head are contiguous in
//     the pool), completion arrives on an mbarrier.
//   * The pool stores tiles pre-swizzled (kernels.h), so the flat copy lands in
//     shared memory bank-conflict-free for ldmatrix / ldmatrix.trans.
//   * S = Q K^T and O += P V run on mma.sync m16n8k16 (bf16 in, fp32 acc) with
//     the G query heads as the (zero-padded) M rows; online softmax uses
//     quad-level warp shuffles; the warp normalises and writes its output
//     itself: no cross-warp merge and no block-wide barrier.
//   * Split-KV for long rows: a row of more than kDecodeSplitTokens tokens is cut at absolute
//     positions s * kDecodeSplitTokens into splits, one warp per (row, kv head, split).  Such a
//     warp writes its unnormalised fp32 partial (O, running max, sum) to a workspace, and a
//     merge kernel combines each row's splits in split order.  A row of at most
//     kDecodeSplitTokens tokens is one split: its warp runs the single-warp path above and
//     writes its output directly.  Either way a row's output depends on the row alone.
#include "common.cuh"
#include "kernels.h"

namespace sb {

namespace {

constexpr int kDecWarps = 4;
constexpr int kDecStages = 3;
constexpr int kStageBytes = 2 * kTileBytes;  // K tile + V tile = 8 KiB
constexpr int kDecSmem = kDecWarps * kDecStages * kStageBytes + 1024;

// Each warp owns a private ring of kDecStages stages of kStageBytes (`ring`) with one mbarrier
// per stage (`bars`); a stage holds one page.
SB_DEVICE void ring_init(uint64_t* bars, int lane) {
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kDecStages; ++s) mbar_init(smem_u32(&bars[s]), 1);
    fence_mbar_init();
  }
  __syncwarp();
}

// Lane 0: one flat bulk copy of the K and V tiles of kv head kvh of `page` into a stage.
SB_DEVICE void issue_page(const __nv_bfloat16* kv_layer, int page, int hkv, int kvh,
                          uint8_t* ring, uint64_t* bars, int stage) {
  const __nv_bfloat16* src = kv_layer + kv_tile_offset(page, hkv, kvh, true);
  const uint32_t bar = smem_u32(&bars[stage]);
  mbar_arrive_expect_tx(bar, kStageBytes);
  bulk_load_1d(smem_u32(ring + stage * kStageBytes), src, kStageBytes, bar);
}

// Q fragments of sequence b: rows = the G query heads of kv head kvh (row >= G is zero padding).
template <int G>
SB_DEVICE void load_q(const __nv_bfloat16* qkv, int b, int kvh, int hq, int hkv, int lane,
                      uint32_t (&qa)[8][2]) {  // [k-step][a0, a2]   (a1 = a3 = 0: rows 8..15 unused)
  const int ldq = (hq + 2 * hkv) * kHeadDim;
  const int qr = lane >> 2;
  const __nv_bfloat16* qp =
      qkv + static_cast<size_t>(b) * ldq + (kvh * G + qr) * kHeadDim + 2 * (lane & 3);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    if (qr < G) {
      qa[kk][0] = *reinterpret_cast<const uint32_t*>(qp + kk * 16);
      qa[kk][1] = *reinterpret_cast<const uint32_t*>(qp + kk * 16 + 8);
    } else {
      qa[kk][0] = 0u;
      qa[kk][1] = 0u;
    }
  }
}

// One page (tokens tile*16 ..) of the online softmax, from the stage at shared address ks:
// S = Q K^T, mask tokens >= L, rescale, O = O * alpha + P V.  o holds rows 0..7 only (c0, c1
// of each n-tile); m_run / l_run are the running max and sum of row lane/4.
SB_DEVICE void decode_tile(uint32_t ks, const uint32_t (&qa)[8][2], int tile, int L,
                           float scale_log2, int lane, float (&o)[16][2], float& m_run,
                           float& l_run) {
  const int lm = lane >> 3;  // ldmatrix: which 8x8 matrix this lane addresses
  const int lr = lane & 7;
  const uint32_t vs = ks + kTileBytes;

  // ---- S = Q K^T : 16 (padded heads) x 16 tokens ----
  float s0[4] = {0.f, 0.f, 0.f, 0.f};  // tokens 0..7
  float s1[4] = {0.f, 0.f, 0.f, 0.f};  // tokens 8..15
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const int tok = (lm >> 1) * 8 + lr;
    const int chunk = kk * 2 + (lm & 1);
    uint32_t b0, b1, b2, b3;
    ldmatrix_x4(ks + tok * 256 + (kv_chunk(tok, chunk) << 4), b0, b1, b2, b3);
    const uint32_t a[4] = {qa[kk][0], 0u, qa[kk][1], 0u};
    mma_bf16_16816(s0, a, b0, b1);
    mma_bf16_16816(s1, a, b2, b3);
  }
  // ---- online softmax on row lane/4 (values c0, c1 of both n-tiles) ----
  const int tok0 = tile * kPageTokens + 2 * (lane & 3);
  float sv[4] = {s0[0], s0[1], s1[0], s1[1]};
  if (tok0 >= L) sv[0] = -INFINITY;
  if (tok0 + 1 >= L) sv[1] = -INFINITY;
  if (tok0 + 8 >= L) sv[2] = -INFINITY;
  if (tok0 + 9 >= L) sv[3] = -INFINITY;
  float mx = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  const float m_new = fmaxf(m_run, mx);  // finite: every visited tile has >= 1 valid token
  const float alpha = exp2f((m_run - m_new) * scale_log2);
  float p[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = exp2f((sv[i] - m_new) * scale_log2);
  float ps = p[0] + p[1] + p[2] + p[3];
  ps += __shfl_xor_sync(0xffffffffu, ps, 1);
  ps += __shfl_xor_sync(0xffffffffu, ps, 2);
  l_run = l_run * alpha + ps;
  m_run = m_new;
  const uint32_t pa[4] = {pack_bf16x2(p[0], p[1]), 0u, pack_bf16x2(p[2], p[3]), 0u};

  // ---- O = O * alpha + P V ----
#pragma unroll
  for (int nt = 0; nt < 16; nt += 2) {
    const int tok = (lm & 1) * 8 + lr;
    const int chunk = nt + (lm >> 1);
    uint32_t b0, b1, b2, b3;
    ldmatrix_x4_trans(vs + tok * 256 + (kv_chunk(tok, chunk) << 4), b0, b1, b2, b3);
    float d0[4] = {o[nt][0] * alpha, o[nt][1] * alpha, 0.f, 0.f};
    float d1[4] = {o[nt + 1][0] * alpha, o[nt + 1][1] * alpha, 0.f, 0.f};
    mma_bf16_16816(d0, pa, b0, b1);
    mma_bf16_16816(d1, pa, b2, b3);
    o[nt][0] = d0[0];
    o[nt][1] = d0[1];
    o[nt + 1][0] = d1[0];
    o[nt + 1][1] = d1[1];
  }
}

// Partial of one (row, kv head, split) unit in the workspace: O[G][128], m[G], l[G] (fp32).
SB_DEVICE float* unit_partial(float* ws, int i, int kvh, int split, int hkv, int max_splits,
                              int G) {
  return ws + (static_cast<size_t>(i * hkv + kvh) * max_splits + split) * G * (kHeadDim + 2);
}

SB_DEVICE int n_splits_of(int L) { return (L + kDecodeSplitTokens - 1) / kDecodeSplitTokens; }

// Warps [0, n_split_units) are split units: unit u is (split row u / hkv / max_splits, kv head,
// split); split row i is batch row split_rows[i] (or i when split_rows is null).  They come first
// so that long rows start early.  The n_pairs warps after them are (row, kv head) pairs; a pair
// whose row has more than one split leaves it to the split units when there are any.
template <int G>
__global__ void __launch_bounds__(kDecWarps * 32)
attn_decode_warp_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                        const __nv_bfloat16* __restrict__ kv_layer,
                        const int32_t* __restrict__ page_table, int max_pages,
                        const int32_t* __restrict__ row_slot, const int32_t* __restrict__ ctx_len,
                        int n_pairs, int hq, int hkv, float scale_log2,
                        const int32_t* __restrict__ split_rows, int n_split_units, int max_splits,
                        float* __restrict__ ws) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~static_cast<uintptr_t>(127));
  __shared__ uint64_t full_bar[kDecWarps][kDecStages];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int pair = blockIdx.x * kDecWarps + warp;
  int b, kvh, split = 0, si = 0;
  const bool split_unit = pair < n_split_units;
  if (split_unit) {
    const int e = pair / hkv;
    kvh = pair - e * hkv;
    si = e / max_splits;
    split = e - si * max_splits;
    b = split_rows != nullptr ? split_rows[si] : si;
  } else {
    pair -= n_split_units;
    if (pair >= n_pairs) return;  // whole warp exits together; no block-wide barriers below
    b = pair / hkv;
    kvh = pair - b * hkv;
  }
  const int slot = row_slot[b];
  const int L = ctx_len[b];
  const int n_splits = n_splits_of(L);
  if (split_unit ? (n_splits == 1 || split >= n_splits) : (n_splits > 1 && n_split_units > 0))
    return;
  const int n_tiles = (L + kPageTokens - 1) / kPageTokens;
  // this warp's tiles: [t0, t1); a pair takes the whole row
  const int t0 = split_unit ? split * (kDecodeSplitTokens / kPageTokens) : 0;
  const int t1 = split_unit ? min(n_tiles, t0 + kDecodeSplitTokens / kPageTokens) : n_tiles;
  const int n_mine = t1 - t0;
  const int32_t* pt = page_table + static_cast<size_t>(slot) * max_pages + t0;

  uint8_t* my_smem = smem + warp * kDecStages * kStageBytes;
  ring_init(full_bar[warp], lane);
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kDecStages; ++s)
      if (s < n_mine) issue_page(kv_layer, pt[s], hkv, kvh, my_smem, full_bar[warp], s);
  }

  const int qr = lane >> 2;
  uint32_t qa[8][2];
  load_q<G>(qkv, b, kvh, hq, hkv, lane, qa);

  float o[16][2];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = 0.f;
  float m_run = -INFINITY, l_run = 0.f;

  for (int j = 0; j < n_mine; ++j) {
    const int stage = j % kDecStages;
    const uint32_t phase = (j / kDecStages) & 1;
    mbar_wait(smem_u32(&full_bar[warp][stage]), phase);
    decode_tile(smem_u32(my_smem + stage * kStageBytes), qa, t0 + j, L, scale_log2, lane, o,
                m_run, l_run);
    __syncwarp();
    const int next = j + kDecStages;
    if (lane == 0 && next < n_mine) {
      fence_proxy_async_smem();  // generic-proxy reads above vs async-proxy write below
      issue_page(kv_layer, pt[next], hkv, kvh, my_smem, full_bar[warp], stage);
    }
  }
  if (qr >= G) return;
  if (split_unit) {  // unnormalised partial; the merge kernel finishes the row
    float* u = unit_partial(ws, si, kvh, split, hkv, max_splits, G);
    float* op = u + qr * kHeadDim + 2 * (lane & 3);
#pragma unroll
    for (int nt = 0; nt < 16; ++nt)
      *reinterpret_cast<float2*>(op + nt * 8) = make_float2(o[nt][0], o[nt][1]);
    if ((lane & 3) == 0) {
      u[G * kHeadDim + qr] = m_run;
      u[G * kHeadDim + G + qr] = l_run;
    }
    return;
  }
  const float inv = 1.0f / l_run;
  __nv_bfloat16* op = out + static_cast<size_t>(b) * hq * kHeadDim + (kvh * G + qr) * kHeadDim +
                      2 * (lane & 3);
#pragma unroll
  for (int nt = 0; nt < 16; ++nt)
    *reinterpret_cast<__nv_bfloat162*>(op + nt * 8) =
        __floats2bfloat162_rn(o[nt][0] * inv, o[nt][1] * inv);
}

// One warp per (split row, query head): combines the row's splits in split order,
//   M = max_s m_s,  w_s = 2^((m_s - M) * scale_log2),  out = bf16(sum_s w_s O_s / sum_s w_s l_s),
// each lane owning 4 of the 128 dims.  Rows of one split were written by the decode kernel.
__global__ void __launch_bounds__(128)
attn_decode_merge_kernel(__nv_bfloat16* __restrict__ out, const int32_t* __restrict__ ctx_len,
                         const int32_t* __restrict__ split_rows, int n_split_rows, int max_splits,
                         int hq, int hkv, float scale_log2, const float* __restrict__ ws) {
  const int w = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_split_rows * hq) return;
  const int si = w / hq;
  const int h = w - si * hq;
  const int b = split_rows != nullptr ? split_rows[si] : si;
  const int n = min(n_splits_of(ctx_len[b]), max_splits);
  if (n <= 1) return;
  const int G = hq / hkv;
  const int kvh = h / G, g = h - kvh * G;
  const size_t unit = static_cast<size_t>(G) * (kHeadDim + 2);
  const float* u0 = ws + static_cast<size_t>(si * hkv + kvh) * max_splits * unit;
  float m = -INFINITY;
  for (int s = 0; s < n; ++s) m = fmaxf(m, u0[s * unit + G * kHeadDim + g]);
  float l = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
  for (int s = 0; s < n; ++s) {
    const float* u = u0 + s * unit;
    const float ws_s = exp2f((u[G * kHeadDim + g] - m) * scale_log2);
    l = fmaf(u[G * kHeadDim + G + g], ws_s, l);
    const float2 a = *reinterpret_cast<const float2*>(u + g * kHeadDim + 4 * lane);
    const float2 c = *reinterpret_cast<const float2*>(u + g * kHeadDim + 4 * lane + 2);
    o[0] = fmaf(a.x, ws_s, o[0]);
    o[1] = fmaf(a.y, ws_s, o[1]);
    o[2] = fmaf(c.x, ws_s, o[2]);
    o[3] = fmaf(c.y, ws_s, o[3]);
  }
  const float inv = 1.0f / l;
  __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(
      out + static_cast<size_t>(b) * hq * kHeadDim + h * kHeadDim + 4 * lane);
  op[0] = __floats2bfloat162_rn(o[0] * inv, o[1] * inv);
  op[1] = __floats2bfloat162_rn(o[2] * inv, o[3] * inv);
}

template <int G>
int launch(const void* qkv, void* out, const void* kv_layer, const int32_t* page_table,
           int max_pages, const int32_t* row_slot, const int32_t* ctx_len, int B, int hq, int hkv,
           float scale, const int32_t* split_rows, int n_split_rows, int max_splits, float* ws,
           cudaStream_t stream) {
  auto* q = static_cast<const __nv_bfloat16*>(qkv);
  auto* o = static_cast<__nv_bfloat16*>(out);
  auto* kv = static_cast<const __nv_bfloat16*>(kv_layer);
  const float scale_log2 = scale * 1.4426950408889634f;
  // One kernel for every batch size: a kernel chosen by the batch would make a row's greedy
  // tokens depend on its neighbours.
  auto kern = attn_decode_warp_kernel<G>;
  SB_SET_MAX_SMEM(kern, kDecSmem);
  const bool split = max_splits > 1 && n_split_rows > 0;
  const int n_split_units = split ? n_split_rows * hkv * max_splits : 0;
  const int n_warps = n_split_units + B * hkv;
  kern<<<(n_warps + kDecWarps - 1) / kDecWarps, kDecWarps * 32, kDecSmem, stream>>>(
      q, o, kv, page_table, max_pages, row_slot, ctx_len, B * hkv, hq, hkv, scale_log2,
      split_rows, n_split_units, max_splits, ws);
  SB_CUDA_CHECK(cudaGetLastError());
  if (split) {
    attn_decode_merge_kernel<<<(n_split_rows * hq + 3) / 4, 128, 0, stream>>>(
        o, ctx_len, split_rows, n_split_rows, max_splits, hq, hkv, scale_log2, ws);
    SB_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

}  // namespace

int attn_decode(const void* qkv, void* out, const void* kv_layer, const int32_t* page_table,
                int max_pages, const int32_t* row_slot, const int32_t* ctx_len, int B, int hq,
                int hkv, float scale, const int32_t* split_rows, int n_split_rows, int max_splits,
                float* ws, cudaStream_t stream) {
  if (B <= 0) return 0;
  return dispatch_gqa("attn_decode", hq, hkv, [&](auto g) {
    return launch<g.value>(qkv, out, kv_layer, page_table, max_pages, row_slot, ctx_len, B, hq,
                           hkv, scale, split_rows, n_split_rows, max_splits, ws, stream);
  });
}

}  // namespace sb
