// sutro_b200 — K3 (tensor-core path): causal varlen prefill attention on Hopper wgmma.
//
// A new token attends to [shared prefix | the row's own tokens].  Both live in DENSE row-major
// buffers here, except the own tokens of a row prefilled in chunks that earlier chunks wrote
// (its history, attn_prefill_chunked): those are gathered from the paged pool by warps 9-11.
// The dense sources:
// the fused QKV epilogue (gemm_wgmma.cu) leaves post-norm / post-RoPE K and V in the qkv
// activation buffer next to q, and the shared prefix's K/V are kept per layer in a small
// dense side buffer.  Dense rows are what TMA wants: every operand tile below is one or a
// few cp.async.bulk.tensor boxes that land in shared memory already in the wgmma canonical
// 128-byte-swizzled layout.  (The paged cache is still written by the epilogue: decode reads it.)
//
// Work item = (sequence, kv head, q tile).  A q tile packs QT = 128/G consecutive tokens x
// the G query heads of the kv head into 128 rows (row = token*G + head), so K/V are read once
// per GQA group and the causal frontier advances in QT-token steps.  At G = 5 that is 25 tokens
// in 125 rows; rows 125-127 are zero padding whose outputs are never stored, and a q tile's
// frontier can fall anywhere inside a KV block.  KV is consumed in blocks
// of up to 128 tokens: first the prefix blocks, then the row's own blocks up to the tile's
// diagonal.  Only the valid tokens (rounded up to 32-row TMA boxes) are loaded, and the MMAs
// cover the same 32, 64, 96 or 128 columns: each width is its own fully unrolled path (a
// data-dependent wgmma count would make ptxas serialise them).  P = 0 on the columns past the
// valid ones (selected, not multiplied, so garbage K rows cannot leak into P); the columns a
// narrower block drops would only have added zero products.  0 * V stays 0 only where V is
// finite, so the CALLER must keep the
// k/v columns of the qkv buffer and the prefix buffer finite in every row a 32-row box can reach
// past a sequence's last token (the engine zeroes both buffers when it allocates them).  Rows
// past the loaded ones hold an earlier block's V or the zeros the V ring starts with.
//
// Persistent CTA, 384 threads, one per SM:
//   warps 8-11  producer warpgroup (gives its registers to the consumers); warp 8 issues the
//               TMA loads: the Q tile, then per block the K and V tiles (2-stage rings)
//   warps 0-7   two consumer warpgroups, warpgroup c owns tile rows [64c, 64c+64):
//               S = Q K^T  (wgmma, both operands from shared memory, S in registers);
//               softmax in registers (a row lives in the four lanes of a quad): running max
//               with lazy rescale (threshold 2^8), exp2, P packed to bf16 A fragments;
//               O += P V   (wgmma, P from registers, V from shared memory MN-major);
//               epilogue O / l -> global.
// While one warpgroup runs its softmax the other one's MMAs keep the tensor cores busy.
//
// Results depend only on the sequence itself (block partition by absolute position, rescale
// decisions per row), never on which other sequences share the batch.
#include <algorithm>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace sb {

namespace {

constexpr int kTcThreads = 384;              // warps 0-7 consumers, warps 8-11 TMA producer
constexpr int kBlk = 128;                    // KV tokens per block
constexpr int kHalfBytes = 128 * 128;        // [128 rows][64 bf16] = 16 KiB, one d-half
constexpr int kTileBytes2 = 2 * kHalfBytes;  // 32 KiB: Q tile, K block, V block
constexpr int kBoxRows = 32;                 // K/V TMA box height
constexpr int kBoxBytes = kBoxRows * 128;    // 4 KiB
constexpr int kTcBarBytes = 256;
constexpr int kTcSmem = 5 * kTileBytes2 + kTcBarBytes + 1024;  // Q K[2] V[2] + barriers + align
constexpr float kRescaleThreshold = 8.0f;    // log2 units: P stays <= 2^8 before a forced rescale

// The Q tile of group size G: QT = 128 / G tokens x G heads.  G * QT = 128 rows for G = 1, 2,
// 4 and 8; at G = 5 the box {64, 5, 25} fills 125 rows and rows 125-127 are padding that no
// TMA load writes.  Q_FULL expects exactly the bytes of the two d-half boxes.
template <int G>
struct QTile {
  static constexpr int kTokens = 128 / G;
  static constexpr int kRows = G * kTokens;
  static constexpr uint32_t kBytes = 2u * 64u * G * kTokens * sizeof(__nv_bfloat16);
  static_assert(kBytes == 2u * kRows * 128u && kBytes <= kTileBytes2 && kBytes % 16 == 0,
                "the Q boxes must fill whole 128-byte rows of the Q tile");
};

// The history of a chunked prefill: each sequence's own tokens [0, hist) were prefilled by
// earlier calls and are read from the paged KV pool (kernels.h layout) of this layer.
struct TcHist {
  const __nv_bfloat16* kv_layer;
  const int32_t* page_table;
  int max_pages;
  const int32_t* seq_slot;
  const int32_t* seq_hist;
};

// Own positions are counted from the row's first own token: the q tile starts at own position
// hist + qt0, and the current call's qkv rows hold own positions [hist, hist + q_len).
struct TcGeom {
  int q_start, q_len, past, qt0, kvh;
  int hist, slot;
  int n_pre, n_blocks;
};

template <int G, bool kHist>
SB_DEVICE TcGeom tc_geom(int item, int hkv, const int32_t* __restrict__ items,
                         const int32_t* __restrict__ seq_q_start,
                         const int32_t* __restrict__ seq_q_len,
                         const int32_t* __restrict__ seq_past, const TcHist& hs) {
  constexpr int QT = 128 / G;
  TcGeom g;
  const int w = item / hkv;
  g.kvh = item - w * hkv;
  const int seq = items[2 * w];
  g.qt0 = items[2 * w + 1];
  g.q_start = seq_q_start[seq];
  g.q_len = seq_q_len[seq];
  g.past = seq_past[seq];
  g.hist = kHist ? hs.seq_hist[seq] : 0;
  g.slot = kHist ? hs.seq_slot[seq] : 0;
  g.n_pre = (g.past + kBlk - 1) / kBlk;
  const int own_end = g.hist + min(g.q_len, g.qt0 + QT);  // exclusive causal frontier of the tile
  g.n_blocks = g.n_pre + (own_end + kBlk - 1) / kBlk;
  return g;
}

// block b of an item: source (prefix / own), first token, tokens the MMA covers (multiple of 16).
// An own block that starts below hist lies wholly in the history (hist is a multiple of kBlk).
template <int G>
SB_DEVICE void tc_block(const TcGeom& g, int b, bool& is_pre, int& j0, int& n16) {
  constexpr int QT = 128 / G;
  is_pre = b < g.n_pre;
  int limit;
  if (is_pre) {
    j0 = b * kBlk;
    limit = g.past - j0;
  } else {
    j0 = (b - g.n_pre) * kBlk;
    limit = g.hist + min(g.q_len, g.qt0 + QT) - j0;
  }
  limit = min(limit, kBlk);
  n16 = (limit + 15) & ~15;
}

SB_DEVICE float ex2_approx(float x) {   // MUFU.EX2: 2^x, flushes denormals (x <= -126 -> 0)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

SB_DEVICE float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
SB_DEVICE float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <int G, bool kHist>
__global__ void __launch_bounds__(kTcThreads, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tm_q,    // 3-D (d, head, token) over qkv
                       const __grid_constant__ CUtensorMap tm_kv,   // 2-D (col, token) over qkv
                       const __grid_constant__ CUtensorMap tm_pre,  // 3-D (col, token, layer)
                       __nv_bfloat16* __restrict__ out, const int32_t* __restrict__ items,
                       int n_items_total, const int32_t* __restrict__ seq_q_start,
                       const int32_t* __restrict__ seq_q_len, const int32_t* __restrict__ seq_past,
                       int hq, int hkv, int layer, float scale_log2, const TcHist hs) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const uint32_t s_q = smem_u32(smem);                       // 32 KiB
  const uint32_t s_k = s_q + kTileBytes2;                    // 2 x 32 KiB
  const uint32_t s_v = s_k + 2 * kTileBytes2;                // 2 x 32 KiB
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * kTileBytes2);
  // H_GO: warp 8 hands a history block's freed stage to the gather warps (chunked prefill)
  enum { Q_FULL = 0, Q_EMPTY = 1, K_FULL = 2, K_EMPTY = 4, V_FULL = 6, V_EMPTY = 8, N_BARS = 10,
         H_GO = 10 };
  auto bar = [&](int i) { return smem_u32(&bars[i]); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_kv);
    tma_prefetch_desc(&tm_pre);
    for (int i = 0; i < N_BARS; ++i) {
      const bool from_consumers = i == Q_EMPTY || (i >= K_EMPTY && i < K_EMPTY + 2) ||
                                  (i >= V_EMPTY && i < V_EMPTY + 2);
      mbar_init(bar(i), from_consumers ? 8 : 1);  // consumer side: one arrival per warp
    }
    if constexpr (kHist) {
      mbar_init(bar(H_GO), 1);
      mbar_init(bar(H_GO + 1), 1);
    }
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < 2 * kTileBytes2 / 16; i += kTcThreads)
    asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(s_v + 16 * i), "r"(0) : "memory");
  if constexpr (QTile<G>::kRows < 128) {
    // Q padding rows: zero once, so that their S / P / O rows stay finite
    constexpr int kPad16 = (128 - QTile<G>::kRows) * 128 / 16;   // 16-byte chunks per d-half
    for (int i = threadIdx.x; i < 2 * kPad16; i += kTcThreads) {
      const int dh = i / kPad16;
      const uint32_t a = s_q + dh * kHalfBytes + QTile<G>::kRows * 128 + 16 * (i - dh * kPad16);
      asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(a), "r"(0) : "memory");
    }
  }
  fence_proxy_async_smem();   // the zeros are visible to the tensor cores' async proxy
  __syncthreads();

  if (warp >= 8) {
    // ===================== TMA producer =====================
    // At most two blocks ahead of the consumers: block g's stage frees once block g-2 is done.
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      uint32_t g = 0;  // global block counter of this CTA
      uint32_t n = 0;  // item counter of this CTA
      for (int item = blockIdx.x; item < n_items_total; item += gridDim.x, ++n) {
        const TcGeom ge =
            tc_geom<G, kHist>(item, hkv, items, seq_q_start, seq_q_len, seq_past, hs);
        mbar_wait_long(bar(Q_EMPTY), (n & 1) ^ 1);
        mbar_arrive_expect_tx(bar(Q_FULL), QTile<G>::kBytes);
        tma_load_3d(s_q, &tm_q, bar(Q_FULL), 0, ge.kvh * G, ge.q_start + ge.qt0);
        tma_load_3d(s_q + kHalfBytes, &tm_q, bar(Q_FULL), 64, ge.kvh * G, ge.q_start + ge.qt0);
        for (int b = 0; b < ge.n_blocks; ++b, ++g) {
          bool is_pre;
          int j0, n16;
          tc_block<G>(ge, b, is_pre, j0, n16);
          const uint32_t st = g & 1, ph = ((g >> 1) & 1) ^ 1;
          if (kHist && !is_pre && j0 < ge.hist) {
            // warps 9-11 gather this block once its stage is free.  Only this thread waits on
            // the EMPTY barriers, for every block in order, so no wait is ever two phases behind
            // or ahead; H_GO cannot be lapped either, since its next arrival on this stage needs
            // this block consumed, hence gathered.
            mbar_wait_long(bar(K_EMPTY + st), ph);
            mbar_wait_long(bar(V_EMPTY + st), ph);
            mbar_arrive(bar(H_GO + st));
            continue;
          }
          const int n32 = (n16 + kBoxRows - 1) / kBoxRows;
          const int kcol = is_pre ? ge.kvh * kHeadDim : (hq + ge.kvh) * kHeadDim;
          const int row0 = is_pre ? j0 : ge.q_start + j0 - ge.hist;
#pragma unroll
          for (int v_flow = 0; v_flow < 2; ++v_flow) {
            const int col = v_flow ? kcol + hkv * kHeadDim : kcol;
            const uint32_t full = bar((v_flow ? V_FULL : K_FULL) + st);
            const uint32_t base = (v_flow ? s_v : s_k) + st * kTileBytes2;
            mbar_wait_long(bar((v_flow ? V_EMPTY : K_EMPTY) + st), ph);
            mbar_arrive_expect_tx(full, n32 * 2 * kBoxBytes);
            for (int i = 0; i < n32; ++i) {
#pragma unroll
              for (int dh = 0; dh < 2; ++dh) {
                const uint32_t dst = base + dh * kHalfBytes + i * kBoxBytes;
                if (is_pre)
                  tma_load_3d(dst, &tm_pre, full, col + dh * 64, row0 + i * kBoxRows, layer);
                else
                  tma_load_2d(dst, &tm_kv, full, col + dh * 64, row0 + i * kBoxRows);
              }
            }
          }
        }
      }
    } else if (kHist && warp > 8) {
      // History blocks: 128 pool rows from 8 pages, 16-byte cp.async copies, each started when
      // warp 8 signals that the block's stage is free (H_GO).  Own token j sits at
      // position past + j; its pool row r = pos % 16 keeps chunk c at c ^ (r & 7), and its tile row
      // i = j - j0 wants chunk c & 7 of d-half c >> 3 at (c & 7) ^ (i & 7) (SWIZZLE_128B).  The two
      // XORs differ whenever past % 8 != 0, so every chunk is re-swizzled.  One thread per 96
      // completes the stage's FULL phase after all copies have landed and been fenced to the async
      // proxy; warp 8 skips these blocks, so each phase still has exactly one arrival.
      const int tid = threadIdx.x - 9 * 32;
      uint32_t g = 0, go_par = 0;  // bit st: parity of the next H_GO phase of stage st
      for (int item = blockIdx.x; item < n_items_total; item += gridDim.x) {
        const TcGeom ge =
            tc_geom<G, kHist>(item, hkv, items, seq_q_start, seq_q_len, seq_past, hs);
        for (int b = 0; b < ge.n_blocks; ++b, ++g) {
          bool is_pre;
          int j0, n16;
          tc_block<G>(ge, b, is_pre, j0, n16);
          if (is_pre || j0 >= ge.hist) continue;
          const uint32_t st = g & 1;
          mbar_wait_long(bar(H_GO + st), (go_par >> st) & 1);
          go_par ^= 1u << st;
          const int32_t* pt = hs.page_table + static_cast<size_t>(ge.slot) * hs.max_pages;
          for (int v_flow = 0; v_flow < 2; ++v_flow) {
            const uint32_t base = (v_flow ? s_v : s_k) + st * kTileBytes2;
            for (int idx = tid; idx < kBlk * 16; idx += 3 * 32) {
              const int i = idx >> 4, c = idx & 15;
              const int pos = ge.past + j0 + i;
              const int r = pos % kPageTokens;
              const __nv_bfloat16* src =
                  hs.kv_layer + kv_tile_offset(pt[pos / kPageTokens], hkv, ge.kvh, v_flow == 0) +
                  r * kHeadDim + kv_chunk(r, c) * 8;
              cp_async_16(base + (c >> 3) * kHalfBytes + i * 128 + (((c & 7) ^ (i & 7)) << 4), src,
                          true);
            }
            cp_async_commit();
            cp_async_wait<0>();
            fence_proxy_async_smem();
            named_bar_sync(1, 3 * 32);
            if (tid == 0) mbar_arrive(bar((v_flow ? V_FULL : K_FULL) + st));
          }
        }
      }
    }
    return;
  }

  // ===================== consumers (warps 0-7) =====================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const int q4 = lane & 3;
  const uint32_t s_qw = s_q + wg * 64 * 128;       // this warpgroup's 64 Q rows
  int t_in[2], h_in[2];                            // token / query head of the thread's 2 rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    t_in[h] = r / G;
    h_in[h] = r - t_in[h] * G;
  }
  uint32_t g = 0, n = 0;
  for (int item = blockIdx.x; item < n_items_total; item += gridDim.x, ++n) {
    const TcGeom ge = tc_geom<G, kHist>(item, hkv, items, seq_q_start, seq_q_len, seq_past, hs);
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float m_used[2] = {0.f, 0.f}, l_run[2] = {0.f, 0.f};   // l_run: this thread's partial sums
    mbar_wait(bar(Q_FULL), n & 1);
    for (int b = 0; b < ge.n_blocks; ++b, ++g) {
      bool is_pre;
      int j0, n16;
      tc_block<G>(ge, b, is_pre, j0, n16);
      const uint32_t st = g & 1, par = (g >> 1) & 1;
      // One block at MMA width W: the n16 valid columns rounded up to 32.  Each width is its own
      // unrolled path (a data-dependent wgmma count would be serialised by ptxas).  Columns in
      // [n16, W) are masked to P = 0 as before; the columns past W, which the full-width MMAs
      // used to cover, would only have added zero products, so O and l are unchanged.
      auto run_block = [&](auto width) {
        constexpr int W = decltype(width)::value;
        // ---- S = Q K^T (64 x W per warpgroup) ----
        float s[W / 2];
        mbar_wait(bar(K_FULL + st), par);
        wgmma_fence();
#pragma unroll
        for (int dh = 0; dh < 2; ++dh)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_ss_n(s, gmma_desc_k_sw128(s_qw + dh * kHalfBytes + 32 * k),
                       gmma_desc_k_sw128(s_k + st * kTileBytes2 + dh * kHalfBytes + 32 * k),
                       (dh | k) != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bar(K_EMPTY + st));
          if (b == ge.n_blocks - 1) mbar_arrive(bar(Q_EMPTY));
        }
        // ---- softmax: s[4j + 2h + e] is row h, column 8j + 2 q4 + e of the block ----
        uint32_t pa[W / 4];   // P as bf16x2: the A fragments of the W/16 K=16 steps of P.V
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // columns c of this block are valid for this row iff c < vlim
          const int vlim = min(is_pre ? ge.past - j0 : ge.hist + ge.qt0 + t_in[h] - j0 + 1, n16);
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < W / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * j + 2 * q4 + e < vlim) mx = fmaxf(mx, s[4 * j + 2 * h + e]);
          mx = quad_max(mx) * scale_log2;   // scale > 0: max commutes with the scaling
          if (b == 0) {
            m_used[h] = (mx == -INFINITY) ? 0.f : mx;
          } else if (mx > m_used[h] + kRescaleThreshold) {
            const float alpha = ex2_approx(m_used[h] - mx);
            m_used[h] = mx;
            l_run[h] *= alpha;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              o[4 * j + 2 * h] *= alpha;
              o[4 * j + 2 * h + 1] *= alpha;
            }
          }
          const float neg_m = -m_used[h];
          float ps = 0.f;
#pragma unroll
          for (int j = 0; j < W / 8; ++j) {
            const int c0 = 8 * j + 2 * q4;
            float p0 = ex2_approx(fmaf(s[4 * j + 2 * h], scale_log2, neg_m));
            float p1 = ex2_approx(fmaf(s[4 * j + 2 * h + 1], scale_log2, neg_m));
            p0 = c0 < vlim ? p0 : 0.f;
            p1 = c0 + 1 < vlim ? p1 : 0.f;
            ps += p0 + p1;
            // K step kk = j / 2: a0/a1 = rows 0/8 at k 2q4, a2/a3 = rows 0/8 at k 8 + 2q4
            pa[4 * (j >> 1) + 2 * (j & 1) + h] = pack_bf16x2(p0, p1);
          }
          l_run[h] += ps;
        }
        // ---- O += P V ----
        mbar_wait(bar(V_FULL + st), par);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < W / 16; ++kk) {
          const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
          wgmma_m64n128k16_rs_tb(
              o, a, gmma_desc_sw128(s_v + st * kTileBytes2 + kk * 2048, kHalfBytes, 1024));
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(V_EMPTY + st));
      };
      switch ((n16 - 1) >> 5) {  // n16 is in [16, 128]
        case 0: run_block(std::integral_constant<int, 32>{}); break;
        case 1: run_block(std::integral_constant<int, 64>{}); break;
        case 2: run_block(std::integral_constant<int, 96>{}); break;
        default: run_block(std::integral_constant<int, 128>{}); break;
      }
    }
    // ---- epilogue: O / l -> bf16 -> global ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float inv = 1.0f / quad_sum(l_run[h]);
      // a padding row's t_in is QT, the first token of the next q tile, which is not ours
      if constexpr (QTile<G>::kRows < 128) {
        if (t_in[h] >= QTile<G>::kTokens) continue;
      }
      const int q_own = ge.qt0 + t_in[h];
      if (q_own >= ge.q_len) continue;
      __nv_bfloat16* dst = out + static_cast<size_t>(ge.q_start + q_own) * (hq * kHeadDim) +
                           (ge.kvh * G + h_in[h]) * kHeadDim + 2 * q4;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) =
            pack_bf16x2(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
    }
  }
}

struct TcMaps {
  CUtensorMap q, kv, pre;
};

struct TcKey {
  const void* qkv;
  const void* pre;
  int t_rows, hq, hkv, pre_rows, n_layers;
  bool operator==(const TcKey& o) const {
    return qkv == o.qkv && pre == o.pre && t_rows == o.t_rows && hq == o.hq && hkv == o.hkv &&
           pre_rows == o.pre_rows && n_layers == o.n_layers;
  }
};
struct TcKeyHash {
  size_t operator()(const TcKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.qkv) * 0x9E3779B97F4A7C15ull;
    h ^= reinterpret_cast<size_t>(k.pre) + (static_cast<size_t>(k.t_rows) << 7) +
         (static_cast<size_t>(k.pre_rows) << 29) + k.hq * 131 + k.hkv * 17 + k.n_layers;
    return h;
  }
};

int tc_maps(const TcKey& key, TcMaps* out) {
  static std::mutex mu;
  static std::unordered_map<TcKey, TcMaps, TcKeyHash> cache;
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return 0;
    }
  }
  const int G = key.hq / key.hkv;
  const uint64_t ldq = static_cast<uint64_t>(key.hq + 2 * key.hkv) * kHeadDim;
  TcMaps m;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(kHeadDim), static_cast<uint64_t>(key.hq),
                              static_cast<uint64_t>(key.t_rows)};
    const uint64_t strides[2] = {kHeadDim * 2ull, ldq * 2ull};
    const uint32_t box[3] = {64u, static_cast<uint32_t>(G), static_cast<uint32_t>(128 / G)};
    if (encode_tmap_bf16(&m.q, key.qkv, 3, dims, strides, box)) return -1;
  }
  {
    const uint64_t dims[2] = {ldq, static_cast<uint64_t>(key.t_rows)};
    const uint64_t strides[1] = {ldq * 2ull};
    const uint32_t box[2] = {64u, static_cast<uint32_t>(kBoxRows)};
    if (encode_tmap_bf16(&m.kv, key.qkv, 2, dims, strides, box)) return -1;
  }
  {
    // the prefix side buffer may be absent (no shared prefix): map the qkv buffer instead so
    // that the descriptor is valid; it is never dereferenced when every past == 0
    const bool have = key.pre != nullptr && key.pre_rows > 0;
    const uint64_t cols = 2ull * key.hkv * kHeadDim;
    const uint64_t rows = have ? key.pre_rows : 1;
    const uint64_t dims[3] = {have ? cols : 64ull, rows,
                              static_cast<uint64_t>(have ? key.n_layers : 1)};
    const uint64_t strides[2] = {(have ? cols : ldq) * 2ull, (have ? cols : ldq) * 2ull * rows};
    const uint32_t box[3] = {64u, static_cast<uint32_t>(kBoxRows), 1u};
    if (encode_tmap_bf16(&m.pre, have ? key.pre : key.qkv, 3, dims, strides, box)) return -1;
  }
  std::lock_guard<std::mutex> g(mu);
  cache.emplace(key, m);
  *out = m;
  return 0;
}

int tc_num_sms() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

template <int G, bool kHist>
int launch_tc(const TcMaps& m, void* out, const int32_t* items, int n_items, const int32_t* qs,
              const int32_t* ql, const int32_t* past, int hq, int hkv, int layer, float scale,
              const TcHist& hs, cudaStream_t stream) {
  auto kern = attn_prefill_tc_kernel<G, kHist>;
  SB_SET_MAX_SMEM(kern, kTcSmem);
  const int total = n_items * hkv;
  const int grid = std::min(total, tc_num_sms());
  kern<<<grid, kTcThreads, kTcSmem, stream>>>(m.q, m.kv, m.pre, static_cast<__nv_bfloat16*>(out),
                                              items, total, qs, ql, past, hq, hkv, layer,
                                              scale * 1.4426950408889634f, hs);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

int attn_prefill_q_tile(int hq, int hkv) { return 128 / (hq / hkv); }

int attn_prefill_dense(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                       int prefix_rows, int n_layers, int layer, const int32_t* items, int n_items,
                       const int32_t* seq_q_start, const int32_t* seq_q_len,
                       const int32_t* seq_past, int hq, int hkv, float scale,
                       cudaStream_t stream) {
  if (n_items <= 0) return 0;
  if (layer < 0 || layer >= std::max(n_layers, 1)) {
    set_last_error("attn_prefill_dense: layer %d out of range", layer);
    return -1;
  }
  return dispatch_gqa("attn_prefill_dense", hq, hkv, [&](auto g) {
    TcMaps m;
    if (tc_maps(TcKey{qkv, prefix_kv, t_rows, hq, hkv, prefix_rows, n_layers}, &m)) return -1;
    return launch_tc<g.value, false>(m, out, items, n_items, seq_q_start, seq_q_len, seq_past,
                                     hq, hkv, prefix_kv ? layer : 0, scale, TcHist{}, stream);
  });
}

int attn_prefill_chunked(const void* qkv, int t_rows, void* out, const void* prefix_kv,
                         int prefix_rows, int n_layers, int layer, const int32_t* items,
                         int n_items, const int32_t* seq_q_start, const int32_t* seq_q_len,
                         const int32_t* seq_past, int hq, int hkv, float scale,
                         const void* kv_layer, const int32_t* page_table, int max_pages,
                         const int32_t* seq_slot, const int32_t* seq_hist, cudaStream_t stream) {
  if (n_items <= 0) return 0;
  if (layer < 0 || layer >= std::max(n_layers, 1)) {
    set_last_error("attn_prefill_chunked: layer %d out of range", layer);
    return -1;
  }
  if (!kv_layer || !page_table || max_pages <= 0 || !seq_slot || !seq_hist) {
    set_last_error("attn_prefill_chunked: the KV pool, page table and history arrays are required");
    return -1;
  }
  const TcHist hs{static_cast<const __nv_bfloat16*>(kv_layer), page_table, max_pages, seq_slot,
                  seq_hist};
  return dispatch_gqa("attn_prefill_chunked", hq, hkv, [&](auto g) {
    TcMaps m;
    if (tc_maps(TcKey{qkv, prefix_kv, t_rows, hq, hkv, prefix_rows, n_layers}, &m)) return -1;
    return launch_tc<g.value, true>(m, out, items, n_items, seq_q_start, seq_q_len, seq_past, hq,
                                    hkv, prefix_kv ? layer : 0, scale, hs, stream);
  });
}

int attn_prefill_hist_align(int hq, int hkv) {
  if (hkv <= 0 || hq % hkv != 0) return 0;
  const int G = hq / hkv;
  if (G != 1 && G != 2 && G != 4 && G != 5 && G != 8) return 0;  // the groups dispatch_gqa serves
  const int qt = attn_prefill_q_tile(hq, hkv);
  int a = kBlk, b = qt;
  while (b) {
    const int t = a % b;
    a = b;
    b = t;
  }
  return kBlk / a * qt;
}

}  // namespace sb
