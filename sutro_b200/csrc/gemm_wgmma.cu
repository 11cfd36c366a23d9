// sutro_b200 — K1: bf16 GEMM  D[M,N] = A[M,K] · W[N,K]^T  on Hopper wgmma tensor cores.
//
// Every projection of the transformer (QKV, O, gate/up, down, lm_head) has this
// shape: activations row-major [tokens, K], weights row-major [N, K] — both
// K-major, which is the native operand layout of wgmma with 128-byte swizzled
// shared-memory tiles.
//
// Kernel anatomy (persistent, warp-specialised, one CTA per SM, 384 threads):
//   warps 0-7  two consumer warpgroups: warpgroup c owns rows [64c, 64c+64) of the 128-row
//              tile and issues wgmma.m64nBLOCK_Nk16 (four per 64-element K block) straight
//              from the shared-memory ring, accumulating in registers; one K block stays in
//              flight while the next is issued.  The accumulators are rounded into the
//              warpgroup's 64-row slab of a staging buffer.  For the store and residual
//              epilogues the warpgroup finishes the slab itself and one thread stores it with
//              TMA; for SwiGLU and QKV (a CTA with more than one tile, K >= 2048) it writes
//              bf16(acc) and hands the slab to the epilogue warps.  Either way it goes on to the
//              next tile's mainloop while the slab drains.
//   warps 8-11 producer warpgroup (gives its registers to the consumers); warp 8 issues the
//              cp.async.bulk.tensor 2-D loads of A (128x64) and W (BLOCK_N x 64) tiles into a
//              kStages-deep ring and runs ahead into the next tile while the consumers are in
//              their epilogue.  For RESIDUAL_BF16, warp 9 loads each slab's residual tile into
//              the staging buffer by TMA as soon as the slab's previous store has read it out,
//              so the load overlaps the tile's mainloop.  For SwiGLU and QKV, warps 9-11 are
//              the epilogue warps: they run the epilogue math in place in each handed-over slab
//              and store it, under the consumers' next mainloop (slab_full / slab_free
//              mbarriers pass each slab back and forth).
//
// Fused epilogues (rounding points mirror the bf16 oracle, oracle/model_ref.py):
//   STORE_BF16     D = bf16(acc)
//   RESIDUAL_BF16  D = bf16(bf16(acc) + R)           (O-proj / down-proj + residual)
//   SWIGLU_BF16    D[:, j] = bf16(silu(bf16(acc[2j])) * bf16(acc[2j+1]))
//                  (gate/up weights interleaved row-wise; output has N/2 columns)
//   STORE_F32      D = acc                             (lm_head logits; stored from the registers:
//                  its 128 x 256 fp32 tile does not fit beside the ring)
//   QKV_ROPE       q/k RMSNorm + RoPE, K/V into the paged cache and into their columns of D
//                  (the dense copy the prefill attention reads; see qkv_head_epilogue)
// TMA clips every store and residual load at the tensor map's dims (M rows, N or N/2 columns),
// so rows >= M and columns past N are never written.
#include <algorithm>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace sb {

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 bf16 = 128 B = one swizzle span
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kGemmThreads = 32 * (kConsumerWarps + 4);

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // The limit is 227 KiB per block: ~192 KiB of ring beside the staging buffer for the 64- and
  // 128-wide tiles; the 256-wide tile gives up its fourth stage to stage the whole tile.
  static constexpr int kStages = (BLOCK_N == 256) ? 3 : (BLOCK_N == 128 ? 6 : 8);
  static constexpr int kSlabBytes = 64 * BLOCK_N * 2;   // one warpgroup's 64 rows, bf16
  static constexpr int kBarBytes = 256;
  static constexpr int kSmemBytes =
      kStages * kStageBytes + 2 * kSlabBytes + kBarBytes + 1024;   // +align slack
  static_assert(kSmemBytes <= 232448, "shared memory per block");
};

// The bf16 output of one tile: kCols columns (N/2 per tile for SwiGLU), staged and stored as
// boxes of 64 rows x kBoxCols columns.
template <int BLOCK_N, int EPI>
struct EpiCfg {
  static constexpr int kCols = EPI == EPI_SWIGLU_BF16 ? BLOCK_N / 2 : BLOCK_N;
  static constexpr int kBoxCols = kCols < 64 ? kCols : 64;
  static constexpr int kBoxes = kCols / kBoxCols;
  static constexpr int kBoxBytes = 64 * kBoxCols * 2;
};

// Byte offset of (row r, column c) in a staging slab: boxes of 64 rows x BOX_COLS columns back
// to back, each in the TMA swizzle of its row width (128-byte rows: SWIZZLE_128B, 64-byte rows:
// SWIZZLE_64B).  The swizzle also puts the 16 bytes a quad writes in each of eight consecutive
// rows into different banks.
template <int BOX_COLS>
SB_DEVICE uint32_t stage_off(int r, int c) {
  const uint32_t off = r * (BOX_COLS * 2) + (c % BOX_COLS) * 2;
  return (c / BOX_COLS) * (64 * BOX_COLS * 2) +
         (off ^ (((off >> 7) & (BOX_COLS == 64 ? 7 : 3)) << 4));
}

template <int BN>
SB_DEVICE void wgmma_ss(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 64) wgmma_m64n64k16_ss(d, adesc, bdesc, 1);
  else if constexpr (BN == 128) wgmma_m64n128k16_ss(d, adesc, bdesc, 1);
  else wgmma_m64n256k16_ss(d, adesc, bdesc, 1);
}

// Tile rasterisation: consecutive tile ids sweep all N tiles of a group of GM row-tiles
// before moving on, so the CTAs running concurrently share a [GM*128, K] slab of A and a
// slab of W that both stay in L2 (M-fastest order would re-read A from HBM once per N tile).
SB_DEVICE void tile_to_mn(int GM, int tile, int num_m, int num_n, int& m_blk, int& n_blk) {
  const int group_tiles = GM * num_n;
  const int g = tile / group_tiles;
  const int first_m = g * GM;
  const int gm = min(GM, num_m - first_m);
  const int within = tile - g * group_tiles;
  m_blk = first_m + within % gm;
  n_blk = within / gm;
}

// The thread's accumulators: acc[4j + 2h + e] is row 8h of the thread's rows, column
// 8j + 2 * (lane % 4) + e of the tile.

// bf16(silu(g) * u) of the bf16-rounded gate and up values
SB_DEVICE uint16_t swiglu_bf16(float g, float u) {
  const float s = bf16_round(g / (1.0f + __expf(-g)));
  return __bfloat16_as_ushort(__float2bfloat16_rn(s * u));
}

// STORE_BF16, SWIGLU_BF16, RESIDUAL_BF16 -> the warpgroup's staging slab; srow is the slab row
// of the thread's first row, q = lane % 4.  For RESIDUAL_BF16 the slab already holds R (loaded
// by TMA), which is read and overwritten in place: D = bf16(bf16(acc) + R).
template <int BLOCK_N, int EPI>
SB_DEVICE void epilogue_stage(const float (&acc)[BLOCK_N / 2], uint32_t slab, int srow, int q) {
  using Epi = EpiCfg<BLOCK_N, EPI>;
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if constexpr (EPI == EPI_SWIGLU_BF16) {
        // gate/up columns 2c, 2c + 1 give output column c = 4j + q
        st_shared_b16(slab + stage_off<Epi::kBoxCols>(srow + 8 * h, 4 * j + q),
                      swiglu_bf16(bf16_round(v0), bf16_round(v1)));
      } else {
        const uint32_t a = slab + stage_off<64>(srow + 8 * h, 8 * j + 2 * q);
        if constexpr (EPI == EPI_RESIDUAL_BF16) {
          const float2 rv = unpack_bf16x2(ld_shared_b32(a));
          st_shared_b32(a, pack_bf16x2(bf16_round(v0) + rv.x, bf16_round(v1) + rv.y));
        } else {
          st_shared_b32(a, pack_bf16x2(v0, v1));
        }
      }
    }
  }
}

// STORE_F32 (rows row0 and row0 + 8, columns col0 + 8j + {0, 1}; col0 includes 2 * (lane % 4)).
template <int BLOCK_N>
SB_DEVICE void epilogue_store_f32(const float (&acc)[BLOCK_N / 2], float* __restrict__ d_out,
                                  int row0, int col0, int M, int N, int ldd) {
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int col = col0 + 8 * j;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (col < N && row < M)
        *reinterpret_cast<float2*>(d_out + static_cast<size_t>(row) * ldd + col) =
            make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

// ---------------------------------------------------------------------------
// EPI_QKV_ROPE: per 128-column head, each row gets exactly what rope_kv_kernel (norm_rope.cu)
// does to the stored bf16 tensor — bf16 rounding of the projection, optional per-head RMSNorm,
// rotate-half RoPE with bf16 op-by-op rounding — then every head goes to the staging slab (q
// heads for the qkv buffer; k/v heads for their columns of it, the dense copy the prefill
// attention reads, stored only with write_dense) and k/v heads straight from the registers into
// the swizzled KV page as well (the page of each row is its own).  A row's head is spread over the four lanes of a
// quad (32 dims each); dim d and its RoPE partner d + 64 sit in the same thread, so only the
// sum of squares needs two shuffles.
// ---------------------------------------------------------------------------
struct QkvRowMeta {
  int pos, r;
  size_t page;
};

SB_DEVICE void qkv_row_meta(const QkvEpiArgs& ea, int row, bool row_ok, QkvRowMeta& rm) {
  rm.pos = 0, rm.r = 0, rm.page = 0;
  if (row_ok) {
    rm.pos = ea.tok_pos[row];
    const int slot = ea.tok_slot[row];
    rm.page = static_cast<size_t>(kv_page(ea.page_table, ea.max_pages, slot, rm.pos));
    rm.r = rm.pos % kPageTokens;
  }
}

// One row of one head.  u[jj] holds dims 8jj + 2q, +1 of the head (q = lane % 4; the quad holds
// the row's 128 dims), the bf16 rounding of the projection.  The result goes to the staging slab
// at (srow, col0 + d) and, for a k/v head, to the row's KV page.  Every lane of the warp calls it
// (the sum of squares is reduced over the quad); with ok = false (row >= M, or a head past N) it
// writes nothing.
SB_DEVICE void qkv_head_epilogue(const uint32_t (&u)[16], const QkvEpiArgs& ea,
                                 const QkvRowMeta& rm, int head, bool ok, uint32_t slab, int srow,
                                 int col0) {
  const int q = threadIdx.x & 3;
  const bool is_q = head < ea.hq;
  const bool is_k = !is_q && head < ea.hq + ea.hkv;
  const __nv_bfloat16* nw =
      static_cast<const __nv_bfloat16*>(is_q ? ea.q_norm_w : (is_k ? ea.k_norm_w : nullptr));
  // Packed bf16x2 arithmetic: a product of two bf16 values is exact in fp32, so HMUL2.BF16
  // (one rounding) equals "fp32 multiply, round to bf16" — the rounding points of the unfused
  // kernel (norm_rope.cu) and of the oracle; sums are HADD2.BF16 (exact sum, one rounding).
  // explicit .rn forms: ptxas must not contract mul + add/sub into one fused (singly rounded) FMA
  auto mul2 = [](uint32_t a, uint32_t b) {
    uint32_t d;
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
  };
  auto add2 = [](uint32_t a, uint32_t b) {
    uint32_t d;
    asm("add.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
  };
  auto sub2 = [](uint32_t a, uint32_t b) {
    uint32_t d;
    asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
  };
  float ss = 0.f;
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) {
    const float2 f = unpack_bf16x2(u[jj]);
    ss += f.x * f.x + f.y * f.y;
  }
  ss += __shfl_xor_sync(0xffffffffu, ss, 1);
  ss += __shfl_xor_sync(0xffffffffu, ss, 2);
  if (!ok) return;
  const float rstd = nw != nullptr ? rsqrtf(ss / static_cast<float>(kHeadDim) + ea.eps) : 1.f;
  // K/V page row; chunk c of the row is stored at c ^ swz: kv_chunk(r, c) == c ^ kv_chunk(r, 0),
  // taken out of the loop below
  __nv_bfloat16* kv_lo = nullptr;
  int swz = 0;
  if (!is_q) {
    const int kvh = is_k ? (head - ea.hq) : (head - ea.hq - ea.hkv);
    kv_lo = static_cast<__nv_bfloat16*>(ea.kv_layer) +
            kv_tile_offset(rm.page, ea.hkv, kvh, is_k) + rm.r * kHeadDim;
    swz = kv_chunk(rm.r, 0);
  }
  const __nv_bfloat16* cosr =
      static_cast<const __nv_bfloat16*>(ea.cos_tab) + static_cast<size_t>(rm.pos) * 64;
  const __nv_bfloat16* sinr =
      static_cast<const __nv_bfloat16*>(ea.sin_tab) + static_cast<size_t>(rm.pos) * 64;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {   // dims d, d+1 of the low half and their +64 partners
    const int d = 8 * jj + 2 * q;
    uint32_t lo = u[jj], hi = u[jj + 8];
    if (nw != nullptr) {   // w * bf16(x * rstd): rstd is fp32, so that product is fp32
      const float2 a = unpack_bf16x2(lo), b = unpack_bf16x2(hi);
      lo = mul2(*reinterpret_cast<const uint32_t*>(nw + d), pack_bf16x2(a.x * rstd, a.y * rstd));
      hi = mul2(*reinterpret_cast<const uint32_t*>(nw + 64 + d),
                pack_bf16x2(b.x * rstd, b.y * rstd));
    }
    if (is_q || is_k) {
      // out[i] = x[i]*cos - x[i+64]*sin ; out[i+64] = x[i+64]*cos + x[i]*sin (bf16 op by op)
      const uint32_t c = *reinterpret_cast<const uint32_t*>(cosr + d);
      const uint32_t s = *reinterpret_cast<const uint32_t*>(sinr + d);
      const uint32_t x = lo, y = hi;
      lo = sub2(mul2(x, c), mul2(y, s));
      hi = add2(mul2(y, c), mul2(x, s));
    }
    st_shared_b32(slab + stage_off<64>(srow, col0 + d), lo);
    st_shared_b32(slab + stage_off<64>(srow, col0 + 64 + d), hi);
    if (!is_q) {
      // the dense prefill attention reads the new tokens' K/V from the qkv buffer through TMA
      // (attn_prefill_tc.cu); decode reads this paged copy
      *reinterpret_cast<uint32_t*>(kv_lo + ((jj ^ swz) << 3) + 2 * q) = lo;
      *reinterpret_cast<uint32_t*>(kv_lo + (((jj + 8) ^ swz) << 3) + 2 * q) = hi;
    }
  }
}

// ---------------------------------------------------------------------------
// Epilogue warps (warps 9-11, SWIGLU_BF16 and QKV_ROPE): the consumers leave bf16(acc) in their
// slab (the STORE_BF16 staging), and these 96 threads finish it in place.
// ---------------------------------------------------------------------------
constexpr int kEpiWarp0 = kProducerWarp + 1;
constexpr int kEpiThreads = 96;
constexpr int kEpiBar = 3;       // named barrier of the epilogue warps (1, 2: the consumers')
constexpr int kQkvPasses = 3;    // 24 quads x 3 passes cover the slab's 64 rows

// The slab row of epilogue quad `quad` (0..23) in pass i; rows >= 64 (the whole of warp 11 in
// the last pass) have no work.
SB_DEVICE int qkv_pass_row(int i, int quad) { return 24 * i + quad; }

// QKV_ROPE: quad g takes slab rows g, g + 24, g + 48 and, in each, every head of the tile; lane
// q loads the 16 words the consumer layout gives lane q, so qkv_head_epilogue sees the same
// values in the same lanes.  Every lane reads its words before it writes them back, and no lane
// touches another's.
template <int BLOCK_N>
SB_DEVICE void qkv_slab_epilogue(const QkvEpiArgs& ea, const QkvRowMeta (&rm)[kQkvPasses],
                                 uint32_t slab, int row_base, int n_blk, int M, int N, int et) {
  const int quad = et >> 2, q = et & 3;
#pragma unroll
  for (int i = 0; i < kQkvPasses; ++i) {
    const int srow = qkv_pass_row(i, quad);
    if (srow >= 64) continue;   // warp-uniform
#pragma unroll
    for (int hh = 0; hh < BLOCK_N / 128; ++hh) {
      const int head = (n_blk * BLOCK_N) / kHeadDim + hh;
      uint32_t u[16];
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        u[jj] = ld_shared_b32(slab + stage_off<64>(srow, 128 * hh + 8 * jj + 2 * q));
      qkv_head_epilogue(u, ea, rm[i], head, head * kHeadDim < N && row_base + srow < M, slab,
                        srow, 128 * hh);
    }
  }
}

// SWIGLU_BF16: item (row r, k) turns input columns [16k, 16k + 16) (8 interleaved gate/up pairs)
// into output columns [8k, 8k + 8), one 16-byte chunk.  The output overwrites the input in place:
// output chunk k of row r lies on input chunk k of row r (BLOCK_N >= 128) or on input row r / 2
// (BLOCK_N = 64, 64-byte output rows), which items of the same or an earlier row read.  So the
// items run in row-major passes, and in each pass every input is read before the barrier and
// every output written after it.
template <int BLOCK_N>
SB_DEVICE void swiglu_slab_epilogue(uint32_t slab, int et) {
  using Epi = EpiCfg<BLOCK_N, EPI_SWIGLU_BF16>;
  constexpr int kChunks = BLOCK_N / 16;   // output chunks per row
  constexpr int kItems = 64 * kChunks;
  auto pair = [](uint32_t w0, uint32_t w1) {
    const float2 a = unpack_bf16x2(w0), b = unpack_bf16x2(w1);
    return static_cast<uint32_t>(swiglu_bf16(a.x, a.y)) |
           (static_cast<uint32_t>(swiglu_bf16(b.x, b.y)) << 16);
  };
#pragma unroll 1
  for (int base = 0; base < kItems; base += kEpiThreads) {
    const int item = base + et;
    const int r = item / kChunks, k = item % kChunks;
    uint4 in0, in1;
    if (item < kItems) {
      in0 = ld_shared_v4(slab + stage_off<64>(r, 16 * k));
      in1 = ld_shared_v4(slab + stage_off<64>(r, 16 * k + 8));
    }
    named_bar_sync(kEpiBar, kEpiThreads);
    if (item < kItems)
      st_shared_v4(slab + stage_off<Epi::kBoxCols>(r, 8 * k),
                   make_uint4(pair(in0.x, in0.y), pair(in0.z, in0.w), pair(in1.x, in1.y),
                              pair(in1.z, in1.w)));
  }
}

// TMA store of one staged slab (rows [row, row + 64) of the tile) into the thread's bulk group.
template <int BLOCK_N, int EPI>
SB_DEVICE void store_slab(const CUtensorMap* tm_d, uint32_t slab, int row, int n_blk, int M,
                          int N, const QkvEpiArgs& ea) {
  using Epi = EpiCfg<BLOCK_N, EPI>;
  const int n_out = EPI == EPI_SWIGLU_BF16 ? N / 2 : N;
  for (int b = 0; b < Epi::kBoxes; ++b) {
    const int col = n_blk * Epi::kCols + b * Epi::kBoxCols;
    // decode (write_dense = 0) leaves the K/V columns of the qkv buffer untouched
    const bool want = EPI != EPI_QKV_ROPE || ea.write_dense || col / kHeadDim < ea.hq;
    if (row < M && col < n_out && want) tma_store_2d(tm_d, slab + b * Epi::kBoxBytes, col, row);
  }
  bulk_commit_group();
}

// EPI_WARPS (SWIGLU_BF16 and QKV_ROPE only): the epilogue warps finish and store each slab, and
// the consumers only write bf16(acc); otherwise the consumers run the whole epilogue.
template <int BLOCK_N, int EPI, bool EPI_WARPS>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tm_a,
                    const __grid_constant__ CUtensorMap tm_b,
                    const __grid_constant__ CUtensorMap tm_d,   // bf16 output (not STORE_F32)
                    const __grid_constant__ CUtensorMap tm_r,   // residual (RESIDUAL_BF16)
                    float* __restrict__ d_f32, int M, int N, int K, int ldd, int ea_gm,
                    const QkvEpiArgs ea) {
  using Cfg = GemmCfg<BLOCK_N>;
  using Epi = EpiCfg<BLOCK_N, EPI>;
  constexpr bool kStaged = EPI != EPI_STORE_F32;
  static_assert(!EPI_WARPS || EPI == EPI_SWIGLU_BF16 || EPI == EPI_QKV_ROPE,
                "epilogue warps run SwiGLU and QKV only");
  // setmaxnreg moves registers between the warpgroups within what the block was launched with
  // (168 per thread, from __launch_bounds__): 2 x consumer + producer <= 3 x 168, or the
  // consumers' setmaxnreg.inc waits forever.  The epilogue warps need more than the loaders, the
  // consumers' bf16 store less than the fused math they no longer run.
  constexpr int kProducerRegs = EPI_WARPS ? 120 : 40;
  constexpr int kConsumerRegs = EPI_WARPS ? 192 : 232;
  static_assert(2 * kConsumerRegs + kProducerRegs <= 3 * 168, "registers of the block");
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* staging = smem + Cfg::kStages * Cfg::kStageBytes;   // two warpgroup slabs
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + 2 * Cfg::kSlabBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;
  uint64_t* slab_free = bars + 2 * Cfg::kStages;   // per slab: its last store has read it out
  uint64_t* resid_full = slab_free + 2;            // per slab: the tile's residual has landed
  uint64_t* slab_full = resid_full + 2;            // per slab: bf16(acc) is staged (EPI_WARPS)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    if constexpr (kStaged) tma_prefetch_desc(&tm_d);
    if constexpr (EPI == EPI_RESIDUAL_BF16) tma_prefetch_desc(&tm_r);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), kConsumerWarps);
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(smem_u32(&slab_free[c]), 1);
      mbar_init(smem_u32(&resid_full[c]), 1);
      if constexpr (EPI_WARPS) mbar_init(smem_u32(&slab_full[c]), kConsumerWarps / 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_m = (M + kBlockM - 1) / kBlockM;
  const int num_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = num_m * num_n;
  const int num_k = K / kBlockK;

  if (warp >= kProducerWarp) {
    // ===== TMA producer =====
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kProducerWarp && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_to_mn(ea_gm, tile, num_m, num_n, m_blk, n_blk);
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait_long(smem_u32(&empty_bar[stage]), phase ^ 1);
          const uint32_t fb = smem_u32(&full_bar[stage]);
          const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
          mbar_arrive_expect_tx(fb, Cfg::kStageBytes);
          tma_load_2d(sa, &tm_a, fb, kb * kBlockK, m_blk * kBlockM);
          tma_load_2d(sa + Cfg::kABytes, &tm_b, fb, kb * kBlockK, n_blk * BLOCK_N);
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (EPI == EPI_RESIDUAL_BF16 && warp == kProducerWarp + 1 && lane == 0) {
      // residual loader: R of each slab, as soon as the slab's previous store has read it out.
      // In place (R == D, as the engine runs it) is safe: tiles are disjoint, and a tile's R is
      // loaded before its D is stored.  Boxes wholly past M or N are not loaded.
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        int m_blk, n_blk;
        tile_to_mn(ea_gm, tile, num_m, num_n, m_blk, n_blk);
        for (int c = 0; c < 2; ++c) {
          const int row = m_blk * kBlockM + 64 * c;
          const uint32_t bar = smem_u32(&resid_full[c]);
          const uint32_t dst = smem_u32(staging + c * Cfg::kSlabBytes);
          int boxes = 0;
          if (row < M) boxes = min(Epi::kBoxes, (N - n_blk * BLOCK_N + 63) / 64);
          mbar_wait_long(smem_u32(&slab_free[c]), (it & 1) ^ 1);
          mbar_arrive_expect_tx(bar, boxes * Epi::kBoxBytes);
          for (int b = 0; b < boxes; ++b)
            tma_load_2d(dst + b * Epi::kBoxBytes, &tm_r, bar, n_blk * BLOCK_N + 64 * b, row);
        }
      }
    } else if (EPI_WARPS && warp >= kEpiWarp0) {
      // epilogue warps: each slab as the consumers hand it over (slab_full), in tile order;
      // once its stores have read it out, it goes back to them (slab_free)
      const int et = threadIdx.x - 32 * kEpiWarp0;
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        int m_blk, n_blk;
        tile_to_mn(ea_gm, tile, num_m, num_n, m_blk, n_blk);
        for (int c = 0; c < 2; ++c) {
          const int row_base = m_blk * kBlockM + 64 * c;
          const uint32_t slab = smem_u32(staging + c * Cfg::kSlabBytes);
          QkvRowMeta rm[kQkvPasses];
          if constexpr (EPI == EPI_QKV_ROPE) {   // overlaps the wait for the slab
#pragma unroll
            for (int i = 0; i < kQkvPasses; ++i) {
              const int srow = qkv_pass_row(i, et >> 2);
              qkv_row_meta(ea, row_base + srow, srow < 64 && row_base + srow < M, rm[i]);
            }
          }
          mbar_wait_long(smem_u32(&slab_full[c]), it & 1);
          if constexpr (EPI == EPI_QKV_ROPE) {
            qkv_slab_epilogue<BLOCK_N>(ea, rm, slab, row_base, n_blk, M, N, et);
          } else {
            swiglu_slab_epilogue<BLOCK_N>(slab, et);
          }
          fence_proxy_async_smem();   // this thread's slab writes, before the async proxy reads them
          named_bar_sync(kEpiBar, kEpiThreads);
          if (et == 0) {
            store_slab<BLOCK_N, EPI>(&tm_d, slab, row_base, n_blk, M, N, ea);
            bulk_wait_group_read<0>();
            mbar_arrive(smem_u32(&slab_free[c]));
          }
        }
      }
      // the stores must finish reading shared memory before the block exits
      if (et == 0) bulk_wait_group<0>();
    }
    return;
  }

  // ===== consumers: MMA + epilogue =====
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2;   // rows [64 wg, 64 wg + 64) of the tile
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t slab = smem_u32(staging + wg * Cfg::kSlabBytes);
  const int srow = (warp & 3) * 16 + (lane >> 2);   // slab row of the thread's first row
  // issues the warpgroup's TMA stores, and waits for them (bulk groups belong to one thread)
  const bool leader = (threadIdx.x & 127) == 0;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    int m_blk, n_blk;
    tile_to_mn(ea_gm, tile, num_m, num_n, m_blk, n_blk);
    const int row0 = m_blk * kBlockM + wg * 64 + srow;
    QkvRowMeta rm[2];
    if constexpr (EPI == EPI_QKV_ROPE && !EPI_WARPS) {   // overlaps the mainloop's loads
      qkv_row_meta(ea, row0, row0 < M, rm[0]);
      qkv_row_meta(ea, row0 + 8, row0 + 8 < M, rm[1]);
    }
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < num_k; ++kb) {
      mbar_wait(smem_u32(&full_bar[stage]), phase);
      const uint32_t sa = smem0 + stage * Cfg::kStageBytes + wg * 64 * 128;
      const uint32_t sb = smem0 + stage * Cfg::kStageBytes + Cfg::kABytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)
        wgmma_ss<BLOCK_N>(acc, gmma_desc_k_sw128(sa + 32 * k), gmma_desc_k_sw128(sb + 32 * k));
      wgmma_commit();
      if constexpr (EPI == EPI_RESIDUAL_BF16) {
        // with the first K block issued, hand the slab to the residual loader once the previous
        // tile's store has read it out
        if (kb == 0 && it > 0 && leader) {
          bulk_wait_group_read<0>();
          mbar_arrive(smem_u32(&slab_free[wg]));
        }
      }
      // the previous K block has retired once at most this one is in flight: free its stage
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
      }
      prev = stage;
      if (++stage == Cfg::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
    }
    if constexpr (EPI == EPI_STORE_F32) {
      epilogue_store_f32<BLOCK_N>(acc, d_f32, row0, n_blk * BLOCK_N + 2 * (lane & 3), M, N, ldd);
      continue;
    }
    if constexpr (EPI_WARPS) {
      // the epilogue warps hand the slab back once its previous store has read it out; stage
      // bf16(acc), hand it over and go straight into the next tile
      mbar_wait(smem_u32(&slab_free[wg]), (it & 1) ^ 1);
      epilogue_stage<BLOCK_N, EPI_STORE_BF16>(acc, slab, srow, lane & 3);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&slab_full[wg]));
      continue;
    }
    if constexpr (EPI == EPI_RESIDUAL_BF16) {
      mbar_wait(smem_u32(&resid_full[wg]), it & 1);
    } else {
      // the slab's previous store has had this tile's mainloop to read it out
      if (leader) bulk_wait_group_read<0>();
      named_bar_sync(1 + wg, 128);
    }
    if constexpr (EPI == EPI_QKV_ROPE) {
      static_assert(BLOCK_N % 128 == 0 || EPI != EPI_QKV_ROPE, "fused QKV needs whole heads");
#pragma unroll
      for (int hh = 0; hh < BLOCK_N / 128; ++hh) {
        const int head = (n_blk * BLOCK_N) / kHeadDim + hh;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // 32 fp32 accumulators -> 16 packed bf16x2 (the rounding of the linear output):
          // u[jj] holds dims 8jj + 2q, +1 of the head
          uint32_t u[16];
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int i = 4 * (16 * hh + jj) + 2 * h;
            u[jj] = pack_bf16x2(acc[i], acc[i + 1]);
          }
          qkv_head_epilogue(u, ea, rm[h], head, head * kHeadDim < N && row0 + 8 * h < M, slab,
                            srow + 8 * h, 128 * hh);
        }
      }
    } else {
      epilogue_stage<BLOCK_N, EPI>(acc, slab, srow, lane & 3);
    }
    fence_proxy_async_smem();   // this thread's slab writes, before the async proxy reads them
    named_bar_sync(1 + wg, 128);
    if (leader) store_slab<BLOCK_N, EPI>(&tm_d, slab, m_blk * kBlockM + 64 * wg, n_blk, M, N, ea);
  }
  // the stores must finish reading shared memory before the block exits
  if (kStaged && !EPI_WARPS && leader) bulk_wait_group<0>();
}

// ---------------------------------------------------------------------------
// host side: tensor maps
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  const void* ptr;
  int rows, cols, box_rows;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h ^= (static_cast<size_t>(k.rows) * 0x9E3779B97F4A7C15ull) ^
         (static_cast<size_t>(k.cols) << 20) ^ (static_cast<size_t>(k.box_rows) << 50);
    return h;
  }
};

// Row-major bf16 [rows, cols] tensor, box = [box_rows, 64 cols], 128B swizzle.
int make_tmap(const void* ptr, int rows, int cols, int box_rows, CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey key{ptr, rows, cols, box_rows};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return 0;
    }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kBlockK), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: %d (ptr=%p rows=%d cols=%d box_rows=%d)",
                   static_cast<int>(r), ptr, rows, cols, box_rows);
    return -1;
  }
  std::lock_guard<std::mutex> g(mu);
  cache.emplace(key, *out);
  return 0;
}

// The bf16 output or residual of a fused epilogue: [rows, cols] with a row stride of ld
// elements, box = 64 rows x box_cols columns in the swizzle of the staging slab (stage_off).
// Encoded per launch, since M changes from call to call.
int make_epi_tmap(const void* ptr, int rows, int cols, int ld, int box_cols, CUtensorMap* out) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (static_cast<long>(ld) * 2) % 16 != 0) {
    set_last_error("gemm_bf16_tn: the bf16 output and residual need 16-byte aligned rows "
                   "(ptr=%p ldd=%d)", ptr, ld);
    return -1;
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: %d (epilogue ptr=%p rows=%d cols=%d ldd=%d)",
                   static_cast<int>(r), ptr, rows, cols, ld);
    return -1;
  }
  return 0;
}

}  // namespace

// Generic bf16 tiled tensor map with 128-byte swizzle (rank 2..5); strides are in bytes for
// dims 1..rank-1 (dim 0 is contiguous).  Used by the attention kernels.
int encode_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable");
    return -1;
  }
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i + 1 < rank) st[i] = strides_bytes[i];
  }
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                   const_cast<void*>(ptr), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled(rank %d) failed: %d (ptr=%p dims=%llu,%llu box=%u,%u)",
                   rank, static_cast<int>(r), ptr, (unsigned long long)dims[0],
                   (unsigned long long)dims[1], box[0], box[1]);
    return -1;
  }
  return 0;
}

namespace {

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 1;
  }
  return cached[dev];
}

int l2_bytes() {
  static long cached = -1;
  if (cached < 0) {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrL2CacheSize, dev);
    cached = n > 0 ? n : (40 << 20);
  }
  return static_cast<int>(cached);
}

// Row-tiles per raster group.  A weight matrix that fits in half the L2 (QKV, Wo, down of the
// smaller models) stays resident whatever the order, so narrow groups are enough: the CTAs of a
// wave then share few A row-tiles and walk W together.  A larger W (gate/up, the LM head) is
// streamed: there the group takes as many row-tiles as keep its A slab (rows x K bf16) within
// ~40 % of the L2, so A is read from HBM once and W once per group.
int raster_group(int tile_rows, int N, int K) {
  const long l2 = l2_bytes();
  if (static_cast<long>(N) * K * 2 <= l2 / 2) return 2;
  const long slab = l2 * 2 / 5;
  long gm = slab / (static_cast<long>(tile_rows) * K * 2);
  if (gm < 2) gm = 2;
  if (gm > 64) gm = 64;
  return static_cast<int>(gm);
}

template <int BLOCK_N, int EPI, bool EPI_WARPS>
int launch_kernel(int grid, cudaStream_t stream, const CUtensorMap& tm_a, const CUtensorMap& tm_b,
                   const CUtensorMap& tm_d, const CUtensorMap& tm_r, void* d, int M, int N, int K,
                   int ldd, int gm, const QkvEpiArgs& ea) {
  using Cfg = GemmCfg<BLOCK_N>;
  auto kern = gemm_bf16_tn_kernel<BLOCK_N, EPI, EPI_WARPS>;
  SB_SET_MAX_SMEM(kern, Cfg::kSmemBytes);
  kern<<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(tm_a, tm_b, tm_d, tm_r,
                                                        reinterpret_cast<float*>(d), M, N, K, ldd,
                                                        gm, ea);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <int BLOCK_N, int EPI>
int launch_cfg(const void* a, int a_rows, const void* w, void* d, const void* resid, int M, int N,
               int K, int ldd, cudaStream_t stream, const QkvEpiArgs& ea) {
  CUtensorMap tm_a, tm_b, tm_d{}, tm_r{};
  if (make_tmap(a, a_rows, K, kBlockM, &tm_a)) return -1;
  if (make_tmap(w, N, K, BLOCK_N, &tm_b)) return -1;
  if constexpr (EPI != EPI_STORE_F32) {
    using Epi = EpiCfg<BLOCK_N, EPI>;
    if (make_epi_tmap(d, M, EPI == EPI_SWIGLU_BF16 ? N / 2 : N, ldd, Epi::kBoxCols, &tm_d))
      return -1;
    if (EPI == EPI_RESIDUAL_BF16 && make_epi_tmap(resid, M, N, ldd, 64, &tm_r)) return -1;
  }
  const int tiles = ((M + kBlockM - 1) / kBlockM) * ((N + BLOCK_N - 1) / BLOCK_N);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  const int gm = raster_group(kBlockM, N, K);
  // The epilogue warps hide the SwiGLU / QKV math under the next tile's mainloop.  A CTA with
  // one tile has no next mainloop, and there the eight consumer warps finish the math sooner
  // (M = 128: 0.119 against 0.131 ms for the four qwen-3-4b shapes).  The math per tile is fixed
  // while the mainloop grows with K: at K = 2,560 it hides under it, at K = 1,024
  // (qwen-3-embedding-0.6b) three warps fall behind and the GEMMs slow down.
  if constexpr (EPI == EPI_SWIGLU_BF16 || EPI == EPI_QKV_ROPE) {
    if (tiles > grid && K >= 2048)
      return launch_kernel<BLOCK_N, EPI, true>(grid, stream, tm_a, tm_b, tm_d, tm_r, d, M, N, K,
                                               ldd, gm, ea);
  }
  return launch_kernel<BLOCK_N, EPI, false>(grid, stream, tm_a, tm_b, tm_d, tm_r, d, M, N, K, ldd,
                                            gm, ea);
}

template <int EPI>
int launch_epi(int block_n, const void* a, int a_rows, const void* w, void* d, const void* resid,
               int M, int N, int K, int ldd, cudaStream_t stream, const QkvEpiArgs& ea) {
  switch (block_n) {
    case 64:
      if constexpr (EPI == EPI_QKV_ROPE) {
        set_last_error("gemm_bf16_tn: the fused QKV epilogue needs block_n >= 128");
        return -1;
      } else {
        return launch_cfg<64, EPI>(a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
      }
    case 128:
      return launch_cfg<128, EPI>(a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    default:   // 256, and 512 (the widest tile)
      return launch_cfg<256, EPI>(a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
  }
}

}  // namespace

int gemm_pick_block_n(int M, int N) {
  // Cost = waves x (tile area / efficiency); pick the cheapest configuration (one CTA per SM,
  // 128 x BLOCK_N tiles).  The relative efficiencies are assumed, not measured: a narrow tile
  // moves more operand bytes per MAC, (128 + BLOCK_N) / (128 * BLOCK_N), which alone would rate
  // the 128- and 64-wide tiles at 0.75 / 0.5 of the 256-wide one; they are rated higher because
  // shared-memory traffic is not the only limit.  Every tile width accumulates in the same order,
  // so the choice changes speed only, never results.
  const int sms = num_sms();
  double best = 1e30;
  int pick = 128;
  struct Cand { int tn; double eff; };
  const Cand cands[] = {{256, 1.0}, {128, 0.85}, {64, 0.6}};
  for (const Cand& c : cands) {
    const long tiles = static_cast<long>((M + kBlockM - 1) / kBlockM) * ((N + c.tn - 1) / c.tn);
    const long waves = (tiles + sms - 1) / sms;
    const double cost = static_cast<double>(waves) * kBlockM * c.tn / c.eff;
    if (cost < best) {
      best = cost;
      pick = c.tn;
    }
  }
  return pick;
}

int gemm_bf16_tn(const void* a, int a_rows, const void* w, void* d, const void* resid, int M,
                 int N, int K, int ldd, int epilogue, int block_n, cudaStream_t stream,
                 const QkvEpiArgs* qkv_args) {
  if (M <= 0) return 0;
  const QkvEpiArgs ea = qkv_args ? *qkv_args : QkvEpiArgs{};
  if (K <= 0 || K % kBlockK != 0 || N % 32 != 0 || a_rows < M) {
    set_last_error("gemm_bf16_tn: unsupported shape M=%d N=%d K=%d a_rows=%d", M, N, K, a_rows);
    return -1;
  }
  if (block_n == 0) block_n = gemm_pick_block_n(M, N);
  if (block_n != 64 && block_n != 128 && block_n != 256 && block_n != 512) {
    set_last_error("gemm_bf16_tn: block_n must be 64/128/256/512, got %d", block_n);
    return -1;
  }
  switch (epilogue) {
    case EPI_STORE_BF16:
      return launch_epi<EPI_STORE_BF16>(block_n, a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    case EPI_RESIDUAL_BF16:
      if (!resid) {
        set_last_error("gemm_bf16_tn: residual epilogue without residual pointer");
        return -1;
      }
      return launch_epi<EPI_RESIDUAL_BF16>(block_n, a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    case EPI_SWIGLU_BF16:
      return launch_epi<EPI_SWIGLU_BF16>(block_n, a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    case EPI_STORE_F32:
      return launch_epi<EPI_STORE_F32>(block_n, a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    case EPI_QKV_ROPE:
      if (!qkv_args || N % kHeadDim != 0 || N != (ea.hq + 2 * ea.hkv) * kHeadDim) {
        set_last_error("gemm_bf16_tn: fused QKV epilogue needs its operands and N = heads*128");
        return -1;
      }
      if (block_n == 64) block_n = 128;
      return launch_epi<EPI_QKV_ROPE>(block_n, a, a_rows, w, d, resid, M, N, K, ldd, stream, ea);
    default:
      set_last_error("gemm_bf16_tn: unknown epilogue %d", epilogue);
      return -1;
  }
}

}  // namespace sb
