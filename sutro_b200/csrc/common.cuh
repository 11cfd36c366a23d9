// sutro_b200 — shared device helpers (sm_90a).
//
// Thin inline-PTX wrappers for the Hopper async machinery used by the kernels in
// this directory: mbarrier and bulk/tensor TMA (the wgmma wrappers are in
// wgmma.cuh), plus the usual warp reductions and bf16 packing.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace sb {

#define SB_DEVICE __device__ __forceinline__

constexpr int kWarpSize = 32;

// ---------------------------------------------------------------------------
// error plumbing for the host side (C-ABI never throws; see capi.cu)
// ---------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
#define SB_CUDA_CHECK(expr)                                                         \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      ::sb::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,            \
                           cudaGetErrorString(_e));                                 \
      return -1;                                                                    \
    }                                                                               \
  } while (0)

// GQA group dispatch of the attention launchers: checks that hq is a multiple of hkv and calls
// f(std::integral_constant<int, G>{}) for G = hq / hkv, one of the group sizes the kernels are
// instantiated for.  Errors are reported as "<who>: ..." and return -1.
template <class F>
int dispatch_gqa(const char* who, int hq, int hkv, F&& f) {
  if (hkv <= 0 || hq % hkv != 0) {
    set_last_error("%s: hq=%d not a multiple of hkv=%d", who, hq, hkv);
    return -1;
  }
  switch (hq / hkv) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 8: return f(std::integral_constant<int, 8>{});
    default:
      set_last_error("%s: unsupported GQA group size %d", who, hq / hkv);
      return -1;
  }
}

// cudaFuncSetAttribute is per device: remember, per call site, on which devices the
// dynamic-shared-memory limit has already been raised (one engine per GPU may live in the
// same process, each driven from its own host thread).
struct PerDeviceOnce {
  unsigned long long done = 0;  // bit d == device d configured (<= 64 devices)
  bool need(int& dev) {
    dev = 0;
    cudaGetDevice(&dev);
    return dev < 0 || dev >= 64 || !((__atomic_load_n(&done, __ATOMIC_ACQUIRE) >> dev) & 1ull);
  }
  void mark(int dev) {
    if (dev >= 0 && dev < 64) __atomic_fetch_or(&done, 1ull << dev, __ATOMIC_RELEASE);
  }
};
#define SB_SET_MAX_SMEM(kernel, bytes)                                                        \
  do {                                                                                        \
    static ::sb::PerDeviceOnce _once;                                                         \
    int _dev;                                                                                 \
    if (_once.need(_dev)) {                                                                   \
      SB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                         bytes));                                             \
      _once.mark(_dev);                                                                       \
    }                                                                                         \
  } while (0)

// ---------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------
SB_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

SB_DEVICE uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

SB_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

SB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

SB_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
SB_DEVICE float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
SB_DEVICE float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// 128-bit streaming global accesses (L1 no-allocate: data is touched once).
SB_DEVICE uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
SB_DEVICE void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// Warpgroup register budget (sm_90a): the TMA producer warpgroup hands its registers to the
// MMA warpgroups.  Executed by every thread of the warpgroup; counts are multiples of 8.
template <int N>
SB_DEVICE void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
SB_DEVICE void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
SB_DEVICE void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
SB_DEVICE void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
SB_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
SB_DEVICE void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
SB_DEVICE void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
SB_DEVICE bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
SB_DEVICE void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// For waits that last microseconds (an epilogue warp waiting for its tile, a producer that is a
// full ring ahead): the same wait with a suspend-time hint, so the thread sleeps in the barrier
// unit instead of re-issuing the poll; it is woken when the phase completes.
SB_DEVICE void mbar_wait_long(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred P;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, P;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(1000000u)
        : "memory");
  } while (!done);
}

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
SB_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates are (inner, outer) element indices.
SB_DEVICE void tma_load_2d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 3-D tiled load: coordinates are (inner, middle, outer) element indices.
SB_DEVICE void tma_load_3d(uint32_t smem_dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                           int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 2-D tiled store shared -> global into the issuing thread's current bulk group; the parts of
// the box outside the tensor map's dims are not written.
SB_DEVICE void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
SB_DEVICE void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Wait until at most N of this thread's bulk groups still read their shared-memory source.
template <int N>
SB_DEVICE void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// Wait until at most N of this thread's bulk groups are incomplete (their writes done).
template <int N>
SB_DEVICE void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// Barrier `id` (1..15; 0 is __syncthreads) over the first `count` threads to arrive.
SB_DEVICE void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
SB_DEVICE void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
SB_DEVICE void st_shared_b16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
SB_DEVICE uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
SB_DEVICE uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "r"(addr)
               : "memory");
  return v;
}
SB_DEVICE void st_shared_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
// 1-D bulk copy global -> shared (no tensor map; size multiple of 16 B).
SB_DEVICE void bulk_load_1d(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_dst),
      "l"(gsrc), "r"(bytes), "r"(bar)
      : "memory");
}

// ---------------------------------------------------------------------------
// mma.sync tensor core helpers used by the paged attention kernels
// ---------------------------------------------------------------------------
SB_DEVICE void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
SB_DEVICE void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                 uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
SB_DEVICE void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

SB_DEVICE void cp_async_16(uint32_t smem_dst, const void* gsrc, bool pred) {
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz)
               : "memory");
}
SB_DEVICE void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
SB_DEVICE void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

}  // namespace sb
