// Shared helpers for the lpb200 CUDA library (sm_90a).
#pragma once
#include <type_traits>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>

#include "../../include/lpb200.h"

namespace lpb {

// ---- error reporting (thread-local message, C-ABI returns the LPB_ERR_* codes of lpb200.h) -------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define LPB_REQUIRE(cond, ...)                       \
  do {                                               \
    if (!(cond)) {                                   \
      ::lpb::set_error(__VA_ARGS__);                 \
      return LPB_ERR_INVALID;                 \
    }                                                \
  } while (0)

#define LPB_CUDA(call)                                                          \
  do {                                                                          \
    cudaError_t e__ = (call);                                                   \
    if (e__ != cudaSuccess) return ::lpb::cuda_fail(e__, #call, __FILE__, __LINE__); \
  } while (0)

extern int g_tuning[];  // abi.cu: kernel-variant switches (LPB_TUNE_*)

// ---- device helpers ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_min_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_max_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---- fp32 pairs -------------------------------------------------------------------------------------
// Code written against pairs of fp32 values (two positions per thread).  sm_90 has no packed fp32 instructions, so each
// pair operation is two scalar IEEE fp32 operations: the same roundings a packed form would give.
struct f32x2 {
  float lo, hi;
};
__device__ __forceinline__ f32x2 pack2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ f32x2 dup2(float x) { return pack2(x, x); }
__device__ __forceinline__ void unpack2(f32x2 a, float& lo, float& hi) {
  lo = a.lo;
  hi = a.hi;
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return f32x2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
// compile-time loop: fn(std::integral_constant<int, I>{}) for I in [0, N)
template <int I, int N, class Fn>
__device__ __forceinline__ void static_for(Fn&& fn) {
  if constexpr (I < N) {
    fn(std::integral_constant<int, I>{});
    static_for<I + 1, N>(fn);
  }
}

// ---- mbarrier + 1-D bulk async copy (TMA engine, no tensor map needed) -------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// the same wait for warps that expect to idle for a long time (epilogue warps during a frame's MMAs, loaders ahead of
// their consumers): poll, then sleep between polls so the spinning does not take issue slots from the working warps
__device__ __forceinline__ void mbar_wait_idle(uint64_t* bar, uint32_t parity, int backoff) {
  if (!backoff) {
    mbar_wait(bar, parity);
    return;
  }
  uint32_t done = 0;
  while (true) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(96);
  }
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// shared -> global bulk copy (TMA store, bulk-group completion); bytes % 16 == 0, both addresses 16-B aligned
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread have finished READING their shared-memory source
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

}  // namespace lpb
