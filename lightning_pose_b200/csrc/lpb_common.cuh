// Shared helpers for the lpb200 CUDA library (sm_90a).
#pragma once
#include <type_traits>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
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

// an LPB_* status: returned as is unless it is LPB_OK
#define LPB_TRY(call)                  \
  do {                                 \
    const int rc__ = (call);           \
    if (rc__ != LPB_OK) return rc__;   \
  } while (0)

// ---- the current device (abi.cu) ----------------------------------------------------------------
struct DeviceLimits {
  int sms;       // streaming multiprocessors
  int max_smem;  // opt-in shared memory per block, bytes (static plus dynamic)
};
// The current device's limits, queried once per device ordinal.  LPB_OK, or LPB_ERR_CUDA with the message set.
int device_limits(DeviceLimits* d);
// For shape planners that must answer without a GPU too: the current device's limits, or an H100 SXM's (132 SMs,
// 227 KB) when there is no device to ask.
DeviceLimits planning_limits();

// ---- launches with dynamic shared memory --------------------------------------------------------
// Every launch with dynamic shared memory first sets its kernel's limit to the bytes it requests.  CUDA refuses that when
// the kernel's static plus dynamic memory exceeds the device's opt-in limit: LPB_ERR_UNSUPPORTED, naming the entry point
// and the bytes, with the refusal cleared so that a later cudaGetLastError does not report it.
int smem_refused(cudaError_t e, const char* entry, size_t bytes);
template <typename Kernel>
int set_dynamic_smem(Kernel* kernel, size_t bytes, const char* entry) {
  const cudaError_t e = bytes <= (size_t)INT32_MAX
                            ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)
                            : cudaErrorInvalidValue;
  return e == cudaSuccess ? LPB_OK : smem_refused(e, entry, bytes);
}

// A caller's device pointer that is null or a multiple of `bytes`.  Entry points check the buffers their kernels move with
// vector accesses, bulk copies or TMA up front: a misaligned one would otherwise fault on the device.
inline bool aligned_to(const void* p, uintptr_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

extern int g_softmax_split;  // abi.cu: LPB_TUNE_SOFTMAX_SPLIT

// ---- output element formats of the ingest entries (LPB_OUT_*, lpb200.h) ----------------------------------------
// element i of `out` in format FMT: fp32 as is, bf16 / fp16 rounded to nearest even (torch's .bfloat16() / .half())
template <int FMT>
__device__ __forceinline__ void store_fmt(void* out, size_t i, float v) {
  static_assert(FMT == LPB_OUT_F32 || FMT == LPB_OUT_BF16 || FMT == LPB_OUT_F16, "output format");
  if constexpr (FMT == LPB_OUT_BF16) static_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(v);
  else if constexpr (FMT == LPB_OUT_F16) static_cast<__half*>(out)[i] = __float2half_rn(v);
  else static_cast<float*>(out)[i] = v;
}
inline bool valid_out_format(int fmt) { return fmt == LPB_OUT_F32 || fmt == LPB_OUT_BF16 || fmt == LPB_OUT_F16; }
// f(integral_constant<int, FMT>) for a run-time format the caller has checked
template <typename F>
inline void with_out_format(int fmt, F&& f) {
  if (fmt == LPB_OUT_BF16) f(std::integral_constant<int, LPB_OUT_BF16>{});
  else if (fmt == LPB_OUT_F16) f(std::integral_constant<int, LPB_OUT_F16>{});
  else f(std::integral_constant<int, LPB_OUT_F32>{});
}

// ---- ragged frame arena of the ingest entries (lpb_frames_normalize_ragged, lpb_frames_crop_normalize_ragged) ---------
// The video of global stream row r: the last entry of videos [n][3] (first row, H, W) whose first row is <= r.  Rows
// past the list's end fall in the last video.  A binary search over a table of a few dozen entries, read through L1.
__device__ __forceinline__ int ragged_video(const int64_t* videos, int n, int64_t r) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (videos[3 * mid] <= r) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Host checks of an arena and its video table, shared by both ragged entries: the arena and slot_bytes 16-byte
// aligned, the device table 8-byte aligned, and in the host copy video 0 starting at row 0, first rows increasing and
// every frame within a slot.
inline int check_ragged(const char* entry, const uint8_t* arena, int64_t slot_bytes, int F, const int64_t* videos,
                        const int64_t* videos_host, int n_videos) {
  LPB_REQUIRE(aligned_to(arena, 16) && aligned_to(videos, 8), "%s: the arena must be 16-byte aligned and the table 8-byte aligned",
              entry);
  LPB_REQUIRE(slot_bytes >= 16 && slot_bytes % 16 == 0, "%s: slot_bytes %lld is not a positive multiple of 16", entry,
              (long long)slot_bytes);
  LPB_REQUIRE(F >= 0 && F <= 65535, "%s: F = %d outside 0..65535", entry, F);
  LPB_REQUIRE(n_videos >= 1, "%s: the video table is empty", entry);
  for (int v = 0; v < n_videos; ++v) {
    const int64_t row0 = videos_host[3 * v], h = videos_host[3 * v + 1], w = videos_host[3 * v + 2];
    LPB_REQUIRE(v == 0 ? row0 == 0 : row0 > videos_host[3 * (v - 1)],
                "%s: video %d starts at row %lld; video 0 starts at row 0 and each later one after it", entry, v, (long long)row0);
    LPB_REQUIRE(h >= 1 && w >= 1 && h <= INT32_MAX / 3 && w <= INT32_MAX / 3, "%s: video %d has frame size %lld x %lld",
                entry, v, (long long)h, (long long)w);
    LPB_REQUIRE(h * w * 3 <= slot_bytes, "%s: video %d's %lld x %lld frames (%lld bytes) do not fit a %lld-byte slot", entry, v,
                (long long)h, (long long)w, (long long)(h * w * 3), (long long)slot_bytes);
  }
  return LPB_OK;
}

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

// Philox4x32-10 (Salmon et al., SC'11): a counter-based generator, so a draw depends only on (key, counter).
// Shared by the augmented ingest's shot noise (ingest.cu) and the patch-masking selection (patchmask.cu).
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const uint32_t lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u, key.y += 0xBB67AE85u;
  }
  return ctr;
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
__device__ __forceinline__ void mbar_wait_idle(uint64_t* bar, uint32_t parity) {
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

// 2-D tiled TMA load of box {x0.., x1..} of tensor map `tm` (a __grid_constant__ CUtensorMap) into shared memory
// (128-B aligned); elements outside the tensor land as zeros
__device__ __forceinline__ void tma_load_2d(void* dst_smem, const void* tm, int x0, int x1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst_smem)),
               "l"(tm), "r"(x0), "r"(x1), "r"(smem_u32(bar))
               : "memory");
}

// warpgroup register budget (sm_90a): every warp of the warpgroup executes the same one
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// shared -> global bulk copy (TMA store, bulk-group completion); bytes % 16 == 0, both addresses 16-B aligned
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread have finished READING their shared-memory source
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

}  // namespace lpb
