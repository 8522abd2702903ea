// Warp-level bf16 / fp16 tensor-core helpers for sm_90a: mma.sync m16n8k16 (fp32 accumulate) fed by ldmatrix straight from
// the library's row layout (row_layout.cuh): 8-element K-chunks of 16 bytes per row, rows linear in memory, so an 8x8
// ldmatrix block is 8 consecutive rows of one K-chunk and a row-shifted operand is just a different start address.
//
// A warp owns a block of 32 accumulator rows (two m16 tiles) x 8*NT columns (NT n8 tiles):
//   acc[mt][nt][0..3] = D(16 mt + g, 8 nt + 2 t + {0, 1}) and D(16 mt + g + 8, ...)   (g = lane / 4, t = lane % 4).
// rows8() turns one n8 tile into "lane = accumulator row" form with shuffles, the layout the head's epilogues read
// (b3a's stores the fragments as they are; the banded kernel's goes through shared memory, rows_store() below).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>
#include <type_traits>

#include "lpb_common.cuh"

namespace lpb {
namespace mma {

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t (&r)[2], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// m16n8k16 on 16-bit operands of type T (__nv_bfloat16 or __half): same fragments, same fp32 accumulators
template <typename T>
__device__ __forceinline__ void mma16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  static_assert(std::is_same_v<T, __nv_bfloat16> || std::is_same_v<T, __half>, "16-bit operands: bf16 or fp16");
  if constexpr (std::is_same_v<T, __half>) mma_f16(d, a, b0, b1);
  else mma_bf16(d, a, b0, b1);
}

// ---- 3xTF32 (fp32-accurate GEMMs on the tf32 tensor cores; the fp32 head, head_f32.cu) ----------------------------
// x = big + small with big = tf32(x) and small = tf32(x - big); a*b ~ a_s*b_b + a_b*b_s + a_b*b_b (the small*small term
// is below fp32 rounding), each product accumulated in fp32 by mma.sync m16n8k8.  Fragments (g = lane / 4, t = lane % 4):
// a0 (g, t), a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4); b0 (k = t, n = g), b1 (k = t + 4, n = g); c as for bf16.
__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r & 0xffffe000u;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& big, uint32_t& small) {
  big = tf32_rna(x);
  small = tf32_rna(x - __uint_as_float(big));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// d += a * b for one k8 step.  The tensor cores' fp32 accumulation truncates, so a long-lived accumulator fed by
// three MMAs per step drifts by up to an ulp of its own size per MMA (~2e-5 relative after K = 1152); the step's
// products are summed in a fresh fragment (small products first) and added to d with a rounded FADD instead.
__device__ __forceinline__ void mma_3xtf32(float (&d)[4], const uint32_t (&ab)[4], const uint32_t (&as)[4], uint32_t bb0, uint32_t bb1,
                                           uint32_t bs0, uint32_t bs1) {
  float p[4];
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
               : "=f"(p[0]), "=f"(p[1]), "=f"(p[2]), "=f"(p[3])
               : "r"(as[0]), "r"(as[1]), "r"(as[2]), "r"(as[3]), "r"(bb0), "r"(bb1), "f"(0.f));
  mma_tf32(p, ab, bs0, bs1);
  mma_tf32(p, ab, bb0, bb1);
#pragma unroll
  for (int i = 0; i < 4; ++i) d[i] += p[i];
}

template <int MT, int NT>
__device__ __forceinline__ void zero(float (&acc)[MT][NT][4]) {
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;
}

// One K = 16 step, both operands K-major: A row r at a + 16 r (K-chunk j at + j * lbo_a), B column n at b + 16 n
// (K-chunk j at + j * lbo_b).  MT m16 tiles of A, NT n8 tiles of B (NT even).  T: the operands' element type (the
// forward's, head_prep.cuh Operand); the backward's operands are bf16.
template <typename T = __nv_bfloat16, int MT, int NT>
__device__ __forceinline__ void kstep(float (&acc)[MT][NT][4], uint32_t a, uint32_t lbo_a, uint32_t b, uint32_t lbo_b, int lane) {
  static_assert(NT % 2 == 0, "n8 tiles are loaded in pairs");
  uint32_t af[MT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) ldsm_x4(af[mt], a + (uint32_t)(16 * mt + ((lane >> 3) & 1) * 8 + (lane & 7)) * 16 + (uint32_t)(lane >> 4) * lbo_a);
#pragma unroll
  for (int np = 0; np < NT / 2; ++np) {
    uint32_t bf[4];
    ldsm_x4(bf, b + (uint32_t)(16 * np + (lane >> 4) * 8 + (lane & 7)) * 16 + (uint32_t)((lane >> 3) & 1) * lbo_b);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      mma16<T>(acc[mt][2 * np], af[mt], bf[0], bf[1]);
      mma16<T>(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
    }
  }
}

// kstep over the n8 tiles set in MASK only (compile time): the others keep their accumulators and cost no B load, and
// a pair with one tile left is loaded with ldmatrix .x2.  MASK == 0 issues nothing, not even the A loads.
template <unsigned MASK, typename T = __nv_bfloat16, int MT, int NT>
__device__ __forceinline__ void kstep_nz(float (&acc)[MT][NT][4], uint32_t a, uint32_t lbo_a, uint32_t b, uint32_t lbo_b, int lane) {
  static_assert(NT % 2 == 0 && (MASK >> NT) == 0, "n8 tiles are loaded in pairs");
  if constexpr (MASK != 0) {
    uint32_t af[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) ldsm_x4(af[mt], a + (uint32_t)(16 * mt + ((lane >> 3) & 1) * 8 + (lane & 7)) * 16 + (uint32_t)(lane >> 4) * lbo_a);
    // one lane offset for both load widths (.x2 reads the addresses of lanes 0-15 only: tile 2 np, or 2 np + 1 one
    // tile further on), so no second per-lane address stays live
    const uint32_t bl = b + (uint32_t)((lane >> 4) * 8 + (lane & 7)) * 16 + (uint32_t)((lane >> 3) & 1) * lbo_b;
#pragma unroll
    for (int np = 0; np < NT / 2; ++np) {
      const bool lo = (MASK >> (2 * np)) & 1u, hi = (MASK >> (2 * np + 1)) & 1u;
      if (lo && hi) {
        uint32_t bf[4];
        ldsm_x4(bf, bl + (uint32_t)(16 * np) * 16);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma16<T>(acc[mt][2 * np], af[mt], bf[0], bf[1]);
          mma16<T>(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
        }
      } else if (lo || hi) {
        const int nt = 2 * np + (hi ? 1 : 0);
        uint32_t bf[2];
        ldsm_x2(bf, bl + (uint32_t)(8 * nt) * 16);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) mma16<T>(acc[mt][nt], af[mt], bf[0], bf[1]);
      }
    }
  }
}

// f(integral_constant<int, sh>) for the four input shifts, so that per-shift tile masks are compile-time
template <typename F>
__device__ __forceinline__ void for_shifts(F&& f) {
  f(std::integral_constant<int, 0>{});
  f(std::integral_constant<int, 1>{});
  f(std::integral_constant<int, 2>{});
  f(std::integral_constant<int, 3>{});
}

// n8 tile `nt` of the 32 rows of m16 tiles M0, M0 + 1 -> v[0..7] = D(16 M0 + lane, 8 nt + 0..7).  A lone last tile
// (M0 + 1 == MT) fills lanes 16..31 with copies of its rows, which the caller ignores.
template <int M0, int MT, int NT>
__device__ __forceinline__ void rows8_at(const float (&acc)[MT][NT][4], int nt, float* v, int lane) {
  constexpr int M1 = M0 + 1 < MT ? M0 + 1 : M0;
  const int g = lane & 7, sel = lane >> 3;  // sel = 2 (tile - M0) + (row >= 8 within the m16 tile)
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int src = g * 4 + t;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const float x0 = __shfl_sync(0xffffffffu, acc[M0][nt][p], src);
      const float x1 = __shfl_sync(0xffffffffu, acc[M0][nt][2 + p], src);
      const float x2 = __shfl_sync(0xffffffffu, acc[M1][nt][p], src);
      const float x3 = __shfl_sync(0xffffffffu, acc[M1][nt][2 + p], src);
      v[2 * t + p] = sel == 0 ? x0 : (sel == 1 ? x1 : (sel == 2 ? x2 : x3));
    }
  }
}
// n8 tile `nt` of a 32-row block -> v[0..7] = D(lane, 8 nt + 0..7)
template <int NT>
__device__ __forceinline__ void rows8(const float (&acc)[2][NT][4], int nt, float* v, int lane) {
  rows8_at<0>(acc, nt, v, lane);
}

// ---- "lane = row" through shared memory (the banded kernel's epilogue; it reads ~34 of a row's 40 columns) --------
// A warp writes n8 tiles NT0 .. NT0 + NTS - 1 of its 32-row block (m16 tiles 0, 1) into its own scratch of ROWS_SCRATCH
// floats with 64-bit stores of the fragment pairs as they lie, then reads D(lane, 8 NT0 + c) at rows_lane(s, lane)[c].
// The scratch is the warp's alone, so a __syncwarp orders its writes before its reads, and its reads before the next
// block's writes.  Element (row r, column c) is at float r * ROWS_STRIDE + 2 (r / 4) + c.  Banks, with
// ROWS_STRIDE = 56 = 24 (mod 32): row r starts at bank 8 (3 r mod 4) + 2 (r / 4) (mod 32), always even, so every pair
// is 8-byte aligned.
//  * st.shared.v2.f32, a wavefront per half-warp: its lanes (g, t) hold rows r0 + g (r0 = 0 mod 4, g / 4 fixed) and
//    columns 8 nt + 2 t, i.e. banks 8 (3 g mod 4) + 2 t + {0, 1} + const: four rows 8 banks apart, four pairs each within
//    8 banks -- 32 distinct banks, conflict-free.
//  * ld.shared.f32, one row per lane: the starts 8 (3 r mod 4) + 2 (r / 4) of rows 0..31 hit each even bank exactly
//    twice, so a column read is 2-way -- the least possible with even (pair-aligned) row starts.
// A row spans 2 * 7 + 8 NTS <= ROWS_STRIDE floats: NTS <= 5.
constexpr int ROWS_STRIDE = 56;
constexpr int ROWS_SCRATCH = 32 * ROWS_STRIDE;

// the tiles j < ntiles (a warp-uniform run-time bound) of NT0 .. NT0 + NTS - 1
template <int NT0, int NTS, int NT>
__device__ __forceinline__ void rows_store(float* s, const float (&acc)[2][NT][4], int ntiles, int lane) {
  static_assert(NT0 + NTS <= NT && 2 * 7 + 8 * NTS <= ROWS_STRIDE, "scratch rows hold 8 NTS columns after the skew");
  const int g = lane >> 2, t = lane & 3;
  float* p = s + g * ROWS_STRIDE + 2 * (g >> 2) + 2 * t;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r0 = 16 * mt + 8 * h;  // compile-time after unrolling; (r0 + g) / 4 = r0 / 4 + g / 4
#pragma unroll
      for (int j = 0; j < NTS; ++j)
        if (j < ntiles)
          *reinterpret_cast<float2*>(p + r0 * ROWS_STRIDE + 2 * (r0 >> 2) + 8 * j) = make_float2(acc[mt][NT0 + j][2 * h], acc[mt][NT0 + j][2 * h + 1]);
    }
}
__device__ __forceinline__ const float* rows_lane(const float* s, int lane) { return s + lane * ROWS_STRIDE + 2 * (lane >> 2); }

}  // namespace mma
}  // namespace lpb
