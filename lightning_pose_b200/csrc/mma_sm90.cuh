// Warp-level bf16 tensor-core helpers for sm_90a: mma.sync m16n8k16 (fp32 accumulate) fed by ldmatrix straight from
// the library's row layout (row_layout.cuh): 8-element K-chunks of 16 bytes per row, rows linear in memory, so an 8x8
// ldmatrix block is 8 consecutive rows of one K-chunk and a row-shifted operand is just a different start address.
//
// A warp owns a block of 32 accumulator rows (two m16 tiles) x 8*NT columns (NT n8 tiles):
//   acc[mt][nt][0..3] = D(16 mt + g, 8 nt + 2 t + {0, 1}) and D(16 mt + g + 8, ...)   (g = lane / 4, t = lane % 4).
// rows8() turns one n8 tile into "lane = accumulator row" form, the layout every epilogue of the head reads.
#pragma once
#include <cstdint>

#include "lpb_common.cuh"

namespace lpb {
namespace mma {

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
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
// (K-chunk j at + j * lbo_b).  MT m16 tiles of A, NT n8 tiles of B (NT even).
template <int MT, int NT>
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
      mma_bf16(acc[mt][2 * np], af[mt], bf[0], bf[1]);
      mma_bf16(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
    }
  }
}

// One K = 16 step, both operands MN-major (the row layout read transposed: K = rows, M / N = channels):
// A element (m, k) at a + (m / 8) * sbo_a + 16 k + 2 (m % 8); B element (n, k) at b + (n / 8) * sbo_b + 16 k + 2 (n % 8).
template <int MT, int NT>
__device__ __forceinline__ void kstep_mn(float (&acc)[MT][NT][4], uint32_t a, uint32_t sbo_a, uint32_t b, uint32_t sbo_b, int lane) {
  static_assert(NT % 2 == 0, "n8 tiles are loaded in pairs");
  uint32_t af[MT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
    ldsm_x4_t(af[mt], a + (uint32_t)(2 * mt + ((lane >> 3) & 1)) * sbo_a + (uint32_t)((lane >> 4) * 8 + (lane & 7)) * 16);
#pragma unroll
  for (int np = 0; np < NT / 2; ++np) {
    uint32_t bf[4];
    ldsm_x4_t(bf, b + (uint32_t)(2 * np + (lane >> 4)) * sbo_b + (uint32_t)(((lane >> 3) & 1) * 8 + (lane & 7)) * 16);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      mma_bf16(acc[mt][2 * np], af[mt], bf[0], bf[1]);
      mma_bf16(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
    }
  }
}

// n8 tile `nt` of a 32-row block -> v[0..7] = D(lane, 8 nt + 0..7)
template <int NT>
__device__ __forceinline__ void rows8(const float (&acc)[2][NT][4], int nt, float* v, int lane) {
  const int g = lane & 7, sel = lane >> 3;  // sel = 2 mt + (row >= 8 within the m16 tile)
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int src = g * 4 + t;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const float x0 = __shfl_sync(0xffffffffu, acc[0][nt][p], src);
      const float x1 = __shfl_sync(0xffffffffu, acc[0][nt][2 + p], src);
      const float x2 = __shfl_sync(0xffffffffu, acc[1][nt][p], src);
      const float x3 = __shfl_sync(0xffffffffu, acc[1][nt][2 + p], src);
      v[2 * t + p] = sel == 0 ? x0 : (sel == 1 ? x1 : (sel == 2 ? x2 : x3));
    }
  }
}

}  // namespace mma
}  // namespace lpb
