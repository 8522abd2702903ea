// Self-test of the tensor-core operand plumbing (mma_sm90.cuh), run by scripts/test_umma_selftest.py.
// One CTA computes a small GEMM from operands stored in the library's "row layout"
//   X[kchunk][row][8] bf16   (element (row, ch) at kchunk = ch/8, 16 bytes per row)
// in two interpretations:
//   mode 0  K-major : D[m][n] = sum_ch  A[row=m][ch] * B[row=n][ch]          (the forward shift-GEMMs)
//   mode 1  MN-major: D[m][n] = sum_row A[row][ch=m] * B[row][ch=n]          (weight-gradient GEMMs:
//           the SAME buffers read transposed, ldmatrix .trans)
// `row_shift` moves A's start address by whole rows (the shift trick); `col_off` is kept by the C ABI and has no effect
// (the accumulators live in registers).
#include <cuda_bf16.h>

#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "mma_sm90.cuh"

namespace lpb {

struct SelfTestParams {
  const __nv_bfloat16* a;  // [kca][rows_a][8]
  const __nv_bfloat16* b;  // [kcb][rows_b][8]
  float* d;                // [128][n]
  int kca, rows_a, kcb, rows_b;
  int mode, n, k, row_shift;
};

__global__ void __launch_bounds__(128, 1) umma_selftest_kernel(const __grid_constant__ SelfTestParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int a_bytes = P.kca * P.rows_a * 16, b_bytes = P.kcb * P.rows_b * 16;
  unsigned char* As = smem;
  unsigned char* Bs = smem + a_bytes;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < a_bytes / 16; i += 128) reinterpret_cast<uint4*>(As)[i] = reinterpret_cast<const uint4*>(P.a)[i];
  for (int i = tid; i < b_bytes / 16; i += 128) reinterpret_cast<uint4*>(Bs)[i] = reinterpret_cast<const uint4*>(P.b)[i];
  __syncthreads();
  const uint32_t a0 = smem_u32(As) + P.row_shift * 16, b0 = smem_u32(Bs);
  const uint32_t kst_a = P.rows_a * 16, kst_b = P.rows_b * 16;  // kchunk strides
  for (int c0 = 0; c0 < P.n; c0 += 16) {  // warp = accumulator rows [32 warp, 32 warp + 32), 16 columns at a time
    float acc[2][2][4];
    mma::zero(acc);
    for (int k16 = 0; k16 < P.k / 16; ++k16) {
      if (P.mode == 0)  // K = channels: two kchunks per step
        mma::kstep(acc, a0 + 2 * k16 * kst_a + 32 * warp * 16, kst_a, b0 + 2 * k16 * kst_b + c0 * 16, kst_b, lane);
      else              // K = rows: 16 rows per step; M / N groups of 8 are the kchunks
        mma::kstep_mn(acc, a0 + k16 * 256 + 4 * warp * kst_a, kst_a, b0 + k16 * 256 + (c0 / 8) * kst_b, kst_b, lane);
    }
    float v[16];
    mma::rows8(acc, 0, v, lane);
    mma::rows8(acc, 1, v + 8, lane);
    for (int i = 0; i < 16 && c0 + i < P.n; ++i) P.d[(size_t)(32 * warp + lane) * P.n + c0 + i] = v[i];
  }
}

}  // namespace lpb

extern "C" int lpb_selftest_umma(const void* a, int kca, int rows_a, const void* b, int kcb, int rows_b, int mode, int n,
                                 int k, int row_shift, int col_off, float* d, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(a && b && d, "selftest_umma: null pointer");
  LPB_REQUIRE(n >= 16 && n <= 256 - col_off && n % 16 == 0 && k % 16 == 0 && k >= 16, "selftest_umma: bad n/k");
  SelfTestParams P;
  P.a = static_cast<const __nv_bfloat16*>(a);
  P.b = static_cast<const __nv_bfloat16*>(b);
  P.d = d;
  P.kca = kca;
  P.rows_a = rows_a;
  P.kcb = kcb;
  P.rows_b = rows_b;
  P.mode = mode;
  P.n = n;
  P.k = k;
  P.row_shift = row_shift;
  (void)col_off;
  const size_t smem = (size_t)(kca * rows_a + kcb * rows_b) * 16 + 64;
  LPB_TRY(set_dynamic_smem(umma_selftest_kernel, smem, "selftest_umma"));
  umma_selftest_kernel<<<1, 128, smem, static_cast<cudaStream_t>(stream)>>>(P);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
