// Shape-generic building blocks of the bf16 head (head_rows_bf16.cu), shared with the C-ABI entry in head_bf16.cu.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "row_layout.cuh"

namespace lpb {

enum { CONVT_ROWS_MID = 0, CONVT_ROWS_PLANES = 1, CONVT_ROWS_SOFTMAX = 2, CONVT_ROWS_SOFTMAX_P0 = 3, CONVT_ROWS_SOFTMAX_P1 = 4 };

struct ConvtRowsParams {
  const __nv_bfloat16* X;    // [B][4*nst][L.rows][8] padded row layout of the conv input
  RowLayout L;
  const __nv_bfloat16* wpk;  // [nst][4 shifts][4 kchunks][80][8] (head_prep_kernel)
  const float* bias;         // [cout] added in the epilogue, or null (bias folded into the GEMM / irrelevant)
  int nst;                   // 32-channel K stages
  int B, cout, mode;
  __nv_bfloat16* mid;        // CONVT_ROWS_MID: [B][4][Lout.rows][8], channel `cout` = 1
  RowLayout Lout;
  float* out;                // planes [B][cout][2Hi][2Wi] (raw or softmaxed)
  float* partials;           // split softmax: [B][nbands][20][2] (max, sum) per (frame, band, plane), or null (fused two-pass form)
  int4* hints;               // optional [B][cout] decode hints {arg-max row, col, bits(max outside the 32x32 box around it), valid}:
                             // written by the fused two-pass softmax (planes up to 128 x 128), zeroed (invalid) by every other form
  int R, rows_alloc, backoff;  // filled by launch_convt_rows
};

int launch_rows_shuffle(const __nv_bfloat16* feat, int B, int C, int H, int W, __nv_bfloat16* xs, cudaStream_t s);
int launch_convt_rows(ConvtRowsParams p, int sms, cudaStream_t s);

// raster rows per band of the banded kernel (its M-tiles x 128)
constexpr int CR_BAND_ROWS = 256;
// bands the banded kernel cuts an (Hi x Wi) conv input into (R = CR_BAND_ROWS / (Wi + 1) image rows each)
inline int convt_rows_bands(int Hi, int Wi) {
  int R = CR_BAND_ROWS / (Wi + 1);
  if (R > Hi) R = Hi;
  if (R < 1) R = 1;
  return (Hi + R - 1) / R;
}
inline size_t convt_rows_partials_bytes(int B, int Hi, int Wi) { return (size_t)B * convt_rows_bands(Hi, Wi) * 20 * 2 * sizeof(float); }

}  // namespace lpb
