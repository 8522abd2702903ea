// Shape-generic building blocks of the bf16 head (head_rows_bf16.cu), shared with the C-ABI entry in head_bf16.cu, and
// the forward's workspace layout, which the backward reads too.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "head_prep.cuh"
#include "row_layout.cuh"

namespace lpb {

enum { CONVT_ROWS_MID = 0, CONVT_ROWS_PLANES = 1, CONVT_ROWS_SOFTMAX = 2, CONVT_ROWS_SOFTMAX_P0 = 3, CONVT_ROWS_SOFTMAX_P1 = 4 };

struct ConvtRowsParams {
  const __nv_bfloat16* X;    // [B][4*nst][L.rows][8] padded row layout of the conv input
  RowLayout L;
  const __nv_bfloat16* wpk;  // [ngroups][nst][4 shifts][4 kchunks][80][8] (head_prep_kernel)
  const float* bias;         // [cout] added in the epilogue, or null (bias folded into the GEMM / irrelevant)
  int nst;                   // 32-channel K stages
  int B, cout, mode;
  __nv_bfloat16* mid;        // CONVT_ROWS_MID: [B][mid_kc][Lout.rows][8], channel `cout` = 1, the rest of the chunks 0
  RowLayout Lout;
  int mid_kc;                // CONVT_ROWS_MID: K-chunks of the next layer's input (4 * head_mid_stages(cout))
  float* out;                // planes [B][cout][2Hi][2Wi] (raw or softmaxed)
  float* partials;           // split softmax: [B][ngroups][nbands][20][2] (max, sum) per (frame, group, band, plane), or
                             // null (fused two-pass form)
  int R, rows_alloc;         // filled by launch_convt_rows
  int ngroups;               // filled by launch_convt_rows: keypoint groups of the output channels (head_prep.cuh)
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
inline size_t convt_rows_partials_bytes(int B, int ngroups, int Hi, int Wi) {
  return (size_t)B * ngroups * convt_rows_bands(Hi, Wi) * HEAD_CLS * 2 * sizeof(float);
}

// Byte offsets into the forward's workspace (lpb_head_fwd_bf16): [packed w1][packed w2][mid activations][split-softmax
// statistics of the last layer].  mid (padded row layout, channel c1 the constant one, 4 * head_mid_stages(c1) K-chunks)
// exists for two-deconv heads only; one w2 stage is reserved for one-deconv heads as well.  Packs and statistics hold
// one block per keypoint group.  The backward reads mid from here.
struct HeadFwdLayout {
  size_t w1, w2, mid, partials, total;
};
inline HeadFwdLayout head_fwd_layout(int B, int C, int H, int W, int c1, int c2) {
  HeadFwdLayout l;
  const int nst2 = c2 > 0 ? head_mid_stages(c1) : 1, g1 = head_groups(c1), g2 = c2 > 0 ? head_groups(c2) : 1;
  l.w1 = 0;
  l.w2 = (size_t)g1 * (C / 4 / HEAD_KSTAGE) * HEAD_BSTAGE_BYTES;
  l.mid = l.w2 + (size_t)g2 * nst2 * HEAD_BSTAGE_BYTES;
  l.partials = l.mid + (c2 > 0 ? (size_t)B * 4 * nst2 * make_row_layout(4 * H, 4 * W).rows * 16 : 0);
  const size_t part = c2 > 0 ? convt_rows_partials_bytes(B, g2, 4 * H, 4 * W) : convt_rows_partials_bytes(B, g1, 2 * H, 2 * W);
  l.total = l.partials + ((part + 255) & ~(size_t)255);
  return l;
}

}  // namespace lpb
