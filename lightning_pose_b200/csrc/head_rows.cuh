// Shape-generic building blocks of the bf16 head (head_rows_bf16.cu), shared with the C-ABI entry in head_bf16.cu, and
// the forward's workspace layout, which the backward reads too.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <type_traits>

#include "head_prep.cuh"
#include "row_layout.cuh"

namespace lpb {

enum { CONVT_ROWS_MID = 0, CONVT_ROWS_PLANES = 1, CONVT_ROWS_SOFTMAX = 2, CONVT_ROWS_SOFTMAX_P0 = 3, CONVT_ROWS_SOFTMAX_P1 = 4 };

// T: the operand element type (head_prep.cuh Operand)
template <typename T>
struct ConvtRowsParams {
  const T* X;                // [B][4*nst][L.rows][8] padded row layout of the conv input
  RowLayout L;
  const T* wpk;              // [ngroups][nst][4 shifts][4 kchunks][80][8] (head_prep_kernel)
  const float* bias;         // [cout] added in the epilogue, or null (bias folded into the GEMM / irrelevant)
  int nst;                   // 32-channel K stages
  int B, cout, mode;
  T* mid;                    // CONVT_ROWS_MID: [B][mid_kc][Lout.rows][8], channel `cout` = 1, the rest of the chunks 0
  RowLayout Lout;
  int mid_kc;                // CONVT_ROWS_MID: K-chunks of the next layer's input (4 * head_mid_stages(cout))
  float* out;                // planes [B][cout][2Hi][2Wi] (raw or softmaxed)
  float* partials;           // split softmax: [B][ngroups][nbands][20][2] (max, sum) per (frame, group, band, plane), or
                             // null (fused two-pass form)
  unsigned* band_max;        // softmax modes that write planes: [B][cout][nbands][8 epilogue warps] the bits of the
                             // largest value each warp stored per (plane, band), or null (not written); see
                             // lpb_head_band_max_dims
  int R, rows_alloc;         // filled by launch_convt_rows
  int ngroups;               // filled by launch_convt_rows: keypoint groups of the output channels (head_prep.cuh)
};

// the C-ABI entry of each operand type, named in its error messages
template <typename T>
constexpr const char* head_fwd_name = std::is_same_v<T, __half> ? "head_fwd_f16" : "head_fwd_bf16";

template <typename T>
int launch_rows_shuffle(const T* feat, int B, int C, int H, int W, T* xs, cudaStream_t s);
template <typename T>
int launch_rows_shuffle_nhwc(const T* feat, int B, int C, int H, int W, T* xs, cudaStream_t s);
template <typename T>
int launch_convt_rows(ConvtRowsParams<T> p, int sms, cudaStream_t s);

// The shuffle stage holds a CTA's 32 channels of one H x W feature map.  Its budget is the public feature-map limit of
// the banded path (lpb_head_bf16_plan): maps up to 56 x 56.
constexpr size_t HEAD_FEATURE_SMEM_BUDGET = 200 * 1024;
inline size_t rows_shuffle_smem_bytes(int H, int W) { return (size_t)32 * H * W * 2; }
// Stage budget of the backward's layer-2 data gradient (b2d, two CTAs per SM): half of an H100 SM's 227 KB.
constexpr size_t HEAD_STAGE_SMEM_BUDGET = 113 * 1024;
// The banded kernel runs one CTA per SM (its accumulators take the register file): stages, statistics and the epilogue
// warps' scratch share an H100 SM's 227 KB.
constexpr size_t CR_SMEM_BUDGET = 227 * 1024;

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

// Byte offsets into the forward's workspace (lpb_head_fwd_bf16, lpb_head3_fwd): [packed w1][packed w2][packed w3][mid
// activations][mid2][split-softmax statistics of the last layer].  mid (padded row layout, channel c1 the constant one,
// 4 * head_mid_stages(c1) K-chunks) exists for two- and three-deconv heads; mid2 (8H x 8W, channel c2 the constant one)
// and the w3 pack for three-deconv heads only (c3 > 0; narrow, head_narrow3), and for every other head the layout is
// the two-layer one.  One w2 stage is reserved for one-deconv heads as well.  Packs and statistics hold one block per
// keypoint group.  The backward reads mid and mid2 from here.
struct HeadFwdLayout {
  size_t w1, w2, w3, mid, mid2, partials, total;
};
inline HeadFwdLayout head_fwd_layout(int B, int C, int H, int W, int c1, int c2, int c3 = 0) {
  HeadFwdLayout l;
  const bool three = c2 > 0 && c3 > 0;
  const int nst2 = c2 > 0 ? head_mid_stages(c1) : 1, g1 = head_groups(c1), g2 = c2 > 0 ? head_groups(c2) : 1;
  const int nst3 = three ? head_mid_stages(c2) : 0;
  l.w1 = 0;
  l.w2 = (size_t)g1 * (C / 4 / HEAD_KSTAGE) * HEAD_BSTAGE_BYTES;
  l.w3 = l.w2 + (size_t)g2 * nst2 * HEAD_BSTAGE_BYTES;
  l.mid = l.w3 + (size_t)nst3 * HEAD_BSTAGE_BYTES;
  l.mid2 = l.mid + (c2 > 0 ? (size_t)B * 4 * nst2 * make_row_layout(4 * H, 4 * W).rows * 16 : 0);
  l.partials = l.mid2 + (three ? (size_t)B * 4 * nst3 * make_row_layout(8 * H, 8 * W).rows * 16 : 0);
  const size_t part = three    ? convt_rows_partials_bytes(B, 1, 8 * H, 8 * W)
                      : c2 > 0 ? convt_rows_partials_bytes(B, g2, 4 * H, 4 * W)
                               : convt_rows_partials_bytes(B, g1, 2 * H, 2 * W);
  l.total = l.partials + ((part + 255) & ~(size_t)255);
  return l;
}

// The three-deconv heads the 16-bit kernels serve, forward and backward alike (lpb200.h lpb_head3_query): narrow
// channels (head_narrow3), feature widths W in {4, 8, 12, 16} -- the backward's data-gradient widths whose layer-3 input
// (8W + 1 raster rows per image row) fits one band of the banded kernel -- H * W a multiple of 8, and H even to train.
// True when covered; otherwise `why` names the first rule the shape breaks.
inline bool head3_covered(int H, int W, int c1, int c2, int c3, bool train, const char** why) {
  if (!head_narrow3(c1, c2, c3)) {
    *why = "channel counts outside the narrow three-deconv set (c1, c2 <= 19, c3 <= 20)";
    return false;
  }
  if (!(W == 4 || W == 8 || W == 12 || W == 16) || 8 * W + 1 > CR_BAND_ROWS) {
    *why = "feature width outside {4, 8, 12, 16}";
    return false;
  }
  if (H < 1 || (H * W) % 8 != 0 || (train && H % 2 != 0)) {
    *why = train ? "feature height must be even to train" : "H * W must be a multiple of 8";
    return false;
  }
  return true;
}

}  // namespace lpb
