// One launch for everything a head call has to prepare: operand packing of the weights (fp32 master -> bf16 / fp16 images),
// clearing the pad rows of freshly allocated row-layout buffers, zeroing gradient accumulators.  Eight tiny launches per
// forward + backward pair became two (each used to cost a launch latency and a tail of its own).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "row_layout.cuh"

namespace lpb {

// The operand element type T of the forward: __nv_bfloat16 (the bf16 head) or __half (the fp16 forward).  Both are
// 2-byte elements in the same layouts below, so packs, workspaces and kernels differ only in how an fp32 value is
// rounded into T (round-to-nearest-even, subnormals kept, overflow to inf: torch's .bfloat16() / .half()), in the bits
// of the constant-one channel that carries a bias, and in the MMA's operand type (mma_sm90.cuh mma16).  Every backward
// operand is bf16.
template <typename T>
struct Operand;
template <>
struct Operand<__nv_bfloat16> {
  static constexpr uint16_t one = 0x3f80;  // bf16 1.0
  static __device__ __forceinline__ __nv_bfloat16 from(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __nv_bfloat162 h2 = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h2);
  }
};
template <>
struct Operand<__half> {
  static constexpr uint16_t one = 0x3c00;  // fp16 1.0
  static __device__ __forceinline__ __half from(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __half2 h2 = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h2);
  }
};

// A stride-2 3x3 transposed convolution in the 4-shift form (head_bf16.cu): output class cls = 2 py + px reads input
// shift sh = 2 dm + dn through a real tap unless (py == 0 && dm == 1) or (px == 0 && dn == 1) -- 9 of the 16 pairs.  The
// packers write exact zeros for the other 7, and the GEMMs skip the tiles that hold nothing else.
__host__ __device__ constexpr bool tap_nonzero(int cls, int sh) {
  return !((cls >> 1) == 0 && (sh >> 1) == 1) && !((cls & 1) == 0 && (sh & 1) == 1);
}

// The operand format of the 4-shift form, shared by the forward, the backward and the packs below.  The forward GEMMs'
// columns and the gradient GEMMs' K are class-major: k = cls * HEAD_CLS + o for output channel o.
constexpr int HEAD_CLS = 20;                                // class stride: output channels per head layer at most (>= 17 keypoints)
constexpr int HEAD_NCOLS = 4 * HEAD_CLS;                    // 80 class-major columns, a multiple of 16
constexpr int HEAD_KC = HEAD_NCOLS / 8;                     // 10 K-chunks of 8 in the gradients' class-major K
constexpr int HEAD_KSTAGE = 32;                             // input channels per forward K stage (4 K-chunks of 8)
constexpr int HEAD_BSTAGE_BYTES = 4 * 4 * HEAD_NCOLS * 16;  // one stage's packed forward weights [shift][kchunk][80][16 B]

// bit i: the `width` class-major columns [width i, width i + width) of the 80 (cls * 20 + o) hold a non-zero weight for shift sh
constexpr unsigned nz_tiles(int sh, int width) {
  unsigned m = 0;
  for (int i = 0; i < HEAD_NCOLS / width; ++i)
    for (int k = width * i; k < width * (i + 1); ++k)
      if (tap_nonzero(k / HEAD_CLS, sh)) m |= 1u << i;
  return m;
}
// per shift: n8 column tiles of the forward GEMMs' B operand, m16 row tiles of the weight gradient's A operand.  Every
// keypoint group (below) is one such 80-column block, so the tables hold for each group alike.
constexpr unsigned NZ_N8[4] = {nz_tiles(0, 8), nz_tiles(1, 8), nz_tiles(2, 8), nz_tiles(3, 8)};
constexpr unsigned NZ_M16[4] = {nz_tiles(0, 16), nz_tiles(1, 16), nz_tiles(2, 16), nz_tiles(3, 16)};
static_assert(NZ_N8[0] == 0x3ffu && NZ_N8[1] == 0x39cu && NZ_N8[2] == 0x3e0u && NZ_N8[3] == 0x380u, "n8 tiles of the 4-shift form");
static_assert(NZ_M16[0] == 0x1fu && NZ_M16[1] == 0x1eu && NZ_M16[2] == 0x1cu && NZ_M16[3] == 0x18u, "m16 tiles of the 4-shift form");

// Keypoint groups.  A layer with more than HEAD_CLS output channels splits them into groups of HEAD_CLS: channel
// o = HEAD_CLS * g + o', and group g is the 80-column class-major block above for its channels o' (a short last group
// leaves its top columns zero).  A wide forward layer is G independent 80-column GEMMs over the same A operand; the
// packed weights are group-major, [group][stage][shift][kchunk][80][8].
constexpr int HEAD_MAX_GROUPS = 4;                            // keypoint groups per layer at most
constexpr int HEAD_MAX_CH = HEAD_MAX_GROUPS * HEAD_CLS;       // 80: output channels per layer at most (LPB_HEAD_MAX_CHANNELS)
__host__ __device__ constexpr int head_groups(int c) { return (c + HEAD_CLS - 1) / HEAD_CLS; }
// 32-channel K stages of the mid activations of a two-deconv head: c1 channels plus the constant-one bias channel, and
// at least the channels of c1's keypoint groups (each group's epilogue writes all of its 20)
__host__ __device__ constexpr int head_mid_stages(int c1) {
  return ((c1 + 1 > HEAD_CLS * head_groups(c1) ? c1 + 1 : HEAD_CLS * head_groups(c1)) + HEAD_KSTAGE - 1) / HEAD_KSTAGE;
}
// Heads the bf16 forward serves.  Narrow: at most HEAD_CLS channels per layer, fewer in the first of two (its mid
// activations then fit one K stage with the ones channel).  Wide: a last layer with more than HEAD_CLS channels, up to
// HEAD_MAX_CH in every layer; wide heads take the banded kernels with keypoint groups.  A two-deconv head with
// c1 >= HEAD_CLS and c2 <= HEAD_CLS is neither.
__host__ __device__ constexpr bool head_narrow(int c1, int c2) { return c2 == 0 ? c1 >= 1 && c1 <= HEAD_CLS : c1 >= 1 && c1 < HEAD_CLS && c2 <= HEAD_CLS; }
__host__ __device__ constexpr bool head_wide(int c1, int c2) {
  return c2 == 0 ? c1 > HEAD_CLS && c1 <= HEAD_MAX_CH : c1 >= 1 && c1 <= HEAD_MAX_CH && c2 > HEAD_CLS && c2 <= HEAD_MAX_CH;
}
static_assert(head_groups(HEAD_CLS) == 1 && head_mid_stages(HEAD_CLS - 1) == 1, "narrow heads: one group, one mid stage");
// Three-deconv heads (downsample factor 1 on a stride-32 backbone) the 16-bit kernels serve: narrow only, every layer one
// keypoint group, and room for the constant-one channel in both mid activations (c1, c2 < HEAD_CLS).
__host__ __device__ constexpr bool head_narrow3(int c1, int c2, int c3) {
  return c1 >= 1 && c1 < HEAD_CLS && c2 >= 1 && c2 < HEAD_CLS && c3 >= 1 && c3 <= HEAD_CLS;
}

struct PrepJobs {
  // forward operand packs: W[Cin][Cout][3][3] -> B[group][stage][shift][kchunk][80][8] of the launch's operand type T
  // (head_bf16.cu); one per deconv (three-deconv heads use the third)
  struct { const float* w; const float* bias; int Cin, Cout, nstages, ngroups; void* out; } fpack[3];
  // data-gradient operand packs: -> [kgroup][tile][shift][kchunk][rows_per_tile][8]    (head_bwd_bf16.cu): K is one
  // keypoint group of the layer's output channels (kgroups of them), row r of tile t is input channel tile_ch t + r
  // (rows r >= tile_ch are zero); always bf16
  struct { const float* w; int Cin, Cout, ntiles, rows_per_tile, tile_ch, kgroups; __nv_bfloat16* out; } dpack[3];
  // pad rows of row-layout buffers of 2-byte elements (zero in either type)
  struct { void* buf; RowLayout L; long long nslabs; } pads[3];
  struct { float* p; long long n; } zero[6];
};

template <typename T = __nv_bfloat16>
int launch_head_prep(const PrepJobs& jobs, int sms, cudaStream_t s);

}  // namespace lpb
