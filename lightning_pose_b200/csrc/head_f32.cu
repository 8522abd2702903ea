// fp32 heatmap head: PixelShuffle(2) -> ConvTranspose2d(k3,s2,p1,op1) [x n] -> spatial softmax (T=1).
// Reference: lightning_pose/models/heads/heatmap.py:20-71 (layer stack), :203-212 (forward).
//
// This is the full-precision path (reference training is fp32, lightning_pose/train.py:411-428).  Every convolution,
// forward and both gradients, is a GEMM on the tensor cores in 3xTF32 (mma_sm90.cuh: each operand split into a tf32
// big part and a tf32 residual, three mma.sync m16n8k8 per product, fp32 accumulate), which keeps fp32 accuracy;
// 1xTF32 would not (its relative error is ~1e-3 at these K).  PixelShuffle is folded into the staging of the first
// layer's input and its inverse into the store of the data gradient.  The bf16 tensor-core path lives in head_bf16.cu.
//
// Pixel blocks.  Every kernel works on blocks of at most 128 conv-input pixels of one frame: RB rows x CB columns,
// RB = 128 / CB, with CB = ceil(Wi / k) for the k in 1..8 that fills the most slots (pixel slot p = (p / CB, p % CB);
// slots outside the frame are masked).  So the shared-memory tiles are bounded for any Hi, Wi, Cin and Cout.
#include <algorithm>
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "mma_sm90.cuh"
#include "reduce_partials.cuh"

namespace lpb {

constexpr int TC_SLOTS = 128;    // pixel slots per block
constexpr int TC_THREADS = 128;  // forward / data gradient: 4 warps x 32 pixel slots (two m16 tiles each)
constexpr int FW_CC = 24;        // forward: input channels staged per pass (three k8 steps; a 17-keypoint input in one)

struct PixBlocks {
  int RB, CB, n;  // rows, columns per block; blocks per frame
};
static PixBlocks pix_blocks(int Hi, int Wi) {
  PixBlocks best{0, 0, 0};
  for (int k = (Wi + TC_SLOTS - 1) / TC_SLOTS; k <= std::max(8, (Wi + TC_SLOTS - 1) / TC_SLOTS); ++k) {
    const int CB = (Wi + k - 1) / k, RB = TC_SLOTS / CB;
    const int n = ((Hi + RB - 1) / RB) * ((Wi + CB - 1) / CB);
    if (best.n == 0 || n < best.n) best = {RB, CB, n};  // fewest blocks = most slots filled
  }
  return best;
}
// a plane stride = 8 (mod 32) floats: the fragment pattern (g + 8 t) of a [k][m] operand falls on 32 distinct banks
__host__ __device__ __forceinline__ int pad8_32(int n) { return ((n + 31) & ~31) + 8; }
// n-stride of a pre-split [k][n] B operand (8 NT columns): = 8 or 24 (mod 32), so (g + t * stride) hits 32 banks
template <int NT>
__host__ __device__ constexpr int bstride() {
  return (NT * 8) % 32 == 8 || (NT * 8) % 32 == 24 ? NT * 8 : NT * 8 + 8;
}

// Shared-memory staging with several global loads in flight per thread (a stage is latency-bound otherwise).
// stage_rows: rows x cols elements, one warp per row and lanes along it, U rows per warp at a time.
template <int U, typename Src, typename Dst>
__device__ __forceinline__ void stage_rows(int rows, int cols, Src src, Dst dst) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int j = lane; j - lane < cols; j += 32)
    for (int r0 = warp; r0 < rows; r0 += nw * U) {
      float v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int r = r0 + u * nw;
        v[u] = (r < rows && j < cols) ? src(r, j) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int r = r0 + u * nw;
        if (r < rows && j < cols) dst(r, j, v[u]);
      }
    }
}
// stage_flat: n elements, U per thread at a time
template <int U, typename Src, typename Dst>
__device__ __forceinline__ void stage_flat(int n, Src src, Dst dst) {
  for (int i0 = threadIdx.x; i0 < n; i0 += U * blockDim.x) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * blockDim.x;
      v[u] = i < n ? src(i) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i < n) dst(i, v[u]);
    }
  }
}

// x / d for 0 <= x, d < 2^16 without a division: (x * ceil(2^32 / d)) >> 32 is exact there (d = 1: no multiplier fits)
struct FastDiv {
  uint32_t m;
  int d;
  __device__ __forceinline__ explicit FastDiv(int d_) : m(d_ > 1 ? (uint32_t)((0x100000000ull + d_ - 1) / d_) : 0u), d(d_) {}
  __device__ __forceinline__ int div(int x) const { return d > 1 ? (int)__umulhi((uint32_t)x, m) : x; }
};

// Channels-last staging of a PixelShuffle(2) source tile.  `feat` is one frame [H][W][C] (C = 4 Cin): the channels
// 4 c0 .. 4 (c0 + ncc) - 1 of a feature pixel are one contiguous run and hold the four sub-pixels (2i + di, 2j + dj) of the
// shuffled channels c0 .. c0 + ncc - 1, so consecutive threads walk that run (coalesced) over the feature pixels that
// cover shuffled rows m0 .. m0 + nm - 1 and columns n0 .. n0 + nn - 1.  dst(cc, m - m0, n - n0, v) receives every element
// of that window, zero outside the frame or past Cin.
template <typename Dst>
__device__ __forceinline__ void stage_shuffled_nhwc(const float* __restrict__ feat, int Cin, int Hi, int Wi, int c0, int ncc, int m0, int nm,
                                                    int n0, int nn, Dst dst) {
  const int i0 = m0 >> 1, ni = ((m0 + nm - 1) >> 1) - i0 + 1, j0 = n0 >> 1, nj = ((n0 + nn - 1) >> 1) - j0 + 1;
  const int run = 4 * ncc, total = ni * nj * run;
  const FastDiv rund(run), jd(nj);
  constexpr int U = 4;
  for (int e0 = threadIdx.x; e0 < total; e0 += U * blockDim.x) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = e0 + u * blockDim.x, px = rund.div(e), k = e - px * run, ii = jd.div(px), i = i0 + ii, j = j0 + px - ii * nj;
      const bool ok = e < total && 4 * c0 + k < 4 * Cin && 2 * i < Hi && 2 * j < Wi;
      v[u] = ok ? __ldg(feat + ((size_t)i * (Wi / 2) + j) * (4 * Cin) + 4 * c0 + k) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int e = e0 + u * blockDim.x, px = rund.div(e), k = e - px * run, ii = jd.div(px);
      const int m = 2 * (i0 + ii) + ((k >> 1) & 1) - m0, n = 2 * (j0 + px - ii * nj) + (k & 1) - n0;
      if (e < total && m >= 0 && m < nm && n >= 0 && n < nn) dst(k >> 2, m, n, v[u]);
    }
  }
}

// ---- forward ------------------------------------------------------------------------------------------------------
// out[o, 2m+py, 2n+px] = bias[o] + sum_c sum_taps in[c, m+dm, n+dn] * Wt[c, o, ky, kx]
//   py=0: (dm,ky)=(0,1);  py=1: (0,2),(1,0)     (y = 2*iy - 1 + ky), same along x.
// SHUFFLE: in[c, m, n] = feat[4c + 2(m&1) + (n&1), m>>1, n>>1]   (PixelShuffle(2)); LPB_SHUFFLE_NHWC: feat is channels-last
// in memory (the staged tile, and so every MMA and every result bit, is the same)
// Each output parity class q = 2 py + px is a GEMM: M = pixels of the block, N = Cout (8 NT per CTA), K = Cin per
// (shift, tap) pair; the 9 pairs below share four shifted A operands, which are constant offsets into the staged tile
// (RB + 1 rows x CB + 1 columns, zero halo).
__device__ constexpr int kFwdShift[9] = {0, 0, 0, 0, 1, 1, 2, 2, 3};  // shift s = 2 dm + dn
__device__ constexpr int kFwdClass[9] = {0, 1, 2, 3, 1, 3, 2, 3, 3};  // output parity q = 2 py + px
__device__ constexpr int kFwdTap[9] = {4, 5, 7, 8, 3, 6, 1, 2, 0};    // ky * 3 + kx

template <int SHUFFLE, int NT>
__global__ void __launch_bounds__(TC_THREADS) convt3x3s2_kernel(const float* __restrict__ in, int Cin, int Hi, int Wi,
                                                                const float* __restrict__ wt, const float* __restrict__ bias,
                                                                int Cout, int RB, int CB, float* __restrict__ out) {
  constexpr int S = bstride<NT>();
  extern __shared__ __align__(16) float sm[];
  const int XR = CB + 1, XP = pad8_32((RB + 1) * XR);
  float* xs = sm;                                                // [FW_CC][XP]: rows r0 .. r0+RB, cols n0 .. n0+CB
  uint32_t* wb = reinterpret_cast<uint32_t*>(sm + FW_CC * XP);  // [9][FW_CC][S] tf32 big
  uint32_t* wsm = wb + 9 * FW_CC * S;                            // [9][FW_CC][S] tf32 small
  const int nbc = (Wi + CB - 1) / CB, nblk = ((Hi + RB - 1) / RB) * nbc;
  const int b = blockIdx.x / nblk, blk = blockIdx.x - b * nblk;
  const int r0 = (blk / nbc) * RB, n0 = (blk - (blk / nbc) * nbc) * CB;
  const int o0 = blockIdx.y * (8 * NT);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;

  int off[2][2];  // staged offset of this lane's A rows (slots g, g + 8 of each m16 tile); 0 for masked slots
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int p = warp * 32 + mt * 16 + h * 8 + g, pr = p / CB, pc = p - pr * CB;
      off[mt][h] = (p < RB * CB && r0 + pr < Hi && n0 + pc < Wi) ? pr * XR + pc : 0;
    }
  float acc[2][4][NT][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) mma::zero(acc[mt]);

  const size_t in_img = (size_t)b * Cin * Hi * Wi;  // = b * 4Cin * (Hi/2) * (Wi/2) with SHUFFLE
  const FastDiv rdiv(RB + 1);
  for (int c0 = 0; c0 < Cin; c0 += FW_CC) {
    __syncthreads();
    if constexpr (SHUFFLE == LPB_SHUFFLE_NHWC)
      stage_shuffled_nhwc(in + in_img, Cin, Hi, Wi, c0, FW_CC, r0, RB + 1, n0, XR, [&](int cc, int m, int n, float v) { xs[cc * XP + m * XR + n] = v; });
    else
    stage_rows<4>(
        FW_CC * (RB + 1), XR,
        [&](int cr, int j) {
          const int cc = rdiv.div(cr), c = c0 + cc, m = r0 + cr - cc * (RB + 1), n = n0 + j;
          if (c >= Cin || m >= Hi || n >= Wi) return 0.f;
          if (SHUFFLE) return __ldg(in + in_img + ((size_t)(4 * c + 2 * (m & 1) + (n & 1)) * (Hi / 2) + (m >> 1)) * (Wi / 2) + (n >> 1));
          return __ldg(in + in_img + ((size_t)c * Hi + m) * Wi + n);
        },
        [&](int cr, int j, float v) {
          const int cc = rdiv.div(cr);
          xs[cc * XP + (cr - cc * (RB + 1)) * XR + j] = v;
        });
    stage_flat<8>(  // weights, global order (c, o, tap) -> [tap][c][o]
        FW_CC * 8 * NT * 9,
        [&](int i) {
          const int tap = i % 9, co = i / 9, ol = co % (8 * NT), cc = co / (8 * NT), c = c0 + cc, o = o0 + ol;
          return (c < Cin && o < Cout) ? __ldg(wt + ((size_t)c * Cout + o) * 9 + tap) : 0.f;
        },
        [&](int i, float v) {
          const int tap = i % 9, co = i / 9, ol = co % (8 * NT), cc = co / (8 * NT);
          mma::split_tf32(v, wb[(tap * FW_CC + cc) * S + ol], wsm[(tap * FW_CC + cc) * S + ol]);
        });
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < FW_CC / 8; ++kk) {
      if (c0 + 8 * kk >= Cin) break;  // an all-zero k8 step (narrow inputs: a second layer's Cin is a keypoint count)
      const float* xk = xs + (kk * 8 + t) * XP;
      uint32_t ab[2][4], as[2][4];
#pragma unroll
      for (int pi = 0; pi < 9; ++pi) {
        const int s = kFwdShift[pi], q = kFwdClass[pi], tap = kFwdTap[pi];
        if (pi == 0 || pi == 4 || pi == 6 || pi == 8) {  // a new shift: its A fragments
          const int so = (s >> 1) * XR + (s & 1);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma::split_tf32(xk[off[mt][0] + so], ab[mt][0], as[mt][0]);
            mma::split_tf32(xk[off[mt][1] + so], ab[mt][1], as[mt][1]);
            mma::split_tf32(xk[4 * XP + off[mt][0] + so], ab[mt][2], as[mt][2]);
            mma::split_tf32(xk[4 * XP + off[mt][1] + so], ab[mt][3], as[mt][3]);
          }
        }
        const int wo = (tap * FW_CC + kk * 8 + t) * S + g;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const uint32_t bb0 = wb[wo + nt * 8], bb1 = wb[wo + 4 * S + nt * 8];
          const uint32_t bs0 = wsm[wo + nt * 8], bs1 = wsm[wo + 4 * S + nt * 8];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) mma::mma_3xtf32(acc[mt][q][nt], ab[mt], as[mt], bb0, bb1, bs0, bs1);
        }
      }
    }
  }
  // c (g [+8], 2t + j): the two x parities of one (pixel, channel, row parity) are one float2 of the output row
  const int Ho = 2 * Hi, Wo = 2 * Wi;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int p = warp * 32 + mt * 16 + h * 8 + g, pr = p / CB, pc = p - pr * CB, m = r0 + pr, n = n0 + pc;
      if (p >= RB * CB || m >= Hi || n >= Wi) continue;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int o = o0 + nt * 8 + 2 * t + j;
          if (o >= Cout) continue;
          const float bv = bias ? __ldg(bias + o) : 0.f;
          float* dst = out + (((size_t)b * Cout + o) * Ho + 2 * m) * Wo + 2 * n;
          *reinterpret_cast<float2*>(dst) = make_float2(acc[mt][0][nt][2 * h + j] + bv, acc[mt][1][nt][2 * h + j] + bv);
          *reinterpret_cast<float2*>(dst + Wo) = make_float2(acc[mt][2][nt][2 * h + j] + bv, acc[mt][3][nt][2 * h + j] + bv);
        }
    }
}

// in-place softmax over each (b, k) plane: one HBM read + one write (plane staged in smem)
__global__ void __launch_bounds__(256) plane_softmax_kernel(float* __restrict__ x, int hw) {
  extern __shared__ float pl[];
  __shared__ float red[8];
  float* p = x + (size_t)blockIdx.x * hw;
  float mx = -3.0e38f;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const float v = p[i];
    pl[i] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
  float s = 0.f;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const float e = expf(pl[i] - mx);
    pl[i] = e;
    s += e;
  }
  s = warp_sum(s);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += red[k];
  const float inv = 1.0f / s;
  for (int i = threadIdx.x; i < hw; i += 256) p[i] = pl[i] * inv;
}

// n_planes >= 1 planes of hw pixels each, softmaxed in place; `entry` names the caller in errors
static int launch_plane_softmax(float* x, int64_t n_planes, int hw, const char* entry, cudaStream_t s) {
  const size_t smem = (size_t)hw * sizeof(float);
  LPB_TRY(set_dynamic_smem(plane_softmax_kernel, smem, entry));
  plane_softmax_kernel<<<(unsigned)n_planes, 256, smem, s>>>(x, hw);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}


template <int SHUFFLE, int NT>
static int launch_fwd_nt(const float* in, int B, int Cin, int Hi, int Wi, const float* wt, const float* bias, int Cout, float* out,
                          cudaStream_t s) {
  const PixBlocks pb = pix_blocks(Hi, Wi);
  const size_t smem = ((size_t)FW_CC * pad8_32((pb.RB + 1) * (pb.CB + 1)) + 2 * 9 * FW_CC * bstride<NT>()) * sizeof(float);
  LPB_TRY(set_dynamic_smem(convt3x3s2_kernel<SHUFFLE, NT>, smem, "convt_fwd_f32"));
  const dim3 grid((unsigned)((size_t)B * pb.n), (unsigned)((Cout + 8 * NT - 1) / (8 * NT)));
  convt3x3s2_kernel<SHUFFLE, NT><<<grid, TC_THREADS, smem, s>>>(in, Cin, Hi, Wi, wt, bias, Cout, pb.RB, pb.CB, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

template <int SHUFFLE>
static int launch_fwd(const float* in, int B, int Cin, int Hi, int Wi, const float* wt, const float* bias, int Cout, float* out,
                      cudaStream_t s) {
  // N tile = Cout rounded up to 8, at most 24 channels (wider heads: more CTAs along y)
  if (Cout <= 8) return launch_fwd_nt<SHUFFLE, 1>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s);
  if (Cout <= 16) return launch_fwd_nt<SHUFFLE, 2>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s);
  return launch_fwd_nt<SHUFFLE, 3>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s);
}

static int launch_convt(int shuffle, const float* in, int B, int Cin, int Hi, int Wi, const float* wt, const float* bias,
                        int Cout, float* out, cudaStream_t s) {
  if (shuffle == LPB_SHUFFLE_NHWC) return launch_fwd<LPB_SHUFFLE_NHWC>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s);
  return shuffle ? launch_fwd<LPB_SHUFFLE_NCHW>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s)
                 : launch_fwd<LPB_SHUFFLE_NONE>(in, B, Cin, Hi, Wi, wt, bias, Cout, out, s);
}

// ---- backward of one transposed convolution -----------------------------------------------------------------------
// In scatter form input pixel (m, n) feeds output pixel (2m - 1 + ky, 2n - 1 + kx), so
//   d in[c, m, n]      = sum_o sum_{ky,kx} g[o, 2m-1+ky, 2n-1+kx] * W[c, o, ky, kx]           (data gradient)
//   d W[c, o, ky, kx]  = sum_{b, m, n} in[c, m, n] * g[o, 2m-1+ky, 2n-1+kx]                   (weight gradient)
//   d bias[o]          = sum g[o]  (= the taps (1..2, 1..2), which partition the output pixels)
// Both kernels stage, per output channel, the gradient tile of a pixel block: output rows 2 r0 - 1 .. 2 (r0 + RB) - 1
// (GR = 2 RB + 1) and columns 2 n0 - 1 .. 2 (n0 + CB) - 1 (GC = 2 CB + 1), zero outside the map.  A row is stored with
// its even columns first (CB + 1 of them) and its odd columns after, so the taps of consecutive pixels are
// consecutive words: tap (ky, kx) of pixel slot (pr, pc) sits at  2 pr GC + pc + ky GC + (kx == 1 ? CB + 1 : kx / 2).
__device__ __forceinline__ int grad_tap_offset(int tap, int GC, int CB) {
  const int ky = tap / 3, kx = tap - 3 * (tap / 3);
  return ky * GC + (kx == 1 ? CB + 1 : kx >> 1);
}

__device__ __forceinline__ void stage_grad_planes(const float* __restrict__ g, int b, int Cout, int Hi, int Wi, int o0, int np, int r0,
                                                  int n0, int RB, int CB, int GP, float* __restrict__ gs) {
  const int Ho = 2 * Hi, Wo = 2 * Wi, GR = 2 * RB + 1, GC = 2 * CB + 1;
  const FastDiv rdiv(GR);
  stage_rows<4>(
      np * GR, GC,
      [&](int orow, int j) {
        const int ol = rdiv.div(orow), o = o0 + ol, y = 2 * r0 - 1 + orow - ol * GR, x = 2 * n0 - 1 + j;
        return (o < Cout && y >= 0 && y < Ho && x >= 0 && x < Wo) ? __ldg(g + (((size_t)b * Cout + o) * Ho + y) * Wo + x) : 0.f;
      },
      [&](int orow, int j, float v) {
        const int ol = rdiv.div(orow);
        gs[ol * GP + (orow - ol * GR) * GC + ((j & 1) ? CB + 1 + (j >> 1) : (j >> 1))] = v;
      });
}

// Data gradient: M = pixels of the block, N = Cin (8 NT per CTA), K = Cout x 9 in stages of 8 output channels
// (72 = 9 k8 steps, k = o_local * 9 + tap; the weights [c][o][tap] are K-contiguous).
template <int SHUFFLE, int NT>
__global__ void __launch_bounds__(TC_THREADS) convt3x3s2_dgrad_kernel(const float* __restrict__ g, int Cout, int Hi, int Wi,
                                                                      const float* __restrict__ wt, int Cin, int RB, int CB,
                                                                      float* __restrict__ din) {
  constexpr int S = bstride<NT>();
  extern __shared__ __align__(16) float sm[];
  const int GC = 2 * CB + 1, GP = pad8_32((2 * RB + 1) * GC);
  float* gs = sm;                                               // [8][GP]
  uint32_t* wb = reinterpret_cast<uint32_t*>(sm + 8 * GP);     // [72][S] tf32 big
  uint32_t* wsm = wb + 72 * S;                                  // [72][S] tf32 small
  const int nbc = (Wi + CB - 1) / CB, nblk = ((Hi + RB - 1) / RB) * nbc;
  const int b = blockIdx.x / nblk, blk = blockIdx.x - b * nblk;
  const int r0 = (blk / nbc) * RB, n0 = (blk - (blk / nbc) * nbc) * CB;
  const int c0 = blockIdx.y * (8 * NT);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g8 = lane >> 2, t = lane & 3;

  int pbase[2][2];  // this lane's A rows: 2 pr GC + pc (0 for masked slots, whose results are never stored)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int p = warp * 32 + mt * 16 + h * 8 + g8, pr = p / CB, pc = p - pr * CB;
      pbase[mt][h] = p < RB * CB ? 2 * pr * GC + pc : 0;
    }
  int koff[9][2];  // this lane's A columns k = 8 ks + t (+4) of a stage
#pragma unroll
  for (int ks = 0; ks < 9; ++ks)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = 8 * ks + t + 4 * h, ol = k / 9;
      koff[ks][h] = ol * GP + grad_tap_offset(k - 9 * ol, GC, CB);
    }
  float acc[2][NT][4];
  mma::zero(acc);

  for (int o0 = 0; o0 < Cout; o0 += 8) {
    __syncthreads();
    stage_grad_planes(g, b, Cout, Hi, Wi, o0, 8, r0, n0, RB, CB, GP, gs);
    stage_flat<8>(  // weights [c][o][tap]: K-contiguous per input channel -> [k][c]
        8 * NT * 72,
        [&](int i) {
          const int k = i % 72, c = c0 + i / 72;
          return (c < Cin && o0 + k / 9 < Cout) ? __ldg(wt + ((size_t)c * Cout + o0) * 9 + k) : 0.f;
        },
        [&](int i, float v) { mma::split_tf32(v, wb[(i % 72) * S + i / 72], wsm[(i % 72) * S + i / 72]); });
    __syncthreads();
    const int nks = min(9, ((Cout - o0) * 9 + 7) / 8);
#pragma unroll
    for (int ks = 0; ks < 9; ++ks) {
      if (ks >= nks) break;
      uint32_t ab[2][4], as[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        mma::split_tf32(gs[pbase[mt][0] + koff[ks][0]], ab[mt][0], as[mt][0]);
        mma::split_tf32(gs[pbase[mt][1] + koff[ks][0]], ab[mt][1], as[mt][1]);
        mma::split_tf32(gs[pbase[mt][0] + koff[ks][1]], ab[mt][2], as[mt][2]);
        mma::split_tf32(gs[pbase[mt][1] + koff[ks][1]], ab[mt][3], as[mt][3]);
      }
      const int wo = (8 * ks + t) * S + g8;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const uint32_t bb0 = wb[wo + nt * 8], bb1 = wb[wo + 4 * S + nt * 8];
        const uint32_t bs0 = wsm[wo + nt * 8], bs1 = wsm[wo + 4 * S + nt * 8];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) mma::mma_3xtf32(acc[mt][nt], ab[mt], as[mt], bb0, bb1, bs0, bs1);
      }
    }
  }
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int p = warp * 32 + mt * 16 + h * 8 + g8, pr = p / CB, pc = p - pr * CB, m = r0 + pr, n = n0 + pc;
      if (p >= RB * CB || m >= Hi || n >= Wi) continue;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int c = c0 + nt * 8 + 2 * t + j;
          if (c >= Cin) continue;
          const float v = acc[mt][nt][2 * h + j];
          if (SHUFFLE == LPB_SHUFFLE_NHWC)
            din[(((size_t)b * (Hi / 2) + (m >> 1)) * (Wi / 2) + (n >> 1)) * (4 * Cin) + 4 * c + 2 * (m & 1) + (n & 1)] = v;
          else if (SHUFFLE)
            din[(((size_t)b * 4 * Cin + 4 * c + 2 * (m & 1) + (n & 1)) * (Hi / 2) + (m >> 1)) * (Wi / 2) + (n >> 1)] = v;
          else
            din[(((size_t)b * Cin + c) * Hi + m) * Wi + n] = v;
        }
    }
}

// Weight gradient: M = Cin (32 WM per CTA), N = Cout x 9 (n = o * 9 + tap, 8 NT WN per CTA), K = pixels.  K is split
// over gridDim.y CTAs ("slots"), each looping over its share of the (frame, pixel block) units with the tile in
// registers.  A = the input [c][slot] (row stride 132 = 4 mod 32: the (g, t) pattern on 32 banks), B = the staged
// gradient planes of the CTA's output channels.  The CTAs of the first channel tile also sum the bias gradient (the four
// taps (1..2, 1..2)) of their channels: warp w takes channels w, w + warps, ...; its lanes sum the unit's pixels and
// the warp's shuffle sum is added to the channel's running total, so that sum has a fixed order too.
// The tile and bias sums are stored into the slot's partial, dw / db + blockIdx.y * slot_stride, one writer per
// element, and reduce_partials adds the slots in slot order (bit-reproducible).
constexpr int WG_PS = TC_SLOTS + 4;

template <int SHUFFLE, int WM, int WN, int NT>
__global__ void __launch_bounds__(32 * WM * WN) convt3x3s2_wgrad_kernel(const float* __restrict__ in, const float* __restrict__ g,
                                                                        int B, int Cin, int Cout, int Hi, int Wi, int RB, int CB,
                                                                        float* __restrict__ dw, float* __restrict__ db, size_t slot_stride) {
  constexpr int CM = 32 * WM, CN = 8 * NT * WN, THREADS = 32 * WM * WN;
  extern __shared__ __align__(16) float sm[];
  const int GC = 2 * CB + 1, GP = pad8_32((2 * RB + 1) * GC);
  const int nct = (Cin + CM - 1) / CM, ct = blockIdx.x % nct, c0 = ct * CM, n0 = (blockIdx.x / nct) * CN;
  const int o_lo = n0 / 9, np = min(Cout, (n0 + CN - 1) / 9 + 1) - o_lo;
  float* xs = sm;                                               // [CM][WG_PS]
  float* gs = xs + CM * WG_PS;                                  // [np][GP]
  int* pbt = reinterpret_cast<int*>(gs + np * GP);             // [TC_SLOTS]: slot -> 2 pr GC + pc
  float* dbs = reinterpret_cast<float*>(pbt + TC_SLOTS);        // [np]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g8 = lane >> 2, t = lane & 3;
  const int wm = warp % WM, wn = warp / WM;
  const bool do_bias = db != nullptr && ct == 0;
  dw += blockIdx.y * slot_stride;
  if (db) db += blockIdx.y * slot_stride;

  for (int i = threadIdx.x; i < CM * WG_PS; i += THREADS) xs[i] = 0.f;  // slots past RB * CB stay zero
  for (int p = threadIdx.x; p < TC_SLOTS; p += THREADS) pbt[p] = p < RB * CB ? 2 * (p / CB) * GC + p % CB : 0;
  for (int i = threadIdx.x; i < np; i += THREADS) dbs[i] = 0.f;
  int koff[NT];  // this lane's B column n = n0 + 8 (NT wn + nt) + g (clamped to plane 0 past Cout x 9: never stored)
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int n = n0 + 8 * (NT * wn + nt) + g8, o = n / 9;
    koff[nt] = n < Cout * 9 ? (o - o_lo) * GP + grad_tap_offset(n - 9 * o, GC, CB) : 0;
  }
  float acc[2][NT][4];
  mma::zero(acc);

  const int nbc = (Wi + CB - 1) / CB, nblk = ((Hi + RB - 1) / RB) * nbc;
  const FastDiv rdiv(RB);
  const long long units = (long long)B * nblk;
  for (long long u = blockIdx.y; u < units; u += gridDim.y) {
    const int b = (int)(u / nblk), blk = (int)(u - (long long)b * nblk);
    const int r0 = (blk / nbc) * RB, q0 = (blk - (blk / nbc) * nbc) * CB;
    __syncthreads();
    if constexpr (SHUFFLE == LPB_SHUFFLE_NHWC)
      stage_shuffled_nhwc(in + (size_t)b * Cin * Hi * Wi, Cin, Hi, Wi, c0, CM, r0, RB, q0, CB, [&](int cc, int m, int n, float v) { xs[cc * WG_PS + m * CB + n] = v; });
    else
    stage_rows<4>(
        CM * RB, CB,
        [&](int cr, int pc) {
          const int cc = rdiv.div(cr), c = c0 + cc, m = r0 + cr - cc * RB, n = q0 + pc;
          if (c >= Cin || m >= Hi || n >= Wi) return 0.f;
          if (SHUFFLE) return __ldg(in + (((size_t)b * 4 * Cin + 4 * c + 2 * (m & 1) + (n & 1)) * (Hi / 2) + (m >> 1)) * (Wi / 2) + (n >> 1));
          return __ldg(in + (((size_t)b * Cin + c) * Hi + m) * Wi + n);
        },
        [&](int cr, int pc, float v) {
          const int cc = rdiv.div(cr);
          xs[cc * WG_PS + (cr - cc * RB) * CB + pc] = v;
        });
    stage_grad_planes(g, b, Cout, Hi, Wi, o_lo, np, r0, q0, RB, CB, GP, gs);
    __syncthreads();
    if (do_bias) {
      const int hw = RB * CB;
      for (int ol = warp; ol < np; ol += WM * WN) {
        float sb = 0.f;
        for (int p = lane; p < hw; p += 32) {
          const int pr = p / CB, pc = p - pr * CB;
          if (r0 + pr >= Hi || q0 + pc >= Wi) continue;
          const float* gp = gs + ol * GP + pbt[p];
          sb += (gp[GC + CB + 1] + gp[GC + 1]) + (gp[2 * GC + CB + 1] + gp[2 * GC + 1]);  // taps 4, 5, 7, 8
        }
        sb = warp_sum(sb);
        if (lane == 0) dbs[ol] += sb;  // only this warp touches dbs[ol]; the units follow one another
      }
    }
#pragma unroll 4
    for (int ks = 0; ks < TC_SLOTS / 8; ++ks) {
      uint32_t ab[2][4], as[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const float* xa = xs + (32 * wm + 16 * mt + g8) * WG_PS + 8 * ks + t;
        mma::split_tf32(xa[0], ab[mt][0], as[mt][0]);
        mma::split_tf32(xa[8 * WG_PS], ab[mt][1], as[mt][1]);
        mma::split_tf32(xa[4], ab[mt][2], as[mt][2]);
        mma::split_tf32(xa[8 * WG_PS + 4], ab[mt][3], as[mt][3]);
      }
      const int p0 = pbt[8 * ks + t], p1 = pbt[8 * ks + t + 4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        uint32_t bb0, bb1, bs0, bs1;
        mma::split_tf32(gs[p0 + koff[nt]], bb0, bs0);
        mma::split_tf32(gs[p1 + koff[nt]], bb1, bs1);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) mma::mma_3xtf32(acc[mt][nt], ab[mt], as[mt], bb0, bb1, bs0, bs1);
      }
    }
  }
  const int nk = Cout * 9;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = c0 + 32 * wm + 16 * mt + 8 * h + g8;
      if (c >= Cin) continue;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = n0 + 8 * (NT * wn + nt) + 2 * t + j;
          if (n >= nk) continue;
          dw[(size_t)c * nk + n] = acc[mt][nt][2 * h + j];
        }
    }
  if (do_bias) {
    __syncthreads();
    for (int ol = threadIdx.x; ol < np; ol += THREADS) {
      const int o = o_lo + ol;
      if (o * 9 < n0) continue;  // channel o belongs to the n tile that holds its tap 0
      db[o] = dbs[ol];
    }
  }
}

// K split of the weight gradient: about `ctas` CTAs in all, each with as many units as that leaves (one tile row of
// partials per CTA).  `ctas` is capped at F32_WG_MAX_CTAS, which bounds the workspace without a device query; on an
// H100 SXM (132 SMs) the cap equals the 2 CTAs per SM asked for, so it does not bind.
constexpr int F32_WG_MAX_CTAS = 264;
constexpr int F32_WG_CN = 160;  // N tile of both tilings below: 8 NT WN
static long long wgrad_f32_slots(int B, int Cin, int Cout, int Hi, int Wi, int ctas) {
  const int CM = Cin > 32 ? 128 : 32;
  const PixBlocks pb = pix_blocks(Hi, Wi);
  const long long tiles = (long long)((Cin + CM - 1) / CM) * ((Cout * 9 + F32_WG_CN - 1) / F32_WG_CN);
  const long long units = (long long)B * pb.n;
  return std::min<long long>(units, std::max<long long>(1, (ctas + tiles - 1) / tiles));
}
// one slot of the partials: its grad_w tile sums [Cin * Cout * 9], then its bias sums [Cout]
static size_t wgrad_f32_part_stride(int Cin, int Cout) { return (size_t)Cin * Cout * 9 + Cout; }

template <int SHUFFLE, int WM, int WN, int NT>
static int launch_wgrad(const float* in, const float* g, int B, int Cin, int Cout, int Hi, int Wi, float* dw, float* db, float* part,
                        cudaStream_t s) {
  constexpr int CM = 32 * WM, CN = 8 * NT * WN;
  static_assert(CN == F32_WG_CN && (CM == 128) == (WM == 4), "wgrad_f32_slots assumes this tiling");
  const PixBlocks pb = pix_blocks(Hi, Wi);
  const int nct = (Cin + CM - 1) / CM, nnt = (Cout * 9 + CN - 1) / CN;
  const int np_max = CN / 9 + 2;
  const size_t smem =
      ((size_t)CM * WG_PS + (size_t)np_max * pad8_32((2 * pb.RB + 1) * (2 * pb.CB + 1)) + TC_SLOTS + np_max) * sizeof(float);
  DeviceLimits dev;
  LPB_TRY(device_limits(&dev));
  const long long ks = wgrad_f32_slots(B, Cin, Cout, Hi, Wi, std::min(2 * dev.sms, F32_WG_MAX_CTAS));
  const dim3 grid((unsigned)(nct * nnt), (unsigned)ks);
  const size_t stride = wgrad_f32_part_stride(Cin, Cout), nw = (size_t)Cin * Cout * 9;
  LPB_TRY(set_dynamic_smem(convt3x3s2_wgrad_kernel<SHUFFLE, WM, WN, NT>, smem, "convt_bwd_f32"));
  convt3x3s2_wgrad_kernel<SHUFFLE, WM, WN, NT><<<grid, 32 * WM * WN, smem, s>>>(in, g, B, Cin, Cout, Hi, Wi, pb.RB, pb.CB, part,
                                                                                db ? part + nw : nullptr, stride);
  reduce_partials<1>(part, (int)ks, stride, (int)nw, dw, dev.sms, s);
  if (db) reduce_partials<1>(part + nw, (int)ks, stride, Cout, db, dev.sms, s);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

template <int SHUFFLE>
static int launch_bwd(const float* in, const float* g, int B, int Cin, int Hi, int Wi, const float* wt, int Cout, float* din, float* dw,
                      float* db, float* part, cudaStream_t s) {
  // M tile: 128 input channels, or 32 for narrow inputs (a second layer's Cin is the first layer's keypoint count)
  const int rc = Cin > 32 ? launch_wgrad<SHUFFLE, 4, 2, 10>(in, g, B, Cin, Cout, Hi, Wi, dw, db, part, s)
                          : launch_wgrad<SHUFFLE, 1, 4, 5>(in, g, B, Cin, Cout, Hi, Wi, dw, db, part, s);
  if (rc || !din) return rc;
  const PixBlocks pb = pix_blocks(Hi, Wi);
  const size_t gfl = (size_t)8 * pad8_32((2 * pb.RB + 1) * (2 * pb.CB + 1));
  auto go = [&](auto kernel, int nt, int stride) -> int {
    const size_t smem = (gfl + (size_t)2 * 72 * stride) * sizeof(float);
    LPB_TRY(set_dynamic_smem(kernel, smem, "convt_bwd_f32"));
    const dim3 grid((unsigned)((size_t)B * pb.n), (unsigned)((Cin + 8 * nt - 1) / (8 * nt)));
    kernel<<<grid, TC_THREADS, smem, s>>>(g, Cout, Hi, Wi, wt, Cin, pb.RB, pb.CB, din);
    LPB_CUDA(cudaGetLastError());
    return LPB_OK;
  };
  // N tile = Cin rounded up to 8, 16, 24, 32 or 64 channels
  if (Cin <= 8) return go(convt3x3s2_dgrad_kernel<SHUFFLE, 1>, 1, bstride<1>());
  if (Cin <= 16) return go(convt3x3s2_dgrad_kernel<SHUFFLE, 2>, 2, bstride<2>());
  if (Cin <= 24) return go(convt3x3s2_dgrad_kernel<SHUFFLE, 3>, 3, bstride<3>());
  if (Cin <= 32) return go(convt3x3s2_dgrad_kernel<SHUFFLE, 4>, 4, bstride<4>());
  return go(convt3x3s2_dgrad_kernel<SHUFFLE, 8>, 8, bstride<8>());
}

// part: the workspace of lpb_convt_bwd_f32_ws (the weight gradient's per-slot partials)
static int convt_bwd_f32(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w, int Cout,
                         float* grad_in, float* grad_w, float* grad_bias, float* part, cudaStream_t s) {
  if (B == 0) {  // no partials to sum: the gradients of an empty batch are zero
    LPB_CUDA(cudaMemsetAsync(grad_w, 0, sizeof(float) * (size_t)Cin * Cout * 9, s));
    if (grad_bias) LPB_CUDA(cudaMemsetAsync(grad_bias, 0, sizeof(float) * Cout, s));
    return LPB_OK;
  }
  if (shuffle == LPB_SHUFFLE_NHWC) return launch_bwd<LPB_SHUFFLE_NHWC>(in, grad_out, B, Cin, Hi, Wi, w, Cout, grad_in, grad_w, grad_bias, part, s);
  return shuffle ? launch_bwd<LPB_SHUFFLE_NCHW>(in, grad_out, B, Cin, Hi, Wi, w, Cout, grad_in, grad_w, grad_bias, part, s)
                 : launch_bwd<LPB_SHUFFLE_NONE>(in, grad_out, B, Cin, Hi, Wi, w, Cout, grad_in, grad_w, grad_bias, part, s);
}

}  // namespace lpb

// one layer at a time: the Python side (models/heads/heatmap.py) chains any number of deconvs
extern "C" int lpb_convt_fwd_f32(const float* in, int B, int Cin, int Hi, int Wi, int shuffle, const float* w, const float* bias,
                                 int Cout, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(in && w && out, "convt_fwd_f32: null pointer");
  LPB_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1 && Hi >= 1 && Wi >= 1 && (!shuffle || (Hi % 2 == 0 && Wi % 2 == 0)), "convt_fwd_f32: bad shape");
  if (B == 0) return LPB_OK;
  return launch_convt(shuffle, in, B, Cin, Hi, Wi, w, bias, Cout, out, static_cast<cudaStream_t>(stream));
}

extern "C" int lpb_plane_softmax_f32(float* x, int64_t n_planes, int hw, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(x && n_planes >= 0 && hw >= 1, "plane_softmax_f32: bad arguments");
  if (n_planes == 0) return LPB_OK;
  return launch_plane_softmax(x, n_planes, hw, "plane_softmax_f32", static_cast<cudaStream_t>(stream));
}

extern "C" int lpb_convt_bwd_f32_workspace_bytes(int B, int Cin, int Hi, int Wi, int Cout, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "convt_bwd_f32_workspace_bytes: null pointer");
  LPB_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1 && Hi >= 1 && Wi >= 1, "convt_bwd_f32_workspace_bytes: bad shape");
  *bytes = B == 0 ? 0 : (size_t)wgrad_f32_slots(B, Cin, Cout, Hi, Wi, F32_WG_MAX_CTAS) * wgrad_f32_part_stride(Cin, Cout) * sizeof(float);
  return LPB_OK;
}

extern "C" int lpb_convt_bwd_f32_ws(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w,
                                    int Cout, float* grad_in, float* grad_w, float* grad_bias, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  using namespace lpb;
  LPB_REQUIRE(in && grad_out && w && grad_w, "convt_bwd_f32_ws: null pointer");
  LPB_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1 && Hi >= 1 && Wi >= 1 && (!shuffle || (Hi % 2 == 0 && Wi % 2 == 0)),
              "convt_bwd_f32_ws: bad shape");
  size_t need = 0;
  LPB_TRY(lpb_convt_bwd_f32_workspace_bytes(B, Cin, Hi, Wi, Cout, &need));
  LPB_REQUIRE(B == 0 || (workspace && aligned_to(workspace, 4)), "convt_bwd_f32_ws: null or unaligned workspace");
  LPB_REQUIRE(workspace_bytes >= need, "convt_bwd_f32_ws: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  return convt_bwd_f32(in, grad_out, B, Cin, Hi, Wi, shuffle, w, Cout, grad_in, grad_w, grad_bias, static_cast<float*>(workspace),
                       static_cast<cudaStream_t>(stream));
}
