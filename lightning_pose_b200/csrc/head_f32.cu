// fp32 heatmap head: PixelShuffle(2) -> ConvTranspose2d(k3,s2,p1,op1) [x2] -> spatial softmax (T=1).
// Reference: lightning_pose/models/heads/heatmap.py:20-71 (layer stack), :203-212 (forward).
//
// This is the full-precision path (reference training is fp32, lightning_pose/train.py:411-428):
// CUDA-core FMA with fp32 accumulation, gather-form transposed convolution (each thread owns one
// input pixel and produces its 2x2 output quad for a group of output channels, so there is no
// scatter / atomics), PixelShuffle folded into the shared-memory staging of the first layer.
// The bf16 tensor-core path lives in head_bf16.cu.
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {

constexpr int CT_CC = 8;        // input channels staged per iteration
constexpr int CT_OG = 5;        // groups of 4 output channels per pass (20 >= 17 keypoints)
constexpr int CT_KO = 4 * CT_OG;
constexpr int CT_MAX_THREADS = 256;

// out[o, 2m+py, 2n+px] = bias[o] + sum_c sum_taps in[c, m+dm, n+dn] * Wt[c, o, ky, kx]
//   py=0: (dm,ky)=(0,1);  py=1: (0,2),(1,0)     (y = 2*iy - 1 + ky), same along x.
// SHUFFLE: in[c, m, n] = feat[4c + 2(m&1) + (n&1), m>>1, n>>1]   (PixelShuffle(2))
template <bool SHUFFLE>
__global__ void __launch_bounds__(CT_MAX_THREADS) convt3x3s2_kernel(const float* __restrict__ in, int Cin, int Hi, int Wi,
                                                                    const float* __restrict__ wt,
                                                                    const float* __restrict__ bias, int Cout, int TR,
                                                                    float* __restrict__ out) {
  // Hi, Wi: spatial size of the (shuffled) conv input; output is (Cout, 2Hi, 2Wi)
  extern __shared__ __align__(16) float sm[];
  const int xs_row = Wi + 1;
  const int xs_plane = (TR + 1) * xs_row;
  float* xs = sm;                                   // [CT_CC][TR+1][Wi+1]
  float* ws = sm + ((CT_CC * xs_plane + 3) & ~3);   // [CT_CC][CT_KO*9], 16-B aligned rows (180 floats)
  const int tiles_per_img = (Hi + TR - 1) / TR;
  const int b = blockIdx.x / tiles_per_img;
  const int m0 = (blockIdx.x - b * tiles_per_img) * TR;
  const int o0 = blockIdx.y * CT_KO;
  const int nquad = TR * Wi;
  const int q = threadIdx.x;
  const int qm = q / Wi, qn = q - qm * Wi;
  const bool active = (q < nquad) && (m0 + qm < Hi);

  float acc[CT_KO][4];
#pragma unroll
  for (int o = 0; o < CT_KO; ++o) acc[o][0] = acc[o][1] = acc[o][2] = acc[o][3] = 0.f;

  const size_t in_img = SHUFFLE ? (size_t)b * (4 * Cin) * (Hi / 2) * (Wi / 2) : (size_t)b * Cin * Hi * Wi;
  for (int c0 = 0; c0 < Cin; c0 += CT_CC) {
    __syncthreads();
    // ---- stage inputs (rows m0 .. m0+TR, cols 0 .. Wi; zero halo) ----
    for (int i = threadIdx.x; i < CT_CC * xs_plane; i += blockDim.x) {
      const int cc = i / xs_plane, r = (i - cc * xs_plane) / xs_row, n = i - cc * xs_plane - r * xs_row;
      const int c = c0 + cc, m = m0 + r;
      float v = 0.f;
      if (c < Cin && m < Hi && n < Wi) {
        if (SHUFFLE) {
          const int ch = 4 * c + 2 * (m & 1) + (n & 1);
          v = __ldg(in + in_img + ((size_t)ch * (Hi / 2) + (m >> 1)) * (Wi / 2) + (n >> 1));
        } else {
          v = __ldg(in + in_img + ((size_t)c * Hi + m) * Wi + n);
        }
      }
      xs[i] = v;
    }
    // ---- stage weights for output channels o0 .. o0+CT_KO ----
    for (int i = threadIdx.x; i < CT_CC * CT_KO * 9; i += blockDim.x) {
      const int cc = i / (CT_KO * 9), r = i - cc * (CT_KO * 9);
      const int o = o0 + r / 9, c = c0 + cc;
      ws[i] = (c < Cin && o < Cout) ? __ldg(wt + ((size_t)c * Cout + o) * 9 + (r % 9)) : 0.f;
    }
    __syncthreads();
    if (active) {
#pragma unroll 2
      for (int cc = 0; cc < CT_CC; ++cc) {
        const float* xp = xs + cc * xs_plane + qm * xs_row + qn;
        const float x00 = xp[0], x01 = xp[1], x10 = xp[xs_row], x11 = xp[xs_row + 1];
        const float4* w4 = reinterpret_cast<const float4*>(ws + cc * (CT_KO * 9));
#pragma unroll
        for (int g = 0; g < CT_OG; ++g) {
          float w[36];
#pragma unroll
          for (int k = 0; k < 9; ++k) {
            const float4 t = w4[g * 9 + k];
            w[4 * k] = t.x;
            w[4 * k + 1] = t.y;
            w[4 * k + 2] = t.z;
            w[4 * k + 3] = t.w;
          }
#pragma unroll
          for (int oo = 0; oo < 4; ++oo) {
            const float* k9 = w + oo * 9;  // [ky][kx]
            float* a = acc[g * 4 + oo];
            a[0] = fmaf(x00, k9[4], a[0]);                                                      // (even, even)
            a[1] = fmaf(x00, k9[5], fmaf(x01, k9[3], a[1]));                                    // (even, odd)
            a[2] = fmaf(x00, k9[7], fmaf(x10, k9[1], a[2]));                                    // (odd, even)
            a[3] = fmaf(x00, k9[8], fmaf(x01, k9[6], fmaf(x10, k9[2], fmaf(x11, k9[0], a[3]))));  // (odd, odd)
          }
        }
      }
    }
  }
  if (!active) return;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const int y = 2 * (m0 + qm), x = 2 * qn;
#pragma unroll
  for (int o = 0; o < CT_KO; ++o) {
    if (o0 + o >= Cout) break;
    const float bv = bias ? __ldg(bias + o0 + o) : 0.f;
    float* dst = out + (((size_t)b * Cout + o0 + o) * Ho + y) * Wo + x;
    *reinterpret_cast<float2*>(dst) = make_float2(acc[o][0] + bv, acc[o][1] + bv);
    *reinterpret_cast<float2*>(dst + Wo) = make_float2(acc[o][2] + bv, acc[o][3] + bv);
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

static int launch_convt(bool shuffle, const float* in, int B, int Cin, int Hi, int Wi, const float* wt, const float* bias,
                        int Cout, float* out, cudaStream_t s) {
  int TR = CT_MAX_THREADS / Wi;
  LPB_REQUIRE(TR >= 1, "head: conv input width %d > %d unsupported", Wi, CT_MAX_THREADS);
  if (TR > Hi) TR = Hi;
  const int threads = ((TR * Wi + 31) / 32) * 32;
  const int tiles = (Hi + TR - 1) / TR;
  const size_t smem = (size_t)(((CT_CC * (TR + 1) * (Wi + 1) + 3) & ~3) + CT_CC * CT_KO * 9) * sizeof(float);
  dim3 grid((unsigned)(B * tiles), (unsigned)((Cout + CT_KO - 1) / CT_KO));
  if (shuffle)
    convt3x3s2_kernel<true><<<grid, threads, smem, s>>>(in, Cin, Hi, Wi, wt, bias, Cout, TR, out);
  else
    convt3x3s2_kernel<false><<<grid, threads, smem, s>>>(in, Cin, Hi, Wi, wt, bias, Cout, TR, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

// ---- backward of one transposed convolution (fp32, CUDA cores) --------------------------------------
// In scatter form input pixel (m, n) feeds output pixel (2m - 1 + ky, 2n - 1 + kx), so
//   d in[c, m, n]      = sum_o sum_{ky,kx} g[o, 2m-1+ky, 2n-1+kx] * W[c, o, ky, kx]           (data gradient)
//   d W[c, o, ky, kx]  = sum_{b, m, n} in[c, m, n] * g[o, 2m-1+ky, 2n-1+kx]                   (weight gradient)
//   d bias[o]          = sum g[o]  (= the taps (1..2, 1..2), which partition the output pixels)
// Both kernels stage the gradient tile of a band of input rows (output rows 2m0-1 .. 2(m0+TR)-1, all Cout planes)
// in shared memory.  SHUFFLE folds PixelShuffle(2) (and its inverse for d in) into the addressing.
constexpr int CB_CG = 32;  // input channels per CTA (data gradient)
constexpr int CB_WC = 8;   // input channels per CTA (weight gradient)

__device__ __forceinline__ void stage_grad_tile(const float* __restrict__ g, int b, int Cout, int Hi, int Wi, int m0, int TR,
                                                float* __restrict__ gs) {
  const int Ho = 2 * Hi, Wo = 2 * Wi, gr = 2 * TR + 1, gc = 2 * Wi + 1;
  for (int i = threadIdx.x; i < Cout * gr * gc; i += blockDim.x) {
    const int o = i / (gr * gc), r = (i - o * gr * gc) / gc, cidx = i - o * gr * gc - r * gc;
    const int y = 2 * m0 - 1 + r, x = cidx - 1;
    gs[i] = (y >= 0 && y < Ho && x >= 0) ? __ldg(g + (((size_t)b * Cout + o) * Ho + y) * Wo + x) : 0.f;
  }
}

template <bool SHUFFLE>
__global__ void __launch_bounds__(CT_MAX_THREADS) convt3x3s2_dgrad_kernel(const float* __restrict__ g, int Cout, int Hi, int Wi,
                                                                          const float* __restrict__ wt, int Cin, int TR,
                                                                          float* __restrict__ din) {
  extern __shared__ __align__(16) float sm[];
  const int gr = 2 * TR + 1, gc = 2 * Wi + 1;
  float* gs = sm;                                        // [Cout][gr][gc]
  float* ws = sm + ((Cout * gr * gc + 3) & ~3);          // [Cout*9][CB_CG]
  const int tiles = (Hi + TR - 1) / TR;
  const int b = blockIdx.x / tiles, m0 = (blockIdx.x - b * tiles) * TR, c0 = blockIdx.y * CB_CG;
  stage_grad_tile(g, b, Cout, Hi, Wi, m0, TR, gs);
  for (int i = threadIdx.x; i < Cout * 9 * CB_CG; i += blockDim.x) {
    const int cc = i % CB_CG, ot = i / CB_CG;  // ot = o*9 + tap
    ws[i] = (c0 + cc < Cin) ? __ldg(wt + (size_t)(c0 + cc) * Cout * 9 + ot) : 0.f;
  }
  __syncthreads();
  const int q = threadIdx.x, qm = q / Wi, qn = q - qm * Wi;
  if (q >= TR * Wi || m0 + qm >= Hi) return;
  const int m = m0 + qm;
  for (int cg = 0; cg < CB_CG; cg += 4) {
    if (c0 + cg >= Cin) break;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int o = 0; o < Cout; ++o) {
      const float* gp = gs + (o * gr + 2 * qm) * gc + 2 * qn;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const float gv = gp[(t / 3) * gc + (t % 3)];
        const float4 w = *reinterpret_cast<const float4*>(ws + (o * 9 + t) * CB_CG + cg);
        a0 = fmaf(gv, w.x, a0);
        a1 = fmaf(gv, w.y, a1);
        a2 = fmaf(gv, w.z, a2);
        a3 = fmaf(gv, w.w, a3);
      }
    }
    const float acc[4] = {a0, a1, a2, a3};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + cg + k;
      if (c >= Cin) break;
      if (SHUFFLE)
        din[(((size_t)b * 4 * Cin + 4 * c + 2 * (m & 1) + (qn & 1)) * (Hi / 2) + (m >> 1)) * (Wi / 2) + (qn >> 1)] = acc[k];
      else
        din[(((size_t)b * Cin + c) * Hi + m) * Wi + qn] = acc[k];
    }
  }
}

template <bool SHUFFLE>
__global__ void __launch_bounds__(CT_MAX_THREADS) convt3x3s2_wgrad_kernel(const float* __restrict__ in, const float* __restrict__ g,
                                                                          int Cin, int Cout, int Hi, int Wi, int TR,
                                                                          float* __restrict__ dw, float* __restrict__ db) {
  extern __shared__ __align__(16) float sm[];
  const int gr = 2 * TR + 1, gc = 2 * Wi + 1;
  float* gs = sm;                                  // [Cout][gr][gc]
  float* xs = sm + ((Cout * gr * gc + 3) & ~3);    // [TR*Wi][CB_WC]
  const int tiles = (Hi + TR - 1) / TR;
  const int b = blockIdx.x / tiles, m0 = (blockIdx.x - b * tiles) * TR, c0 = blockIdx.y * CB_WC;
  stage_grad_tile(g, b, Cout, Hi, Wi, m0, TR, gs);
  const int npix = TR * Wi;
  for (int i = threadIdx.x; i < npix * CB_WC; i += blockDim.x) {
    const int cc = i % CB_WC, pix = i / CB_WC, qm = pix / Wi, qn = pix - qm * Wi, c = c0 + cc, m = m0 + qm;
    float v = 0.f;
    if (c < Cin && m < Hi) {
      if (SHUFFLE) v = __ldg(in + (((size_t)b * 4 * Cin + 4 * c + 2 * (m & 1) + (qn & 1)) * (Hi / 2) + (m >> 1)) * (Wi / 2) + (qn >> 1));
      else v = __ldg(in + (((size_t)b * Cin + c) * Hi + m) * Wi + qn);
    }
    xs[i] = v;
  }
  __syncthreads();
  const int ot = threadIdx.x;  // o*9 + tap
  if (ot >= Cout * 9) return;
  const int o = ot / 9, t = ot - o * 9;
  const float* gp = gs + o * gr * gc + (t / 3) * gc + (t % 3);
  float acc[CB_WC], gsum = 0.f;
#pragma unroll
  for (int k = 0; k < CB_WC; ++k) acc[k] = 0.f;
  const int rows = min(TR, Hi - m0);
  for (int qm = 0; qm < rows; ++qm)
    for (int qn = 0; qn < Wi; ++qn) {
      const float gv = gp[2 * qm * gc + 2 * qn];
      gsum += gv;
      const float4 x0 = *reinterpret_cast<const float4*>(xs + (qm * Wi + qn) * CB_WC);
      const float4 x1 = *reinterpret_cast<const float4*>(xs + (qm * Wi + qn) * CB_WC + 4);
      acc[0] = fmaf(gv, x0.x, acc[0]);
      acc[1] = fmaf(gv, x0.y, acc[1]);
      acc[2] = fmaf(gv, x0.z, acc[2]);
      acc[3] = fmaf(gv, x0.w, acc[3]);
      acc[4] = fmaf(gv, x1.x, acc[4]);
      acc[5] = fmaf(gv, x1.y, acc[5]);
      acc[6] = fmaf(gv, x1.z, acc[6]);
      acc[7] = fmaf(gv, x1.w, acc[7]);
    }
#pragma unroll
  for (int k = 0; k < CB_WC; ++k)
    if (c0 + k < Cin && acc[k] != 0.f) atomicAdd(dw + (size_t)(c0 + k) * Cout * 9 + ot, acc[k]);
  if (db && blockIdx.y == 0 && (t == 4 || t == 5 || t == 7 || t == 8) && gsum != 0.f) atomicAdd(db + o, gsum);
}

}  // namespace lpb

// one layer at a time: the Python side (models/heads/heatmap.py) chains any number of deconvs
extern "C" int lpb_convt_fwd_f32(const float* in, int B, int Cin, int Hi, int Wi, int shuffle, const float* w, const float* bias,
                                 int Cout, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(in && w && out, "convt_fwd_f32: null pointer");
  LPB_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1 && Hi >= 1 && Wi >= 1 && (!shuffle || (Hi % 2 == 0 && Wi % 2 == 0)), "convt_fwd_f32: bad shape");
  if (B == 0) return LPB_OK;
  return launch_convt(shuffle != 0, in, B, Cin, Hi, Wi, w, bias, Cout, out, static_cast<cudaStream_t>(stream));
}

extern "C" int lpb_plane_softmax_f32(float* x, int64_t n_planes, int hw, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(x && n_planes >= 0 && hw >= 1, "plane_softmax_f32: bad arguments");
  if (n_planes == 0) return LPB_OK;
  const size_t smem = (size_t)hw * sizeof(float);
  LPB_REQUIRE(smem <= 200 * 1024, "plane_softmax_f32: plane of %d pixels too large for the softmax stage", hw);
  if (smem > 48 * 1024) LPB_CUDA(cudaFuncSetAttribute(plane_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  plane_softmax_kernel<<<(unsigned)n_planes, 256, smem, static_cast<cudaStream_t>(stream)>>>(x, hw);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_convt_bwd_f32(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w,
                                 int Cout, float* grad_in, float* grad_w, float* grad_bias, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(in && grad_out && w && grad_w, "convt_bwd_f32: null pointer");
  LPB_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1 && Cout * 9 <= CT_MAX_THREADS && Hi >= 1 && Wi >= 1 && Wi <= CT_MAX_THREADS &&
                  (!shuffle || (Hi % 2 == 0 && Wi % 2 == 0)),
              "convt_bwd_f32: bad shape (Cout <= 28, Wi <= 256)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  LPB_CUDA(cudaMemsetAsync(grad_w, 0, sizeof(float) * (size_t)Cin * Cout * 9, s));
  if (grad_bias) LPB_CUDA(cudaMemsetAsync(grad_bias, 0, sizeof(float) * Cout, s));
  if (B == 0) return LPB_OK;
  int TR = CT_MAX_THREADS / Wi;
  if (TR > Hi) TR = Hi;
  // shrink the band until the staged gradient tile fits
  auto tile_floats = [&](int tr) { return (size_t)((Cout * (2 * tr + 1) * (2 * Wi + 1) + 3) & ~3); };
  while (TR > 1 && (tile_floats(TR) + (size_t)Cout * 9 * CB_CG) * sizeof(float) > 200 * 1024) --TR;
  const int tiles = (Hi + TR - 1) / TR;
  const size_t smem_w = (tile_floats(TR) + (size_t)TR * Wi * CB_WC) * sizeof(float);
  const size_t smem_d = (tile_floats(TR) + (size_t)Cout * 9 * CB_CG) * sizeof(float);
  LPB_REQUIRE(smem_w <= 220 * 1024 && smem_d <= 220 * 1024, "convt_bwd_f32: gradient tile too large (Wi = %d, Cout = %d)", Wi, Cout);
  const int threads_w = ((max(Cout * 9, 32) + 31) / 32) * 32;
  const int threads_d = ((TR * Wi + 31) / 32) * 32;
  dim3 gw((unsigned)(B * tiles), (unsigned)((Cin + CB_WC - 1) / CB_WC)), gd((unsigned)(B * tiles), (unsigned)((Cin + CB_CG - 1) / CB_CG));
  if (shuffle) {
    LPB_CUDA(cudaFuncSetAttribute(convt3x3s2_wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_w));
    convt3x3s2_wgrad_kernel<true><<<gw, threads_w, smem_w, s>>>(in, grad_out, Cin, Cout, Hi, Wi, TR, grad_w, grad_bias);
    if (grad_in) {
      LPB_CUDA(cudaFuncSetAttribute(convt3x3s2_dgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_d));
      convt3x3s2_dgrad_kernel<true><<<gd, threads_d, smem_d, s>>>(grad_out, Cout, Hi, Wi, w, Cin, TR, grad_in);
    }
  } else {
    LPB_CUDA(cudaFuncSetAttribute(convt3x3s2_wgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_w));
    convt3x3s2_wgrad_kernel<false><<<gw, threads_w, smem_w, s>>>(in, grad_out, Cin, Cout, Hi, Wi, TR, grad_w, grad_bias);
    if (grad_in) {
      LPB_CUDA(cudaFuncSetAttribute(convt3x3s2_dgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_d));
      convt3x3s2_dgrad_kernel<false><<<gd, threads_d, smem_d, s>>>(grad_out, Cout, Hi, Wi, w, Cin, TR, grad_in);
    }
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_head_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "head_workspace_bytes: null pointer");
  LPB_REQUIRE(B >= 0 && C >= 4 && C % 4 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 0, "head_workspace_bytes: bad shape");
  *bytes = c2 > 0 ? (size_t)B * c1 * (4 * H) * (4 * W) * sizeof(float) : 0;
  return LPB_OK;
}

extern "C" int lpb_head_fwd_f32(const float* features, int B, int C, int H, int W, const float* w1, const float* b1,
                                int c1, const float* w2, const float* b2, int c2, int final_softmax, float* out,
                                void* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(features && w1 && out, "head_fwd_f32: null pointer");
  LPB_REQUIRE(B >= 0 && C >= 4 && C % 4 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 0, "head_fwd_f32: bad shape");
  LPB_REQUIRE(c2 == 0 || (w2 && workspace), "head_fwd_f32: two-layer head needs w2 and workspace");
  if (B == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int Hs = 2 * H, Ws = 2 * W;  // after PixelShuffle(2)
  int K, Ho, Wo;
  if (c2 == 0) {
    int rc = launch_convt(true, features, B, C / 4, Hs, Ws, w1, b1, c1, out, s);
    if (rc) return rc;
    K = c1;
    Ho = 2 * Hs;
    Wo = 2 * Ws;
  } else {
    float* mid = static_cast<float*>(workspace);
    int rc = launch_convt(true, features, B, C / 4, Hs, Ws, w1, b1, c1, mid, s);
    if (rc) return rc;
    rc = launch_convt(false, mid, B, c1, 2 * Hs, 2 * Ws, w2, b2, c2, out, s);
    if (rc) return rc;
    K = c2;
    Ho = 4 * Hs;
    Wo = 4 * Ws;
  }
  if (final_softmax) {
    const int hw = Ho * Wo;
    const size_t smem = (size_t)hw * sizeof(float);
    LPB_REQUIRE(smem <= 200 * 1024, "head_fwd_f32: plane %dx%d too large for the softmax stage", Ho, Wo);
    if (smem > 48 * 1024)
      LPB_CUDA(cudaFuncSetAttribute(plane_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    plane_softmax_kernel<<<(unsigned)((size_t)B * K), 256, smem, s>>>(out, hw);
    LPB_CUDA(cudaGetLastError());
  }
  return LPB_OK;
}
