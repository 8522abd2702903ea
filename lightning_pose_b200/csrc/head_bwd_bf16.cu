// Backward of the bf16 heatmap head on tensor-core (data gradients), mirroring head_bf16.cu.
// Reference: autograd of lightning_pose/models/heads/heatmap.py:203-212 (PixelShuffle + 2 x ConvTranspose2d).
//
// Gradients travel in the "class-major row layout"  G[b][kchunk = k/8][row = m*Wi + n][8] bf16  with
// k = cls*20 + o, cls = (py, px): row (m, n) carries, for every output class and channel, the gradient at
// output pixel (2m+py, 2n+px).  In this layout the data gradient of a stride-2 3x3 transposed convolution
//   d in[c, m', n'] = sum_{cls, (dm,dn) valid} G[(m'-dm, n'-dn)][(cls, o)] * W[c, o, ky, kx]
// is again a 4-shift GEMM (negative row shifts of the same smem operand, mma_sm90.cuh), K = 80:
//   b2d: G2 (48x48 rows)  x W2  -> d mid (48x48 x 17)  written straight into G1 (24x24 rows) for the next stage
//   b3a: W1 (M = 128 channels) x G1^T -> d Xs[c][row]   un-shuffled in the epilogue into d features (bf16, NCHW or
//        channels-last [B][H][W][C])
#include <cuda_bf16.h>

#include <cstdint>

#include "../../include/lpb200.h"
#include "head_prep.cuh"
#include "head_rows.cuh"
#include <cstring>

#include "lpb_common.cuh"
#include "tensor_map.cuh"
#include "row_layout.cuh"
#include "mma_sm90.cuh"
#include "targets.cuh"
#include "reduce_partials.cuh"

namespace lpb {

// ---- gradient front end: everything upstream of the second deconv's output, fused into the G2 writer --------
// The gradient w.r.t. the head output arrives as a sum of
//   g_out   dense [B, c2, Ho, Wo] fp32 (heatmap losses)                      -- optional
//   win     sparse 32x32 windows of the soft-argmax decode (decode.cu)        -- optional, flag 2 = dense plane in gov
// and, when the head ends in the spatial softmax, is pulled back through it on the fly:
//   g_logit = p * (g - dot),  dot = sum_plane(g * p) = ddot (dense part, plane_dot_kernel) + window dot (meta).
// Neither the dense decode gradient, nor its sum with g_out, nor g_logit ever exist in memory.
// The dense part may instead come from keypoint targets (lpb_mse_targets): the fused target + MSE loss's gradient
// (p - t) * scale, rebuilt per pixel from each plane's target mode and axis factors.  plane_dot_targets_kernel computes
// those once per plane into fac, and the G2 writers (TGT forms) read them with the probabilities, so that gradient is
// never in memory either.
struct G2Src {
  const float* g_out;   // or null
  const float* probs;   // head output when it ends in softmax, else null
  const float* win;     // [planes][32*32] or null
  const int* meta;      // [planes][4] {row0, col0, flag, bits(dot)}
  const float* gov;     // dense fallback planes (flag 2)
  const float* ddot;    // [planes] dense part of the softmax dot (valid when probs && (g_out || win || kp))
  // keypoint targets (kp non-null): the MSE's keypoints / visibility, target geometry, its forward's out (out[1] =
  // kept planes) and upstream gradient, and fac [planes][fac_stride] = {mode, 3 unused, ex[Wo], er[Ho]}
  const float* kp;
  const int32_t* vis;
  float sx, sy, two_s2;
  const float* mse_out;
  const float* mse_gout;
  float* fac;
  int fac_stride;
};

// floats per plane of the target factors: {mode, 3 unused} + ex[ow] + er[oh], a multiple of 4 (16-byte rows)
inline int mse_fac_stride(int oh, int ow) { return (4 + ow + oh + 3) & ~3; }

// ddot[plane] = sum(p * (g_out + [flag == 2] gov)); one CTA per plane
__global__ void __launch_bounds__(256) plane_dot_kernel(G2Src S, int hw, float* __restrict__ ddot) {
  const size_t plane = blockIdx.x;
  const bool ov = S.meta && S.meta[4 * plane + 2] == 2;
  float acc = 0.f;
  if (S.g_out || ov) {
    const float4* p4 = reinterpret_cast<const float4*>(S.probs + plane * hw);
    const float4* g4 = S.g_out ? reinterpret_cast<const float4*>(S.g_out + plane * hw) : nullptr;
    const float4* o4 = ov ? reinterpret_cast<const float4*>(S.gov + plane * hw) : nullptr;
    for (int i = threadIdx.x; i < hw / 4; i += 256) {
      const float4 p = __ldg(p4 + i);
      float4 g = g4 ? __ldg(g4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (o4) {
        const float4 o = __ldg(o4 + i);
        g.x += o.x, g.y += o.y, g.z += o.z, g.w += o.w;
      }
      acc += p.x * g.x + p.y * g.y + p.z * g.z + p.w * g.w;
    }
  }
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    ddot[plane] = t;
  }
}

// Keypoint-target form: the dense gradient is rebuilt per element as heatmap_mse_from_kp_bwd_kernel (losses.cu) computes
// it -- the same 256-thread axis factors, so norm has the same bits, and the same mse_target_grad -- and ddot sums it in
// plane_dot_kernel's loop and expression order, so the result is what that kernel gives on the materialised gradient.
// Also writes the plane's mode and factor rows (ex[c], er[r] = ey[r] * norm; uniform planes 1/n and 1) to S.fac.
// ow % 4 == 0 (the head's output widths): a float4 of pixels lies in one row.
__global__ void __launch_bounds__(256) plane_dot_targets_kernel(G2Src S, int oh, int ow, float* __restrict__ ddot) {
  extern __shared__ float sm[];  // ex[ow], ey[oh] (then er), red[16]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  __shared__ float dred[8];
  const size_t plane = blockIdx.x;
  const int hw = oh * ow;
  const TargetPlane tp = classify_target(S.kp, S.vis, plane, S.sx, S.sy, oh, ow);
  float* fac = S.fac + plane * S.fac_stride;
  if (threadIdx.x == 0) reinterpret_cast<int*>(fac)[0] = tp.mode;
  if (tp.mode != TARGET_ZERO) {
    const float norm = tp.mode == TARGET_GAUSS ? target_axis_factors(tp, oh, ow, S.two_s2, ex, ey, red, 256) : 1.f;
    const float u = mse_target_uniform(hw);
    for (int c = threadIdx.x; c < ow; c += 256) {
      if (tp.mode == TARGET_UNIFORM) ex[c] = u;
      fac[4 + c] = ex[c];
    }
    for (int r = threadIdx.x; r < oh; r += 256) {
      const float er = tp.mode == TARGET_UNIFORM ? 1.f : ey[r] * norm;
      ey[r] = er;
      fac[4 + ow + r] = er;
    }
    __syncthreads();
  }
  const float scale = mse_target_scale(S.mse_gout[0], S.mse_out[1]);
  const bool ov = S.meta && S.meta[4 * plane + 2] == 2;
  const float4* p4 = reinterpret_cast<const float4*>(S.probs + plane * hw);
  const float4* o4 = ov ? reinterpret_cast<const float4*>(S.gov + plane * hw) : nullptr;
  float acc = 0.f;
  for (int i = threadIdx.x; i < hw / 4; i += 256) {
    const float4 p = __ldg(p4 + i);
    const int r = (4 * i) / ow, c = 4 * i - r * ow;
    const float er = ey[r];
    float4 g = make_float4(mse_target_grad(tp.mode, p.x, ex[c], er, scale), mse_target_grad(tp.mode, p.y, ex[c + 1], er, scale),
                           mse_target_grad(tp.mode, p.z, ex[c + 2], er, scale), mse_target_grad(tp.mode, p.w, ex[c + 3], er, scale));
    if (o4) {
      const float4 o = __ldg(o4 + i);
      g.x += o.x, g.y += o.y, g.z += o.z, g.w += o.w;
    }
    acc += p.x * g.x + p.y * g.y + p.z * g.z + p.w * g.w;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) dred[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += dred[i];
    ddot[plane] = t;
  }
}

// Window-only form (no dense gradient): ddot is zero except for the few planes whose decode gradient is dense (flag 2).
// A CTA looks after 8 planes and sweeps only the flagged ones, all 256 threads on one plane at a time -- an eighth of the
// CTAs of the per-plane launch and no single-warp tail.
__global__ void __launch_bounds__(256) plane_dot_sparse_kernel(G2Src S, long long n_planes, int hw, float* __restrict__ ddot) {
  __shared__ float red[8];
  const long long p0 = (long long)blockIdx.x * 8;
  for (long long plane = p0; plane < p0 + 8 && plane < n_planes; ++plane) {
    if (S.meta[4 * plane + 2] != 2) {  // uniform over the CTA
      if (threadIdx.x == 0) ddot[plane] = 0.f;
      continue;
    }
    const float4* p4 = reinterpret_cast<const float4*>(S.probs + plane * hw);
    const float4* o4 = reinterpret_cast<const float4*>(S.gov + plane * hw);
    float acc = 0.f;
    for (int i = threadIdx.x; i < hw / 4; i += 256) {
      const float4 p = __ldg(p4 + i), o = __ldg(o4 + i);
      acc += p.x * o.x + p.y * o.y + p.z * o.z + p.w * o.w;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < 8; ++i) t += red[i];
      ddot[plane] = t;
    }
    __syncthreads();
  }
}

// Thread t of a frame handles input-grid pixel (m, n) = divmod(t, Wi): the 2x2 output block x all channels.
// Loads are issued as independent batches (probs, dense gradient) before any dependent work; the decode windows are
// added afterwards by g2_patch_kernel.
constexpr int G2B_THREADS = 128;

// HAS_OV (pass ahead of the patch kernel): planes whose decode gradient is dense (flag 2, the decode's overflow buffer) are
// added here, in the streaming pass -- in the fresh-init regime that is every plane.  blockIdx.y is the keypoint group
// (head_prep.cuh): planes [20 g, 20 g + 20) of the C, written to the group's 10 K-chunks of the frame's gridDim.y * 10.
// TGT (with HAS_G, HAS_P): the dense gradient is the keypoint targets' (G2Src), from the probabilities and the factor rows.
template <bool HAS_G, bool HAS_P, bool HAS_OV, bool TGT>
__global__ void __launch_bounds__(G2B_THREADS, 4) g2_build_kernel(G2Src S, int B, int C, int Hi, int Wi, int ctas_per_frame,
                                                               __nv_bfloat16* __restrict__ G, RowLayout L) {
  static_assert(!TGT || (HAS_G && HAS_P), "the keypoint-target source is a dense gradient of a softmax head");
  const int b = blockIdx.x / ctas_per_frame, t0 = (blockIdx.x - b * ctas_per_frame) * G2B_THREADS, t = t0 + threadIdx.x;
  const int Wo = 2 * Wi, Ho = 2 * Hi;
  const int g = blockIdx.y, o0 = HEAD_CLS * g, cg = min(HEAD_CLS, C - o0);
  __shared__ float sdot[HEAD_CLS];
  __shared__ int smode[HEAD_CLS];
  __shared__ float sscale;
  __shared__ unsigned sov;
  if (threadIdx.x < HEAD_CLS) {
    float d = 0.f;
    int4 mt = make_int4(0, 0, 0, 0);
    int mode = TARGET_ZERO;
    if (threadIdx.x < cg) {
      const size_t plane = (size_t)b * C + o0 + threadIdx.x;
      if (S.meta) mt = reinterpret_cast<const int4*>(S.meta)[plane];
      if (HAS_P) {
        if (mt.z == 1) d = __int_as_float(mt.w);
        if (S.ddot) d += S.ddot[plane];
      }
      if (TGT) mode = reinterpret_cast<const int*>(S.fac + plane * S.fac_stride)[0];
    }
    sdot[threadIdx.x] = d;
    if (TGT) {
      smode[threadIdx.x] = mode;
      if (threadIdx.x == 0) sscale = mse_target_scale(S.mse_gout[0], S.mse_out[1]);
    }
    if (HAS_OV) {
      const unsigned bov = __ballot_sync((1u << HEAD_CLS) - 1, mt.z == 2);
      if (threadIdx.x == 0) sov = bov;
    }
  }
  __syncthreads();
  if (t >= Hi * Wi) return;
  const int m = t / Wi, n = t - m * Wi;
#pragma unroll
  for (int py = 0; py < 2; ++py) {
    const int y = 2 * m + py, x = 2 * n;
    const size_t off0 = (((size_t)b * C + o0) * Ho + y) * Wo + x;
    const size_t pstride = (size_t)Ho * Wo;
    float2 pv[HEAD_CLS], gv[HEAD_CLS];
#pragma unroll
    for (int o = 0; o < HEAD_CLS; ++o) {
      pv[o] = make_float2(0.f, 0.f);
      gv[o] = make_float2(0.f, 0.f);
      if (o < cg) {
        if (HAS_P) pv[o] = __ldg(reinterpret_cast<const float2*>(S.probs + off0 + o * pstride));
        if (HAS_G && !TGT) gv[o] = __ldg(reinterpret_cast<const float2*>(S.g_out + off0 + o * pstride));
      }
    }
    if (TGT) {
      // plane by plane to the softmax term, so that each plane's operands die at once (the same operations in the same
      // order as the three passes below)
      const float scale = sscale;
      const unsigned ovm = HAS_OV ? sov : 0u;
      const float* f0 = S.fac + ((size_t)b * C + o0) * S.fac_stride + 4;
#pragma unroll
      for (int o = 0; o < HEAD_CLS; ++o) {
        if (o < cg) {
          const float* f = f0 + (size_t)o * S.fac_stride;
          const float2 e = __ldg(reinterpret_cast<const float2*>(f + x));
          const float er = __ldg(f + Wo + y);
          float2 gt = make_float2(mse_target_grad(smode[o], pv[o].x, e.x, er, scale), mse_target_grad(smode[o], pv[o].y, e.y, er, scale));
          if (HAS_OV && ((ovm >> o) & 1u)) {
            const float2 u = __ldg(reinterpret_cast<const float2*>(S.gov + off0 + o * pstride));
            gt.x += u.x, gt.y += u.y;
          }
          const float d = sdot[o];
          gv[o] = make_float2(pv[o].x * (gt.x - d), pv[o].y * (gt.y - d));
        }
      }
    } else if (HAS_OV && sov) {  // uniform per frame
      const unsigned ovm = sov;
#pragma unroll
      for (int o = 0; o < HEAD_CLS; ++o) {
        if (o < cg && ((ovm >> o) & 1u)) {
          const float2 u = __ldg(reinterpret_cast<const float2*>(S.gov + off0 + o * pstride));
          gv[o].x += u.x, gv[o].y += u.y;
        }
      }
    }
    if (HAS_P && !TGT) {
#pragma unroll
      for (int o = 0; o < HEAD_CLS; ++o) {
        const float d = sdot[o];
        gv[o].x = pv[o].x * (gv[o].x - d);
        gv[o].y = pv[o].y * (gv[o].y - d);
      }
    }
    // k = (2*py + px) * 20 + o : 40 consecutive k values = K-chunks 5py .. 5py+4
#pragma unroll
    for (int ch = 0; ch < 5; ++ch) {
      uint32_t pk[4];
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) {
        const int k0 = ch * 8 + 2 * e2, k1 = k0 + 1;  // 0..39 within this py
        const float f0 = k0 < HEAD_CLS ? gv[k0].x : gv[k0 - HEAD_CLS].y;
        const float f1 = k1 < HEAD_CLS ? gv[k1].x : gv[k1 - HEAD_CLS].y;
        __nv_bfloat162 h2 = __floats2bfloat162_rn(f0, f1);
        pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(G + ((((size_t)(b * gridDim.y + g) * HEAD_KC + 5 * py + ch) * L.rows) + L.lead + (size_t)m * L.Pp + n) * 8) =
          make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  }
}

// Window patch: after a window-less g2_build pass (which already folds each window's dot into the softmax term and adds the
// dense-overflow planes), one warp per plane re-evaluates the <= 32 x 32 pixels under its window and overwrites those
// bf16 entries.  The streaming pass then runs at the DRAM roofline with no look-ups in it, and this pass touches 4 KB of
// probabilities per plane (a ninth of it).
// Window rows go eight at a time: 8 independent window loads, then 8 independent probability loads per lane.
template <bool HAS_G, bool HAS_P, bool TGT>
__global__ void __launch_bounds__(128) g2_patch_kernel(G2Src S, long long n_planes, int C, int Hi, int Wi,
                                                      __nv_bfloat16* __restrict__ G, RowLayout L) {
  const int lane = threadIdx.x & 31;
  const int Wo = 2 * Wi, Ho = 2 * Hi;
  {
    const long long plane = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
    int4 mt = make_int4(0, 0, 0, 0);
    if (plane < n_planes) mt = reinterpret_cast<const int4*>(S.meta)[plane];
    if (mt.z == 1) {
      const int b = (int)(plane / C), oc = (int)(plane - (long long)b * C), g = oc / HEAD_CLS, o = oc - g * HEAD_CLS;
      float dot = 0.f;
      if (HAS_P) dot = __int_as_float(mt.w) + (S.ddot ? S.ddot[plane] : 0.f);
      // keypoint targets: this plane's mode and factor rows, the loss's scale
      const float* fac = TGT ? S.fac + (size_t)plane * S.fac_stride : nullptr;
      const int tmode = TGT ? reinterpret_cast<const int*>(fac)[0] : TARGET_ZERO;
      const float tscale = TGT ? mse_target_scale(S.mse_gout[0], S.mse_out[1]) : 0.f;
      const size_t poff = (size_t)plane * Ho * Wo;
      const float* wp = S.win + (size_t)plane * 1024 + lane;
      const int x = mt.y + lane;
      const bool xin = (unsigned)x < (unsigned)Wo;
      // k = cls * 20 + o with cls = 2 (y & 1) + (x & 1): the K-chunk / element of this lane for even and odd rows
      const int kx = (x & 1) * HEAD_CLS + o;
      __nv_bfloat16* gcol = G + ((size_t)(b * head_groups(C) + g) * HEAD_KC * L.rows + L.lead + (x >> 1)) * 8;
#pragma unroll 1
      for (int r0 = 0; r0 < 32; r0 += 8) {
        float gw[8], pv[8], go[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) gw[k] = __ldg(wp + (r0 + k) * 32);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int y = mt.x + r0 + k;
          const bool ok = xin && gw[k] != 0.f && (unsigned)y < (unsigned)Ho;
          pv[k] = (HAS_P && ok) ? __ldg(S.probs + poff + (size_t)y * Wo + x) : 0.f;
          if (TGT) go[k] = ok ? mse_target_grad(tmode, pv[k], __ldg(fac + 4 + x), __ldg(fac + 4 + Wo + y), tscale) : 0.f;
          else go[k] = (HAS_G && ok) ? __ldg(S.g_out + poff + (size_t)y * Wo + x) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int y = mt.x + r0 + k;
          if (!(xin && gw[k] != 0.f && (unsigned)y < (unsigned)Ho)) continue;
          float g = gw[k] + go[k];
          if (HAS_P) g = pv[k] * (g - dot);
          const int kk = kx + 2 * HEAD_CLS * (y & 1);
          gcol[((size_t)(kk >> 3) * L.rows + (size_t)(y >> 1) * L.Pp) * 8 + (kk & 7)] = __float2bfloat16_rn(g);
        }
      }
    }
  }
}

template <bool HAS_G, bool HAS_P, bool TGT = false>
static void launch_g2_build(const G2Src& S, int B, int C, int Hi, int Wi, __nv_bfloat16* G, RowLayout L, cudaStream_t s) {
  const int cpf = (Hi * Wi + G2B_THREADS - 1) / G2B_THREADS;
  const dim3 grid((unsigned)(B * cpf), (unsigned)head_groups(C));
  if (!S.win) {
    g2_build_kernel<HAS_G, HAS_P, false, TGT><<<grid, G2B_THREADS, 0, s>>>(S, B, C, Hi, Wi, cpf, G, L);
    return;
  }
  g2_build_kernel<HAS_G, HAS_P, true, TGT><<<grid, G2B_THREADS, 0, s>>>(S, B, C, Hi, Wi, cpf, G, L);
  const long long np = (long long)B * C;
  g2_patch_kernel<HAS_G, HAS_P, TGT><<<(unsigned)((np + 3) / 4), 128, 0, s>>>(S, np, C, Hi, Wi, G, L);
}

// (the data-gradient operand packs  out[tile][shift][kchunk][r][8]: element (r, k) = W[tile*rows_per_tile + r][o][ky][kx]
// for k = cls*20 + o when (cls, shift) is a valid tap, else 0  are produced by head_prep_kernel, head_bf16.cu)

// =====================================================================================================
// b2d: data gradient of the second deconv:  G2 -> d mid, emitted as G1 (+ bias gradient of layer 1)
// =====================================================================================================
constexpr int B2D_THREADS = 192;  // warp 0 loader, warp 1 idle, warps 2-5 MMA + epilogue (K of a chunk is resident)
constexpr int B2D_TILES = 3;       // M-tiles per chunk: R2 = 384 / (Wi + 1) image rows (7 * 49 = 343 raster rows at Wi = 48)

struct B2dParams {
  const __nv_bfloat16* G2;    // [B][10][L2.rows][8] padded row layout
  const __nv_bfloat16* wpk;   // [4][10][32][8]
  __nv_bfloat16* G1;          // [B][10][L1.rows][8] padded row layout of the (Hi/2 x Wi/2) grid
  RowLayout L2, L1;
  float* db1_part;            // [gridDim.x * 4 MMA warps][HEAD_CLS]: each warp's bias-gradient sum (reduced in a fixed order)
  int B, Hi, Wi, c1;
  int R2;                     // image rows per chunk
  // WIDE (keypoint groups): one launch per (c1 group, c2 group), c2 groups in order.  K is c2 group kc0 / 10 of the
  // frame's kc_frame K-chunks of G2; the columns are mid channels [o0, o0 + cg); the result goes to (accumulate = 0) or is
  // added to (1) the fp32 planes dmid, which the G1 writer reads afterwards.
  float* dmid;                // [B][c1][Hi * Wi]
  int kc_frame, kc0, o0, cg, accumulate;
};

template <bool WIDE>
__global__ void __launch_bounds__(B2D_THREADS, 2) b2d_dgrad_kernel(const __grid_constant__ B2dParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1;
  const int LEAD = Pp + 1;  // one zero row + the previous image row
  const int rows_alloc = (LEAD + B2D_TILES * 128 + 7) & ~7;
  const int a_bytes = HEAD_KC * rows_alloc * 16;
  const int w_bytes = 4 * HEAD_KC * 32 * 16;
  unsigned char* As = smem;
  unsigned char* Ws = smem + a_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Ws + w_bytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + 1;
  uint64_t* w_full = bars + 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int i = tid; i < a_bytes / 16; i += B2D_THREADS) reinterpret_cast<uint4*>(As)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, 4);  // one arrival per MMA warp
    mbar_init(w_full, 1);
    fence_mbar_init();
  }
  fence_proxy_async();
  __syncthreads();
  const int B2D_ROWS = P.R2;
  const int nchunk = (Hi + B2D_ROWS - 1) / B2D_ROWS;

  if (warp == 0) {
    if (lane == 0) {
      mbar_expect_tx(w_full, (uint32_t)w_bytes);
      bulk_g2s(Ws, P.wpk, (uint32_t)w_bytes, w_full);
    }
    int it = 0;
    for (int b = blockIdx.x; b < P.B; b += gridDim.x) {
      for (int ck = 0; ck < nchunk; ++ck, ++it) {
        const int y0 = ck * B2D_ROWS;
        mbar_wait(a_empty, (it & 1) ^ 1);
        // per K-chunk ONE copy: the zero entry before image row y0-1, that row, and the chunk's rows (zero columns
        // included); the row above the image comes from the layout's zero lead rows.  A short last chunk copies only its
        // own rows (stale rows further down feed accumulator rows the epilogue skips).
        const uint32_t nbytes = (uint32_t)((1 + (min(B2D_ROWS, Hi - y0) + 1) * Pp) * 16);
        if (lane < HEAD_KC) {
          if (lane == 0) mbar_expect_tx(a_full, HEAD_KC * nbytes);
          __syncwarp((1u << HEAD_KC) - 1);
          bulk_g2s(As + (size_t)lane * rows_alloc * 16,
                   P.G2 + (((size_t)b * (WIDE ? P.kc_frame : HEAD_KC) + (WIDE ? P.kc0 : 0) + lane) * P.L2.rows + P.L2.lead + (size_t)(y0 - 1) * Pp - 1) * 8,
                   nbytes, a_full);
        }
      }
    }
  } else if (warp >= 2) {
    const int q = warp & 3;
    const uint32_t lbo_a = rows_alloc * 16, lbo_b = 32 * 16;
    const uint32_t a0 = smem_u32(As), b0 = smem_u32(Ws);
    mbar_wait(w_full, 0);
    float dbs[HEAD_CLS];
#pragma unroll
    for (int o = 0; o < HEAD_CLS; ++o) dbs[o] = 0.f;
    int it = 0;
    for (int b = blockIdx.x; b < P.B; b += gridDim.x) {
      for (int ck = 0; ck < nchunk; ++ck, ++it) {
        const int y0 = ck * B2D_ROWS, nrow = min(B2D_ROWS, Hi - y0);
        mbar_wait(a_full, it & 1);
        for (int t = 0; t < B2D_TILES; ++t) {
          float d[32];
          {
            float acc[2][4][4];
            mma::zero(acc);
#pragma unroll
            for (int sh = 0; sh < 4; ++sh) {
              const int shift_rows = (sh >> 1) * Pp + (sh & 1);
#pragma unroll
              for (int k16 = 0; k16 < HEAD_NCOLS / 16; ++k16) {
                if (k16 < sh) continue;  // all-zero weight chunks of this shift (see b3a)
                mma::kstep(acc, a0 + (2 * k16) * lbo_a + (LEAD + t * 128 + 32 * q - shift_rows) * 16, lbo_a, b0 + (sh * HEAD_KC + 2 * k16) * lbo_b,
                           lbo_b, lane);
              }
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) mma::rows8(acc, nt, &d[8 * nt], lane);
          }
          const int row = t * 128 + 32 * q + lane;
          const int ml = row / Pp, n = row - ml * Pp;
          if (WIDE && ml < nrow && n < Wi) {
            // same sum order per element as the narrow form within a group; the groups are added in launch order
            const size_t hw = (size_t)Hi * Wi;
            float* dst = P.dmid + ((size_t)b * P.c1 + P.o0) * hw + (size_t)(y0 + ml) * Wi + n;
#pragma unroll
            for (int o = 0; o < HEAD_CLS; ++o)
              if (o < P.cg) dst[o * hw] = P.accumulate ? dst[o * hw] + d[o] : d[o];
          } else if (ml < nrow && n < Wi) {
            const int y = y0 + ml;
            const int row1 = P.L1.lead + (y >> 1) * P.L1.Pp + (n >> 1);
            const int k0 = HEAD_CLS * (((y & 1) << 1) | (n & 1));
#pragma unroll
            for (int o = 0; o < HEAD_CLS; ++o)
              if (o < P.c1) dbs[o] += d[o];
#pragma unroll
            for (int i = 0; i < HEAD_CLS / 4; ++i) {
              uint32_t pk[2];
#pragma unroll
              for (int e2 = 0; e2 < 2; ++e2) {
                const int c0 = 4 * i + 2 * e2;
                __nv_bfloat162 h2 = __floats2bfloat162_rn(c0 < P.c1 ? d[c0] : 0.f, c0 + 1 < P.c1 ? d[c0 + 1] : 0.f);
                pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
              }
              const int k = k0 + 4 * i;
              *reinterpret_cast<uint2*>(P.G1 + (((size_t)b * HEAD_KC + (k >> 3)) * P.L1.rows + row1) * 8 + (k & 7)) = make_uint2(pk[0], pk[1]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(a_empty);
      }
    }
    if (!WIDE) {
      float* part = P.db1_part + ((size_t)blockIdx.x * 4 + q) * HEAD_CLS;
#pragma unroll
      for (int o = 0; o < HEAD_CLS; ++o) {
        const float s = warp_sum(dbs[o]);
        if (lane == 0) part[o] = s;
      }
    }
  }
}

// =====================================================================================================
// b3a: data gradient of the first deconv + inverse PixelShuffle:  G1 -> d features (NCHW bf16)
// =====================================================================================================
// 8 MMA + epilogue warps, two per 32-channel quarter of the CTA's 128 channels; lane 0-9 of warp 0 also issue the
// operand copies.  Two warps per SM sub-partition leave each thread up to 255 registers (10 warps would cap it at 168),
// which the weight fragments held in registers need.
constexpr int B3A_THREADS = 256;

struct B3aParams {
  const __nv_bfloat16* G1;   // [B][10][L.rows][8] padded row layout
  RowLayout L;
  const __nv_bfloat16* wpk;  // [ceil(C4/128)][4][10][128][8]
  __nv_bfloat16* dfeat;      // [B][4*C4][(Hi/2)*(Wi/2)], or [B][Hi/2][Wi/2][4*C4] in the NHWC instantiations
  int B, C4, Hi, Wi;         // shuffled-image geometry (Hi = 2H, Wi = 2W)
  int Hh;                    // image rows per band (multiple of 4)
  int ncols;                 // accumulator columns per band = Hh * (Wi + 1) rounded up to 16 (<= 304)
  int tma_store;             // 1: the epilogue stages bf16 rows in shared memory and a TMA tensor store writes them (below)
  // ACC (keypoint groups): one launch per c1 group, in order.  K is group kc0 / 10 of the frame's kc_frame K-chunks of G1;
  // the group's d features are added to the fp32 partial sums acc32 [B][4 C4][HW] of the groups before it (acc_in) and
  // stored there (acc_out) or, for the last group, rounded to bf16 into dfeat.
  float* acc32;
  int acc_in, acc_out, kc_frame, kc0;
};

// TMA tensor store of d features.  The tensor maps view the NCHW gradient as [b][c'][pl][px] (source plane 4c' + pl,
// px = H*W pixels); a box is {2 or 4 feature rows, one pl, 128 c', one frame}: in shared memory 128 rows of 4*WS2 or
// 8*WS2 bytes, and the copy engine does the plane-strided scatter.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, const void* smem_src, int x0, int x1, int x2, int x3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tm), "r"(smem_u32(smem_src)), "r"(x0),
               "r"(x1), "r"(x2), "r"(x3)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// Column tiling of b3a (W = WS2, the feature width).  A work item is (di, pair of feature rows i, i + 1) of one frame:
// shuffled rows m = 2i + di and m + 2 of the band.  Its columns go in plane order: for dj = 0, 1, the 2W pixels
// (2i' + di, 2j + dj), i' = i, i + 1, j < W, which are 2W consecutive elements of source plane 4c + 2di + dj in NCHW.
// So an item is B3aCols::NTI = W / 2 n8 tiles (W / 4 per dj) with no padding or wasted column, and the accumulator pair
// (2t, 2t + 1) of a thread is two adjacent pixels of one plane.  ldmatrix takes one row address per lane, so the G1 rows
// of a tile can be any 8 raster rows.  The tiles are computed in chunks of NT, with the chunk sized from W so that the
// accumulators fit beside the 112 registers of weights without spilling (larger chunks spill at W = 32).
template <int WS2>
struct B3aCols {
  static constexpr int TPD = WS2 / 4;  // n8 tiles per dj
  static constexpr int NTI = 2 * TPD;  // n8 tiles per item
  static constexpr int NT_MAX = 6;
  static constexpr int nt() {
    int n = 2;
    for (int d = 2; d <= NT_MAX && d <= NTI; d += 2)
      if (NTI % d == 0) n = d;
    return n;
  }
  static constexpr int NT = nt();  // n8 tiles per chunk: the largest even divisor of NTI up to NT_MAX
  static constexpr int NCHUNK = NTI / NT;
  static_assert(WS2 % 4 == 0 && NTI % NT == 0 && NT % 2 == 0, "b3a column tiling");
  // band column of tile T's column n (T < NTI, n < 8), relative to the item's first accumulator row
  __device__ static int col(int T, int n) {
    const int dj = T / TPD, x = 8 * (T % TPD) + n;  // x: index into the plane's 2W run
    return (x / WS2) * 2 * (2 * WS2 + 1) + 2 * (x % WS2) + dj;
  }
};
// the 14 non-zero (shift, k16) steps in issue order: shift 0..3, k16 = shift..4
__host__ __device__ constexpr int b3a_kstep(int sh, int k16) { return 5 * sh - sh * (sh - 1) / 2 + k16 - sh; }
constexpr int B3A_KSTEPS = b3a_kstep(3, 4) + 1;
static_assert(B3A_KSTEPS == 14, "b3a: 14 non-zero (shift, k16) weight steps");

// f(channel row within the warp, dj, x, D(x), D(x + 1)) for every accumulator pair of chunk ch: x indexes the plane's
// 2W run, and the pair is two adjacent pixels of it
template <int WS2, typename F>
__device__ __forceinline__ void b3a_each_pair(int ch, const float (&acc)[2][B3aCols<WS2>::NT][4], int lane, F&& f) {
  constexpr int NT = B3aCols<WS2>::NT, TPD = B3aCols<WS2>::TPD;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int T = ch * NT + t, dj = T / TPD, x = 8 * (T % TPD) + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) f(16 * m + 8 * h + (lane >> 2), dj, x, acc[m][t][2 * h], acc[m][t][2 * h + 1]);
    }
}

// Channels-last d features (NHWC): [B][H][W][C] with C = 4 C4.  The accumulator rows are channels and the columns pixels,
// so the store transposes through shared memory.  The two items (di = 0, 1) of a feature-row pair, which the two warp
// groups e = 0, 1 compute side by side, cover every source channel 4c + 2 di + dj of the CTA's 128 shuffled channels at the
// pair's 2W feature pixels: both groups round their values into one staging tile [2W pixels][128 c][4 planes] bf16, and
// after a CTA barrier all threads copy it out with 16-byte vectors -- per pixel one contiguous run of up to 1024 bytes
// (the tile's 512 channels), whole 32-byte sectors.  B3A_NHWC_PX is the tile's pixel stride: 16 bytes past the 1024 so
// that the 2-byte staging stores of a warp (8 channels x 4 pixel pairs) spread over the banks.
constexpr int B3A_NHWC_PX = 1024 + 16;
inline size_t b3a_nhwc_stage_bytes(int W) { return (size_t)2 * W * B3A_NHWC_PX + 128; }

// A frame is processed in bands of Hh image rows (the band's gradient rows plus the halo row above are double-buffered
// in shared memory).
template <int WS2, bool ACC = false, bool NHWC = false>
__global__ void __launch_bounds__(B3A_THREADS, 1) b3a_dgrad_kernel(const __grid_constant__ B3aParams P, const __grid_constant__ CUtensorMap TM,
                                                                   const __grid_constant__ CUtensorMap TM_PAIR) {
  using Cols = B3aCols<WS2>;
  constexpr int NT = Cols::NT;
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1, LEAD = Pp + 1;
  const int Hh = P.Hh, nbands = (Hi + Hh - 1) / Hh;
  const int rows_alloc = (LEAD + P.ncols + 7) & ~7;
  const int g_bytes = HEAD_KC * rows_alloc * 16;
  const int w_bytes = 4 * HEAD_KC * 128 * 16;
  unsigned char* Gs = smem;                 // [2 stages][10][rows_alloc][16 B]
  unsigned char* Ws = smem + 2 * g_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Ws + w_bytes);
  uint64_t* g_full = bars;       // [2]
  uint64_t* g_empty = bars + 2;  // [2]
  uint64_t* w_full = bars + 4;
  // staging slices of the TMA store: [pl][128 channels][2 items][4 * WS2 bytes]
  unsigned char* Ss = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(bars + 12) + 127) & ~(uintptr_t)127);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntile = (P.C4 + 127) / 128;
  const int mt = blockIdx.x % ntile, slot = blockIdx.x / ntile, nslot = gridDim.x / ntile;

  for (int i = tid; i < 2 * g_bytes / 16; i += B3A_THREADS) reinterpret_cast<uint4*>(Gs)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int st = 0; st < 2; ++st) {
      mbar_init(&g_full[st], 1);
      mbar_init(&g_empty[st], 8);  // one arrival per MMA warp
    }
    mbar_init(w_full, 1);
    fence_mbar_init();
  }
  fence_proxy_async();
  __syncthreads();

  // operand copies, issued by warp 0: the weights once, then the bands in (frame, band) order, each into stage j % 2 once
  // every warp has arrived on that stage's g_empty for band j - 2
  int lb = slot, lband = 0;  // the next band to copy
  auto load_next = [&](int j) {
    const int st = j & 1, y0 = lband * Hh, hb = min(Hh, Hi - y0);
    // one copy per K-chunk: the zero entry before image row y0 - 1, that row (zero lead rows of the layout when
    // y0 = 0), and the band's rows, zero columns included
    const uint32_t nbytes = (uint32_t)((1 + (hb + 1) * Pp) * 16);
    if (lane < HEAD_KC) {
      if (lane == 0) mbar_expect_tx(&g_full[st], HEAD_KC * nbytes);
      __syncwarp((1u << HEAD_KC) - 1);
      bulk_g2s(Gs + (size_t)st * g_bytes + (size_t)lane * rows_alloc * 16,
               P.G1 + (((size_t)lb * (ACC ? P.kc_frame : HEAD_KC) + (ACC ? P.kc0 : 0) + lane) * P.L.rows + P.L.lead + (size_t)(y0 - 1) * Pp - 1) * 8,
               nbytes, &g_full[st]);
    }
    if (++lband == nbands) lband = 0, lb += nslot;
  };
  if (warp == 0) {
    if (lane == 0) {
      mbar_expect_tx(w_full, (uint32_t)w_bytes);
      bulk_g2s(Ws, reinterpret_cast<const unsigned char*>(P.wpk) + (size_t)mt * w_bytes, (uint32_t)w_bytes, w_full);
    }
    for (int j = 0; j < 2 && lb < P.B; ++j) load_next(j);
  }
  {
    // MMA + epilogue: D[c][pixel] = sum_{shift, k} W1[shift][c][k] * G1[pixel - shift][k], M = channels, N = pixels.  Warp
    // (q, e) owns the 32 channels 32 q .. 32 q + 31 of the CTA's 128-channel tile (two m16 tiles) and the items with di = e;
    // the band's whole K is resident, and the warp's weight fragments sit in registers for the whole launch.
    const int q = warp & 3, e = warp >> 2;
    const int HW = (Hi / 2) * WS2;
    const uint32_t lbo_g = rows_alloc * 16, lbo_w = 128 * 16;
    mbar_wait(w_full, 0);
    uint32_t af[B3A_KSTEPS][2][4];  // A fragments of the 14 non-zero (shift, k16) steps x 2 m16 tiles
#pragma unroll
    for (int sh = 0; sh < 4; ++sh)
#pragma unroll
      for (int k16 = sh; k16 < HEAD_NCOLS / 16; ++k16)
#pragma unroll
        for (int m = 0; m < 2; ++m)
          mma::ldsm_x4(af[b3a_kstep(sh, k16)][m], smem_u32(Ws) + ((sh * HEAD_KC + 2 * k16) * 128 + 32 * q + 16 * m + ((lane >> 3) & 1) * 8 + (lane & 7)) * 16 +
                                                     (lane >> 4) * lbo_w);
    // this lane's ldmatrix row of tile pair np of chunk ch: tile 2 np + lane / 16 of the chunk, column lane % 8, K-chunk
    // (lane / 8) % 2 of the k16 step
    auto b_row = [&](int ch, int np) { return (uint32_t)(LEAD + Cols::col(ch * NT + 2 * np + (lane >> 4), lane & 7)) * 16 + ((lane >> 3) & 1) * lbo_g; };
    // one chunk of an item: each element is the same mma.sync sequence from zero, shift 0..3, k16 ascending, the
    // all-zero k16 < shift steps skipped (K = (cls, o), cls = 2 py + px at stride 20: shift (dm, dn) has no tap for the
    // classes with py < dm or px < dn, so its packed weights are zero for k < 20 (dn), k < 40 (dm), k < 60 (both))
    auto mma_chunk = [&](uint32_t g_item, int ch, float (&acc)[2][NT][4]) {
      mma::zero(acc);
#pragma unroll
      for (int sh = 0; sh < 4; ++sh) {
        const int shift_rows = (sh >> 1) * Pp + (sh & 1);
#pragma unroll
        for (int k16 = sh; k16 < HEAD_NCOLS / 16; ++k16) {
          const uint32_t g_k = g_item + (2 * k16) * lbo_g - shift_rows * 16;
#pragma unroll
          for (int np = 0; np < NT / 2; ++np) {
            uint32_t bf[4];
            mma::ldsm_x4(bf, g_k + b_row(ch, np));
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              mma::mma_bf16(acc[m][2 * np], af[b3a_kstep(sh, k16)][m], bf[0], bf[1]);
              mma::mma_bf16(acc[m][2 * np + 1], af[b3a_kstep(sh, k16)][m], bf[2], bf[3]);
            }
          }
        }
      }
    };
    int it = 0;
    for (int b = slot; b < P.B; b += nslot)
      for (int band = 0; band < nbands; ++band, ++it) {
        const int st = it & 1, y0 = band * Hh, hb = min(Hh, Hi - y0);
        const int nitems = 2 * (hb / 4);  // (di, feature-row pair) items of this band
        mbar_wait_idle(&g_full[st], (it >> 1) & 1);
        const uint32_t g0 = smem_u32(Gs + (size_t)st * g_bytes);
        for (int item = e; item < nitems; item += 2) {
          const int ip = item >> 1, ml = 4 * ip + e;  // ml: the item's first accumulator row within the band
          const uint32_t g_item = g0 + (uint32_t)(ml * Pp) * 16;
          if (NHWC && !(ACC && P.acc_out)) {
            // (keypoint groups: only the last group's rounding store is channels-last; the fp32 partial sums keep their
            // plane layout)
            const int c0 = mt * 128 + 32 * q, i0 = y0 / 2 + 2 * ip;
            const size_t base = ((size_t)b * 4 * P.C4 + 4 * c0 + 2 * e) * HW + (size_t)i0 * WS2;
            uint16_t* st = reinterpret_cast<uint16_t*>(Ss) + (32 * q) * 4 + 2 * e;
#pragma unroll 1
            for (int ch = 0; ch < Cols::NCHUNK; ++ch) {
              float acc[2][NT][4];
              mma_chunk(g_item, ch, acc);
              b3a_each_pair<WS2>(ch, acc, lane, [&](int r, int dj, int x, float v0, float v1) {
                if (c0 + r >= P.C4) return;
                if constexpr (ACC) {
                  if (P.acc_in) {
                    const float2 p = *reinterpret_cast<const float2*>(P.acc32 + base + (size_t)((4 * r + dj) * HW + x));
                    v0 = p.x + v0, v1 = p.y + v1;
                  }
                }
                uint16_t* d = st + (size_t)x * (B3A_NHWC_PX / 2) + 4 * r + dj;
                d[0] = __bfloat16_as_ushort(__float2bfloat16_rn(v0));
                d[B3A_NHWC_PX / 2] = __bfloat16_as_ushort(__float2bfloat16_rn(v1));
              });
            }
            named_bar_sync(3, B3A_THREADS);  // both groups' halves of the tile are staged
            const int nv = min(128, P.C4 - mt * 128) / 2;  // 16-byte vectors per pixel: this tile's channels
            unsigned char* out = reinterpret_cast<unsigned char*>(P.dfeat + (((size_t)b * (Hi / 2) + i0) * WS2) * 4 * P.C4 + (size_t)mt * 512);
            for (int idx = tid; idx < 2 * WS2 * nv; idx += B3A_THREADS) {
              const int px = idx / nv, v = idx - px * nv;
              *reinterpret_cast<uint4*>(out + (size_t)px * 8 * P.C4 + v * 16) = *reinterpret_cast<const uint4*>(Ss + (size_t)px * B3A_NHWC_PX + v * 16);
            }
            named_bar_sync(3, B3A_THREADS);  // the tile may be overwritten
          } else if (!ACC && P.tma_store) {
            // The 4 warps of this e form a group of 128 channels that owns the slices pl = 2e, 2e + 1.  Items go out in
            // pairs (ip even, ip + 1): a slice row holds both items' 2W pixels of a channel's plane, 8W consecutive bytes
            // of d features, and one tensor store per plane class writes them.  Single items' 4W-byte rows (48 bytes at
            // W = 12) split 32-byte sectors between two stores, which made the stores take twice as long on an H100
            // (DESIGN.md K4).  A band's last item without a partner (odd pair count) is stored alone, from a dense
            // [128][4W bytes] slice.
            constexpr int PB = 4 * WS2, SLICE = 128 * 2 * PB;  // bytes per channel and item / per slice
            const bool issuer = (q == 0 && lane == 0);
            const bool alone = ip + 1 == nitems / 2 && (ip & 1) == 0, last = alone || (ip & 1);
            // row stride and offset of this item in the slice
            const int rs = alone ? PB : 2 * PB, ro = (ip & 1) * PB;
            unsigned char* sl = Ss + (size_t)(2 * e) * SLICE + (size_t)(32 * q) * rs + ro;
#pragma unroll
            for (int ch = 0; ch < Cols::NCHUNK; ++ch) {
              float acc[2][NT][4];
              mma_chunk(g_item, ch, acc);
              if (ch == 0 && (ip & 1) == 0) {
                if (issuer) bulk_wait_group_read0();  // the group's last stores have read the slices
                named_bar_sync(1 + e, 128);
              }
              b3a_each_pair<WS2>(ch, acc, lane, [&](int r, int dj, int x, float v0, float v1) {
                *reinterpret_cast<__nv_bfloat162*>(sl + dj * SLICE + r * rs + 2 * x) = __floats2bfloat162_rn(v0, v1);
              });
            }
            if (last) {
              fence_proxy_async();
              named_bar_sync(1 + e, 128);
              if (issuer) {
                const int px0 = (y0 / 2 + 2 * (ip & ~1)) * WS2;
                const CUtensorMap* tm = alone ? &TM : &TM_PAIR;
                tma_store_4d(tm, Ss + (size_t)(2 * e) * SLICE, px0, 2 * e, mt * 128, b);
                tma_store_4d(tm, Ss + (size_t)(2 * e + 1) * SLICE, px0, 2 * e + 1, mt * 128, b);
                bulk_commit_group();
              }
            }
          } else {
            const int c0 = mt * 128 + 32 * q, i0 = y0 / 2 + 2 * ip;  // the warp's first channel, the pair's first feature row
            const size_t base = ((size_t)b * 4 * P.C4 + 4 * c0 + 2 * e) * HW + (size_t)i0 * WS2;
            // (not unrolled: the chunks' operand addresses would stay live together and spill at W >= 24)
#pragma unroll 1
            for (int ch = 0; ch < Cols::NCHUNK; ++ch) {
              float acc[2][NT][4];
              mma_chunk(g_item, ch, acc);
              b3a_each_pair<WS2>(ch, acc, lane, [&](int r, int dj, int x, float v0, float v1) {
                if (c0 + r >= P.C4) return;
                const size_t off = base + (size_t)((4 * r + dj) * HW + x);
                __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(P.dfeat + off);
                if constexpr (ACC) {
                  float2* a32 = reinterpret_cast<float2*>(P.acc32 + off);
                  if (P.acc_in) {
                    const float2 p = *a32;
                    v0 = p.x + v0, v1 = p.y + v1;
                  }
                  if (P.acc_out) *a32 = make_float2(v0, v1);
                  else *dst = __floats2bfloat162_rn(v0, v1);
                } else {
                  *dst = __floats2bfloat162_rn(v0, v1);
                }
              });
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&g_empty[st]);  // this warp's reads of the band are done
        if (warp == 0 && lb < P.B) {
          mbar_wait(&g_empty[st], (it >> 1) & 1);  // every warp's are: band it + 2 may overwrite the stage
          load_next(it + 2);
        }
      }
    if (!ACC && P.tma_store && q == 0 && lane == 0) bulk_wait_group0();  // the stores have landed before the kernel ends
  }
}


// =====================================================================================================
// wg: weight gradient of a stride-2 3x3 transposed convolution (both layers)
// =====================================================================================================
//   dW[c, o, ky, kx] = sum_{frames, rows} X[row + shift][c] * G[row][(cls, o)]      ((cls, shift) -> tap)
// a GEMM whose K dimension is the pixel raster.  Both operands are the row layout read TRANSPOSED (ldmatrix .trans,
// mma_sm90.cuh ldsm_x4_t): A = G (M = the 80 (cls, o) rows), B = X at a row offset (the shift), N = this CTA's channel
// group.  Of the 4 shifts x 5 m16 tiles of A, 14 hold a real tap (NZ_M16, head_prep.cuh);
// MMA warp w takes half w / 4 of the channel group and the (shift, m16 tile) units of role w % 4 (wg_unit) of it -- at most 4 each,
// where one warp per shift would carry 5.  Its accumulators stay in registers across every (frame, row-chunk) unit of
// the CTA, and one epilogue at the end writes them to the CTA's slot of the partials.  An all-ones input channel (the
// bias lane of the mid activations) yields the bias gradient from the same GEMM.
constexpr int WG_THREADS = 288;  // warp 0 loader, warps 1-8 MMA + epilogue
constexpr int WG_UNITS = 4;
struct WgUnit { int sh, mt; };  // sh = -1: unused
// role r: shift r's non-zero tiles, except (shift 0, tile 3), which the shift-3 role takes: it shares that tile's A
// fragment with its own (shift 3, tile 3)
__host__ __device__ constexpr WgUnit wg_unit(int r, int v) {
  constexpr WgUnit role[4][WG_UNITS] = {
      {{0, 0}, {0, 1}, {0, 2}, {0, 4}},
      {{1, 1}, {1, 2}, {1, 3}, {1, 4}},
      {{2, 2}, {2, 3}, {2, 4}, {-1, 0}},
      {{3, 3}, {0, 3}, {3, 4}, {-1, 0}},
  };
  return role[r][v];
}
// m16 tiles (sh_bits = false) or shifts (true) a role reads
__host__ __device__ constexpr unsigned wg_role_set(int r, bool sh_bits) {
  unsigned m = 0;
  for (int v = 0; v < WG_UNITS; ++v)
    if (wg_unit(r, v).sh >= 0) m |= 1u << (sh_bits ? wg_unit(r, v).sh : wg_unit(r, v).mt);
  return m;
}
// the roles cover exactly the non-zero units, each once
constexpr bool wg_roles_exact() {
  unsigned seen[4] = {0, 0, 0, 0};
  for (int r = 0; r < 4; ++r)
    for (int v = 0; v < WG_UNITS; ++v) {
      const WgUnit u = wg_unit(r, v);
      if (u.sh < 0) continue;
      if (seen[u.sh] & (1u << u.mt)) return false;
      seen[u.sh] |= 1u << u.mt;
    }
  for (int sh = 0; sh < 4; ++sh)
    if (seen[sh] != NZ_M16[sh]) return false;
  return true;
}
static_assert(wg_roles_exact(), "weight-gradient warp roles must cover each non-zero (shift, m16 tile) unit exactly once");

struct WgParams {
  const __nv_bfloat16* X;     // [B][kcx_total][L.rows][8] padded row layout
  const __nv_bfloat16* G;     // [B][10][L.rows][8]
  RowLayout L;
  float* part;                // [slots][Cin * Cout * 9 + 4 * Cout]: this slot's dW, then its bias gradient per output class
  int has_bias;               // 1: the bias gradient is taken from input channel ones_c
  int B, Hi, Wi;
  int R;                      // image rows per unit
  int KR;                     // GEMM-K rows per unit = R*(Wi+1) rounded up to 16
  int XR;                     // X rows per K-chunk in smem (KR + Wi + 2, multiple of 8)
  int kcx, kcx_total;         // K-chunks (8 channels) per CTA group / per frame
  int Cin, Cout, ones_c;
  int ngo;                    // keypoint groups of Cout: G holds ngo * 10 K-chunks per frame, and a CTA takes one group
  int smem_bytes;
};

// The gradients are summed over the CTAs in a fixed order (per-CTA partials, then reduce_partials_kernel), so that a
// backward pass gives bit-identical results from run to run.
constexpr int WG_MAX_CTAS = 132;   // weight-gradient CTAs per layer (one per SM of an H100 SXM; fewer on smaller devices)
constexpr int B2D_MAX_CTAS = 264;  // b2d CTAs (two per SM)
// Budget of the one-CTA-per-SM kernels (weight gradient, layer-1 data gradient b3a): an H100 SM's 227 KB less 2 KB.  It
// picks the weight gradient's rows per unit R and whether b3a stages its d features for TMA stores.
constexpr size_t HEAD_BWD_SMEM_BUDGET = 225 * 1024;
__host__ __device__ inline size_t wgrad_part_stride(int Cin, int Cout) { return (size_t)Cin * Cout * 9 + 4 * (size_t)Cout; }
// weight-gradient channel group (K-chunks of 8 channels per CTA) of a layer with nkc K-chunks of input
inline int wgrad_kcx(int nkc) { return nkc % 8 == 0 ? 8 : 4; }
inline int wgrad_max_slots(int nkc) {
  const int slots = WG_MAX_CTAS / (nkc / wgrad_kcx(nkc));
  return slots < 1 ? 1 : slots;
}

// NT = n8 tiles per warp = kcx / 2
template <int NT>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_kernel(const __grid_constant__ WgParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1, R = P.R, KR = P.KR, XR = P.XR;
  const int g_bytes = HEAD_KC * KR * 16, x_bytes = P.kcx * XR * 16;
  unsigned char* Gs = smem;
  unsigned char* Xs = smem + 2 * g_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P.smem_bytes - 64);
  uint64_t* full = bars;       // [2]
  uint64_t* empty = bars + 2;  // [2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = P.kcx * 8;
  const int ngroups = P.kcx_total / P.kcx;  // kcx_total may include K-chunks beyond the last group (ignored)
  // CTA tile = (channel group grp, output keypoint group go), slot = its share of the (frame, row-chunk) units
  const int ntile = ngroups * P.ngo, tile = blockIdx.x % ntile, grp = tile % ngroups, go = tile / ngroups;
  const int slot = blockIdx.x / ntile, nslot = gridDim.x / ntile;
  const int nchunk = Hi / R, nunits = P.B * nchunk;  // R divides Hi (host)

  for (int i = tid; i < (P.smem_bytes - 64) / 16; i += WG_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], WG_THREADS / 32 - 1);  // one arrival per MMA warp
    }
    fence_mbar_init();
  }
  fence_proxy_async();
  __syncthreads();

  if (warp == 0) {
    int j = 0;
    for (int u = slot; u < nunits; u += nslot, ++j) {
      const int s = j & 1, b = u / nchunk, y0 = (u - b * nchunk) * R;
      mbar_wait(&empty[s], ((j >> 1) & 1) ^ 1);
      // one copy per K-chunk: R image rows of G; R + 1 rows of X (the row below is the shifts' halo)
      const uint32_t gbytes = (uint32_t)(R * Pp * 16), xbytes = (uint32_t)((R + 1) * Pp * 16);
      if (lane == 0) mbar_expect_tx(&full[s], HEAD_KC * gbytes + P.kcx * xbytes);
      __syncwarp();
      const size_t row0 = (size_t)P.L.lead + (size_t)y0 * Pp;
      if (lane < HEAD_KC)
        bulk_g2s(Gs + (size_t)s * g_bytes + (size_t)lane * KR * 16, P.G + (((size_t)(b * P.ngo + go) * HEAD_KC + lane) * P.L.rows + row0) * 8, gbytes,
                 &full[s]);
      if (lane < P.kcx)
        bulk_g2s(Xs + (size_t)s * x_bytes + (size_t)lane * XR * 16,
                 P.X + (((size_t)b * P.kcx_total + (size_t)grp * P.kcx + lane) * P.L.rows + row0) * 8, xbytes, &full[s]);
    }
  } else if (slot < nunits) {
    const int cw = warp - 1, half = cw >> 2;
    const uint32_t g0 = smem_u32(Gs), x0 = smem_u32(Xs) + (uint32_t)(half * NT) * XR * 16;  // n8 tile = one K-chunk of X
    float* part = P.part + (size_t)slot * wgrad_part_stride(P.Cin, P.Cout);
    // warp role r = cw % 4 owns the (shift, m16 tile) units wg_unit(r, .) of channel half `half`
    auto run = [&](auto rc) {
      constexpr int ROLE = decltype(rc)::value;
      constexpr unsigned mt_set = wg_role_set(ROLE, false), sh_set = wg_role_set(ROLE, true);
      float acc[WG_UNITS][NT][4];
      mma::zero(acc);
      int j = 0;
      for (int u = slot; u < nunits; u += nslot, ++j) {
        const int s = j & 1;
        mbar_wait(&full[s], (j >> 1) & 1);
        const uint32_t a = g0 + s * g_bytes, b = x0 + s * x_bytes;
        for (int k16 = 0; k16 < KR / 16; ++k16) {
          // A (G) fragments of the role's m16 tiles, B (X) fragments of its shifts; each loaded once per K step
          uint32_t af[HEAD_NCOLS / 16][4], bf[4][NT / 2][4];
#pragma unroll
          for (int mt = 0; mt < HEAD_NCOLS / 16; ++mt)
            if ((mt_set >> mt) & 1u)
              mma::ldsm_x4_t(af[mt], a + k16 * 256 + (uint32_t)(2 * mt + ((lane >> 3) & 1)) * KR * 16 + (uint32_t)((lane >> 4) * 8 + (lane & 7)) * 16);
#pragma unroll
          for (int sh = 0; sh < 4; ++sh)
            if ((sh_set >> sh) & 1u)
#pragma unroll
              for (int np = 0; np < NT / 2; ++np)
                mma::ldsm_x4_t(bf[sh][np], b + (k16 * 16 + (sh >> 1) * Pp + (sh & 1)) * 16 + (uint32_t)(2 * np + (lane >> 4)) * XR * 16 +
                                               (uint32_t)(((lane >> 3) & 1) * 8 + (lane & 7)) * 16);
#pragma unroll
          for (int v = 0; v < WG_UNITS; ++v) {
            const int ush = wg_unit(ROLE, v).sh, umt = wg_unit(ROLE, v).mt;
            if (ush < 0) continue;
#pragma unroll
            for (int np = 0; np < NT / 2; ++np) {
              mma::mma_bf16(acc[v][2 * np], af[umt], bf[ush][np][0], bf[ush][np][1]);
              mma::mma_bf16(acc[v][2 * np + 1], af[umt], bf[ush][np][2], bf[ush][np][3]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      }
      // accumulator (k = 16 mt + g (+8), c = 8 nt + 2 t (+1)) of unit (shift, mt) -> this slot's partial of dW[c][o][ky][kx]
      const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
      for (int v = 0; v < WG_UNITS; ++v) {
        const int sh = wg_unit(ROLE, v).sh, mt = wg_unit(ROLE, v).mt;
        if (sh < 0) continue;
        const int dm = sh >> 1, dn = sh & 1;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int k = 16 * mt + gq + 8 * (i >> 1);
          const int cls = k / HEAD_CLS, o = go * HEAD_CLS + k - cls * HEAD_CLS, py = cls >> 1, px = cls & 1;
          if (o >= P.Cout || !tap_nonzero(cls, sh)) continue;
          const int ky = py == 0 ? 1 : (dm ? 0 : 2), kx = px == 0 ? 1 : (dn ? 0 : 2);
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const int c = grp * N + (half * NT + nt) * 8 + 2 * tq + (i & 1);
            const float val = acc[v][nt][i];
            // (cls, shift) -> tap is one-to-one and every unit has one owner, so every element of the slot's partial has
            // exactly one writer
            if (c < P.Cin) part[((size_t)c * P.Cout + o) * 9 + ky * 3 + kx] = val;
            else if (P.has_bias && c == P.ones_c && sh == 0) part[(size_t)P.Cin * P.Cout * 9 + cls * P.Cout + o] = val;
          }
        }
      }
    };
    switch (cw & 3) {
      case 0: run(std::integral_constant<int, 0>{}); break;
      case 1: run(std::integral_constant<int, 1>{}); break;
      case 2: run(std::integral_constant<int, 2>{}); break;
      default: run(std::integral_constant<int, 3>{}); break;
    }
  }
}

static int launch_wgrad(const __nv_bfloat16* X, const __nv_bfloat16* G, float* dW, float* dbias, float* part, int B, int Hi, int Wi,
                        int kcx_total, int Cin, int Cout, int ones_c, int sms, cudaStream_t s) {
  const int ngo = head_groups(Cout);
  const int kcx = wgrad_kcx(kcx_total);
  // image rows per unit: the largest divisor of Hi (<= 8) whose two stages fit in shared memory
  int R = 0;
  for (int r = Hi < 8 ? Hi : 8; r >= 1; --r) {
    if (Hi % r) continue;
    const int kr = (r * (Wi + 1) + 15) & ~15, xr = (kr + Wi + 2 + 7) & ~7;
    if ((size_t)2 * HEAD_KC * kr * 16 + (size_t)2 * kcx * xr * 16 + 64 <= HEAD_BWD_SMEM_BUDGET) {
      R = r;
      break;
    }
  }
  LPB_REQUIRE(R >= 1, "head_bwd_bf16: image width %d too large for the weight-gradient stages", Wi);
  WgParams p;
  p.X = X;
  p.G = G;
  p.L = make_row_layout(Hi, Wi);
  p.part = part;
  p.has_bias = dbias != nullptr;
  p.B = B;
  p.Hi = Hi;
  p.Wi = Wi;
  p.R = R;
  p.KR = (R * (Wi + 1) + 15) & ~15;
  p.XR = (p.KR + Wi + 2 + 7) & ~7;
  p.kcx = kcx;
  p.kcx_total = kcx_total;
  p.Cin = Cin;
  p.Cout = Cout;
  p.ones_c = ones_c;
  p.ngo = ngo;
  const size_t body = ((size_t)2 * HEAD_KC * p.KR * 16 + (size_t)2 * kcx * p.XR * 16 + 15) & ~(size_t)15;
  p.smem_bytes = (int)(body + 64);  // within the budget: R was chosen so
  const int ngroups = kcx_total / kcx * ngo;  // CTA tiles
  const int nunits = B * (Hi / R);
  int slots = sms / ngroups;
  if (slots > wgrad_max_slots(kcx_total)) slots = wgrad_max_slots(kcx_total);  // the partials' workspace
  if (slots < 1) slots = 1;
  if (slots > nunits) slots = nunits;
  auto kern = kcx == 8 ? wgrad_kernel<4> : wgrad_kernel<2>;
  LPB_TRY(set_dynamic_smem(kern, p.smem_bytes, "head_bwd_bf16"));
  kern<<<slots * ngroups, WG_THREADS, p.smem_bytes, s>>>(p);
  const size_t stride = wgrad_part_stride(Cin, Cout);
  reduce_partials<1>(part, slots, stride, Cin * Cout * 9, dW, sms, s);
  if (dbias) reduce_partials<4>(part + (size_t)Cin * Cout * 9, slots, stride, Cout, dbias, sms, s);  // 4 output classes per slot
  return LPB_OK;
}


// bias gradient of a one-deconv head: column sums of the gradient rows, folded over the four classes.  Stage 1 writes
// the eight column sums of every (frame, K-chunk); stage 2 adds them per output channel in a fixed order, so the bias
// gradient is bit-reproducible like every other gradient of this file (no atomics).
__global__ void __launch_bounds__(256) rows_colsum_kernel(const __nv_bfloat16* __restrict__ G, RowLayout L, float* __restrict__ part) {
  // one CTA per (frame, K-chunk): thread = (row stripe, e); the frame's chunks are consecutive, so block = b * nkc + kc
  const __nv_bfloat16* slab = G + (size_t)blockIdx.x * (size_t)L.rows * 8;
  const int e = threadIdx.x & 7;
  float acc = 0.f;
  for (int r = L.lead + (threadIdx.x >> 3); r < L.lead + L.Hi * L.Pp; r += 32) acc += __bfloat162float(slab[(size_t)r * 8 + e]);
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float t = 0.f;
    for (int i = threadIdx.x; i < 256; i += 8) t += red[i];
    part[(size_t)blockIdx.x * 8 + threadIdx.x] = t;
  }
}

// one CTA per output channel o = 20 g + o': the partials of K entries k = kc * 8 + e of group g (k / 80 == g of the
// frame's nkc * 8) with k % HEAD_CLS == o', in a fixed order
__global__ void __launch_bounds__(256) rows_colsum_reduce_kernel(const float* __restrict__ part, long long n, int nkc, float* __restrict__ db) {
  const int o = blockIdx.x;
  float acc = 0.f;
  for (long long j = threadIdx.x; j < n; j += 256) {
    const int k = (int)(j % (nkc * 8));
    if ((k / HEAD_NCOLS) * HEAD_CLS + (k % HEAD_NCOLS) % HEAD_CLS == o) acc += part[j];
  }
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) db[o] = red[0];
}

// largest rows-per-band Hh (multiple of 4) whose band fits the b3a shared-memory stages
static int b3a_band_rows(int Hi1, int Wi1) {
  int hh = (256 / (Wi1 + 1)) & ~3;  // two accumulator buffers fit
  if (hh < 4) hh = (304 / (Wi1 + 1)) & ~3;  // wide maps: one buffer
  if (hh > Hi1) hh = Hi1;
  return hh;
}

// shared memory of b3a's operands: two band stages of G1 and the CTA's weights
static size_t b3a_operand_smem_bytes(int Hi1, int Wi1) {
  const int ncols = (b3a_band_rows(Hi1, Wi1) * (Wi1 + 1) + 15) & ~15, rows_alloc = (Wi1 + 2 + ncols + 7) & ~7;
  return (size_t)2 * HEAD_KC * rows_alloc * 16 + (size_t)4 * HEAD_KC * 128 * 16 + 160;
}

// d features [B][4*C4][HW] bf16 viewed as [b][c'][pl][px]; box = {box_px pixels, one pl, 128 c', one frame}.
static bool make_dfeat_tensor_map(CUtensorMap* tm, void* dfeat, int B, int C4, int HW, int box_px) {
  const TensorMapEncodeFn encode = tensor_map_encoder();
  if (!encode || (HW * 2) % 16 != 0 || (box_px * 2) % 16 != 0 || box_px > 256) return false;
  const cuuint64_t gdim[4] = {(cuuint64_t)HW, 4, (cuuint64_t)C4, (cuuint64_t)B};
  const cuuint64_t gstride[3] = {(cuuint64_t)HW * 2, (cuuint64_t)HW * 2 * 4, (cuuint64_t)HW * 2 * 4 * (cuuint64_t)C4};  // bytes, dims 1..3
  const cuuint32_t box[4] = {(cuuint32_t)box_px, 1, 128, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  return encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dfeat, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The shapes the backward serves (lpb200.h): H even, W one of the widths b3a_dgrad_kernel is instantiated for, and the
// forward's channel limits.  LPB_OK, or LPB_ERR_UNSUPPORTED with the message set.
static int head_bwd_covers(const char* who, int H, int W, int c1, int c2, int feature_layout) {
  const bool width = W == 4 || W == 8 || W == 12 || W == 16 || W == 24 || W == 32;
  if (feature_layout != LPB_FEATURES_NCHW && feature_layout != LPB_FEATURES_NHWC) {
    set_error("%s: unknown feature layout %d", who, feature_layout);
    return LPB_ERR_INVALID;
  }
  if (feature_layout == LPB_FEATURES_NHWC && width && b3a_operand_smem_bytes(2 * H, 2 * W) + b3a_nhwc_stage_bytes(W) > HEAD_BWD_SMEM_BUDGET) {
    // (W = 32: the operands leave no room for the transposing tile; such features train through an NCHW copy)
    set_error("%s: channels-last d features of width %d do not fit the data gradient's shared memory", who, W);
    return LPB_ERR_UNSUPPORTED;
  }
  if (H % 2 == 0 && width && (head_narrow(c1, c2) || head_wide(c1, c2))) return LPB_OK;
  set_error("%s: head %dx%d with %d/%d channels outside this build's set (H even, W in {4, 8, 12, 16, 24, 32}, the "
            "forward's channel counts)", who, H, W, c1, c2);
  return LPB_ERR_UNSUPPORTED;
}

// Byte offsets into the backward's workspace: [W1 dgrad pack][W2 dgrad pack][G2][G1][plane dots, 256-byte rounded] and
// the fixed-order reduction partials [layer-1 wgrad][layer-2 wgrad][b2d bias].  G2 / G1 are padded row layouts
// (row_layout.cuh).  A one-deconv head (c2 = 0) has no G2 (its output gradient is G1 directly) but keeps the W2 pack's
// space, and its partials are [layer-1 wgrad][bias column sums: eight per (frame, K-chunk)].  Members a head does not
// have are 0.
// Keypoint groups (wide heads, head_prep.cuh): the packs hold one block per (K group, tile), G2 / G1 hold 10 K-chunks per
// group of c2 / c1, and two fp32 buffers follow the narrow layout: dmid [B][c1][4H * 4W] (the mid activations' gradient,
// summed over the c2 groups, two-deconv heads) and acc32 [B][C][H * W] (the d features of the c1 groups before the last,
// when c1 has more than one group).  Narrow heads have one group everywhere and neither buffer.
// Three-deconv heads (c3 > 0, narrow: head_narrow3) append [W3 dgrad pack][G3 (8H x 8W grid)][layer-3 wgrad partials]
// [layer-3 b2d bias partials] to the two-deconv layout; every other head has none of them.
// With keypoint targets, the per-plane target factors (mse_fac_stride floats per output plane) come last.
struct HeadBwdLayout {
  size_t wp1, wp2, G2, G1, ddot, part1, part2, part_db1, part_cs, dmid, acc32, wp3, G3, part3, part_db2, fac, total;
};
static HeadBwdLayout head_bwd_layout(int B, int C, int H, int W, int c1, int c2, bool targets, int c3 = 0) {
  const int C4 = C / 4;
  const bool two = c2 > 0, wide = head_wide(c1, c2), three = two && c3 > 0;
  const int kout = three ? c3 : two ? c2 : c1;  // planes of the head's output
  const int g1 = head_groups(c1), g2 = two ? head_groups(c2) : 1, nst2 = two ? head_mid_stages(c1) : 1;
  HeadBwdLayout l{};
  l.wp1 = 0;
  l.wp2 = l.wp1 + (size_t)g1 * ((C4 + 127) / 128) * 4 * HEAD_KC * 128 * 16;
  l.G2 = l.wp2 + (size_t)(two ? g1 * g2 : 1) * 4 * HEAD_KC * 32 * 16;
  l.G1 = l.G2 + (two ? (size_t)B * g2 * HEAD_KC * make_row_layout(4 * H, 4 * W).rows * 16 : 0);
  l.ddot = l.G1 + (size_t)B * g1 * HEAD_KC * make_row_layout(2 * H, 2 * W).rows * 16;
  l.part1 = l.ddot + (((size_t)B * kout * 4 + 255) & ~(size_t)255);
  const size_t part1_end = l.part1 + (size_t)wgrad_max_slots(C4 / 8) * wgrad_part_stride(C4, c1) * sizeof(float);
  if (two) {
    l.part2 = part1_end;
    l.part_db1 = l.part2 + (size_t)wgrad_max_slots(4 * nst2) * wgrad_part_stride(c1, c2) * sizeof(float);
    l.total = l.part_db1 + (size_t)B2D_MAX_CTAS * 4 * HEAD_CLS * sizeof(float);
  } else {
    l.part_cs = part1_end;
    l.total = l.part_cs + (size_t)B * HEAD_KC * 8 * sizeof(float);
  }
  if (wide) {
    l.part_cs = l.total;  // the bias column sums of G1 (db1 of every wide head)
    l.dmid = l.part_cs + (((size_t)B * g1 * HEAD_KC * 8 * sizeof(float) + 255) & ~(size_t)255);
    l.acc32 = l.dmid + (two ? (size_t)B * c1 * 16 * H * W * sizeof(float) : 0);
    l.total = l.acc32 + (g1 > 1 ? (size_t)B * C * H * W * sizeof(float) : 0);
  }
  if (three) {
    l.wp3 = (l.total + 255) & ~(size_t)255;
    l.G3 = l.wp3 + (size_t)4 * HEAD_KC * 32 * 16;
    l.part3 = l.G3 + (size_t)B * HEAD_KC * make_row_layout(8 * H, 8 * W).rows * 16;
    l.part_db2 = l.part3 + (size_t)wgrad_max_slots(4 * head_mid_stages(c2)) * wgrad_part_stride(c2, c3) * sizeof(float);
    l.total = l.part_db2 + (size_t)B2D_MAX_CTAS * 4 * HEAD_CLS * sizeof(float);
  }
  if (targets) {
    const int up = three ? 16 : two ? 8 : 4;  // output grid: (up H) x (up W)
    l.fac = (l.total + 255) & ~(size_t)255;
    l.total = l.fac + (size_t)B * kout * mse_fac_stride(up * H, up * W) * sizeof(float);
  }
  return l;
}

}  // namespace lpb

extern "C" int lpb_head_bwd_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes) {
  return lpb_head_bwd_bf16_workspace_bytes_layout(B, C, H, W, c1, c2, LPB_FEATURES_NCHW, bytes);
}

extern "C" int lpb_head_bwd_bf16(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                                 const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H,
                                 int W, const float* w1, int c1, const float* w2, int c2, void* dfeat, float* dw1, float* db1,
                                 float* dw2, float* db2, void* workspace, void* stream) {
  return lpb_head_bwd_bf16_layout(g_out, probs, win, win_meta, g_overflow, saved_xs, fwd_workspace, B, C, H, W, w1, c1, w2, c2,
                                  LPB_FEATURES_NCHW, dfeat, dw1, db1, dw2, db2, workspace, stream);
}

extern "C" int lpb_head_bwd_bf16_workspace_bytes_layout(int B, int C, int H, int W, int c1, int c2, int feature_layout, size_t* bytes) {
  return lpb_head_bwd_bf16_workspace_bytes_targets(B, C, H, W, c1, c2, feature_layout, 0, bytes);
}

extern "C" int lpb_head_bwd_bf16_workspace_bytes_targets(int B, int C, int H, int W, int c1, int c2, int feature_layout, int with_targets,
                                                         size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "head_bwd_bf16_workspace_bytes: null pointer");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 0, "head_bwd_bf16_workspace_bytes: bad shape");
  if (const int rc = head_bwd_covers("head_bwd_bf16_workspace_bytes", H, W, c1, c2, feature_layout); rc != LPB_OK) return rc;
  *bytes = head_bwd_layout(B, C, H, W, c1, c2, with_targets != 0).total;
  return LPB_OK;
}

extern "C" int lpb_head_bwd_bf16_layout(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                                        const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C,
                                        int H, int W, const float* w1, int c1, const float* w2, int c2, int feature_layout,
                                        void* dfeat, float* dw1, float* db1, float* dw2, float* db2, void* workspace, void* stream) {
  return lpb_head_bwd_bf16_targets(g_out, nullptr, probs, win, win_meta, g_overflow, saved_xs, fwd_workspace, B, C, H, W, w1, c1, w2, c2,
                                   feature_layout, dfeat, dw1, db1, dw2, db2, workspace, stream);
}

// lpb_head_bwd_bf16_targets (c3 = 0) and lpb_head3_bwd (c3 > 0, a narrow three-deconv head).  A third layer runs ahead of
// the two-deconv sequence: the front end writes G3 on the 8H x 8W grid, the layer-3 weight gradient reads mid2, and b2d
// takes G3 to G2 (the mid2 gradient, whose column sums are db2); from G2 on, the two-deconv kernels run unchanged.
static int head_bwd(const float* g_out, const lpb_mse_targets* mse, const float* probs, const float* win, const int32_t* win_meta,
                    const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H, int W,
                    const float* w1, int c1, const float* w2, int c2, int feature_layout, void* dfeat, float* dw1, float* db1,
                    float* dw2, float* db2, void* workspace, void* stream, const float* w3 = nullptr, int c3 = 0,
                    float* dw3 = nullptr, float* db3 = nullptr) {
  using namespace lpb;
  const bool two = c2 > 0, three = c3 > 0, nhwc = feature_layout == LPB_FEATURES_NHWC;
  LPB_REQUIRE(saved_xs && fwd_workspace && w1 && dw1 && db1 && workspace, "head_bwd_bf16: null pointer");
  LPB_REQUIRE(!two || (w2 && dw2 && db2), "head_bwd_bf16: a two-deconv head needs w2, dw2, db2");
  LPB_REQUIRE(!three || (two && w3 && dw3 && db3), "head_bwd_bf16: a three-deconv head needs w2, w3, dw2, db2, dw3, db3");
  LPB_REQUIRE(g_out || mse || win, "head_bwd_bf16: neither a dense gradient nor decode windows given");
  if (mse) {
    LPB_REQUIRE(!g_out, "head_bwd_bf16: keypoint targets stand for the dense gradient; g_out must be null");
    LPB_REQUIRE(probs, "head_bwd_bf16: keypoint targets need the softmax head's output (probs)");
    LPB_REQUIRE(mse->keypoints && mse->fwd_out && mse->grad_out, "head_bwd_bf16: keypoint targets: null pointer");
    LPB_REQUIRE(mse->img_height > 0.f && mse->img_width > 0.f && mse->sigma > 0.f, "head_bwd_bf16: keypoint targets: bad image size or sigma");
  }
  LPB_REQUIRE(!win || (win_meta && g_overflow), "head_bwd_bf16: windows need their meta and overflow buffers");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1, "head_bwd_bf16: bad shape C=%d H=%d W=%d c1=%d", C, H, W, c1);
  if (const int rc = head_bwd_covers("head_bwd_bf16", H, W, c1, c2, feature_layout); rc != LPB_OK) return rc;
  if (const char* why = nullptr; three && !head3_covered(H, W, c1, c2, c3, true, &why)) {
    set_error("head_bwd_bf16: three-deconv head %dx%d with %d/%d/%d channels: %s", H, W, c1, c2, c3, why);
    return LPB_ERR_UNSUPPORTED;
  }
  {
    // read or written with 16-byte vectors (g_out, probs, g_overflow: float4 plane dots; win_meta: int4; dfeat: uint4 or
    // TMA stores) or bulk copies (saved_xs, fwd_workspace, workspace)
    const struct { const void* p; const char* name; } bufs[] = {{g_out, "g_out"}, {probs, "probs"}, {win_meta, "win_meta"},
        {g_overflow, "g_overflow"}, {saved_xs, "saved_xs"}, {fwd_workspace, "fwd_workspace"}, {dfeat, "dfeat"}, {workspace, "workspace"}};
    for (const auto& b : bufs) LPB_REQUIRE(aligned_to(b.p, 16), "head_bwd_bf16: %s must be 16-byte aligned", b.name);
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int C4 = C / 4, Hi1 = 2 * H, Wi1 = 2 * W, Hi2 = 4 * H, Wi2 = 4 * W, Hi3 = 8 * H, Wi3 = 8 * W;
  const int kout = three ? c3 : two ? c2 : c1;
  if (B == 0) {
    LPB_CUDA(cudaMemsetAsync(dw1, 0, sizeof(float) * (size_t)C4 * c1 * 9, s));
    LPB_CUDA(cudaMemsetAsync(db1, 0, sizeof(float) * c1, s));
    if (two) {
      LPB_CUDA(cudaMemsetAsync(dw2, 0, sizeof(float) * (size_t)c1 * c2 * 9, s));
      LPB_CUDA(cudaMemsetAsync(db2, 0, sizeof(float) * c2, s));
    }
    if (three) {
      LPB_CUDA(cudaMemsetAsync(dw3, 0, sizeof(float) * (size_t)c2 * c3 * 9, s));
      LPB_CUDA(cudaMemsetAsync(db3, 0, sizeof(float) * c3, s));
    }
    return LPB_OK;
  }
  const int Hh = b3a_band_rows(Hi1, Wi1);
  if (Hh < 4) {
    set_error("head_bwd_bf16: feature map %dx%d outside this build's band tiling", H, W);
    return LPB_ERR_UNSUPPORTED;
  }
  DeviceLimits dev;
  LPB_TRY(device_limits(&dev));
  const int sms = dev.sms;
  const RowLayout L3 = make_row_layout(Hi3, Wi3), L2 = make_row_layout(Hi2, Wi2), L1 = make_row_layout(Hi1, Wi1);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const int ntile1 = (C4 + 127) / 128;
  const HeadBwdLayout wl = head_bwd_layout(B, C, H, W, c1, c2, mse != nullptr, c3);
  __nv_bfloat16* wp1 = reinterpret_cast<__nv_bfloat16*>(ws + wl.wp1);
  __nv_bfloat16* wp2 = reinterpret_cast<__nv_bfloat16*>(ws + wl.wp2);
  __nv_bfloat16* G2 = reinterpret_cast<__nv_bfloat16*>(ws + wl.G2);
  __nv_bfloat16* G1 = reinterpret_cast<__nv_bfloat16*>(ws + wl.G1);
  float* ddot = reinterpret_cast<float*>(ws + wl.ddot);
  float* part1 = reinterpret_cast<float*>(ws + wl.part1);
  float* part2 = two ? reinterpret_cast<float*>(ws + wl.part2) : nullptr;
  float* part_db1 = two ? reinterpret_cast<float*>(ws + wl.part_db1) : nullptr;
  const bool wide = head_wide(c1, c2);
  const int g1 = head_groups(c1), g2 = two ? head_groups(c2) : 1, nst2 = two ? head_mid_stages(c1) : 1;
  float* part_cs = two && !wide ? nullptr : reinterpret_cast<float*>(ws + wl.part_cs);
  float* dmid = wide && two ? reinterpret_cast<float*>(ws + wl.dmid) : nullptr;
  float* acc32 = wide && g1 > 1 ? reinterpret_cast<float*>(ws + wl.acc32) : nullptr;
  __nv_bfloat16* wp3 = three ? reinterpret_cast<__nv_bfloat16*>(ws + wl.wp3) : nullptr;
  __nv_bfloat16* G3 = three ? reinterpret_cast<__nv_bfloat16*>(ws + wl.G3) : nullptr;
  float* part3 = three ? reinterpret_cast<float*>(ws + wl.part3) : nullptr;
  float* part_db2 = three ? reinterpret_cast<float*>(ws + wl.part_db2) : nullptr;
  const int nst3 = three ? head_mid_stages(c2) : 0;
  // the forward pass's mid activations
  const HeadFwdLayout fl = head_fwd_layout(B, C, H, W, c1, c2, c3);
  const __nv_bfloat16* mid = reinterpret_cast<const __nv_bfloat16*>(static_cast<const unsigned char*>(fwd_workspace) + fl.mid);
  const __nv_bfloat16* mid2 = reinterpret_cast<const __nv_bfloat16*>(static_cast<const unsigned char*>(fwd_workspace) + fl.mid2);

  {
    // one launch: gradient accumulators zeroed, both data-gradient operand packs, pad rows of G2 / G1
    PrepJobs jobs{};
    jobs.dpack[0] = {w1, C4, c1, ntile1, 128, 128, g1, wp1};
    jobs.pads[0] = {G1, L1, (long long)B * g1 * HEAD_KC};
    jobs.zero[0] = {dw1, (long long)C4 * c1 * 9};
    jobs.zero[1] = {db1, (long long)c1};
    if (two) {
      // wide: tile t = the mid channels of c1 group t (20 of the 32 rows), K = one c2 group
      if (wide) jobs.dpack[1] = {w2, c1, c2, g1, 32, HEAD_CLS, g2, wp2};
      else jobs.dpack[1] = {w2, c1, c2, 1, 32, 32, 1, wp2};
      jobs.pads[1] = {G2, L2, (long long)B * g2 * HEAD_KC};
      jobs.zero[2] = {dw2, (long long)c1 * c2 * 9};
      jobs.zero[3] = {db2, (long long)c2};
    }
    if (three) {
      jobs.dpack[2] = {w3, c2, c3, 1, 32, 32, 1, wp3};
      jobs.pads[2] = {G3, L3, (long long)B * HEAD_KC};
      jobs.zero[4] = {dw3, (long long)c2 * c3 * 9};
      jobs.zero[5] = {db3, (long long)c3};
    }
    launch_head_prep(jobs, sms, s);
  }
  {
    // gradient front end on the head's OUTPUT grid: G3 / G2 / G1 for a three- / two- / one-deconv head
    const int Hio = three ? Hi3 : two ? Hi2 : Hi1, Wio = three ? Wi3 : two ? Wi2 : Wi1;
    __nv_bfloat16* Gout = three ? G3 : two ? G2 : G1;
    const RowLayout Lo = three ? L3 : two ? L2 : L1;
    G2Src src{};
    src.g_out = g_out;
    src.probs = probs;
    src.win = win;
    src.meta = win ? win_meta : nullptr;
    src.gov = g_overflow;
    src.ddot = nullptr;
    if (mse) {
      const int oh = 2 * Hio, ow = 2 * Wio;  // ow is a multiple of 4 (W even)
      const TargetGeom tg = target_geom(mse->img_height, mse->img_width, oh, ow, mse->sigma);
      src.kp = mse->keypoints;
      src.vis = mse->visibility;
      src.sx = tg.sx, src.sy = tg.sy, src.two_s2 = tg.two_s2;
      src.mse_out = mse->fwd_out;
      src.mse_gout = mse->grad_out;
      src.fac = reinterpret_cast<float*>(ws + wl.fac);
      src.fac_stride = mse_fac_stride(oh, ow);
      plane_dot_targets_kernel<<<(unsigned)(B * kout), 256, (size_t)(oh + ow + 16) * sizeof(float), s>>>(src, oh, ow, ddot);
      src.ddot = ddot;
      launch_g2_build<true, true, true>(src, B, kout, Hio, Wio, Gout, Lo, s);
    } else {
      if (probs) {
        LPB_REQUIRE(((4 * Hio * Wio) % 4) == 0, "head_bwd_bf16: plane size");
        if (!g_out && win)
          plane_dot_sparse_kernel<<<(unsigned)(((long long)B * kout + 7) / 8), 256, 0, s>>>(src, (long long)B * kout, 4 * Hio * Wio, ddot);
        else
          plane_dot_kernel<<<(unsigned)(B * kout), 256, 0, s>>>(src, 4 * Hio * Wio, ddot);
        src.ddot = ddot;
      }
      if (g_out && probs) launch_g2_build<true, true>(src, B, kout, Hio, Wio, Gout, Lo, s);
      else if (g_out) launch_g2_build<true, false>(src, B, kout, Hio, Wio, Gout, Lo, s);
      else if (probs) launch_g2_build<false, true>(src, B, kout, Hio, Wio, Gout, Lo, s);
      else launch_g2_build<false, false>(src, B, kout, Hio, Wio, Gout, Lo, s);
    }
  }
  // b2d over a (Hi x Wi) gradient grid Gin: the data gradient at the layer's input, written as the gradient rows Gnext
  // of the layer before (grid Lnext) with the bias-gradient partials of that layer's cmid channels in db_part
  int grid = B < 2 * sms ? B : 2 * sms;
  if (grid > B2D_MAX_CTAS) grid = B2D_MAX_CTAS;  // the bias partials' workspace
  auto b2d_params = [&](const __nv_bfloat16* Gin, RowLayout Lin, const __nv_bfloat16* wpk, __nv_bfloat16* Gnext, RowLayout Lnext, int Hi, int Wi,
                        int cmid, float* db_part, size_t* smem) {
    B2dParams p{};
    p.G2 = Gin;
    p.wpk = wpk;
    p.G1 = Gnext;
    p.L2 = Lin;
    p.L1 = Lnext;
    p.db1_part = db_part;
    p.B = B;
    p.Hi = Hi;
    p.Wi = Wi;
    p.c1 = cmid;
    p.R2 = (B2D_TILES * 128) / (Wi + 1);
    if (p.R2 > Hi) p.R2 = Hi;
    const int rows_alloc = (Wi + 2 + B2D_TILES * 128 + 7) & ~7;
    *smem = (size_t)HEAD_KC * rows_alloc * 16 + (size_t)4 * HEAD_KC * 32 * 16 + 64;
    return p;
  };
  if (three) {
    // layer 3: weight + bias gradient (bias from the all-ones channel c2 of mid2), then data gradient -> G2 (+ db2)
    const int rc = launch_wgrad(mid2, G3, dw3, db3, part3, B, Hi3, Wi3, 4 * nst3, c2, c3, c2, sms, s);
    if (rc != LPB_OK) return rc;
    size_t smem = 0;
    const B2dParams p = b2d_params(G3, L3, wp3, G2, L2, Hi3, Wi3, c2, part_db2, &smem);
    LPB_REQUIRE(smem <= HEAD_STAGE_SMEM_BUDGET && p.R2 >= 1, "head_bwd_bf16: layer-3 width %d too large", Wi3);
    LPB_TRY(set_dynamic_smem(b2d_dgrad_kernel<false>, smem, "head_bwd_bf16"));
    b2d_dgrad_kernel<false><<<grid, B2D_THREADS, smem, s>>>(p);
    reduce_partials<1>(part_db2, grid * 4, HEAD_CLS, c2, db2, sms, s);
  }
  if (two) {
    // layer 2: weight gradient and, for a two-deconv head, the bias gradient (from the all-ones channel c1 of mid; a
    // three-deconv head has db2 from layer 3's b2d), then data gradient -> G1 (+ db1)
    const int rc = launch_wgrad(mid, G2, dw2, three ? nullptr : db2, part2, B, Hi2, Wi2, 4 * nst2, c1, c2, c1, sms, s);
    if (rc != LPB_OK) return rc;
    size_t smem = 0;
    B2dParams p = b2d_params(G2, L2, wp2, G1, L1, Hi2, Wi2, c1, part_db1, &smem);
    LPB_REQUIRE(smem <= HEAD_STAGE_SMEM_BUDGET && p.R2 >= 1, "head_bwd_bf16: layer-2 width %d too large", Wi2);
    if (!wide) {
      LPB_TRY(set_dynamic_smem(b2d_dgrad_kernel<false>, smem, "head_bwd_bf16"));
      b2d_dgrad_kernel<false><<<grid, B2D_THREADS, smem, s>>>(p);
      reduce_partials<1>(part_db1, grid * 4, HEAD_CLS, c1, db1, sms, s);
    } else {
      // keypoint groups: the mid activations' gradient in fp32 planes, the c2 groups added in order per c1 group, then
      // written as G1 by the front end's writer (a dense gradient, no softmax) and the bias gradient from G1's columns
      LPB_TRY(set_dynamic_smem(b2d_dgrad_kernel<true>, smem, "head_bwd_bf16"));
      p.dmid = dmid;
      p.kc_frame = g2 * HEAD_KC;
      for (int t = 0; t < g1; ++t)
        for (int k = 0; k < g2; ++k) {
          p.wpk = wp2 + (size_t)(k * g1 + t) * 4 * HEAD_KC * 32 * 8;
          p.kc0 = k * HEAD_KC;
          p.o0 = t * HEAD_CLS;
          p.cg = c1 - p.o0 < HEAD_CLS ? c1 - p.o0 : HEAD_CLS;
          p.accumulate = k > 0;
          b2d_dgrad_kernel<true><<<grid, B2D_THREADS, smem, s>>>(p);
        }
      G2Src src{};
      src.g_out = dmid;
      launch_g2_build<true, false>(src, B, c1, Hi1, Wi1, G1, L1, s);
    }
  }
  if (!two || wide) {
    rows_colsum_kernel<<<(unsigned)(B * g1 * HEAD_KC), 256, 0, s>>>(G1, L1, part_cs);
    rows_colsum_reduce_kernel<<<(unsigned)c1, 256, 0, s>>>(part_cs, (long long)B * g1 * HEAD_KC * 8, g1 * HEAD_KC, db1);
  }
  // layer 1: weight gradient from the saved shuffled features, data gradient -> d features
  {
    const int nkc = C4 / 8;  // multiple of 4
    const int rc = launch_wgrad(static_cast<const __nv_bfloat16*>(saved_xs), G1, dw1, nullptr, part1, B, Hi1, Wi1, nkc, C4, c1, -1, sms, s);
    if (rc != LPB_OK) return rc;
  }
  if (dfeat) {
    B3aParams p;
    p.G1 = G1;
    p.L = L1;
    p.wpk = wp1;
    p.dfeat = static_cast<__nv_bfloat16*>(dfeat);
    p.B = B;
    p.C4 = C4;
    p.Hi = Hi1;
    p.Wi = Wi1;
    p.Hh = Hh;
    p.ncols = (Hh * (Wi1 + 1) + 15) & ~15;
    p.acc32 = acc32;
    p.kc_frame = g1 * HEAD_KC;
    p.acc_in = p.acc_out = p.kc0 = 0;
    size_t smem = b3a_operand_smem_bytes(Hi1, Wi1);
    LPB_REQUIRE(smem <= HEAD_BWD_SMEM_BUDGET, "head_bwd_bf16: layer-1 operands need %zu B shared memory", smem);
    // TMA tensor stores of d features when their staging slices (4 x 128 channels x 2 items x 4W bytes) still fit and the
    // tensor maps (boxes of one item and of an item pair) encode; otherwise direct stores (dfeat's alignment was checked
    // with the arguments)
    CUtensorMap tmap, tmap_pair;
    memset(&tmap, 0, sizeof(tmap));
    memset(&tmap_pair, 0, sizeof(tmap_pair));
    p.tma_store = 0;
    if (nhwc) {
      smem += b3a_nhwc_stage_bytes(W);
      LPB_REQUIRE(smem <= HEAD_BWD_SMEM_BUDGET, "head_bwd_bf16: the channels-last d-feature tile of width %d needs %zu B shared memory", W, smem);
    } else if (!acc32) {  // (the groups' fp32 sums take the direct stores)
      const size_t stage = (size_t)4 * 128 * 2 * 4 * W + 128;
      if (smem + stage <= HEAD_BWD_SMEM_BUDGET && make_dfeat_tensor_map(&tmap, dfeat, B, C4, H * W, 2 * W) &&
          make_dfeat_tensor_map(&tmap_pair, dfeat, B, C4, H * W, 4 * W)) {
        p.tma_store = 1;
        smem += stage;
      }
    }
    int slots = sms / ntile1;
    if (slots < 1) slots = 1;
    if (slots > B) slots = B;
    auto run = [&](auto kern, auto kern_acc) -> int {
      if (!acc32) {
        LPB_TRY(set_dynamic_smem(kern, smem, "head_bwd_bf16"));
        kern<<<slots * ntile1, B3A_THREADS, smem, s>>>(p, tmap, tmap_pair);
        return LPB_OK;
      }
      // keypoint groups of c1: one launch per group, in order, each adding its d features to the groups' fp32 sums
      LPB_TRY(set_dynamic_smem(kern_acc, smem, "head_bwd_bf16"));
      for (int g = 0; g < g1; ++g) {
        p.wpk = wp1 + (size_t)g * ntile1 * 4 * HEAD_KC * 128 * 8;
        p.kc0 = g * HEAD_KC;
        p.acc_in = g > 0;
        p.acc_out = g < g1 - 1;
        kern_acc<<<slots * ntile1, B3A_THREADS, smem, s>>>(p, tmap, tmap_pair);
      }
      return LPB_OK;
    };
    int rc = LPB_ERR_UNSUPPORTED;
    switch (W) {
#define LPB_B3A_CASE(WS2) \
  case WS2: \
    rc = nhwc ? run(b3a_dgrad_kernel<WS2, false, true>, b3a_dgrad_kernel<WS2, true, true>) : run(b3a_dgrad_kernel<WS2>, b3a_dgrad_kernel<WS2, true>); \
    break;
      LPB_B3A_CASE(4)
      LPB_B3A_CASE(8)
      LPB_B3A_CASE(12)
      LPB_B3A_CASE(16)
      LPB_B3A_CASE(24)
      LPB_B3A_CASE(32)
#undef LPB_B3A_CASE
      default: set_error("head_bwd_bf16: feature width %d not in this build's epilogue set", W);
    }
    if (rc != LPB_OK) return rc;
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_head_bwd_bf16_targets(const float* g_out, const lpb_mse_targets* mse, const float* probs, const float* win,
                                         const int32_t* win_meta, const float* g_overflow, const void* saved_xs,
                                         const void* fwd_workspace, int B, int C, int H, int W, const float* w1, int c1,
                                         const float* w2, int c2, int feature_layout, void* dfeat, float* dw1, float* db1,
                                         float* dw2, float* db2, void* workspace, void* stream) {
  return head_bwd(g_out, mse, probs, win, win_meta, g_overflow, saved_xs, fwd_workspace, B, C, H, W, w1, c1, w2, c2, feature_layout, dfeat,
                  dw1, db1, dw2, db2, workspace, stream);
}

// ---- three-deconv heads (lpb200.h) -----------------------------------------------------------------------------------
extern "C" int lpb_head3_query(int B, int C, int H, int W, int c1, int c2, int c3, int feature_layout, int train, lpb_head3_sizes* sizes) {
  using namespace lpb;
  LPB_REQUIRE(sizes, "head3_query: null pointer");
  LPB_REQUIRE(feature_layout == LPB_FEATURES_NCHW || feature_layout == LPB_FEATURES_NHWC, "head3_query: unknown feature layout %d", feature_layout);
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 1 && c3 >= 1, "head3_query: bad shape");
  memset(sizes, 0, sizeof(*sizes));
  const char* why = nullptr;
  if (!head3_covered(H, W, c1, c2, c3, train != 0, &why)) {
    set_error("head3_query: %dx%d features, channels %d/%d/%d: %s", H, W, c1, c2, c3, why);
    return LPB_ERR_UNSUPPORTED;
  }
  LPB_TRY(lpb_head_bf16_plan_layout(C, H, W, c1, c2, feature_layout, &sizes->plan));
  sizes->fwd_workspace = head_fwd_layout(B, C, H, W, c1, c2, c3).total;
  LPB_TRY(lpb_head_bf16_saved_bytes(B, C, H, W, &sizes->saved));
  if (train) {
    LPB_TRY(head_bwd_covers("head3_query", H, W, c1, c2, feature_layout));
    sizes->bwd_workspace = head_bwd_layout(B, C, H, W, c1, c2, false, c3).total;
    sizes->bwd_workspace_targets = head_bwd_layout(B, C, H, W, c1, c2, true, c3).total;
  }
  return LPB_OK;
}

extern "C" int lpb_head3_bwd(const float* g_out, const lpb_mse_targets* mse, const float* probs, const float* win, const int32_t* win_meta,
                             const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int feature_layout, int B, int C,
                             int H, int W, const float* w1, int c1, const float* w2, int c2, const float* w3, int c3, void* dfeat, float* dw1,
                             float* db1, float* dw2, float* db2, float* dw3, float* db3, void* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(w2 && w3 && dw2 && db2 && dw3 && db3, "head3_bwd: null pointer");
  LPB_REQUIRE(c1 >= 1 && c2 >= 1 && c3 >= 1, "head3_bwd: bad channel counts %d/%d/%d", c1, c2, c3);
  return head_bwd(g_out, mse, probs, win, win_meta, g_overflow, saved_xs, fwd_workspace, B, C, H, W, w1, c1, w2, c2, feature_layout, dfeat,
                  dw1, db1, dw2, db2, workspace, stream, w3, c3, dw3, db3);
}
