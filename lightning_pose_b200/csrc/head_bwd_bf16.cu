// Backward of the bf16 heatmap head on tensor-core (data gradients), mirroring head_bf16.cu.
// Reference: autograd of lightning_pose/models/heads/heatmap.py:203-212 (PixelShuffle + 2 x ConvTranspose2d).
//
// Gradients travel in the "class-major row layout"  G[b][kchunk = k/8][row = m*Wi + n][8] bf16  with
// k = cls*20 + o, cls = (py, px): row (m, n) carries, for every output class and channel, the gradient at
// output pixel (2m+py, 2n+px).  In this layout the data gradient of a stride-2 3x3 transposed convolution
//   d in[c, m', n'] = sum_{cls, (dm,dn) valid} G[(m'-dm, n'-dn)][(cls, o)] * W[c, o, ky, kx]
// is again a 4-shift GEMM (negative row shifts of the same smem operand, mma_sm90.cuh), K = 80:
//   b2d: G2 (48x48 rows)  x W2  -> d mid (48x48 x 17)  written straight into G1 (24x24 rows) for the next stage
//   b3a: W1 (M = 128 channels) x G1^T -> d Xs[c][row]   un-shuffled in the epilogue into d features (NCHW bf16)
#include <cuda_bf16.h>

#include <cstdint>

#include "../../include/lpb200.h"
#include "head_prep.cuh"
#include <cstring>
#include <cuda.h>  // CUtensorMap (the encoder is fetched through cudaGetDriverEntryPoint: no libcuda link)

#include "lpb_common.cuh"
#include "row_layout.cuh"
#include "mma_sm90.cuh"

namespace lpb {

constexpr int GB_CLS = 20;            // class stride in K
constexpr int GB_K = 4 * GB_CLS;      // 80
constexpr int GB_KC = GB_K / 8;       // 10 K-chunks

// ---- gradient front end: everything upstream of the second deconv's output, fused into the G2 writer --------
// The gradient w.r.t. the head output arrives as a sum of
//   g_out   dense [B, c2, Ho, Wo] fp32 (heatmap losses)                      -- optional
//   win     sparse 32x32 windows of the soft-argmax decode (decode.cu)        -- optional, flag 2 = dense plane in gov
// and, when the head ends in the spatial softmax, is pulled back through it on the fly:
//   g_logit = p * (g - dot),  dot = sum_plane(g * p) = ddot (dense part, plane_dot_kernel) + window dot (meta).
// Neither the dense decode gradient, nor its sum with g_out, nor g_logit ever exist in memory.
struct G2Src {
  const float* g_out;   // or null
  const float* probs;   // head output when it ends in softmax, else null
  const float* win;     // [planes][32*32] or null
  const int* meta;      // [planes][4] {row0, col0, flag, bits(dot)}
  const float* gov;     // dense fallback planes (flag 2)
  const float* ddot;    // [planes] dense part of the softmax dot (valid when probs && (g_out || win))
};

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
// Loads are issued as independent batches (probs, dense gradient) before any dependent work; the window
// look-ups are rare (a 32x32 patch of a 96x96 plane) and come last.
constexpr int G2B_THREADS = 128;

// HAS_WIN: the decode windows are staged per CTA into shared memory first (the CTA's 128 input-grid pixels span at
// most G2B_MROWS rows m, i.e. 2 * G2B_MROWS output rows; a window contributes 32 columns of each), so the main loop
// adds them with branch-free shared-memory reads instead of divergent global gathers.
constexpr int G2B_MROWS = 4;  // input-grid rows a CTA can touch: ceil(128 / Wi) + 1 for Wi >= 43 (host checks)

// HAS_OV (window-less pass ahead of the patch kernel): planes whose decode gradient is dense (flag 2, the decode's overflow
// buffer) are added here, in the streaming pass -- in the fresh-init regime that is every plane.
template <bool HAS_G, bool HAS_P, bool HAS_WIN, bool HAS_OV = false>
__global__ void __launch_bounds__(G2B_THREADS, 4) g2_build_kernel(G2Src S, int B, int C, int Hi, int Wi, int ctas_per_frame,
                                                               __nv_bfloat16* __restrict__ G, RowLayout L) {
  const int b = blockIdx.x / ctas_per_frame, t0 = (blockIdx.x - b * ctas_per_frame) * G2B_THREADS, t = t0 + threadIdx.x;
  const int Wo = 2 * Wi, Ho = 2 * Hi;
  __shared__ float sdot[GB_CLS];
  __shared__ int4 smeta[GB_CLS];
  __shared__ float wtile[HAS_WIN ? GB_CLS * 2 * G2B_MROWS * 32 : 1];
  __shared__ unsigned shit, sov;
  const int m0 = t0 / Wi;
  if (threadIdx.x < GB_CLS) {
    float d = 0.f;
    int4 mt = make_int4(0, 0, 0, 0);
    if (threadIdx.x < C) {
      const size_t plane = (size_t)b * C + threadIdx.x;
      if (S.meta) mt = reinterpret_cast<const int4*>(S.meta)[plane];
      if (HAS_P) {
        if (mt.z == 1) d = __int_as_float(mt.w);
        if (S.ddot) d += S.ddot[plane];
      }
    }
    sdot[threadIdx.x] = d;
    smeta[threadIdx.x] = mt;
    if (HAS_OV) {
      const unsigned bov = __ballot_sync((1u << GB_CLS) - 1, mt.z == 2);
      if (threadIdx.x == 0) sov = bov;
    }
    if (HAS_WIN) {
      // does this plane's window (or its dense fallback) touch the CTA's output rows [2 m0, 2 m0 + 2 MROWS)?  A 32x32
      // window covers a ninth of a 96x96 plane: most (CTA, plane) pairs skip the look-ups altogether (uniform branch)
      const bool hit = mt.z == 2 || (mt.z == 1 && mt.x < 2 * m0 + 2 * G2B_MROWS && mt.x + 32 > 2 * m0);
      const unsigned bal = __ballot_sync((1u << GB_CLS) - 1, hit);
      if (threadIdx.x == 0) shit = bal;
    }
  }
  if (HAS_WIN) {
    __syncthreads();
    // wtile[o][yl][lx] = win[o][2*m0 + yl - row0][lx] (0 outside the window / for planes without one)
    // one window row (32 floats) per warp and step, all steps unrolled: the predicated loads are independent
    const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
    constexpr int NROW = GB_CLS * 2 * G2B_MROWS, NSTEP = NROW / (G2B_THREADS / 32), NB = 10;  // NB loads in flight per thread
    static_assert(NSTEP % NB == 0, "window staging batches");
#pragma unroll 1
    for (int k0 = 0; k0 < NSTEP; k0 += NB) {
      float stage[NB];
#pragma unroll
      for (int k = 0; k < NB; ++k) {
        const int r = wq + (k0 + k) * (G2B_THREADS / 32), o = r / (2 * G2B_MROWS), yl = r - o * (2 * G2B_MROWS);
        float v = 0.f;
        if (o < C && ((shit >> o) & 1u)) {
          const int4 mt = smeta[o];
          const int ly = 2 * m0 + yl - mt.x;
          if (mt.z == 1 && (unsigned)ly < 32u) v = __ldg(S.win + ((size_t)b * C + o) * 1024 + ly * 32 + lane);
        }
        stage[k] = v;
      }
#pragma unroll
      for (int k = 0; k < NB; ++k) wtile[(wq + (k0 + k) * (G2B_THREADS / 32)) * 32 + lane] = stage[k];
    }
  }
  __syncthreads();
  if (t >= Hi * Wi) return;
  const int m = t / Wi, n = t - m * Wi;
#pragma unroll
  for (int py = 0; py < 2; ++py) {
    const int y = 2 * m + py, x = 2 * n;
    const size_t off0 = (((size_t)b * C) * Ho + y) * Wo + x;
    const size_t pstride = (size_t)Ho * Wo;
    float2 pv[GB_CLS], gv[GB_CLS];
#pragma unroll
    for (int o = 0; o < GB_CLS; ++o) {
      pv[o] = make_float2(0.f, 0.f);
      gv[o] = make_float2(0.f, 0.f);
      if (o < C) {
        if (HAS_P) pv[o] = __ldg(reinterpret_cast<const float2*>(S.probs + off0 + o * pstride));
        if (HAS_G) gv[o] = __ldg(reinterpret_cast<const float2*>(S.g_out + off0 + o * pstride));
      }
    }
    if (HAS_WIN) {
      const float* wrow = wtile + (2 * (m - m0) + py) * 32;
      const unsigned hits = shit;
#pragma unroll
      for (int o = 0; o < GB_CLS; ++o) {
        if (o < C && ((hits >> o) & 1u)) {
          const int4 mt = smeta[o];
          const int lx = x - mt.y;  // window column of output pixel x; x + 1 -> lx + 1
          const float w0 = wrow[o * (64 * G2B_MROWS) + min(max(lx, 0), 31)];
          const float w1 = wrow[o * (64 * G2B_MROWS) + min(max(lx + 1, 0), 31)];
          gv[o].x += (unsigned)lx < 32u ? w0 : 0.f;
          gv[o].y += (unsigned)(lx + 1) < 32u ? w1 : 0.f;
          if (mt.z == 2) {  // dense fallback plane (rare; uniform per CTA)
            const float2 u = __ldg(reinterpret_cast<const float2*>(S.gov + off0 + o * pstride));
            gv[o].x += u.x, gv[o].y += u.y;
          }
        }
      }
    }
    if (HAS_OV && sov) {  // uniform per frame
      const unsigned ovm = sov;
#pragma unroll
      for (int o = 0; o < GB_CLS; ++o) {
        if (o < C && ((ovm >> o) & 1u)) {
          const float2 u = __ldg(reinterpret_cast<const float2*>(S.gov + off0 + o * pstride));
          gv[o].x += u.x, gv[o].y += u.y;
        }
      }
    }
    if (HAS_P) {
#pragma unroll
      for (int o = 0; o < GB_CLS; ++o) {
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
        const float f0 = k0 < GB_CLS ? gv[k0].x : gv[k0 - GB_CLS].y;
        const float f1 = k1 < GB_CLS ? gv[k1].x : gv[k1 - GB_CLS].y;
        __nv_bfloat162 h2 = __floats2bfloat162_rn(f0, f1);
        pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(G + ((((size_t)b * GB_KC + 5 * py + ch) * L.rows) + L.lead + (size_t)m * L.Pp + n) * 8) =
          make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
  }
}

// Window patch: after a window-less g2_build pass (which already folds each window's dot into the softmax term and adds the
// dense-overflow planes), one warp per plane re-evaluates the <= 32 x 32 pixels under its window and overwrites those
// bf16 entries.  The streaming pass then runs at the DRAM roofline with no look-ups in it, and this pass touches 4 KB of
// probabilities per plane (a ninth of it).
// Window rows go eight at a time: 8 independent window loads, then 8 independent probability loads per lane.
template <bool HAS_G, bool HAS_P>
__global__ void __launch_bounds__(128) g2_patch_kernel(G2Src S, long long n_planes, int C, int Hi, int Wi,
                                                      __nv_bfloat16* __restrict__ G, RowLayout L) {
  const int lane = threadIdx.x & 31;
  const int Wo = 2 * Wi, Ho = 2 * Hi;
  {
    const long long plane = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
    int4 mt = make_int4(0, 0, 0, 0);
    if (plane < n_planes) mt = reinterpret_cast<const int4*>(S.meta)[plane];
    if (mt.z == 1) {
      const int b = (int)(plane / C), o = (int)(plane - (long long)b * C);
      float dot = 0.f;
      if (HAS_P) dot = __int_as_float(mt.w) + (S.ddot ? S.ddot[plane] : 0.f);
      const size_t poff = (size_t)plane * Ho * Wo;
      const float* wp = S.win + (size_t)plane * 1024 + lane;
      const int x = mt.y + lane;
      const bool xin = (unsigned)x < (unsigned)Wo;
      // k = cls * 20 + o with cls = 2 (y & 1) + (x & 1): the K-chunk / element of this lane for even and odd rows
      const int kx = (x & 1) * GB_CLS + o;
      __nv_bfloat16* gcol = G + ((size_t)b * GB_KC * L.rows + L.lead + (x >> 1)) * 8;
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
          go[k] = (HAS_G && ok) ? __ldg(S.g_out + poff + (size_t)y * Wo + x) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int y = mt.x + r0 + k;
          if (!(xin && gw[k] != 0.f && (unsigned)y < (unsigned)Ho)) continue;
          float g = gw[k] + go[k];
          if (HAS_P) g = pv[k] * (g - dot);
          const int kk = kx + 2 * GB_CLS * (y & 1);
          gcol[((size_t)(kk >> 3) * L.rows + (size_t)(y >> 1) * L.Pp) * 8 + (kk & 7)] = __float2bfloat16_rn(g);
        }
      }
    }
  }
}

template <bool HAS_G, bool HAS_P>
static void launch_g2_build(const G2Src& S, int B, int C, int Hi, int Wi, __nv_bfloat16* G, RowLayout L, cudaStream_t s) {
  const int cpf = (Hi * Wi + G2B_THREADS - 1) / G2B_THREADS;
  const bool fits = (G2B_THREADS + Wi - 1) / Wi + 1 <= G2B_MROWS;  // rows m a CTA's pixels can span
  if (S.win && fits && !g_tuning[LPB_TUNE_G2_PATCH]) {
    g2_build_kernel<HAS_G, HAS_P, true><<<(unsigned)(B * cpf), G2B_THREADS, 0, s>>>(S, B, C, Hi, Wi, cpf, G, L);
    return;
  }
  if (!S.win) {
    g2_build_kernel<HAS_G, HAS_P, false><<<(unsigned)(B * cpf), G2B_THREADS, 0, s>>>(S, B, C, Hi, Wi, cpf, G, L);
    return;
  }
  g2_build_kernel<HAS_G, HAS_P, false, true><<<(unsigned)(B * cpf), G2B_THREADS, 0, s>>>(S, B, C, Hi, Wi, cpf, G, L);
  {
    const long long np = (long long)B * C;
    g2_patch_kernel<HAS_G, HAS_P><<<(unsigned)((np + 3) / 4), 128, 0, s>>>(S, np, C, Hi, Wi, G, L);
  }
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
  float* db1_part;            // [gridDim.x * 4 MMA warps][GB_CLS]: each warp's bias-gradient sum (reduced in a fixed order)
  int B, Hi, Wi, c1;
  int R2;                     // image rows per chunk
};

__global__ void __launch_bounds__(B2D_THREADS, 2) b2d_dgrad_kernel(const __grid_constant__ B2dParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1;
  const int LEAD = Pp + 1;  // one zero row + the previous image row
  const int rows_alloc = (LEAD + B2D_TILES * 128 + 7) & ~7;
  const int a_bytes = GB_KC * rows_alloc * 16;
  const int w_bytes = 4 * GB_KC * 32 * 16;
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
        if (lane < GB_KC) {
          if (lane == 0) mbar_expect_tx(a_full, GB_KC * nbytes);
          __syncwarp((1u << GB_KC) - 1);
          bulk_g2s(As + (size_t)lane * rows_alloc * 16,
                   P.G2 + (((size_t)b * GB_KC + lane) * P.L2.rows + P.L2.lead + (size_t)(y0 - 1) * Pp - 1) * 8, nbytes, a_full);
        }
      }
    }
  } else if (warp >= 2) {
    const int q = warp & 3;
    const uint32_t lbo_a = rows_alloc * 16, lbo_b = 32 * 16;
    const uint32_t a0 = smem_u32(As), b0 = smem_u32(Ws);
    mbar_wait(w_full, 0);
    float dbs[GB_CLS];
#pragma unroll
    for (int o = 0; o < GB_CLS; ++o) dbs[o] = 0.f;
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
              for (int k16 = 0; k16 < GB_K / 16; ++k16) {
                if (k16 < sh) continue;  // all-zero weight chunks of this shift (see b3a)
                mma::kstep(acc, a0 + (2 * k16) * lbo_a + (LEAD + t * 128 + 32 * q - shift_rows) * 16, lbo_a, b0 + (sh * GB_KC + 2 * k16) * lbo_b,
                           lbo_b, lane);
              }
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) mma::rows8(acc, nt, &d[8 * nt], lane);
          }
          const int row = t * 128 + 32 * q + lane;
          const int ml = row / Pp, n = row - ml * Pp;
          if (ml < nrow && n < Wi) {
            const int y = y0 + ml;
            const int row1 = P.L1.lead + (y >> 1) * P.L1.Pp + (n >> 1);
            const int k0 = GB_CLS * (((y & 1) << 1) | (n & 1));
#pragma unroll
            for (int o = 0; o < GB_CLS; ++o)
              if (o < P.c1) dbs[o] += d[o];
#pragma unroll
            for (int i = 0; i < GB_CLS / 4; ++i) {
              uint32_t pk[2];
#pragma unroll
              for (int e2 = 0; e2 < 2; ++e2) {
                const int c0 = 4 * i + 2 * e2;
                __nv_bfloat162 h2 = __floats2bfloat162_rn(c0 < P.c1 ? d[c0] : 0.f, c0 + 1 < P.c1 ? d[c0 + 1] : 0.f);
                pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
              }
              const int k = k0 + 4 * i;
              *reinterpret_cast<uint2*>(P.G1 + (((size_t)b * GB_KC + (k >> 3)) * P.L1.rows + row1) * 8 + (k & 7)) = make_uint2(pk[0], pk[1]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(a_empty);
      }
    }
    float* part = P.db1_part + ((size_t)blockIdx.x * 4 + q) * GB_CLS;
#pragma unroll
    for (int o = 0; o < GB_CLS; ++o) {
      const float s = warp_sum(dbs[o]);
      if (lane == 0) part[o] = s;
    }
  }
}

// =====================================================================================================
// b3a: data gradient of the first deconv + inverse PixelShuffle:  G1 -> d features (NCHW bf16)
// =====================================================================================================
constexpr int B3A_THREADS = 320;  // warp 0 loader, warp 1 idle, warps 2-9 MMA + epilogue (lane = channel, two warps per 32-channel quarter)

struct B3aParams {
  const __nv_bfloat16* G1;   // [B][10][L.rows][8] padded row layout
  RowLayout L;
  const __nv_bfloat16* wpk;  // [ceil(C4/128)][4][10][128][8]
  __nv_bfloat16* dfeat;      // [B][4*C4][(Hi/2)*(Wi/2)]
  int B, C4, Hi, Wi;         // shuffled-image geometry (Hi = 2H, Wi = 2W)
  int Hh;                    // image rows per band (multiple of 4)
  int ncols;                 // accumulator columns per band = Hh * (Wi + 1) rounded up to 16 (<= 304)
  int backoff, prefetch;
  int tma_store;             // 1: the epilogue stages bf16 rows in shared memory and a TMA tensor store writes them (below)
};

// TMA tensor store of d features.  The tensor map views the NCHW gradient as [b][c'][pl][px] (source plane 4c' + pl,
// px = H*W pixels); a box is {2 feature rows, one pl, 128 c', one frame}: in shared memory 128 rows of 4*WS2 bytes, so
// thread c' writes at a 4*WS2-byte stride (conflict-free for WS2 = 12) and the copy engine does the 1152-byte-strided
// scatter that cost the epilogue 32 half-used sectors per store instruction.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* tm, const void* smem_src, int x0, int x1, int x2, int x3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tm), "r"(smem_u32(smem_src)), "r"(x0),
               "r"(x1), "r"(x2), "r"(x3)
               : "memory");
}
__device__ __forceinline__ void bulk_wait_group_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// A frame is processed in bands of Hh image rows (N = Hh * (Wi + 1) accumulator columns per band; the band's gradient
// rows plus the halo row above are double-buffered in shared memory).
template <int WS2>
__global__ void __launch_bounds__(B3A_THREADS, 1) b3a_dgrad_kernel(const __grid_constant__ B3aParams P, const __grid_constant__ CUtensorMap TM) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1, LEAD = Pp + 1;
  const int Hh = P.Hh, nbands = (Hi + Hh - 1) / Hh;
  const int rows_alloc = (LEAD + P.ncols + 7) & ~7;
  const int g_bytes = GB_KC * rows_alloc * 16;
  const int w_bytes = 4 * GB_KC * 128 * 16;
  unsigned char* Gs = smem;                 // [2 stages][10][rows_alloc][16 B]
  unsigned char* Ws = smem + 2 * g_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Ws + w_bytes);
  uint64_t* g_full = bars;       // [2]
  uint64_t* g_empty = bars + 2;  // [2]
  uint64_t* w_full = bars + 4;
  // staging slices of the TMA store: [ip & 1][pl][128 lanes][4 * WS2 bytes]
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

  if (warp == 0) {
    if (lane == 0) {
      mbar_expect_tx(w_full, (uint32_t)w_bytes);
      bulk_g2s(Ws, reinterpret_cast<const unsigned char*>(P.wpk) + (size_t)mt * w_bytes, (uint32_t)w_bytes, w_full);
    }
    int it = 0;
    for (int b = slot; b < P.B; b += nslot)
      for (int band = 0; band < nbands; ++band, ++it) {
        const int st = it & 1, y0 = band * Hh, hb = min(Hh, Hi - y0);
        mbar_wait(&g_empty[st], ((it >> 1) & 1) ^ 1);
        // one copy per K-chunk: the zero entry before image row y0 - 1, that row (zero lead rows of the layout when
        // y0 = 0), and the band's rows, zero columns included
        const uint32_t nbytes = (uint32_t)((1 + (hb + 1) * Pp) * 16);
        if (lane < GB_KC) {
          if (lane == 0) mbar_expect_tx(&g_full[st], GB_KC * nbytes);
          __syncwarp((1u << GB_KC) - 1);
          bulk_g2s(Gs + (size_t)st * g_bytes + (size_t)lane * rows_alloc * 16,
                   P.G1 + (((size_t)b * GB_KC + lane) * P.L.rows + P.L.lead + (size_t)(y0 - 1) * Pp - 1) * 8, nbytes, &g_full[st]);
        }
      }
  } else if (warp >= 2) {
    // MMA + epilogue.  The band's whole K (4 shifts x 80) is resident, so a warp computes each 16-pixel block of its 32
    // channels (accumulator rows) when the epilogue needs it.  Thread = shuffled channel c (accumulator row); shuffled pixel (m, n) = (2i + di, 2j + dj) belongs to source
    // plane 4c + 2di + dj.  A work item is (di, pair of feature rows i, i+1): two accumulator rows m = 2i + di and m + 2,
    // i.e. 2 * WS2 consecutive elements of each of the planes dj = 0, 1 -> aligned 16-byte stores.  The two warps of a
    // lane quarter take alternate items.
    const int q = warp & 3, e = (warp - 2) >> 2;
    const int c = mt * 128 + 32 * q + lane;
    const int HW = (Hi / 2) * WS2;
    constexpr int NCH = (2 * WS2 + 15) / 16;  // 16-column blocks per accumulator row
    const uint32_t lbo_g = rows_alloc * 16, lbo_w = 128 * 16;
    const uint32_t w0 = smem_u32(Ws);
    mbar_wait(w_full, 0);
    int it = 0, tma_cnt = 0;
    for (int b = slot; b < P.B; b += nslot)
      for (int band = 0; band < nbands; ++band, ++it) {
        const int st = it & 1, y0 = band * Hh, hb = min(Hh, Hi - y0);
        const int npairs = hb / 4;  // feature-row pairs in this band
        mbar_wait_idle(&g_full[st], (it >> 1) & 1, P.backoff);
        const uint32_t g0 = smem_u32(Gs + (size_t)st * g_bytes);
        auto issue = [&](int item, float (&buf)[2][NCH * 16]) {
          const int ml = 4 * (item >> 1) + (item & 1);  // first accumulator row of the item within this band
#pragma unroll
          for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int k = 0; k < NCH; ++k) {
              const int col0 = (ml + 2 * r) * Pp + 16 * k;  // first accumulator column (band pixel) of the block
              float acc[2][2][4];
              mma::zero(acc);
#pragma unroll
              for (int sh = 0; sh < 4; ++sh) {
                const int shift_rows = (sh >> 1) * Pp + (sh & 1);
#pragma unroll
                for (int k16 = 0; k16 < GB_K / 16; ++k16) {
                  // K = (cls, o), cls = 2 py + px at stride 20: shift (dm, dn) has no tap for classes with py < dm or px < dn,
                  // so its packed weights are zero for k < 20 (dn), k < 40 (dm), k < 60 (both): the 16-wide chunks k16 < sh
                  // are all-zero and skipped (14 of 20 remain)
                  if (k16 < sh) continue;
                  mma::kstep(acc, w0 + ((sh * GB_KC + 2 * k16) * 128 + 32 * q) * 16, lbo_w,
                             g0 + (2 * k16) * lbo_g + (LEAD - shift_rows + col0) * 16, lbo_g, lane);
                }
              }
              mma::rows8(acc, 0, &buf[r][16 * k], lane);
              mma::rows8(acc, 1, &buf[r][16 * k + 8], lane);
            }
        };
        auto emit = [&](int item, const float (&v)[2][NCH * 16]) {
          if (c >= P.C4) return;
          const int di = item & 1, ip = item >> 1;
          const int i0 = y0 / 2 + 2 * ip;  // first feature row of the pair
#pragma unroll
          for (int dj = 0; dj < 2; ++dj) {
            __nv_bfloat16* dst = P.dfeat + ((size_t)b * 4 * P.C4 + 4 * c + 2 * di + dj) * HW + (size_t)i0 * WS2;
#pragma unroll
            for (int s4 = 0; s4 < (2 * WS2) / 8; ++s4) {  // 8 consecutive elements of [row r][j]
              uint32_t pk[4];
#pragma unroll
              for (int e2 = 0; e2 < 4; ++e2) {
                const int x0 = 8 * s4 + 2 * e2, x1 = x0 + 1;  // index into the 2*WS2 run
                const float f0 = v[x0 / WS2][2 * (x0 % WS2) + dj];
                const float f1 = v[x1 / WS2][2 * (x1 % WS2) + dj];
                __nv_bfloat162 h2 = __floats2bfloat162_rn(f0, f1);
                pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
              }
              *reinterpret_cast<uint4*>(dst + 8 * s4) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
          }
        };
        const int nitems = 2 * npairs;
        if (P.tma_store) {
          // warps with the same e (= di) form a group of 128 lanes that owns the slices pl = 2e, 2e + 1; per item:
          //   the group's issuer makes sure the copy that last read these slices is done, the group writes its
          //   2 x (2 * WS2 / 8) 16-byte pieces per lane, and the issuer launches one tensor store per plane class
          constexpr int PB = 4 * WS2, SLICE = 128 * PB;  // bytes per lane and slice / per slice
          const bool issuer = (q == 0 && lane == 0);
          float va[2][NCH * 16];
          for (int item = e; item < nitems; item += 2, ++tma_cnt) {
            issue(item, va);
            const int ip = item >> 1, par = tma_cnt & 1;  // the group's slices alternate item by item
            unsigned char* sl = Ss + (size_t)(par * 4 + 2 * e) * SLICE + (size_t)(32 * q + lane) * PB;
            if (issuer) bulk_wait_group_read1();  // at most the previous item's stores (the other ip parity) still read smem
            named_bar_sync(1 + e, 128);
#pragma unroll
            for (int dj = 0; dj < 2; ++dj) {
#pragma unroll
              for (int s4 = 0; s4 < (2 * WS2) / 8; ++s4) {
                uint32_t pk[4];
#pragma unroll
                for (int e2 = 0; e2 < 4; ++e2) {
                  const int x0 = 8 * s4 + 2 * e2, x1 = x0 + 1;
                  __nv_bfloat162 h2 = __floats2bfloat162_rn(va[x0 / WS2][2 * (x0 % WS2) + dj], va[x1 / WS2][2 * (x1 % WS2) + dj]);
                  pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
                }
                *reinterpret_cast<uint4*>(sl + dj * SLICE + 16 * s4) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
              }
            }
            fence_proxy_async();
            named_bar_sync(1 + e, 128);
            if (issuer) {
              const int px0 = (y0 / 2 + 2 * ip) * WS2;
              tma_store_4d(&TM, Ss + (size_t)(par * 4 + 2 * e) * SLICE, px0, 2 * e, mt * 128, b);
              tma_store_4d(&TM, Ss + (size_t)(par * 4 + 2 * e + 1) * SLICE, px0, 2 * e + 1, mt * 128, b);
              bulk_commit_group();
            }
          }
        } else if (NCH <= 2 && P.prefetch) {
          // the next item's blocks are computed before the current item is converted and stored
          float va[2][NCH * 16], vb[2][NCH * 16];
          if (e < nitems) issue(e, va);
          for (int item = e; item < nitems; item += 4) {
            if (item + 2 < nitems) issue(item + 2, vb);
            emit(item, va);
            if (item + 2 < nitems) {
              if (item + 4 < nitems) issue(item + 4, va);
              emit(item + 2, vb);
            }
          }
        } else {
          for (int item = e; item < nitems; item += 2) {
            float v[2][NCH * 16];
            issue(item, v);
            emit(item, v);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&g_empty[st]);  // this warp's reads of the band are done
      }
    if (P.tma_store && q == 0 && lane == 0) bulk_wait_group0();  // the stores have landed before the kernel ends
  }
}


// =====================================================================================================
// wg: weight gradient of a stride-2 3x3 transposed convolution (both layers)
// =====================================================================================================
//   dW[c, o, ky, kx] = sum_{frames, rows} X[row + shift][c] * G[row][(cls, o)]      ((cls, shift) -> tap)
// a GEMM whose K dimension is the pixel raster.  Both operands are the row layout read TRANSPOSED (ldmatrix .trans,
// mma_sm90.cuh kstep_mn / umma_selftest.cu mode 1): A = G (M = the 80 (cls, o) rows), B = X at a row offset (the
// shift), N = this CTA's channel group.  MMA warp w owns shift w % 4 and half w / 4 of the channel group; its
// accumulators D_sh[k][c] stay in registers across every (frame, row-chunk) unit of the CTA, and one epilogue at the
// end adds them into dW with atomics.  An all-ones input channel (the bias lane of the mid activations) yields the bias
// gradient from the same GEMM.
constexpr int WG_THREADS = 288;  // warp 0 loader, warps 1-8 MMA + epilogue

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
  int smem_bytes;
};

// The gradients are summed over the CTAs in a fixed order (per-CTA partials, then reduce_partials_kernel), so that a
// backward pass gives bit-identical results from run to run.
constexpr int WG_MAX_CTAS = 132;   // weight-gradient CTAs per layer (one per SM of an H100 SXM; fewer on smaller devices)
constexpr int B2D_MAX_CTAS = 264;  // b2d CTAs (two per SM)
__host__ __device__ inline size_t wgrad_part_stride(int Cin, int Cout) { return (size_t)Cin * Cout * 9 + 4 * (size_t)Cout; }
// weight-gradient channel group (K-chunks of 8 channels per CTA) of a layer with nkc K-chunks of input
inline int wgrad_kcx(int nkc) { return nkc % 8 == 0 ? 8 : 4; }
inline int wgrad_max_slots(int nkc) {
  const int slots = WG_MAX_CTAS / (nkc / wgrad_kcx(nkc));
  return slots < 1 ? 1 : slots;
}

// out[i] = sum_{p < nparts} sum_{j < nsub} part[p * stride + j * n + i], in that order (i < n)
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ part, int nparts, size_t stride, int nsub, int n,
                                                              float* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p)
      for (int j = 0; j < nsub; ++j) s += part[(size_t)p * stride + (size_t)j * n + i];
    out[i] = s;
  }
}
static void reduce_partials(const float* part, int nparts, size_t stride, int nsub, int n, float* out, cudaStream_t s) {
  int blocks = (n + 255) / 256;
  if (blocks > 4 * WG_MAX_CTAS) blocks = 4 * WG_MAX_CTAS;
  reduce_partials_kernel<<<blocks, 256, 0, s>>>(part, nparts, stride, nsub, n, out);
}

// NT = n8 tiles per warp = kcx / 2
template <int NT>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_kernel(const __grid_constant__ WgParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Wi = P.Wi, Hi = P.Hi, Pp = Wi + 1, R = P.R, KR = P.KR, XR = P.XR;
  const int g_bytes = GB_KC * KR * 16, x_bytes = P.kcx * XR * 16;
  unsigned char* Gs = smem;
  unsigned char* Xs = smem + 2 * g_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P.smem_bytes - 64);
  uint64_t* full = bars;       // [2]
  uint64_t* empty = bars + 2;  // [2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = P.kcx * 8;
  const int ngroups = P.kcx_total / P.kcx;  // kcx_total may include K-chunks beyond the last group (ignored)
  const int grp = blockIdx.x % ngroups, slot = blockIdx.x / ngroups, nslot = gridDim.x / ngroups;
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
      if (lane == 0) mbar_expect_tx(&full[s], GB_KC * gbytes + P.kcx * xbytes);
      __syncwarp();
      const size_t row0 = (size_t)P.L.lead + (size_t)y0 * Pp;
      if (lane < GB_KC)
        bulk_g2s(Gs + (size_t)s * g_bytes + (size_t)lane * KR * 16, P.G + (((size_t)b * GB_KC + lane) * P.L.rows + row0) * 8, gbytes, &full[s]);
      if (lane < P.kcx)
        bulk_g2s(Xs + (size_t)s * x_bytes + (size_t)lane * XR * 16,
                 P.X + (((size_t)b * P.kcx_total + (size_t)grp * P.kcx + lane) * P.L.rows + row0) * 8, xbytes, &full[s]);
    }
  } else if (slot < nunits) {
    const int cw = warp - 1, sh = cw & 3, half = cw >> 2;
    const int dm = sh >> 1, dn = sh & 1, shift_rows = dm * Pp + dn;
    const uint32_t g0 = smem_u32(Gs), x0 = smem_u32(Xs) + (uint32_t)(half * NT) * XR * 16;  // n8 tile = one K-chunk of X
    float acc[GB_K / 16][NT][4];
    mma::zero(acc);
    int j = 0;
    for (int u = slot; u < nunits; u += nslot, ++j) {
      const int s = j & 1;
      mbar_wait(&full[s], (j >> 1) & 1);
      for (int k16 = 0; k16 < KR / 16; ++k16)
        mma::kstep_mn(acc, g0 + s * g_bytes + k16 * 256, KR * 16, x0 + s * x_bytes + (k16 * 16 + shift_rows) * 16, XR * 16, lane);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // accumulator (k = 16 mt + g (+8), c = 8 nt + 2 t (+1)) of shift sh -> this slot's partial of dW[c][o][ky][kx]
    float* part = P.part + (size_t)slot * wgrad_part_stride(P.Cin, P.Cout);
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int mt = 0; mt < GB_K / 16; ++mt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int k = 16 * mt + gq + 8 * (i >> 1);
        const int cls = k / GB_CLS, o = k - cls * GB_CLS, py = cls >> 1, px = cls & 1;
        if (o >= P.Cout || (py == 0 && dm == 1) || (px == 0 && dn == 1)) continue;
        const int ky = py == 0 ? 1 : (dm ? 0 : 2), kx = px == 0 ? 1 : (dn ? 0 : 2);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const int c = grp * N + (half * NT + nt) * 8 + 2 * tq + (i & 1);
          const float v = acc[mt][nt][i];
          // (cls, shift) -> tap is one-to-one, so every element of the slot's partial has exactly one writer
          if (c < P.Cin) part[((size_t)c * P.Cout + o) * 9 + ky * 3 + kx] = v;
          else if (P.has_bias && c == P.ones_c && sh == 0) part[(size_t)P.Cin * P.Cout * 9 + cls * P.Cout + o] = v;
        }
      }
  }
}

static int launch_wgrad(const __nv_bfloat16* X, const __nv_bfloat16* G, float* dW, float* dbias, float* part, int B, int Hi, int Wi,
                        int kcx_total, int Cin, int Cout, int ones_c, int sms, cudaStream_t s) {
  const int kcx = wgrad_kcx(kcx_total);
  // image rows per unit: the largest divisor of Hi (<= 8) whose two stages fit in shared memory
  int R = 0;
  for (int r = Hi < 8 ? Hi : 8; r >= 1; --r) {
    if (Hi % r) continue;
    const int kr = (r * (Wi + 1) + 15) & ~15, xr = (kr + Wi + 2 + 7) & ~7;
    if ((size_t)2 * GB_KC * kr * 16 + (size_t)2 * kcx * xr * 16 + 64 <= 225 * 1024) {
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
  const size_t body = ((size_t)2 * GB_KC * p.KR * 16 + (size_t)2 * kcx * p.XR * 16 + 15) & ~(size_t)15;
  p.smem_bytes = (int)(body + 64);
  LPB_REQUIRE(p.smem_bytes <= 225 * 1024, "head_bwd_bf16: weight-gradient stages need %d B shared memory", p.smem_bytes);
  const int ngroups = kcx_total / kcx;
  const int nunits = B * (Hi / R);
  int slots = sms / ngroups;
  if (slots > wgrad_max_slots(kcx_total)) slots = wgrad_max_slots(kcx_total);  // the partials' workspace
  if (slots < 1) slots = 1;
  if (slots > nunits) slots = nunits;
  auto kern = kcx == 8 ? wgrad_kernel<4> : wgrad_kernel<2>;
  LPB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, p.smem_bytes));
  kern<<<slots * ngroups, WG_THREADS, p.smem_bytes, s>>>(p);
  const size_t stride = wgrad_part_stride(Cin, Cout);
  reduce_partials(part, slots, stride, 1, Cin * Cout * 9, dW, s);
  if (dbias) reduce_partials(part + (size_t)Cin * Cout * 9, slots, stride, 4, Cout, dbias, s);
  return LPB_OK;
}


// bias gradient of a one-deconv head: column sums of the gradient rows, folded over the four classes
__global__ void __launch_bounds__(256) rows_colsum_kernel(const __nv_bfloat16* __restrict__ G, RowLayout L, int B, int cout,
                                                          float* __restrict__ db) {
  // one CTA per (frame, K-chunk): thread = (row stripe, e)
  const int b = blockIdx.x / GB_KC, kc = blockIdx.x - b * GB_KC;
  const __nv_bfloat16* slab = G + ((size_t)b * GB_KC + kc) * (size_t)L.rows * 8;
  const int e = threadIdx.x & 7;
  float acc = 0.f;
  for (int r = L.lead + (threadIdx.x >> 3); r < L.lead + L.Hi * L.Pp; r += 32) acc += __bfloat162float(slab[(size_t)r * 8 + e]);
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float t = 0.f;
    for (int i = threadIdx.x; i < 256; i += 8) t += red[i];
    const int k = kc * 8 + threadIdx.x, o = k % GB_CLS;
    if (o < cout && t != 0.f) atomicAdd(db + o, t);
  }
}

// largest rows-per-band Hh (multiple of 4) whose band fits the b3a shared-memory stages
static int b3a_band_rows(int Hi1, int Wi1) {
  int hh = (256 / (Wi1 + 1)) & ~3;  // two accumulator buffers fit
  if (hh < 4) hh = (304 / (Wi1 + 1)) & ~3;  // wide maps: one buffer
  if (hh > Hi1) hh = Hi1;
  return hh;
}

// d features [B][4*C4][HW] bf16 viewed as [b][c'][pl][px]; box = {box_px pixels, one pl, 128 c', one frame}.
// The encoder is a driver entry point; it is looked up once (no link-time dependency on libcuda).
static bool make_dfeat_tensor_map(CUtensorMap* tm, void* dfeat, int B, int C4, int HW, int box_px) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  static bool looked_up = false;
  if (!looked_up) {
    looked_up = true;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      encode = reinterpret_cast<EncodeFn>(fn);
    (void)cudaGetLastError();
  }
  if (!encode || (HW * 2) % 16 != 0 || (box_px * 2) % 16 != 0 || box_px > 256) return false;
  const cuuint64_t gdim[4] = {(cuuint64_t)HW, 4, (cuuint64_t)C4, (cuuint64_t)B};
  const cuuint64_t gstride[3] = {(cuuint64_t)HW * 2, (cuuint64_t)HW * 2 * 4, (cuuint64_t)HW * 2 * 4 * (cuuint64_t)C4};  // bytes, dims 1..3
  const cuuint32_t box[4] = {(cuuint32_t)box_px, 1, 128, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  return encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, dfeat, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace lpb

// workspace: [W1 dgrad pack][W2 dgrad pack][G2][G1][plane dots]   (G2 / G1: padded row layouts, row_layout.cuh);
// a one-deconv head (c2 = 0) has no W2 pack and no G2: its output gradient is G1 directly
// fixed-order reduction partials: [layer-1 wgrad][layer-2 wgrad][b2d bias]
static size_t bwd_partials_bytes(int C, int c1, int c2) {
  using namespace lpb;
  const int nkc1 = C / 4 / 8;
  size_t n = (size_t)wgrad_max_slots(nkc1) * wgrad_part_stride(C / 4, c1);
  if (c2 > 0) n += (size_t)wgrad_max_slots(4) * wgrad_part_stride(c1, c2) + (size_t)B2D_MAX_CTAS * 4 * GB_CLS;
  return n * sizeof(float);
}

extern "C" int lpb_head_bwd_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "head_bwd_bf16_workspace_bytes: null pointer");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 0, "head_bwd_bf16_workspace_bytes: bad shape");
  const int C4 = C / 4;
  const size_t w1 = (size_t)((C4 + 127) / 128) * 4 * GB_KC * 128 * 16, w2 = (size_t)4 * GB_KC * 32 * 16;
  const size_t g2 = c2 > 0 ? (size_t)B * GB_KC * make_row_layout(4 * H, 4 * W).rows * 16 : 0;
  const size_t g1 = (size_t)B * GB_KC * make_row_layout(2 * H, 2 * W).rows * 16;
  *bytes = w1 + w2 + g2 + g1 + (((size_t)B * (c2 > 0 ? c2 : c1) * 4 + 255) & ~(size_t)255) + bwd_partials_bytes(C, c1, c2);
  return LPB_OK;
}

extern "C" int lpb_head_bwd_bf16(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                                 const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H,
                                 int W, const float* w1, int c1, const float* w2, int c2, void* dfeat, float* dw1, float* db1,
                                 float* dw2, float* db2, void* workspace, void* stream) {
  using namespace lpb;
  const bool two = c2 > 0;
  LPB_REQUIRE(saved_xs && fwd_workspace && w1 && dw1 && db1 && workspace, "head_bwd_bf16: null pointer");
  LPB_REQUIRE(!two || (w2 && dw2 && db2), "head_bwd_bf16: a two-deconv head needs w2, dw2, db2");
  LPB_REQUIRE(g_out || win, "head_bwd_bf16: neither a dense gradient nor decode windows given");
  LPB_REQUIRE(!win || (win_meta && g_overflow), "head_bwd_bf16: windows need their meta and overflow buffers");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1, "head_bwd_bf16: bad feature shape C=%d H=%d W=%d", C, H, W);
  LPB_REQUIRE(two ? (c1 >= 1 && c1 < GB_CLS && c2 <= GB_CLS) : (c1 >= 1 && c1 <= GB_CLS), "head_bwd_bf16: channel counts %d/%d exceed %d", c1, c2, GB_CLS);
  if ((W % 4) != 0 || (H % 2) != 0 || !(W == 4 || W == 8 || W == 12 || W == 16 || W == 24 || W == 32)) {
    set_error("head_bwd_bf16: feature map %dx%d outside this build's epilogue set (H even, W in {4, 8, 12, 16, 24, 32})", H, W);
    return LPB_ERR_UNSUPPORTED;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int C4 = C / 4, Hi1 = 2 * H, Wi1 = 2 * W, Hi2 = 4 * H, Wi2 = 4 * W;
  const int kout = two ? c2 : c1;
  if (B == 0) {
    LPB_CUDA(cudaMemsetAsync(dw1, 0, sizeof(float) * (size_t)C4 * c1 * 9, s));
    LPB_CUDA(cudaMemsetAsync(db1, 0, sizeof(float) * c1, s));
    if (two) {
      LPB_CUDA(cudaMemsetAsync(dw2, 0, sizeof(float) * (size_t)c1 * c2 * 9, s));
      LPB_CUDA(cudaMemsetAsync(db2, 0, sizeof(float) * c2, s));
    }
    return LPB_OK;
  }
  const int Hh = b3a_band_rows(Hi1, Wi1);
  if (Hh < 4) {
    set_error("head_bwd_bf16: feature map %dx%d outside this build's band tiling", H, W);
    return LPB_ERR_UNSUPPORTED;
  }
  int dev = 0, sms = 0;
  LPB_CUDA(cudaGetDevice(&dev));
  LPB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const RowLayout L2 = make_row_layout(Hi2, Wi2), L1 = make_row_layout(Hi1, Wi1);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const int ntile1 = (C4 + 127) / 128;
  const size_t w1b = (size_t)ntile1 * 4 * GB_KC * 128 * 16, w2b = (size_t)4 * GB_KC * 32 * 16;
  const size_t g2b = two ? (size_t)B * GB_KC * L2.rows * 16 : 0, g1b = (size_t)B * GB_KC * L1.rows * 16;
  __nv_bfloat16* wp1 = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* wp2 = reinterpret_cast<__nv_bfloat16*>(ws + w1b);
  __nv_bfloat16* G2 = reinterpret_cast<__nv_bfloat16*>(ws + w1b + w2b);
  __nv_bfloat16* G1 = reinterpret_cast<__nv_bfloat16*>(ws + w1b + w2b + g2b);
  float* ddot = reinterpret_cast<float*>(ws + w1b + w2b + g2b + g1b);
  float* part1 = reinterpret_cast<float*>(ws + w1b + w2b + g2b + g1b + ((((size_t)B * kout * 4) + 255) & ~(size_t)255));
  float* part2 = part1 + (size_t)wgrad_max_slots(C4 / 8) * wgrad_part_stride(C4, c1);
  float* part_db1 = two ? part2 + (size_t)wgrad_max_slots(4) * wgrad_part_stride(c1, c2) : nullptr;
  // the forward pass's mid activations (head_bf16.cu workspace layout: [packed w1][packed w2][mid])
  const size_t fwd_mid_off = (size_t)(C4 / 32 + 1) * (4 * 4 * 80 * 16);
  const __nv_bfloat16* mid = reinterpret_cast<const __nv_bfloat16*>(static_cast<const unsigned char*>(fwd_workspace) + fwd_mid_off);

  {
    // one launch: gradient accumulators zeroed, both data-gradient operand packs, pad rows of G2 / G1
    PrepJobs jobs{};
    jobs.dpack[0] = {w1, C4, c1, ntile1, 128, wp1};
    jobs.pads[0] = {G1, L1, (long long)B * GB_KC};
    jobs.zero[0] = {dw1, (long long)C4 * c1 * 9};
    jobs.zero[1] = {db1, (long long)c1};
    if (two) {
      jobs.dpack[1] = {w2, c1, c2, 1, 32, wp2};
      jobs.pads[1] = {G2, L2, (long long)B * GB_KC};
      jobs.zero[2] = {dw2, (long long)c1 * c2 * 9};
      jobs.zero[3] = {db2, (long long)c2};
    }
    launch_head_prep(jobs, s);
  }
  {
    // gradient front end on the head's OUTPUT grid: G2 for a two-deconv head, G1 for a one-deconv head
    const int Hio = two ? Hi2 : Hi1, Wio = two ? Wi2 : Wi1;
    __nv_bfloat16* Gout = two ? G2 : G1;
    const RowLayout Lo = two ? L2 : L1;
    G2Src src;
    src.g_out = g_out;
    src.probs = probs;
    src.win = win;
    src.meta = win ? win_meta : nullptr;
    src.gov = g_overflow;
    src.ddot = nullptr;
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
  if (two) {
    // layer 2: weight + bias gradient (bias from the all-ones channel c1 of mid), then data gradient -> G1 (+ db1)
    const int rc = launch_wgrad(mid, G2, dw2, db2, part2, B, Hi2, Wi2, 4, c1, c2, c1, sms, s);
    if (rc != LPB_OK) return rc;
    B2dParams p;
    p.G2 = G2;
    p.wpk = wp2;
    p.G1 = G1;
    p.L2 = L2;
    p.L1 = L1;
    p.db1_part = part_db1;
    p.B = B;
    p.Hi = Hi2;
    p.Wi = Wi2;
    p.c1 = c1;
    p.R2 = (B2D_TILES * 128) / (Wi2 + 1);
    if (p.R2 > Hi2) p.R2 = Hi2;
    const int rows_alloc = (Wi2 + 2 + B2D_TILES * 128 + 7) & ~7;
    const size_t smem = (size_t)GB_KC * rows_alloc * 16 + (size_t)4 * GB_KC * 32 * 16 + 64;
    LPB_REQUIRE(smem <= 113 * 1024 && p.R2 >= 1, "head_bwd_bf16: layer-2 width %d too large", Wi2);
    LPB_CUDA(cudaFuncSetAttribute(b2d_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = B < 2 * sms ? B : 2 * sms;
    if (grid > B2D_MAX_CTAS) grid = B2D_MAX_CTAS;  // the bias partials' workspace
    b2d_dgrad_kernel<<<grid, B2D_THREADS, smem, s>>>(p);
    reduce_partials(part_db1, grid * 4, GB_CLS, 1, c1, db1, s);
  } else {
    rows_colsum_kernel<<<(unsigned)(B * GB_KC), 256, 0, s>>>(G1, L1, B, c1, db1);
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
    p.backoff = g_tuning[LPB_TUNE_WAIT_BACKOFF];
    p.prefetch = g_tuning[LPB_TUNE_B3A_PREFETCH];
    const int rows_alloc = (Wi1 + 2 + p.ncols + 7) & ~7;
    size_t smem = (size_t)2 * GB_KC * rows_alloc * 16 + (size_t)4 * GB_KC * 128 * 16 + 160;
    LPB_REQUIRE(smem <= 225 * 1024, "head_bwd_bf16: layer-1 operands need %zu B shared memory", smem);
    // TMA tensor store of d features when its staging slices (2 x 4 x 128 lanes x 4W bytes) still fit
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    p.tma_store = 0;
    {
      const size_t stage = (size_t)2 * 4 * 128 * 4 * W + 128;
      if (g_tuning[LPB_TUNE_B3A_TMA_STORE] && smem + stage <= 225 * 1024 && (reinterpret_cast<uintptr_t>(dfeat) % 16) == 0 &&
          make_dfeat_tensor_map(&tmap, dfeat, B, C4, H * W, 2 * W)) {
        p.tma_store = 1;
        smem += stage;
      }
    }
    int slots = sms / ntile1;
    if (slots < 1) slots = 1;
    if (slots > B) slots = B;
    auto run = [&](auto kern) -> int {
      LPB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kern<<<slots * ntile1, B3A_THREADS, smem, s>>>(p, tmap);
      return LPB_OK;
    };
    int rc = LPB_ERR_UNSUPPORTED;
    switch (W) {
      case 4: rc = run(b3a_dgrad_kernel<4>); break;
      case 8: rc = run(b3a_dgrad_kernel<8>); break;
      case 12: rc = run(b3a_dgrad_kernel<12>); break;
      case 16: rc = run(b3a_dgrad_kernel<16>); break;
      case 24: rc = run(b3a_dgrad_kernel<24>); break;
      case 32: rc = run(b3a_dgrad_kernel<32>); break;
      default: set_error("head_bwd_bf16: feature width %d not in this build's epilogue set", W);
    }
    if (rc != LPB_OK) return rc;
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
