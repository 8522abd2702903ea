// Multi-frame (context) branch of the MHCRNN head: bidirectional convolutional RNN over 5 context frames.
// Reference: UpsamplingCRNN.forward  lightning_pose/models/heads/heatmap_mhcrnn.py:268-316
//   x_f = W_f(x_0);  x_f = W_f(x_s) + H_f(x_f)  for s = 1..4        (and mirrored with W_b / H_b on the flipped sequence)
//   heatmaps = spatial_softmax2d((x_f + x_b) / 2)
// and get_context_from_sequence  lightning_pose/models/base.py:159-196.
//
// What makes this cheap on any hardware: H_f = ConvTranspose2d(16K -> K, k2, s2, groups=K) o Conv2d(K -> 16K, k2, s2,
// groups=K) has kernel == stride == 2 and one group per keypoint, so it acts on every 2x2 block of every keypoint plane
// independently and, having no nonlinearity, is a 4x4 affine map per keypoint:
//   H(x)[block] = L_k x[block] + h_k,   L_k = sum_f T_kf C_kf^T,   h_k = sum_f T_kf cb_kf + tb_k.
// The recurrence therefore needs no convolution at all: per output frame, keypoint and 2x2 block it is five 4x4
// matrix-vector steps per direction on the per-frame deconv maps WF[t] = W_f(x_t), WB[t] = W_b(x_t).  Those maps are
// computed ONCE per frame by the head's tensor-core GEMM (head_rows_bf16.cu) -- a frame that sits in five overlapping windows
// of a video sequence is never duplicated (the reference tiles the features 5x, base.py:380-390) -- and the windows are
// an index table idx[m][s] into them.  HBM-bound: 10 plane reads (mostly L2 hits between neighbouring windows) + 1 write.
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "reduce_partials.cuh"

namespace lpb {

constexpr int CRNN_CTX = 5;

// L[k][o][i] (4x4, o = output position 2a+b of the transposed conv, i = input position of the conv), h[k][o]
__global__ void crnn_prepare_kernel(const float* __restrict__ cw, const float* __restrict__ cb, const float* __restrict__ tw,
                                    const float* __restrict__ tb, int K, int F, float* __restrict__ L, float* __restrict__ h) {
  const int k = blockIdx.x, t = threadIdx.x;  // 20 threads: 16 entries of L + 4 of h
  if (t < 16) {
    const int o = t >> 2, i = t & 3;
    float acc = 0.f;
    for (int f = 0; f < F; ++f) acc = fmaf(tw[(size_t)(k * F + f) * 4 + o], cw[(size_t)(k * F + f) * 4 + i], acc);
    L[k * 16 + t] = acc;
  } else if (t < 20) {
    const int o = t - 16;
    float acc = tb[k];
    for (int f = 0; f < F; ++f) acc = fmaf(tw[(size_t)(k * F + f) * 4 + o], cb[k * F + f], acc);
    h[k * 4 + o] = acc;
  }
}

// gradients of the four parameter tensors from (dL, dh):
//   dT[f][o] = sum_i dL[o][i] C[f][i] + dh[o] cb[f];  dC[f][i] = sum_o dL[o][i] T[f][o];  dcb[f] = sum_o dh[o] T[f][o];  dtb = sum_o dh[o]
__global__ void crnn_prepare_bwd_kernel(const float* __restrict__ cw, const float* __restrict__ cb, const float* __restrict__ tw,
                                        const float* __restrict__ dL, const float* __restrict__ dh, int K, int F,
                                        float* __restrict__ dcw, float* __restrict__ dcb, float* __restrict__ dtw,
                                        float* __restrict__ dtb) {
  const int k = blockIdx.x;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const size_t r = (size_t)(k * F + f) * 4;
    float db = 0.f;
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      float a = dh[k * 4 + o] * cb[k * F + f];
#pragma unroll
      for (int i = 0; i < 4; ++i) a = fmaf(dL[k * 16 + o * 4 + i], cw[r + i], a);
      dtw[r + o] = a;
      db = fmaf(dh[k * 4 + o], tw[r + o], db);
    }
    dcb[k * F + f] = db;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a = 0.f;
#pragma unroll
      for (int o = 0; o < 4; ++o) a = fmaf(dL[k * 16 + o * 4 + i], tw[r + o], a);
      dcw[r + i] = a;
    }
  }
  if (threadIdx.x == 0) dtb[k] = dh[k * 4] + dh[k * 4 + 1] + dh[k * 4 + 2] + dh[k * 4 + 3];
}

struct CrnnParams {
  const float* WF;   // [N][K][H][W] deconv maps of the forward direction
  const float* WB;
  const int32_t* idx;  // [M][5] frame index of each context slot
  const float *Lf, *hf, *Lb, *hb;  // [K][16], [K][4]
  int M, N, K, H, W;
};

__device__ __forceinline__ void load_block(const float* __restrict__ plane, int W, int by, int bx, float (&v)[4]) {
  const float2 r0 = __ldg(reinterpret_cast<const float2*>(plane + (size_t)(2 * by) * W + 2 * bx));
  const float2 r1 = __ldg(reinterpret_cast<const float2*>(plane + (size_t)(2 * by + 1) * W + 2 * bx));
  v[0] = r0.x, v[1] = r0.y, v[2] = r1.x, v[3] = r1.y;
}
__device__ __forceinline__ void affine(const float (&L)[16], const float (&h)[4], const float (&x)[4], const float (&w)[4], float (&y)[4]) {
#pragma unroll
  for (int o = 0; o < 4; ++o) y[o] = w[o] + h[o] + L[o * 4] * x[0] + L[o * 4 + 1] * x[1] + L[o * 4 + 2] * x[2] + L[o * 4 + 3] * x[3];
}

// one thread per 2x2 block of one (m, k) plane; grid.y = m * K + k
__global__ void __launch_bounds__(256) crnn_combine_fwd_kernel(const __grid_constant__ CrnnParams P, float* __restrict__ out) {
  const int plane = blockIdx.y, m = plane / P.K, k = plane - m * P.K;
  const int Wb = P.W / 2, nblk = (P.H / 2) * Wb;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nblk) return;
  const int by = t / Wb, bx = t - by * Wb;
  float Lf[16], Lb[16], hf[4], hb[4];
#pragma unroll
  for (int i = 0; i < 16; ++i) Lf[i] = __ldg(P.Lf + k * 16 + i), Lb[i] = __ldg(P.Lb + k * 16 + i);
#pragma unroll
  for (int i = 0; i < 4; ++i) hf[i] = __ldg(P.hf + k * 4 + i), hb[i] = __ldg(P.hb + k * 4 + i);
  int fr[CRNN_CTX];
#pragma unroll
  for (int s = 0; s < CRNN_CTX; ++s) fr[s] = __ldg(P.idx + m * CRNN_CTX + s);
  const size_t hw = (size_t)P.H * P.W;
  float xf[4], xb[4], w[4], y[4];
  load_block(P.WF + ((size_t)fr[0] * P.K + k) * hw, P.W, by, bx, xf);
  load_block(P.WB + ((size_t)fr[CRNN_CTX - 1] * P.K + k) * hw, P.W, by, bx, xb);
#pragma unroll
  for (int s = 1; s < CRNN_CTX; ++s) {
    load_block(P.WF + ((size_t)fr[s] * P.K + k) * hw, P.W, by, bx, w);
    affine(Lf, hf, xf, w, y);
#pragma unroll
    for (int o = 0; o < 4; ++o) xf[o] = y[o];
    load_block(P.WB + ((size_t)fr[CRNN_CTX - 1 - s] * P.K + k) * hw, P.W, by, bx, w);
    affine(Lb, hb, xb, w, y);
#pragma unroll
    for (int o = 0; o < 4; ++o) xb[o] = y[o];
  }
  float* dst = out + (size_t)plane * hw;
  *reinterpret_cast<float2*>(dst + (size_t)(2 * by) * P.W + 2 * bx) = make_float2(0.5f * (xf[0] + xb[0]), 0.5f * (xf[1] + xb[1]));
  *reinterpret_cast<float2*>(dst + (size_t)(2 * by + 1) * P.W + 2 * bx) = make_float2(0.5f * (xf[2] + xb[2]), 0.5f * (xf[3] + xb[3]));
}

// Backward: recompute the two chains, then walk them in reverse.
// FIXED = false (lpb_crnn_combine_bwd): dWF / dWB are accumulated with atomics (a frame can sit in several windows); dL /
//   dh are reduced per warp, then added with atomics.  The order of those adds is not fixed.
// FIXED = true (lpb_crnn_combine_bwd_ws): dWF / dWB are left to crnn_dmaps_kernel; each CTA sums dL / dh over its warps
//   in warp order and stores them as partial row m * gridDim.x + blockIdx.x of `part` ([dLf | dhf | dLb | dhb], 40 K
//   floats a row; the CTA writes its keypoint's 40), which reduce_partials adds in row order.
template <bool FIXED>
__global__ void __launch_bounds__(256) crnn_combine_bwd_kernel(const __grid_constant__ CrnnParams P, const float* __restrict__ g,
                                                               float* __restrict__ dWF, float* __restrict__ dWB,
                                                               float* __restrict__ dLf, float* __restrict__ dhf,
                                                               float* __restrict__ dLb, float* __restrict__ dhb, float* __restrict__ part) {
  __shared__ float red[8][40];  // FIXED: [warp][dLf 16 | dhf 4 | dLb 16 | dhb 4]
  const int plane = blockIdx.y, m = plane / P.K, k = plane - m * P.K;
  const int Wb = P.W / 2, nblk = (P.H / 2) * Wb;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = t < nblk;
  const int by = active ? t / Wb : 0, bx = active ? t - by * Wb : 0;
  const size_t hw = (size_t)P.H * P.W;
  int fr[CRNN_CTX];
#pragma unroll
  for (int s = 0; s < CRNN_CTX; ++s) fr[s] = __ldg(P.idx + m * CRNN_CTX + s);
#pragma unroll
  for (int dir = 0; dir < 2; ++dir) {
    const float* Wm = dir ? P.WB : P.WF;
    float* dWm = dir ? dWB : dWF;
    float L[16], h[4];
#pragma unroll
    for (int i = 0; i < 16; ++i) L[i] = __ldg((dir ? P.Lb : P.Lf) + k * 16 + i);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __ldg((dir ? P.hb : P.hf) + k * 4 + i);
    // chain states x_0 .. x_3 (x_4 is the output and is not needed); slot order: dir 0 -> 0..4, dir 1 -> 4..0
    float xs[CRNN_CTX - 1][4], w[4], y[4];
    float dL[16], dh[4], gg[4];
#pragma unroll
    for (int i = 0; i < 16; ++i) dL[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) dh[i] = 0.f, gg[i] = 0.f;
    if (active) {
      load_block(Wm + ((size_t)fr[dir ? CRNN_CTX - 1 : 0] * P.K + k) * hw, P.W, by, bx, xs[0]);
#pragma unroll
      for (int s = 1; s < CRNN_CTX - 1; ++s) {
        load_block(Wm + ((size_t)fr[dir ? CRNN_CTX - 1 - s : s] * P.K + k) * hw, P.W, by, bx, w);
        affine(L, h, xs[s - 1], w, y);
#pragma unroll
        for (int o = 0; o < 4; ++o) xs[s][o] = y[o];
      }
      const float* gp = g + (size_t)plane * hw;
      const float2 r0 = __ldg(reinterpret_cast<const float2*>(gp + (size_t)(2 * by) * P.W + 2 * bx));
      const float2 r1 = __ldg(reinterpret_cast<const float2*>(gp + (size_t)(2 * by + 1) * P.W + 2 * bx));
      gg[0] = 0.5f * r0.x, gg[1] = 0.5f * r0.y, gg[2] = 0.5f * r1.x, gg[3] = 0.5f * r1.y;
#pragma unroll
      for (int s = CRNN_CTX - 1; s >= 0; --s) {
        if constexpr (!FIXED) {
          float* dp = dWm + ((size_t)fr[dir ? CRNN_CTX - 1 - s : s] * P.K + k) * hw;
          atomicAdd(dp + (size_t)(2 * by) * P.W + 2 * bx, gg[0]);
          atomicAdd(dp + (size_t)(2 * by) * P.W + 2 * bx + 1, gg[1]);
          atomicAdd(dp + (size_t)(2 * by + 1) * P.W + 2 * bx, gg[2]);
          atomicAdd(dp + (size_t)(2 * by + 1) * P.W + 2 * bx + 1, gg[3]);
        }
        if (s == 0) break;
        float gn[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          dh[o] += gg[o];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            dL[o * 4 + i] = fmaf(gg[o], xs[s - 1][i], dL[o * 4 + i]);
            gn[i] = fmaf(L[o * 4 + i], gg[o], gn[i]);
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) gg[i] = gn[i];
      }
    }
    if constexpr (FIXED) {
#pragma unroll
      for (int i = 0; i < 20; ++i) {
        const float v = warp_sum(i < 16 ? dL[i] : dh[i - 16]);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][20 * dir + i] = v;
      }
    } else {
      float* dLg = (dir ? dLb : dLf) + k * 16;
      float* dhg = (dir ? dhb : dhf) + k * 4;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float v = warp_sum(dL[i]);
        if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(dLg + i, v);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float v = warp_sum(dh[i]);
        if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(dhg + i, v);
      }
    }
  }
  if constexpr (FIXED) {
    __syncthreads();
    if (threadIdx.x < 40) {
      const int i = threadIdx.x, dir = i / 20, j = i - 20 * dir;
      float v = 0.f;
      for (int wp = 0; wp < (int)(blockDim.x >> 5); ++wp) v += red[wp][i];
      // section offsets in a row: dLf 0, dhf 16 K, dLb 20 K, dhb 36 K
      const size_t col = (size_t)20 * P.K * dir + (j < 16 ? (size_t)k * 16 + j : (size_t)16 * P.K + k * 4 + (j - 16));
      part[((size_t)m * gridDim.x + blockIdx.x) * 40 * P.K + col] = v;
    }
  }
}

// The (window, slot) pairs that read each frame, in ascending window-then-slot order: pairs[start[f] .. start[f + 1]) holds
// e = 5 m + s for every idx[m][s] == f.  One CTA: counts (integer atomics), exclusive scan, placement (integer atomics),
// then each frame's list is sorted, so the result does not depend on the order of the placements.  Entries outside
// [0, N) belong to no frame.
__global__ void __launch_bounds__(1024) crnn_pairs_kernel(const int32_t* __restrict__ idx, int M, int N, int* __restrict__ start,
                                                          int* __restrict__ cnt, int* __restrict__ pairs) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int t = threadIdx.x, E = M * CRNN_CTX;
  for (int f = t; f < N; f += blockDim.x) cnt[f] = 0;
  if (t == 0) carry = 0, start[0] = 0;
  __syncthreads();
  for (int e = t; e < E; e += blockDim.x) {
    const int f = __ldg(idx + e);
    if ((unsigned)f < (unsigned)N) atomicAdd(cnt + f, 1);
  }
  __syncthreads();
  for (int base = 0; base < N; base += blockDim.x) {  // start[f + 1] = sum of cnt[0 .. f]
    const int f = base + t;
    int v = f < N ? cnt[f] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if ((t & 31) >= o) v += u;
    }
    if ((t & 31) == 31) wsum[t >> 5] = v;
    __syncthreads();
    int pre = carry;
    for (int wp = 0; wp < (t >> 5); ++wp) pre += wsum[wp];
    if (f < N) start[f + 1] = pre + v;
    __syncthreads();
    if (t == blockDim.x - 1) carry = pre + v;
    __syncthreads();
  }
  for (int f = t; f < N; f += blockDim.x) cnt[f] = 0;
  __syncthreads();
  for (int e = t; e < E; e += blockDim.x) {
    const int f = __ldg(idx + e);
    if ((unsigned)f < (unsigned)N) pairs[start[f] + atomicAdd(cnt + f, 1)] = e;
  }
  __syncthreads();
  for (int f = t; f < N; f += blockDim.x) {
    int* l = pairs + start[f];
    const int n = start[f + 1] - start[f];
    for (int i = 1; i < n; ++i) {
      const int v = l[i];
      int j = i - 1;
      for (; j >= 0 && l[j] > v; --j) l[j + 1] = l[j];
      l[j + 1] = v;
    }
  }
}

// dWF / dWB of lpb_crnn_combine_bwd_ws, one thread per 2x2 block of one (frame, keypoint) plane: the sum over the frame's
// (window, slot) pairs, in pair order, of the slot's chain gradient.  That gradient needs no chain state: at chain step
// q it is (L^T)^(4 - q) 0.5 g[m], computed here with the backward kernel's own fma sequence, so each term has the bits
// of the term the atomic form adds.  Window slot s is chain step s forward and 4 - s backward.
__global__ void __launch_bounds__(256) crnn_dmaps_kernel(const __grid_constant__ CrnnParams P, const float* __restrict__ g,
                                                         const int* __restrict__ start, const int* __restrict__ pairs,
                                                         float* __restrict__ dWF, float* __restrict__ dWB) {
  const int Wb = P.W / 2, nblk = (P.H / 2) * Wb;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)P.N * P.K * nblk) return;
  const int64_t fk = t / nblk;
  const int blk = (int)(t - fk * nblk), k = (int)(fk % P.K), f = (int)(fk / P.K);
  const int by = blk / Wb, bx = blk - by * Wb;
  const size_t hw = (size_t)P.H * P.W, o0 = (size_t)(2 * by) * P.W + 2 * bx, o1 = o0 + P.W;
  const int p0 = __ldg(start + f), p1 = __ldg(start + f + 1);
#pragma unroll
  for (int dir = 0; dir < 2; ++dir) {
    float L[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) L[i] = __ldg((dir ? P.Lb : P.Lf) + k * 16 + i);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = p0; p < p1; ++p) {
      const int e = __ldg(pairs + p), m = e / CRNN_CTX, s = e - m * CRNN_CTX;
      const float* gp = g + ((size_t)m * P.K + k) * hw;
      const float2 r0 = __ldg(reinterpret_cast<const float2*>(gp + o0)), r1 = __ldg(reinterpret_cast<const float2*>(gp + o1));
      float gg[4] = {0.5f * r0.x, 0.5f * r0.y, 0.5f * r1.x, 0.5f * r1.y};
      for (int q = CRNN_CTX - 1; q > (dir ? CRNN_CTX - 1 - s : s); --q) {
        float gn[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
          for (int i = 0; i < 4; ++i) gn[i] = fmaf(L[o * 4 + i], gg[o], gn[i]);
#pragma unroll
        for (int i = 0; i < 4; ++i) gg[i] = gn[i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] += gg[i];
    }
    float* dp = (dir ? dWB : dWF) + ((size_t)f * P.K + k) * hw;
    *reinterpret_cast<float2*>(dp + o0) = make_float2(acc[0], acc[1]);
    *reinterpret_cast<float2*>(dp + o1) = make_float2(acc[2], acc[3]);
  }
}

// workspace of lpb_crnn_combine_bwd_ws: start [N + 1], cnt [N], pairs [5 M] (ints), then at a 16-byte boundary the
// dL / dh partials [M * ceil(blocks / 256)][40 K] (floats)
struct CrnnWs {
  size_t ints, rows, bytes;
};
static CrnnWs crnn_ws(int M, int N, int K, int H, int W) {
  CrnnWs w;
  w.ints = (((size_t)2 * N + 1 + (size_t)CRNN_CTX * M) + 3) & ~(size_t)3;
  w.rows = (size_t)M * (((size_t)(H / 2) * (W / 2) + 255) / 256);
  w.bytes = w.ints * sizeof(int) + w.rows * 40 * (size_t)K * sizeof(float);
  return w;
}

// get_context_from_sequence: out[i][s] = seq[clamp(i + s - ctx/2, 0, n - 1)]   (16-byte vectors)
__global__ void context_gather_kernel(const uint4* __restrict__ seq, int64_t n, int64_t vec_per_item, int ctx, uint4* __restrict__ out) {
  const int64_t total = n * ctx * vec_per_item;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i % vec_per_item, r = i / vec_per_item;
    const int s = (int)(r % ctx);
    const int64_t fi = r / ctx;
    int64_t src = fi + s - ctx / 2;
    src = src < 0 ? 0 : (src > n - 1 ? n - 1 : src);
    out[i] = __ldg(seq + src * vec_per_item + v);
  }
}

template <int FMT>
__device__ __forceinline__ float load_fmt(const void* p, int64_t i) {
  if constexpr (FMT == LPB_OUT_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  else if constexpr (FMT == LPB_OUT_F16) return __half2float(static_cast<const __half*>(p)[i]);
  else return static_cast<const float*>(p)[i];
}

// adjoint of context_gather_kernel: d_seq[f] = sum of grad[i][s] over the slots with clamp(i + s - ctx/2) == f.  Only the
// windows i in [f - ctx/2, f + ctx/2] can read frame f (the edge frames' repeats included); they are summed in ascending
// (i, s) order in fp32, one thread per element of d_seq, so the result does not depend on the launch.
template <int FMT>
__global__ void context_gather_bwd_kernel(const void* __restrict__ grad, int64_t n, int64_t elems, int ctx, void* __restrict__ d_seq) {
  const int half = ctx / 2;
  const int64_t total = n * elems;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = i / elems, e = i - f * elems;
    const int64_t lo = f - half < 0 ? 0 : f - half, hi = f + half > n - 1 ? n - 1 : f + half;
    float acc = 0.f;
    for (int64_t w = lo; w <= hi; ++w)
      for (int s = 0; s < ctx; ++s) {
        int64_t src = w + s - half;
        src = src < 0 ? 0 : (src > n - 1 ? n - 1 : src);
        if (src == f) acc += load_fmt<FMT>(grad, (w * ctx + s) * elems + e);
      }
    store_fmt<FMT>(d_seq, (size_t)i, acc);
  }
}

}  // namespace lpb

extern "C" int lpb_crnn_prepare(const float* conv_w, const float* conv_b, const float* convt_w, const float* convt_b, int K, int F,
                                float* L, float* h, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(conv_w && conv_b && convt_w && convt_b && L && h && K >= 1 && F >= 1, "crnn_prepare: bad arguments");
  crnn_prepare_kernel<<<K, 32, 0, static_cast<cudaStream_t>(stream)>>>(conv_w, conv_b, convt_w, convt_b, K, F, L, h);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_crnn_prepare_bwd(const float* conv_w, const float* conv_b, const float* convt_w, const float* dL, const float* dh,
                                    int K, int F, float* d_conv_w, float* d_conv_b, float* d_convt_w, float* d_convt_b, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(conv_w && conv_b && convt_w && dL && dh && d_conv_w && d_conv_b && d_convt_w && d_convt_b && K >= 1 && F >= 1,
              "crnn_prepare_bwd: bad arguments");
  crnn_prepare_bwd_kernel<<<K, 32, 0, static_cast<cudaStream_t>(stream)>>>(conv_w, conv_b, convt_w, dL, dh, K, F, d_conv_w, d_conv_b, d_convt_w,
                                                                            d_convt_b);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

static int crnn_check(const void* a, const void* b, const void* idx, int M, int N, int K, int H, int W) {
  using namespace lpb;
  LPB_REQUIRE(a && b && idx, "crnn_combine: null pointer");
  LPB_REQUIRE(M >= 0 && N >= 1 && K >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && (int64_t)M * K < 65536,
              "crnn_combine: bad shape (even H, W; M * K < 65536 per call)");
  return LPB_OK;
}

extern "C" int lpb_crnn_combine_fwd(const float* WF, const float* WB, const int32_t* idx, int M, int N, int K, int H, int W,
                                    const float* Lf, const float* hf, const float* Lb, const float* hb, float* out_logits, void* stream) {
  using namespace lpb;
  if (int rc = crnn_check(WF, WB, idx, M, N, K, H, W)) return rc;
  LPB_REQUIRE(Lf && hf && Lb && hb && out_logits, "crnn_combine_fwd: null pointer");
  if (M == 0) return LPB_OK;
  CrnnParams p{WF, WB, idx, Lf, hf, Lb, hb, M, N, K, H, W};
  const int nblk = (H / 2) * (W / 2);
  dim3 grid((unsigned)((nblk + 255) / 256), (unsigned)(M * K));
  crnn_combine_fwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, out_logits);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_crnn_combine_bwd(const float* WF, const float* WB, const int32_t* idx, const float* grad_logits, int M, int N, int K,
                                    int H, int W, const float* Lf, const float* hf, const float* Lb, const float* hb, float* dWF,
                                    float* dWB, float* dLf, float* dhf, float* dLb, float* dhb, void* stream) {
  using namespace lpb;
  if (int rc = crnn_check(WF, WB, idx, M, N, K, H, W)) return rc;
  LPB_REQUIRE(grad_logits && Lf && hf && Lb && hb && dWF && dWB && dLf && dhf && dLb && dhb, "crnn_combine_bwd: null pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t nmap = (size_t)N * K * H * W * sizeof(float);
  LPB_CUDA(cudaMemsetAsync(dWF, 0, nmap, s));
  LPB_CUDA(cudaMemsetAsync(dWB, 0, nmap, s));
  LPB_CUDA(cudaMemsetAsync(dLf, 0, sizeof(float) * K * 16, s));
  LPB_CUDA(cudaMemsetAsync(dLb, 0, sizeof(float) * K * 16, s));
  LPB_CUDA(cudaMemsetAsync(dhf, 0, sizeof(float) * K * 4, s));
  LPB_CUDA(cudaMemsetAsync(dhb, 0, sizeof(float) * K * 4, s));
  if (M == 0) return LPB_OK;
  CrnnParams p{WF, WB, idx, Lf, hf, Lb, hb, M, N, K, H, W};
  const int nblk = (H / 2) * (W / 2);
  dim3 grid((unsigned)((nblk + 255) / 256), (unsigned)(M * K));
  crnn_combine_bwd_kernel<false><<<grid, 256, 0, s>>>(p, grad_logits, dWF, dWB, dLf, dhf, dLb, dhb, nullptr);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_crnn_combine_bwd_workspace_bytes(int M, int N, int K, int H, int W, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "crnn_combine_bwd_workspace_bytes: null pointer");
  LPB_REQUIRE(M >= 0 && N >= 1 && K >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && (int64_t)M * K < 65536,
              "crnn_combine_bwd_workspace_bytes: bad shape (even H, W; M * K < 65536 per call)");
  *bytes = crnn_ws(M, N, K, H, W).bytes;
  return LPB_OK;
}

extern "C" int lpb_crnn_combine_bwd_ws(const float* WF, const float* WB, const int32_t* idx, const float* grad_logits, int M, int N,
                                       int K, int H, int W, const float* Lf, const float* hf, const float* Lb, const float* hb,
                                       float* dWF, float* dWB, float* dLf, float* dhf, float* dLb, float* dhb, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  using namespace lpb;
  if (int rc = crnn_check(WF, WB, idx, M, N, K, H, W)) return rc;
  LPB_REQUIRE(grad_logits && Lf && hf && Lb && hb && dWF && dWB && dLf && dhf && dLb && dhb, "crnn_combine_bwd_ws: null pointer");
  const CrnnWs ws = crnn_ws(M, N, K, H, W);
  LPB_REQUIRE(workspace && aligned_to(workspace, 16), "crnn_combine_bwd_ws: null or unaligned workspace (16 bytes)");
  LPB_REQUIRE(workspace_bytes >= ws.bytes, "crnn_combine_bwd_ws: workspace of %zu bytes, %zu needed", workspace_bytes, ws.bytes);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (M == 0) {
    const size_t nmap = (size_t)N * K * H * W * sizeof(float);
    LPB_CUDA(cudaMemsetAsync(dWF, 0, nmap, s));
    LPB_CUDA(cudaMemsetAsync(dWB, 0, nmap, s));
    LPB_CUDA(cudaMemsetAsync(dLf, 0, sizeof(float) * K * 16, s));
    LPB_CUDA(cudaMemsetAsync(dLb, 0, sizeof(float) * K * 16, s));
    LPB_CUDA(cudaMemsetAsync(dhf, 0, sizeof(float) * K * 4, s));
    LPB_CUDA(cudaMemsetAsync(dhb, 0, sizeof(float) * K * 4, s));
    return LPB_OK;
  }
  DeviceLimits dev;
  LPB_TRY(device_limits(&dev));
  int* start = static_cast<int*>(workspace);
  int* cnt = start + N + 1;
  int* pairs = cnt + N;
  float* part = reinterpret_cast<float*>(start + ws.ints);
  CrnnParams p{WF, WB, idx, Lf, hf, Lb, hb, M, N, K, H, W};
  const int nblk = (H / 2) * (W / 2);
  crnn_pairs_kernel<<<1, 1024, 0, s>>>(idx, M, N, start, cnt, pairs);
  const dim3 grid((unsigned)((nblk + 255) / 256), (unsigned)(M * K));
  crnn_combine_bwd_kernel<true><<<grid, 256, 0, s>>>(p, grad_logits, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, part);
  const int64_t nthreads = (int64_t)N * K * nblk;
  crnn_dmaps_kernel<<<(unsigned)((nthreads + 255) / 256), 256, 0, s>>>(p, grad_logits, start, pairs, dWF, dWB);
  const size_t stride = (size_t)40 * K;
  const int rows = (int)ws.rows;
  reduce_partials<1>(part, rows, stride, 16 * K, dLf, dev.sms, s);
  reduce_partials<1>(part + (size_t)16 * K, rows, stride, 4 * K, dhf, dev.sms, s);
  reduce_partials<1>(part + (size_t)20 * K, rows, stride, 16 * K, dLb, dev.sms, s);
  reduce_partials<1>(part + (size_t)36 * K, rows, stride, 4 * K, dhb, dev.sms, s);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_context_gather(const void* seq, int64_t n, int64_t item_bytes, int ctx, void* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(seq && out && n >= 1 && ctx >= 1 && (ctx & 1) && item_bytes >= 16 && item_bytes % 16 == 0,
              "context_gather: bad arguments (odd context length, item size a multiple of 16 bytes)");
  const int64_t total = n * ctx * (item_bytes / 16);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;  // 32 CTAs per SM of an H100 SXM
  context_gather_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint4*>(seq), n, item_bytes / 16, ctx,
                                                                                        static_cast<uint4*>(out));
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_context_gather_bwd(const void* grad, int64_t n, int64_t elems, int ctx, int format, void* d_seq, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(grad && d_seq && n >= 1 && elems >= 1 && ctx >= 1 && (ctx & 1) && valid_out_format(format),
              "context_gather_bwd: bad arguments (odd context length, element format LPB_OUT_F32 / BF16 / F16)");
  DeviceLimits dev;
  LPB_TRY(device_limits(&dev));
  int64_t blocks = (n * elems + 255) / 256;
  if (blocks > (int64_t)dev.sms * 16) blocks = (int64_t)dev.sms * 16;
  with_out_format(format, [&](auto fmt) {
    context_gather_bwd_kernel<decltype(fmt)::value><<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(grad, n, elems, ctx, d_seq);
  });
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
