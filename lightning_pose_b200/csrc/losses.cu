// Loss stack of the hot path.
//   heatmap MSE / KL / JS         lightning_pose/losses/losses.py:229-289, :314-335, :360-378, :404-423
//   coordinate remap              lightning_pose/data/utils.py:142-234, lightning_pose/data/bboxes.py:74-105,222-288
//   temporal + PCA losses         lightning_pose/losses/losses.py:548-573, :608-703; lightning_pose/utils/pca.py:97-190,266-309
//
// Design notes: the reference's boolean-mask gathers (targets[~idxs_ignore], masked_select) are
// data-dependent-shape ops that force a host sync; here "dropped" planes are a per-plane flag and
// the mean's denominator is reduced on the device.  All reductions are two-stage and atomic-free,
// hence run-to-run deterministic.
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "targets.cuh"

namespace lpb {

constexpr int HL_THREADS = 256;

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int k = 0; k < HL_THREADS / 32; ++k) t += red[k];
  return t;
}

// F.relu as torch computes it: NaN stays NaN (fmaxf would return the 0), every other value gets fmaxf's bits
__device__ __forceinline__ float relu_keep_nan(float x) { return isnan(x) ? x : fmaxf(x, 0.f); }

__device__ __forceinline__ float hm_term(int kind, float t, float p) {
  if (kind == LPB_HM_MSE) {
    const float d = t - p;
    return d * d;
  }
  const float tt = t + 1e-10f, pp = p + 1e-10f;  // losses.py:375-376, :420-421
  if (kind == LPB_HM_KL) return tt * (logf(tt) - logf(pp));
  const float m = 0.5f * (tt + pp);
  const float lm = logf(m);
  return 0.5f * (tt * (logf(tt) - lm) + pp * (logf(pp) - lm));
}

// d hm_term / d p for KL and JS (losses.py:375-376, :420-421 through autograd)
__device__ __forceinline__ float hm_div_grad(int kind, float t, float p) {
  const float tt = t + 1e-10f, pp = p + 1e-10f;
  return (kind == LPB_HM_KL) ? -tt / pp : 0.5f * (logf(pp) - logf(0.5f * (tt + pp)));
}

// stage 1: one CTA per plane -> ws[2*plane] = sum of terms, ws[2*plane+1] = 1 if target not all-zero
__global__ void __launch_bounds__(HL_THREADS) heatmap_loss_plane_kernel(const float* __restrict__ targ,
                                                                        const float* __restrict__ pred, int hw,
                                                                        int kind, float* __restrict__ ws) {
  __shared__ float red[HL_THREADS / 32];
  const size_t plane = blockIdx.x;
  const float* __restrict__ t = targ + plane * (size_t)hw;
  const float* __restrict__ p = pred + plane * (size_t)hw;
  float acc = 0.f, nz = 0.f;
  if ((hw & 3) == 0 && ((reinterpret_cast<uintptr_t>(t) | reinterpret_cast<uintptr_t>(p)) & 15) == 0) {
    const float4* t4 = reinterpret_cast<const float4*>(t);
    const float4* p4 = reinterpret_cast<const float4*>(p);
    for (int i = threadIdx.x; i < (hw >> 2); i += HL_THREADS) {
      const float4 a = __ldg(t4 + i), b = __ldg(p4 + i);
      acc += hm_term(kind, a.x, b.x) + hm_term(kind, a.y, b.y) + hm_term(kind, a.z, b.z) + hm_term(kind, a.w, b.w);
      if (a.x != 0.f || a.y != 0.f || a.z != 0.f || a.w != 0.f) nz = 1.f;
    }
  } else {
    for (int i = threadIdx.x; i < hw; i += HL_THREADS) {
      const float a = __ldg(t + i);
      acc += hm_term(kind, a, __ldg(p + i));
      if (a != 0.f) nz = 1.f;
    }
  }
  acc = block_sum_256(acc, red);
  nz = block_sum_256(nz, red);
  if (threadIdx.x == 0) {
    ws[2 * plane] = acc;
    ws[2 * plane + 1] = nz > 0.f ? 1.f : 0.f;
  }
}

// stage 2: out[0] = sum_kept(ws) / n_kept (NaN when nothing is kept, like torch.mean of an empty tensor)
__global__ void __launch_bounds__(HL_THREADS) heatmap_loss_final_kernel(const float* __restrict__ ws, int64_t n_planes,
                                                                        float* __restrict__ out) {
  __shared__ float red[HL_THREADS / 32];
  float acc = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n_planes; i += HL_THREADS) {
    const float k = ws[2 * i + 1];
    if (k > 0.f) {
      acc += ws[2 * i];
      cnt += 1.f;
    }
  }
  acc = block_sum_256(acc, red);
  cnt = block_sum_256(cnt, red);
  if (threadIdx.x == 0) {
    out[0] = acc / cnt;
    out[1] = cnt;
  }
}

__global__ void __launch_bounds__(HL_THREADS) heatmap_loss_bwd_kernel(const float* __restrict__ targ,
                                                                      const float* __restrict__ pred, int hw, int kind,
                                                                      const float* __restrict__ ws,
                                                                      const float* __restrict__ fwd_out,
                                                                      const float* __restrict__ gout,
                                                                      float* __restrict__ gpred) {
  const size_t plane = blockIdx.x;
  const float* __restrict__ t = targ + plane * (size_t)hw;
  const float* __restrict__ p = pred + plane * (size_t)hw;
  float* __restrict__ g = gpred + plane * (size_t)hw;
  const float scale = (ws[2 * plane + 1] > 0.f) ? gout[0] / fwd_out[1] : 0.f;
  for (int i = threadIdx.x; i < hw; i += HL_THREADS) {
    float d;
    if (scale == 0.f) {
      d = 0.f;
    } else if (kind == LPB_HM_MSE) {
      d = 2.f * (p[i] - t[i]);
    } else {
      d = hm_div_grad(kind, t[i], p[i]);
    }
    g[i] = d * scale;
  }
}

// fused target generation + MSE: the target plane only ever exists as two 1-D factors in smem
__global__ void __launch_bounds__(HL_THREADS) heatmap_mse_from_kp_kernel(const float* __restrict__ kp,
                                                                         const int32_t* __restrict__ vis,
                                                                         const float* __restrict__ pred, float sx,
                                                                         float sy, int oh, int ow, float two_s2,
                                                                         float* __restrict__ ws) {
  extern __shared__ float sm[];  // ex[ow], ey[oh], red[16]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  const size_t plane = blockIdx.x;
  const int n = oh * ow;
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  if (tp.mode == TARGET_ZERO) {  // dropped plane: the prediction is not even read
    if (threadIdx.x == 0) {
      ws[2 * plane] = 0.f;
      ws[2 * plane + 1] = 0.f;
    }
    return;
  }
  const float* __restrict__ p = pred + plane * (size_t)n;
  float acc = 0.f;
  if (tp.mode == TARGET_UNIFORM) {
    const float u = 1.0f / (float)n;
    for (int i = threadIdx.x; i < n; i += HL_THREADS) {
      const float d = u - __ldg(p + i);
      acc = fmaf(d, d, acc);
    }
  } else {
    const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, HL_THREADS);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < oh; r += HL_THREADS / 32) {
      const float er = ey[r] * norm;
      const float* __restrict__ pr = p + (size_t)r * ow;
      for (int c = lane; c < ow; c += 32) {
        const float d = ex[c] * er - __ldg(pr + c);
        acc = fmaf(d, d, acc);
      }
    }
  }
  acc = block_sum_256(acc, red + 8);
  if (threadIdx.x == 0) {
    ws[2 * plane] = acc;
    ws[2 * plane + 1] = 1.f;  // a Gaussian / uniform target is never all-zero (NaN planes are kept too)
  }
}


// backward of the fused target + MSE: d loss / d pred = 2 (pred - target) / n_kept on kept planes
__global__ void __launch_bounds__(HL_THREADS) heatmap_mse_from_kp_bwd_kernel(const float* __restrict__ kp,
                                                                             const int32_t* __restrict__ vis,
                                                                             const float* __restrict__ pred, float sx,
                                                                             float sy, int oh, int ow, float two_s2,
                                                                             const float* __restrict__ fwd_out,
                                                                             const float* __restrict__ gout,
                                                                             float* __restrict__ gpred) {
  extern __shared__ float sm[];  // ex[ow], ey[oh], red[16]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  const size_t plane = blockIdx.x;
  const int n = oh * ow;
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  float* __restrict__ g = gpred + plane * (size_t)n;
  if (tp.mode == TARGET_ZERO) {
    for (int i = threadIdx.x; i < n; i += HL_THREADS) g[i] = 0.f;
    return;
  }
  const float scale = mse_target_scale(gout[0], fwd_out[1]);
  const float* __restrict__ p = pred + plane * (size_t)n;
  if (tp.mode == TARGET_UNIFORM) {
    const float u = mse_target_uniform(n);
    for (int i = threadIdx.x; i < n; i += HL_THREADS) g[i] = mse_target_grad(TARGET_UNIFORM, __ldg(p + i), u, 1.f, scale);
    return;
  }
  const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, HL_THREADS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < oh; r += HL_THREADS / 32) {
    const float er = ey[r] * norm;
    for (int c = lane; c < ow; c += 32) g[(size_t)r * ow + c] = mse_target_grad(TARGET_GAUSS, __ldg(p + (size_t)r * ow + c), ex[c], er, scale);
  }
}

// fused target generation + KL / JS: each target value is made in registers where the prediction is read
// (losses.py:338-423 on the planes of data/heatmaps.py:37-87).  A dropped plane's prediction is not read.
__global__ void __launch_bounds__(HL_THREADS) heatmap_div_from_kp_kernel(const float* __restrict__ kp,
                                                                         const int32_t* __restrict__ vis,
                                                                         const float* __restrict__ pred, float sx,
                                                                         float sy, int oh, int ow, float two_s2,
                                                                         int kind, float* __restrict__ ws) {
  extern __shared__ float sm[];  // ex[ow], ey[oh], red[16]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  const size_t plane = blockIdx.x;
  const int n = oh * ow;
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  if (tp.mode == TARGET_ZERO) {
    if (threadIdx.x == 0) {
      ws[2 * plane] = 0.f;
      ws[2 * plane + 1] = 0.f;
    }
    return;
  }
  const float* __restrict__ p = pred + plane * (size_t)n;
  float acc = 0.f;
  if (tp.mode == TARGET_UNIFORM) {
    const float u = mse_target_uniform(n);
    for (int i = threadIdx.x; i < n; i += HL_THREADS) acc += hm_term(kind, u, __ldg(p + i));
  } else {
    const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, HL_THREADS);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < oh; r += HL_THREADS / 32) {
      const float er = ey[r] * norm;
      const float* __restrict__ pr = p + (size_t)r * ow;
      for (int c = lane; c < ow; c += 32) acc += hm_term(kind, ex[c] * er, __ldg(pr + c));
    }
  }
  acc = block_sum_256(acc, red + 8);
  if (threadIdx.x == 0) {
    ws[2 * plane] = acc;
    ws[2 * plane + 1] = 1.f;  // a Gaussian / uniform target is never all-zero (NaN planes are kept too)
  }
}

// backward of the kernel above: d loss / d pred = hm_div_grad(target, pred) * grad_out / n_kept on kept planes, 0 on
// dropped ones (and everywhere when the scale is 0, as heatmap_loss_bwd_kernel does)
__global__ void __launch_bounds__(HL_THREADS) heatmap_div_from_kp_bwd_kernel(const float* __restrict__ kp,
                                                                             const int32_t* __restrict__ vis,
                                                                             const float* __restrict__ pred, float sx,
                                                                             float sy, int oh, int ow, float two_s2,
                                                                             int kind, const float* __restrict__ fwd_out,
                                                                             const float* __restrict__ gout,
                                                                             float* __restrict__ gpred) {
  extern __shared__ float sm[];  // ex[ow], ey[oh], red[16]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  const size_t plane = blockIdx.x;
  const int n = oh * ow;
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  float* __restrict__ g = gpred + plane * (size_t)n;
  const float scale = tp.mode == TARGET_ZERO ? 0.f : gout[0] / fwd_out[1];
  if (scale == 0.f) {
    for (int i = threadIdx.x; i < n; i += HL_THREADS) g[i] = 0.f;
    return;
  }
  const float* __restrict__ p = pred + plane * (size_t)n;
  if (tp.mode == TARGET_UNIFORM) {
    const float u = mse_target_uniform(n);
    for (int i = threadIdx.x; i < n; i += HL_THREADS) g[i] = hm_div_grad(kind, u, __ldg(p + i)) * scale;
    return;
  }
  const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, HL_THREADS);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < oh; r += HL_THREADS / 32) {
    const float er = ey[r] * norm;
    for (int c = lane; c < ow; c += 32) g[(size_t)r * ow + c] = hm_div_grad(kind, ex[c] * er, __ldg(p + (size_t)r * ow + c)) * scale;
  }
}

// ---- TemporalHeatmapLoss (lightning_pose/losses/losses.py:793-854) ------------------------------------
// stage 1: one CTA per (t, k) pair of consecutive planes -> ws[t*K+k] = mean-pixel MSE or
// KL(pred = h[t] + 1e-10, target = h[t+1] + 1e-10)  (argument order of :818-822)
__global__ void __launch_bounds__(HL_THREADS) temporal_heatmap_pair_kernel(const float* __restrict__ hm, int K, int hw,
                                                                           int kind, float* __restrict__ ws) {
  __shared__ float red[HL_THREADS / 32];
  const int t = blockIdx.x / K, k = blockIdx.x - t * K;
  const float* __restrict__ a = hm + ((size_t)t * K + k) * hw;
  const float* __restrict__ b = hm + ((size_t)(t + 1) * K + k) * hw;
  float acc = 0.f;
  for (int i = threadIdx.x; i < hw; i += HL_THREADS) {
    const float x = __ldg(a + i), y = __ldg(b + i);
    if (kind == LPB_HM_MSE) {
      const float d = x - y;
      acc = fmaf(d, d, acc);
    } else {
      const float q = x + 1e-10f, p = y + 1e-10f;
      acc += p * (logf(p) - logf(q));
    }
  }
  acc = block_sum_256(acc, red);
  if (threadIdx.x == 0) ws[blockIdx.x] = (kind == LPB_HM_MSE) ? acc / (float)hw : acc;
}

__global__ void __launch_bounds__(HL_THREADS) temporal_heatmap_final_kernel(const float* __restrict__ ws,
                                                                            const float* __restrict__ conf, int T, int K,
                                                                            const float* __restrict__ eps, float thr,
                                                                            float* __restrict__ out) {
  __shared__ float red[HL_THREADS / 32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < (T - 1) * K; i += HL_THREADS) {
    const int t = i / K, k = i - t * K;
    float d = ws[i];
    if (conf[(size_t)t * K + k] < thr || conf[(size_t)(t + 1) * K + k] < thr) d = 0.f;
    acc += relu_keep_nan(d - eps[k]);
  }
  acc = block_sum_256(acc, red);
  if (threadIdx.x == 0) out[0] = acc / (float)((T - 1) * K);
}

// backward of the two kernels above: one CTA per plane (t, k).  With a = h[t], b = h[t+1]:
//   MSE  d = mean((a-b)^2):                 dd/da = 2(a-b)/hw,          dd/db = -2(a-b)/hw
//   KL   d = sum p (log p - log q), q = a + 1e-10, p = b + 1e-10:   dd/da = -p/q,   dd/db = log p - log q + 1
// a pair (t, k) carries gradient iff neither confidence is below the threshold (the reference zeroes those
// entries in place, losses.py:789) and d > eps_k or d is NaN (F.relu, :761, passes the gradient of a NaN); the mean
// runs over all (T-1)*K entries (:851).  A pair without gradient whose d is NaN still gives NaN where either of its
// pixels is NaN, as autograd's 0 * NaN does in the per-pixel backward; its other pixels get 0.
__global__ void __launch_bounds__(HL_THREADS) temporal_heatmap_bwd_kernel(const float* __restrict__ hm,
                                                                          const float* __restrict__ conf,
                                                                          const float* __restrict__ ws, int T, int K,
                                                                          int hw, int kind, const float* __restrict__ eps,
                                                                          float thr, const float* __restrict__ gout,
                                                                          float* __restrict__ grad) {
  const int t = blockIdx.x / K, k = blockIdx.x - t * K;
  const float scale = __ldg(gout) / (float)((T - 1) * K);
  enum { PAIR_OFF, PAIR_GRAD, PAIR_NAN_ONLY };
  auto state = [&](int tt) {  // pair (tt, tt + 1)
    if (tt < 0 || tt >= T - 1) return PAIR_OFF;
    const float d = ws[(size_t)tt * K + k];
    if (conf[(size_t)tt * K + k] < thr || conf[(size_t)(tt + 1) * K + k] < thr) return isnan(d) ? PAIR_NAN_ONLY : PAIR_OFF;
    return d - eps[k] > 0.f || isnan(d) ? PAIR_GRAD : PAIR_OFF;
  };
  const int fwd = state(t), bwd = state(t - 1);  // this plane is `a` of pair t and `b` of pair t - 1
  const float* __restrict__ cur = hm + ((size_t)t * K + k) * hw;
  const float* __restrict__ nxt = fwd != PAIR_OFF ? hm + ((size_t)(t + 1) * K + k) * hw : cur;
  const float* __restrict__ prv = bwd != PAIR_OFF ? hm + ((size_t)(t - 1) * K + k) * hw : cur;
  float* __restrict__ g = grad + ((size_t)t * K + k) * hw;
  const float inv_hw = 1.0f / (float)hw;
  for (int i = threadIdx.x; i < hw; i += HL_THREADS) {
    const float x = __ldg(cur + i);
    float acc = 0.f;
    if (fwd == PAIR_GRAD) {
      const float y = __ldg(nxt + i);
      acc += kind == LPB_HM_MSE ? 2.f * (x - y) * inv_hw : -(y + 1e-10f) / (x + 1e-10f);
    } else if (fwd == PAIR_NAN_ONLY) {
      acc += 0.f * (x - __ldg(nxt + i));
    }
    if (bwd == PAIR_GRAD) {
      const float z = __ldg(prv + i);
      acc += kind == LPB_HM_MSE ? -2.f * (z - x) * inv_hw : logf(x + 1e-10f) - logf(z + 1e-10f) + 1.f;
    } else if (bwd == PAIR_NAN_ONLY) {
      acc += 0.f * (__ldg(prv + i) - x);
    }
    g[i] = acc * scale;
  }
}

// ---- coordinate remap ---------------------------------------------------------------------------
__global__ void remap_kernel(const float* __restrict__ in, int64_t n, int K, const float* __restrict__ tf, int per_frame,
                             int num_views, const float* __restrict__ bbox, int bbox_row_off, float inv_mh, float inv_mw,
                             float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * K) return;
  const int64_t f = idx / K;
  const int k = (int)(idx - f * K);
  const int per = K / num_views;
  const int v = min(k / per, num_views - 1);
  float x = in[2 * idx], y = in[2 * idx + 1];
  if (tf) {
    // [A | t] (2x3): undo = A^-1 (p - t)   (data/utils.py:164-167)
    const float* m = tf + (per_frame ? f * 6 : (num_views > 1 ? (int64_t)v * 6 : 0));
    const float a = m[0], b = m[1], tx = m[2], c = m[3], d = m[4], ty = m[5];
    const float idet = 1.0f / (a * d - b * c);
    const float px = x - tx, py = y - ty;
    x = (d * px - b * py) * idet;
    y = (-c * px + a * py) * idet;
  }
  const float* bb = bbox + (f + bbox_row_off) * (int64_t)(4 * num_views) + 4 * v;  // [x, y, h, w]
  out[2 * idx] = (x * inv_mw) * bb[3] + bb[0];      // data/bboxes.py:94-97
  out[2 * idx + 1] = (y * inv_mh) * bb[2] + bb[1];
}


// backward of remap_kernel: out = S * A^-1 (p - t) + b  =>  d/dp = (A^-1)^T S g
__global__ void remap_bwd_kernel(const float* __restrict__ gout, int64_t n, int K, const float* __restrict__ tf,
                                 int per_frame, int num_views, const float* __restrict__ bbox, int bbox_row_off,
                                 float inv_mh, float inv_mw, float* __restrict__ gin) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * K) return;
  const int64_t f = idx / K;
  const int k = (int)(idx - f * K);
  const int per = K / num_views;
  const int v = min(k / per, num_views - 1);
  const float* bb = bbox + (f + bbox_row_off) * (int64_t)(4 * num_views) + 4 * v;
  float gx = gout[2 * idx] * inv_mw * bb[3], gy = gout[2 * idx + 1] * inv_mh * bb[2];
  if (tf) {
    const float* m = tf + (per_frame ? f * 6 : (num_views > 1 ? (int64_t)v * 6 : 0));
    const float a = m[0], b = m[1], c = m[3], d = m[4];
    const float idet = 1.0f / (a * d - b * c);
    // A^-1 = idet * [[d, -b], [-c, a]];  transpose applied to (gx, gy)
    const float ox = (d * gx - c * gy) * idet;
    const float oy = (-b * gx + a * gy) * idet;
    gx = ox;
    gy = oy;
  }
  gin[2 * idx] = gx;
  gin[2 * idx + 1] = gy;
}

// plane softmax backward: out = p * (g - sum(g * p)) per plane; one HBM read of p and g, one write
__global__ void __launch_bounds__(HL_THREADS) plane_softmax_bwd_kernel(const float* __restrict__ p,
                                                                       const float* __restrict__ g, int hw,
                                                                       float* __restrict__ out) {
  extern __shared__ float sm[];  // pp[hw], gg[hw]
  __shared__ float red[HL_THREADS / 32];
  float* pp = sm;
  float* gg = sm + hw;
  const size_t base = (size_t)blockIdx.x * hw;
  float acc = 0.f;
  for (int i = threadIdx.x; i < hw; i += HL_THREADS) {
    const float a = __ldg(p + base + i), b = __ldg(g + base + i);
    pp[i] = a;
    gg[i] = b;
    acc = fmaf(a, b, acc);
  }
  const float dot = block_sum_256(acc, red);
  for (int i = threadIdx.x; i < hw; i += HL_THREADS) out[base + i] = pp[i] * (gg[i] - dot);
}

// ---- unsupervised losses on (T, K, 2) ------------------------------------------------------------
struct PcaDev {
  const int32_t* kp_index;
  const float* mean;
  const float* kept;
  int n_sel, n_views, centering, n_comp;
  float eps;
};

constexpr int UL_THREADS = 256;
constexpr int UL_MAX_SEL = 64;

__device__ __forceinline__ float block_sum_ul(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int k = 0; k < UL_THREADS / 32; ++k) t += red[k];
  return t;
}

// quantile(0.5) with linear interpolation over n values read through `get(i)`; also returns the
// two ranks' source positions and the interpolation fraction (for the backward pass).  Ties rank by position, as a
// stable sort orders them.  Any NaN makes the median NaN, as torch.quantile does: it sorts NaN last and takes the last
// sorted value, so both positions are the last NaN's and the fraction is 0.
template <typename Get>
__device__ float median_interp(int n, Get get, int* lo_src, int* hi_src, float* frac) {
  for (int i = n - 1; i >= 0; --i) {
    const float vi = get(i);
    if (isnan(vi)) {
      *lo_src = *hi_src = i;
      *frac = 0.f;
      return vi;
    }
  }
  const float pos = 0.5f * (float)(n - 1);
  const int lo = (int)floorf(pos), hi = (int)ceilf(pos);
  float vlo = 0.f, vhi = 0.f;
  int slo = 0, shi = 0;
  for (int i = 0; i < n; ++i) {
    const float vi = get(i);
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float vj = get(j);
      rank += (vj < vi || (vj == vi && j < i)) ? 1 : 0;
    }
    if (rank == lo) {
      vlo = vi;
      slo = i;
    }
    if (rank == hi) {
      vhi = vi;
      shi = i;
    }
  }
  *lo_src = slo;
  *hi_src = shi;
  *frac = pos - (float)lo;
  return vlo + (vhi - vlo) * (pos - (float)lo);
}

// Builds the PCA observation matrix X [rows][D] in smem for one clip and returns rows.
//   singleview: rows = T, D = 2*n_sel, X[t][2i+c] = kp[t][idx[i]][c] - center[t][c]
//   multiview:  rows = T*n_sel, D = 2*n_views, X[t*n_sel+j][2v+c] = kp[t][idx[v*n_sel+j]][c]
__device__ void pca_format(const float* __restrict__ kp, int T, int K, const PcaDev& d, float* X, float* center) {
  const int D = d.n_views > 0 ? 2 * d.n_views : 2 * d.n_sel;
  if (d.n_views > 0) {
    const int rows = T * d.n_sel;
    for (int i = threadIdx.x; i < rows * D; i += UL_THREADS) {
      const int row = i / D, col = i - row * D;
      const int t = row / d.n_sel, j = row - t * d.n_sel;
      const int v = col >> 1, c = col & 1;
      X[i] = kp[((size_t)t * K + d.kp_index[v * d.n_sel + j]) * 2 + c];
    }
  } else {
    if (d.centering != 0) {
      for (int i = threadIdx.x; i < T * 2; i += UL_THREADS) {
        const int t = i >> 1, c = i & 1;
        auto get = [&](int q) { return kp[((size_t)t * K + d.kp_index[q]) * 2 + c]; };
        float ctr;
        if (d.centering == 1) {
          float s = 0.f;
          for (int q = 0; q < d.n_sel; ++q) s += get(q);
          ctr = s / (float)d.n_sel;
        } else {
          int a, b;
          float fr;
          ctr = median_interp(d.n_sel, get, &a, &b, &fr);
        }
        center[i] = ctr;
      }
      __syncthreads();
    }
    for (int i = threadIdx.x; i < T * D; i += UL_THREADS) {
      const int t = i / D, col = i - t * D;
      const int q = col >> 1, c = col & 1;
      float v = kp[((size_t)t * K + d.kp_index[q]) * 2 + c];
      if (d.centering != 0) v -= center[2 * t + c];
      X[i] = v;
    }
  }
  __syncthreads();
}

// proj[row][c] = sum_d (X[row][d] - mean[d]) * kept[c][d]
__device__ void pca_project(const float* X, int rows, int D, const PcaDev& d, float* proj) {
  for (int i = threadIdx.x; i < rows * d.n_comp; i += UL_THREADS) {
    const int row = i / d.n_comp, c = i - row * d.n_comp;
    const float* x = X + (size_t)row * D;
    const float* vv = d.kept + (size_t)c * D;
    float s = 0.f;
    for (int k = 0; k < D; ++k) s = fmaf(x[k] - __ldg(d.mean + k), __ldg(vv + k), s);
    proj[i] = s;
  }
  __syncthreads();
}

// residual of element (row, col): x - (proj . kept[:, col] + mean[col])
__device__ __forceinline__ float pca_residual(const float* X, const float* proj, int row, int col, int D,
                                              const PcaDev& d) {
  float rp = __ldg(d.mean + col);
  for (int c = 0; c < d.n_comp; ++c) rp = fmaf(proj[row * d.n_comp + c], __ldg(d.kept + (size_t)c * D + col), rp);
  return X[(size_t)row * D + col] - rp;
}

__device__ float pca_loss_clip(const float* __restrict__ kp, int T, int K, const PcaDev& d, float* scratch, float* red) {
  const int D = d.n_views > 0 ? 2 * d.n_views : 2 * d.n_sel;
  const int rows = d.n_views > 0 ? T * d.n_sel : T;
  float* X = scratch;
  float* proj = X + (size_t)rows * D;
  float* center = proj + (size_t)rows * d.n_comp;
  pca_format(kp, T, K, d, X, center);
  pca_project(X, rows, D, d, proj);
  float acc = 0.f;
  const int npairs = rows * (D / 2);
  for (int i = threadIdx.x; i < npairs; i += UL_THREADS) {
    const int row = i / (D / 2), pr = i - row * (D / 2);
    const float rx = pca_residual(X, proj, row, 2 * pr, D, d);
    const float ry = pca_residual(X, proj, row, 2 * pr + 1, D, d);
    acc += relu_keep_nan(sqrtf(rx * rx + ry * ry) - d.eps);  // rectify_epsilon, losses.py:125-136
  }
  acc = block_sum_ul(acc, red);
  return acc / (float)npairs;
}

__global__ void __launch_bounds__(UL_THREADS) unsup_losses_fwd_kernel(const float* __restrict__ kps,
                                                                      const float* __restrict__ confs, int T, int K,
                                                                      const float* __restrict__ teps, float thr,
                                                                      int temporal_on, PcaDev sv, PcaDev mv,
                                                                      float* __restrict__ out) {
  extern __shared__ float scratch[];
  __shared__ float red[UL_THREADS / 32];
  const size_t clip = blockIdx.x;
  const float* __restrict__ kp = kps + clip * (size_t)T * K * 2;
  const float* __restrict__ cf = confs ? confs + clip * (size_t)T * K : nullptr;
  float* o = out + clip * LPB_UNSUP_NOUT;
  float lt = 0.f;
  if (temporal_on && T > 1) {
    float acc = 0.f;
    for (int i = threadIdx.x; i < (T - 1) * K; i += UL_THREADS) {
      const int t = i / K, k = i - t * K;
      const float dx = kp[((size_t)(t + 1) * K + k) * 2] - kp[((size_t)t * K + k) * 2];
      const float dy = kp[((size_t)(t + 1) * K + k) * 2 + 1] - kp[((size_t)t * K + k) * 2 + 1];
      float d = sqrtf(dx * dx + dy * dy);
      if (cf && (cf[(size_t)t * K + k] < thr || cf[(size_t)(t + 1) * K + k] < thr)) d = 0.f;  // losses.py:636-649
      acc += relu_keep_nan(d - teps[k]);
    }
    acc = block_sum_ul(acc, red);
    lt = acc / (float)((T - 1) * K);
  } else if (temporal_on) {
    lt = __int_as_float(0x7fc00000);  // mean of an empty tensor
  }
  float lsv = 0.f, lmv = 0.f;
  if (sv.n_sel > 0) lsv = pca_loss_clip(kp, T, K, sv, scratch, red);
  __syncthreads();
  if (mv.n_sel > 0) lmv = pca_loss_clip(kp, T, K, mv, scratch, red);
  if (threadIdx.x == 0) {
    o[0] = lt;
    o[1] = lsv;
    o[2] = lmv;
    o[3] = 0.f;
  }
}

// gradient of one PCA loss wrt the clip's keypoints, accumulated into gkp (smem, [T*K*2])
__device__ void pca_loss_clip_bwd(const float* __restrict__ kp, int T, int K, const PcaDev& d, float gscale,
                                  float* scratch, float* gkp) {
  const int D = d.n_views > 0 ? 2 * d.n_views : 2 * d.n_sel;
  const int rows = d.n_views > 0 ? T * d.n_sel : T;
  float* X = scratch;
  float* proj = X + (size_t)rows * D;
  float* center = proj + (size_t)rows * d.n_comp;
  float* gr = center + 2 * T;           // [rows][D] gradient wrt the residual
  float* gproj = gr + (size_t)rows * D;  // [rows][n_comp] = kept . gr
  pca_format(kp, T, K, d, X, center);
  pca_project(X, rows, D, d, proj);
  const int npairs = rows * (D / 2);
  const float g = gscale / (float)npairs;
  for (int i = threadIdx.x; i < npairs; i += UL_THREADS) {
    const int row = i / (D / 2), pr = i - row * (D / 2);
    const float rx = pca_residual(X, proj, row, 2 * pr, D, d);
    const float ry = pca_residual(X, proj, row, 2 * pr + 1, D, d);
    const float e = sqrtf(rx * rx + ry * ry);
    // autograd: relu passes the gradient where e > eps and where e is NaN, and the norm's backward (r / e) g is 0 at
    // e == 0; a NaN e makes both entries NaN (not only the NaN coordinate's)
    const float s = (isnan(e) || (e > d.eps && e > 0.f)) ? g / e : 0.f;
    gr[(size_t)row * D + 2 * pr] = rx * s;
    gr[(size_t)row * D + 2 * pr + 1] = ry * s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < rows * d.n_comp; i += UL_THREADS) {
    const int row = i / d.n_comp, c = i - row * d.n_comp;
    float s = 0.f;
    for (int k = 0; k < D; ++k) s = fmaf(gr[(size_t)row * D + k], __ldg(d.kept + (size_t)c * D + k), s);
    gproj[i] = s;
  }
  __syncthreads();
  // gX = gr - kept^T (kept gr); reuse X for gX
  for (int i = threadIdx.x; i < rows * D; i += UL_THREADS) {
    const int row = i / D, col = i - row * D;
    float s = gr[i];
    for (int c = 0; c < d.n_comp; ++c) s = fmaf(-gproj[row * d.n_comp + c], __ldg(d.kept + (size_t)c * D + col), s);
    X[i] = s;
  }
  __syncthreads();
  if (d.n_views > 0) {
    for (int i = threadIdx.x; i < rows * D; i += UL_THREADS) {
      const int row = i / D, col = i - row * D;
      const int t = row / d.n_sel, j = row - t * d.n_sel;
      const int v = col >> 1, c = col & 1;
      atomicAdd(&gkp[((size_t)t * K + d.kp_index[v * d.n_sel + j]) * 2 + c], X[i]);
    }
  } else {
    // centring: x = sel - center(sel)  =>  gsel = gX - d center/d sel applied to sum_q gX
    for (int i = threadIdx.x; i < T * 2; i += UL_THREADS) {
      const int t = i >> 1, c = i & 1;
      float tot = 0.f;
      for (int q = 0; q < d.n_sel; ++q) tot += X[(size_t)t * D + 2 * q + c];
      int lo = 0, hi = 0;
      float fr = 0.f;
      if (d.centering == 2) {
        auto get = [&](int q) { return kp[((size_t)t * K + d.kp_index[q]) * 2 + c]; };
        median_interp(d.n_sel, get, &lo, &hi, &fr);
      }
      for (int q = 0; q < d.n_sel; ++q) {
        float gq = X[(size_t)t * D + 2 * q + c];
        if (d.centering == 1) gq -= tot / (float)d.n_sel;
        if (d.centering == 2) gq -= tot * ((q == lo ? 1.f - fr : 0.f) + (q == hi ? fr : 0.f));
        atomicAdd(&gkp[((size_t)t * K + d.kp_index[q]) * 2 + c], gq);
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(UL_THREADS) unsup_losses_bwd_kernel(const float* __restrict__ kps,
                                                                      const float* __restrict__ confs, int T, int K,
                                                                      const float* __restrict__ teps, float thr,
                                                                      int temporal_on, PcaDev sv, PcaDev mv,
                                                                      const float* __restrict__ gout,
                                                                      float* __restrict__ gkps) {
  extern __shared__ float smem[];
  const size_t clip = blockIdx.x;
  const float* __restrict__ kp = kps + clip * (size_t)T * K * 2;
  const float* __restrict__ cf = confs ? confs + clip * (size_t)T * K : nullptr;
  const float* go = gout + clip * LPB_UNSUP_NOUT;
  float* gkp = smem;                        // [T*K*2]
  float* scratch = smem + (size_t)T * K * 2;
  for (int i = threadIdx.x; i < T * K * 2; i += UL_THREADS) gkp[i] = 0.f;
  __syncthreads();
  if (temporal_on && T > 1 && go[0] != 0.f) {
    const float g = go[0] / (float)((T - 1) * K);
    for (int i = threadIdx.x; i < (T - 1) * K; i += UL_THREADS) {
      const int t = i / K, k = i - t * K;
      const float dx = kp[((size_t)(t + 1) * K + k) * 2] - kp[((size_t)t * K + k) * 2];
      const float dy = kp[((size_t)(t + 1) * K + k) * 2 + 1] - kp[((size_t)t * K + k) * 2 + 1];
      const float d = sqrtf(dx * dx + dy * dy);
      const bool masked = cf && (cf[(size_t)t * K + k] < thr || cf[(size_t)(t + 1) * K + k] < thr);
      if (isnan(d)) {
        // autograd: the norm's backward (dx, dy) * (g / d) is NaN in both coordinates, whatever the mask and the
        // rectification pass on (a masked pair gets 0 * NaN)
        const float nan = __int_as_float(0x7fc00000);
        atomicAdd(&gkp[((size_t)(t + 1) * K + k) * 2], nan);
        atomicAdd(&gkp[((size_t)(t + 1) * K + k) * 2 + 1], nan);
        atomicAdd(&gkp[((size_t)t * K + k) * 2], nan);
        atomicAdd(&gkp[((size_t)t * K + k) * 2 + 1], nan);
      } else if (!masked && d > teps[k] && d > 0.f) {
        const float sx = g * dx / d, sy = g * dy / d;
        atomicAdd(&gkp[((size_t)(t + 1) * K + k) * 2], sx);
        atomicAdd(&gkp[((size_t)(t + 1) * K + k) * 2 + 1], sy);
        atomicAdd(&gkp[((size_t)t * K + k) * 2], -sx);
        atomicAdd(&gkp[((size_t)t * K + k) * 2 + 1], -sy);
      }
    }
    __syncthreads();
  }
  if (sv.n_sel > 0 && go[1] != 0.f) pca_loss_clip_bwd(kp, T, K, sv, go[1], scratch, gkp);
  if (mv.n_sel > 0 && go[2] != 0.f) pca_loss_clip_bwd(kp, T, K, mv, go[2], scratch, gkp);
  __syncthreads();
  float* __restrict__ dst = gkps + clip * (size_t)T * K * 2;
  for (int i = threadIdx.x; i < T * K * 2; i += UL_THREADS) dst[i] = gkp[i];
}

static int make_pca_dev(const lpb_pca_desc* d, int K, PcaDev* out, const char* name) {
  PcaDev p{};
  if (d && d->n_sel > 0) {
    // no components: the reprojection is the mean and `kept` (0 x D, an empty tensor's null pointer) is never read
    LPB_REQUIRE(d->kp_index && d->mean && (d->kept || d->n_components == 0), "%s: null pointer in pca desc", name);
    LPB_REQUIRE(d->n_sel <= UL_MAX_SEL * 4 && d->n_components >= 0 && d->n_views >= 0 && d->n_views <= 32,
                "%s: bad pca desc n_sel=%d n_components=%d n_views=%d", name, d->n_sel, d->n_components, d->n_views);
    LPB_REQUIRE(d->centering >= 0 && d->centering <= 2 && !(d->n_views > 0 && d->centering != 0),
                "%s: bad centering", name);
    p.kp_index = d->kp_index;
    p.mean = d->mean;
    p.kept = d->kept;
    p.n_sel = d->n_sel;
    p.n_views = d->n_views;
    p.centering = d->centering;
    p.n_comp = d->n_components;
    p.eps = d->epsilon;
  }
  (void)K;
  *out = p;
  return LPB_OK;
}

static size_t pca_scratch_floats(const PcaDev& p, int T, bool bwd) {
  if (p.n_sel == 0) return 0;
  const size_t D = p.n_views > 0 ? 2 * p.n_views : 2 * p.n_sel;
  const size_t rows = p.n_views > 0 ? (size_t)T * p.n_sel : (size_t)T;
  size_t f = rows * D + rows * p.n_comp + 2 * (size_t)T;
  if (bwd) f += rows * D + rows * p.n_comp;
  return f;
}

}  // namespace lpb

extern "C" int lpb_heatmap_loss_fwd(const float* targets, const float* preds, int64_t n_planes, int h, int w, int kind,
                                    float* out, float* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(targets && preds && out && workspace, "heatmap_loss_fwd: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && kind >= 0 && kind <= 2, "heatmap_loss_fwd: bad shape/kind");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_loss_fwd: bad n_planes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  heatmap_loss_plane_kernel<<<(unsigned)n_planes, HL_THREADS, 0, s>>>(targets, preds, h * w, kind, workspace);
  heatmap_loss_final_kernel<<<1, HL_THREADS, 0, s>>>(workspace, n_planes, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_heatmap_loss_bwd(const float* targets, const float* preds, int64_t n_planes, int h, int w, int kind,
                                    const float* workspace, const float* fwd_out, const float* grad_out,
                                    float* grad_preds, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(targets && preds && workspace && fwd_out && grad_out && grad_preds, "heatmap_loss_bwd: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && kind >= 0 && kind <= 2, "heatmap_loss_bwd: bad shape/kind");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_loss_bwd: bad n_planes");
  heatmap_loss_bwd_kernel<<<(unsigned)n_planes, HL_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      targets, preds, h * w, kind, workspace, fwd_out, grad_out, grad_preds);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_heatmap_mse_from_keypoints_fwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                                  int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                                  float sigma, float* out, float* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && preds && out && workspace, "heatmap_mse_from_keypoints_fwd: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "heatmap_mse_from_keypoints_fwd: bad shape");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_mse_from_keypoints_fwd: bad n_planes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)(oh + ow + 16) * sizeof(float);
  const TargetGeom tg = target_geom(img_height, img_width, oh, ow, sigma);
  heatmap_mse_from_kp_kernel<<<(unsigned)n_planes, HL_THREADS, smem, s>>>(keypoints, visibility, preds, tg.sx, tg.sy, oh, ow,
                                                                          tg.two_s2, workspace);
  heatmap_loss_final_kernel<<<1, HL_THREADS, 0, s>>>(workspace, n_planes, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_remap_keypoints(const float* keypoints_in, int64_t n, int K, const float* transforms, int per_frame,
                                   int num_views, const float* bbox, int64_t n_bbox, float model_height,
                                   float model_width, float* keypoints_out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints_in && keypoints_out && bbox, "remap_keypoints: null pointer");
  LPB_REQUIRE(n >= 0 && K >= 1 && num_views >= 1 && K % num_views == 0, "remap_keypoints: bad shape n=%lld K=%d V=%d",
              (long long)n, K, num_views);
  LPB_REQUIRE(n_bbox == n || n_bbox == n + 4, "remap_keypoints: bbox rows %lld vs %lld frames", (long long)n_bbox,
              (long long)n);
  LPB_REQUIRE(model_height > 0.f && model_width > 0.f, "remap_keypoints: bad model dims");
  if (n == 0) return LPB_OK;
  const int64_t total = n * K;
  remap_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      keypoints_in, n, K, transforms, per_frame, num_views, bbox, n_bbox == n ? 0 : 2, 1.0f / model_height,
      1.0f / model_width, keypoints_out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_unsup_losses_fwd(const float* keypoints, const float* confidences, int64_t n_clips, int T, int K,
                                    const float* temporal_eps, float prob_threshold, int temporal_enabled,
                                    const lpb_pca_desc* pca_singleview, const lpb_pca_desc* pca_multiview, float* out,
                                    void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && out, "unsup_losses_fwd: null pointer");
  LPB_REQUIRE(n_clips >= 1 && n_clips < (1ll << 31) && T >= 1 && K >= 1, "unsup_losses_fwd: bad shape");
  LPB_REQUIRE(!temporal_enabled || temporal_eps, "unsup_losses_fwd: temporal enabled without epsilon");
  PcaDev sv, mv;
  int rc = make_pca_dev(pca_singleview, K, &sv, "unsup_losses_fwd(singleview)");
  if (rc) return rc;
  rc = make_pca_dev(pca_multiview, K, &mv, "unsup_losses_fwd(multiview)");
  if (rc) return rc;
  size_t fl = pca_scratch_floats(sv, T, false);
  const size_t fl2 = pca_scratch_floats(mv, T, false);
  fl = fl > fl2 ? fl : fl2;
  const size_t smem = (fl + 4) * sizeof(float);
  LPB_TRY(set_dynamic_smem(unsup_losses_fwd_kernel, smem, "unsup_losses_fwd"));
  unsup_losses_fwd_kernel<<<(unsigned)n_clips, UL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, confidences, T, K, temporal_eps, prob_threshold, temporal_enabled, sv, mv, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_unsup_losses_bwd(const float* keypoints, const float* confidences, int64_t n_clips, int T, int K,
                                    const float* temporal_eps, float prob_threshold, int temporal_enabled,
                                    const lpb_pca_desc* pca_singleview, const lpb_pca_desc* pca_multiview,
                                    const float* grad_out, float* grad_keypoints, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && grad_out && grad_keypoints, "unsup_losses_bwd: null pointer");
  LPB_REQUIRE(n_clips >= 1 && n_clips < (1ll << 31) && T >= 1 && K >= 1, "unsup_losses_bwd: bad shape");
  LPB_REQUIRE(!temporal_enabled || temporal_eps, "unsup_losses_bwd: temporal enabled without epsilon");
  PcaDev sv, mv;
  int rc = make_pca_dev(pca_singleview, K, &sv, "unsup_losses_bwd(singleview)");
  if (rc) return rc;
  rc = make_pca_dev(pca_multiview, K, &mv, "unsup_losses_bwd(multiview)");
  if (rc) return rc;
  size_t fl = pca_scratch_floats(sv, T, true);
  const size_t fl2 = pca_scratch_floats(mv, T, true);
  fl = fl > fl2 ? fl : fl2;
  const size_t smem = (fl + (size_t)T * K * 2 + 4) * sizeof(float);
  LPB_TRY(set_dynamic_smem(unsup_losses_bwd_kernel, smem, "unsup_losses_bwd"));
  unsup_losses_bwd_kernel<<<(unsigned)n_clips, UL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, confidences, T, K, temporal_eps, prob_threshold, temporal_enabled, sv, mv, grad_out, grad_keypoints);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_temporal_heatmap_loss_fwd(const float* heatmaps, const float* confidences, int64_t T, int K, int h,
                                             int w, int kind, const float* eps, float prob_threshold, float* out,
                                             float* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && confidences && eps && out && workspace, "temporal_heatmap_loss_fwd: null pointer");
  LPB_REQUIRE(T >= 2 && K >= 1 && h >= 1 && w >= 1 && (kind == LPB_HM_MSE || kind == LPB_HM_KL) &&
                  (T - 1) * K < (1ll << 31),
              "temporal_heatmap_loss_fwd: bad shape/kind");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  temporal_heatmap_pair_kernel<<<(unsigned)((T - 1) * K), HL_THREADS, 0, s>>>(heatmaps, K, h * w, kind, workspace);
  temporal_heatmap_final_kernel<<<1, HL_THREADS, 0, s>>>(workspace, confidences, (int)T, K, eps, prob_threshold, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_temporal_heatmap_loss_bwd(const float* heatmaps, const float* confidences, const float* workspace,
                                             int64_t T, int K, int h, int w, int kind, const float* eps,
                                             float prob_threshold, const float* grad_out, float* grad_heatmaps,
                                             void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && confidences && workspace && eps && grad_out && grad_heatmaps, "temporal_heatmap_loss_bwd: null pointer");
  LPB_REQUIRE(T >= 2 && K >= 1 && h >= 1 && w >= 1 && (kind == LPB_HM_MSE || kind == LPB_HM_KL) && T * K < (1ll << 31),
              "temporal_heatmap_loss_bwd: bad shape/kind");
  temporal_heatmap_bwd_kernel<<<(unsigned)(T * K), HL_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      heatmaps, confidences, workspace, (int)T, K, h * w, kind, eps, prob_threshold, grad_out, grad_heatmaps);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_heatmap_mse_from_keypoints_bwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                                  int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                                  float sigma, const float* fwd_out, const float* grad_out,
                                                  float* grad_preds, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && preds && fwd_out && grad_out && grad_preds, "heatmap_mse_from_keypoints_bwd: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "heatmap_mse_from_keypoints_bwd: bad shape");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_mse_from_keypoints_bwd: bad n_planes");
  const size_t smem = (size_t)(oh + ow + 16) * sizeof(float);
  const TargetGeom tg = target_geom(img_height, img_width, oh, ow, sigma);
  heatmap_mse_from_kp_bwd_kernel<<<(unsigned)n_planes, HL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, visibility, preds, tg.sx, tg.sy, oh, ow, tg.two_s2, fwd_out, grad_out, grad_preds);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_heatmap_loss_from_keypoints_fwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                                   int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                                   float sigma, int kind, float* out, float* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(kind >= 0 && kind <= 2, "heatmap_loss_from_keypoints_fwd: bad kind %d", kind);
  if (kind == LPB_HM_MSE)
    return lpb_heatmap_mse_from_keypoints_fwd(keypoints, visibility, preds, n_planes, img_height, img_width, oh, ow, sigma,
                                              out, workspace, stream);
  LPB_REQUIRE(keypoints && preds && out && workspace, "heatmap_loss_from_keypoints_fwd: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "heatmap_loss_from_keypoints_fwd: bad shape");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_loss_from_keypoints_fwd: bad n_planes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)(oh + ow + 16) * sizeof(float);
  const TargetGeom tg = target_geom(img_height, img_width, oh, ow, sigma);
  heatmap_div_from_kp_kernel<<<(unsigned)n_planes, HL_THREADS, smem, s>>>(keypoints, visibility, preds, tg.sx, tg.sy, oh, ow,
                                                                          tg.two_s2, kind, workspace);
  heatmap_loss_final_kernel<<<1, HL_THREADS, 0, s>>>(workspace, n_planes, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_heatmap_loss_from_keypoints_bwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                                   int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                                   float sigma, int kind, const float* fwd_out, const float* grad_out,
                                                   float* grad_preds, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(kind >= 0 && kind <= 2, "heatmap_loss_from_keypoints_bwd: bad kind %d", kind);
  if (kind == LPB_HM_MSE)
    return lpb_heatmap_mse_from_keypoints_bwd(keypoints, visibility, preds, n_planes, img_height, img_width, oh, ow, sigma,
                                              fwd_out, grad_out, grad_preds, stream);
  LPB_REQUIRE(keypoints && preds && fwd_out && grad_out && grad_preds, "heatmap_loss_from_keypoints_bwd: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "heatmap_loss_from_keypoints_bwd: bad shape");
  LPB_REQUIRE(n_planes >= 1 && n_planes < (1ll << 31), "heatmap_loss_from_keypoints_bwd: bad n_planes");
  const size_t smem = (size_t)(oh + ow + 16) * sizeof(float);
  const TargetGeom tg = target_geom(img_height, img_width, oh, ow, sigma);
  heatmap_div_from_kp_bwd_kernel<<<(unsigned)n_planes, HL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, visibility, preds, tg.sx, tg.sy, oh, ow, tg.two_s2, kind, fwd_out, grad_out, grad_preds);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_remap_keypoints_bwd(const float* grad_out, int64_t n, int K, const float* transforms, int per_frame,
                                       int num_views, const float* bbox, int64_t n_bbox, float model_height,
                                       float model_width, float* grad_in, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(grad_out && grad_in && bbox, "remap_keypoints_bwd: null pointer");
  LPB_REQUIRE(n >= 0 && K >= 1 && num_views >= 1 && K % num_views == 0, "remap_keypoints_bwd: bad shape");
  LPB_REQUIRE(n_bbox == n || n_bbox == n + 4, "remap_keypoints_bwd: bbox rows %lld vs %lld frames", (long long)n_bbox,
              (long long)n);
  if (n == 0) return LPB_OK;
  const int64_t total = n * K;
  remap_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      grad_out, n, K, transforms, per_frame, num_views, bbox, n_bbox == n ? 0 : 2, 1.0f / model_height, 1.0f / model_width,
      grad_in);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_plane_softmax_bwd(const float* probs, const float* grad_probs, int64_t n_planes, int hw,
                                     float* grad_logits, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(probs && grad_probs && grad_logits, "plane_softmax_bwd: null pointer");
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31) && hw >= 1, "plane_softmax_bwd: bad shape");
  if (n_planes == 0) return LPB_OK;
  const size_t smem = (size_t)2 * hw * sizeof(float);
  LPB_TRY(set_dynamic_smem(plane_softmax_bwd_kernel, smem, "plane_softmax_bwd"));
  plane_softmax_bwd_kernel<<<(unsigned)n_planes, HL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(probs, grad_probs, hw,
                                                                                                      grad_logits);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
