// Device helpers shared by target generation and the fused target+loss kernel.
// Rules restated from lightning_pose/data/heatmaps.py:37-87.
#pragma once
#include "lpb_common.cuh"

namespace lpb {

enum : int { TARGET_ZERO = 0, TARGET_UNIFORM = 1, TARGET_GAUSS = 2 };

struct TargetPlane {
  int mode;
  float x, y;  // clamped heatmap-grid coordinates (NaN propagates, as torch.clamp does)
};

// Plane `plane` of keypoints kp (x, y image pixels); vis null means "visibility is None".  With a visibility, only 0, 1 and
// 2 change the plane: any other value (3, -1, ...) keeps the clamped Gaussian, NaN included.
__device__ __forceinline__ TargetPlane classify_target(const float* kp, const int32_t* vis, size_t plane, float sx, float sy,
                                                       int oh, int ow) {
  TargetPlane t;
  const float x = kp[2 * plane] * sx, y = kp[2 * plane + 1] * sy;  // :41-42
  // :43-49 - only x is tested for NaN; NaN comparisons are false
  const bool bad = isnan(x) || (x < -1.f) || (x > (float)(ow + 1)) || (y < -1.f) || (y > (float)(oh + 1));
  t.x = isnan(x) ? x : fminf(fmaxf(x, -1.f), (float)(ow + 1));  // :52-53
  t.y = isnan(y) ? y : fminf(fmaxf(y, -1.f), (float)(oh + 1));
  if (!vis) {
    t.mode = bad ? TARGET_ZERO : TARGET_GAUSS;  // :78-79
    return t;
  }
  const int v = vis[plane];
  if (v == 0) {
    t.mode = TARGET_ZERO;  // :81
  } else if (v == 1) {
    t.mode = TARGET_UNIFORM;  // :82
  } else {
    t.mode = (v == 2 && bad) ? TARGET_ZERO : TARGET_GAUSS;  // :83
  }
  return t;
}

// Fills ex[0..ow), ey[0..oh) with the separable Gaussian factors and returns 1/(sum ex * sum ey).
// `red` needs 2 * (nthreads/32) floats.  All threads of the block must call; ends synchronised.
__device__ __forceinline__ float target_axis_factors(const TargetPlane& tp, int oh, int ow, float two_s2, float* ex,
                                                     float* ey, float* red, int nthreads) {
  float px = 0.f, py = 0.f;
  for (int c = threadIdx.x; c < ow; c += nthreads) {
    const float d = (float)c - tp.x;
    const float e = expf(-(d * d) / two_s2);
    ex[c] = e;
    px += e;
  }
  for (int r = threadIdx.x; r < oh; r += nthreads) {
    const float d = (float)r - tp.y;
    const float e = expf(-(d * d) / two_s2);
    ey[r] = e;
    py += e;
  }
  px = warp_sum(px);
  py = warp_sum(py);
  const int warp = threadIdx.x >> 5, nw = nthreads >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[warp] = px;
    red[nw + warp] = py;
  }
  __syncthreads();
  float sxs = 0.f, sys = 0.f;
  for (int k = 0; k < nw; ++k) {
    sxs += red[k];
    sys += red[nw + k];
  }
  return 1.0f / (sxs * sys);
}

// grid scale (sx, sy) and 2 sigma^2 of the targets, from the image size and sigma the loss entries take
struct TargetGeom {
  float sx, sy, two_s2;
};
inline TargetGeom target_geom(float img_height, float img_width, int oh, int ow, float sigma) {
  return {(float)((double)ow / (double)img_width), (float)((double)oh / (double)img_height), (float)(2.0 * (double)sigma * (double)sigma)};
}

// ---- gradient of the fused target + MSE (lpb_heatmap_mse_from_keypoints_bwd, and the head backward's target source) --
// d loss / d pred = 2 (pred - target) / n_kept * grad_out = (pred - target) * scale on kept planes, 0 on dropped ones.
__device__ __forceinline__ float mse_target_scale(float grad_out, float n_kept) { return 2.f * grad_out / n_kept; }
// the uniform target of a plane of n pixels
__device__ __forceinline__ float mse_target_uniform(int n) { return 1.0f / (float)n; }
// One pixel: target = exc * er with exc = ex[column], er = ey[row] * norm for a Gaussian plane, and exc = 1/n, er = 1 for a
// uniform one (the fma is then exactly pred - 1/n).  The intrinsics pin the rounding: one fused multiply-add, then a
// separate multiply that no caller may fuse with what it does next, so every user gets the same bits.
__device__ __forceinline__ float mse_target_grad(int mode, float p, float exc, float er, float scale) {
  if (mode == TARGET_ZERO) return 0.f;
  return __fmul_rn(__fmaf_rn(-exc, er, p), scale);
}

}  // namespace lpb
