// Gaussian target generation and windowed heatmap evaluation.
//   generate_heatmaps            lightning_pose/data/heatmaps.py:11-87
//   evaluate_heatmaps_at_location lightning_pose/data/heatmaps.py:90-142
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "targets.cuh"

namespace lpb {

constexpr int TGT_THREADS = 128;

__global__ void __launch_bounds__(TGT_THREADS) generate_heatmaps_kernel(const float* __restrict__ kp,
                                                                        const int32_t* __restrict__ vis,
                                                                        float sx, float sy, int oh, int ow,
                                                                        float two_s2, float* __restrict__ out) {
  extern __shared__ float sm[];  // ex[ow], ey[oh], red[8]
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;
  const size_t plane = blockIdx.x;
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  float* __restrict__ dst = out + plane * (size_t)oh * ow;
  const int n = oh * ow;
  if (tp.mode != TARGET_GAUSS) {
    const float v = (tp.mode == TARGET_UNIFORM) ? 1.0f / (float)n : 0.f;
    for (int i = threadIdx.x; i < n; i += TGT_THREADS) dst[i] = v;
    return;
  }
  const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, TGT_THREADS);
  for (int i = threadIdx.x; i < n; i += TGT_THREADS) {
    const int r = i / ow, c = i - r * ow;
    dst[i] = ex[c] * ey[r] * norm;
  }
}


// d loss / d keypoints of the normalised Gaussian:  d g_rc / d x = g_rc (c - xbar) / sigma^2 with
// xbar = sum g c  (softmax-like Jacobian); chain through the clamp (zero outside [-1, size+1]) and the
// image->grid scale.  Used by keep_gradients=True (lightning_pose/data/heatmaps.py:37-40).
// The sums take c and r relative to the grid point (c0, r0) nearest the centre: sum G g (c - xbar) is unchanged by the
// shift, and its two terms stay of the size of the result instead of c times larger (in fp32, sum G g c - xbar sum G g
// at c ~ 190 loses the gradient of a sharp target, and most of it when the centre is clamped off the grid's edge).
__global__ void __launch_bounds__(TGT_THREADS) generate_heatmaps_bwd_kernel(const float* __restrict__ kp,
                                                                            const int32_t* __restrict__ vis,
                                                                            const float* __restrict__ gout, float sx,
                                                                            float sy, int oh, int ow, float two_s2,
                                                                            float* __restrict__ gkp) {
  extern __shared__ float sm[];
  float* ex = sm;
  float* ey = sm + ow;
  float* red = ey + oh;  // 16 floats
  const size_t plane = blockIdx.x;
  const float xr = kp[2 * plane], yr = kp[2 * plane + 1];
  const TargetPlane tp = classify_target(kp, vis, plane, sx, sy, oh, ow);
  if (tp.mode != TARGET_GAUSS) {
    if (threadIdx.x == 0) gkp[2 * plane] = gkp[2 * plane + 1] = 0.f;
    return;
  }
  const float norm = target_axis_factors(tp, oh, ow, two_s2, ex, ey, red, TGT_THREADS);
  const float* __restrict__ g = gout + plane * (size_t)oh * ow;
  // (a NaN centre gives NaN sums whatever c0, r0 are)
  const int c0 = (int)fminf(fmaxf(rintf(tp.x), 0.f), (float)(ow - 1)), r0 = (int)fminf(fmaxf(rintf(tp.y), 0.f), (float)(oh - 1));
  // sum G g, sum G g (c - c0), sum G g (r - r0), sum g (c - c0), sum g (r - r0)
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, m1 = 0.f, m2 = 0.f;
  for (int i = threadIdx.x; i < oh * ow; i += TGT_THREADS) {
    const int r = i / ow, c = i - r * ow;
    const float gv = ex[c] * ey[r] * norm;
    const float Gg = g[i] * gv;
    s0 += Gg;
    s1 = fmaf(Gg, (float)(c - c0), s1);
    s2 = fmaf(Gg, (float)(r - r0), s2);
    m1 = fmaf(gv, (float)(c - c0), m1);
    m2 = fmaf(gv, (float)(r - r0), m2);
  }
  float vals[5] = {s0, s1, s2, m1, m2};
  __shared__ float acc[5][TGT_THREADS / 32];
  for (int k = 0; k < 5; ++k) {
    const float v = warp_sum(vals[k]);
    if ((threadIdx.x & 31) == 0) acc[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t[5];
    for (int k = 0; k < 5; ++k) {
      t[k] = 0.f;
      for (int q = 0; q < TGT_THREADS / 32; ++q) t[k] += acc[k][q];
    }
    const float inv_s2 = 2.0f / two_s2;
    const float xs = xr * sx, ys = yr * sy;
    const bool inx = xs >= -1.f && xs <= (float)(ow + 1), iny = ys >= -1.f && ys <= (float)(oh + 1);
    gkp[2 * plane] = inx ? (t[1] - t[3] * t[0]) * inv_s2 * sx : 0.f;
    gkp[2 * plane + 1] = iny ? (t[2] - t[4] * t[0]) * inv_s2 * sy : 0.f;
  }
}

__global__ void evaluate_at_location_kernel(const float* __restrict__ heat, const float* __restrict__ locs,
                                            int64_t n_planes, int h, int w, int radius, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t plane = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (plane >= n_planes) return;
  const float* hp = heat + plane * (size_t)h * w;
  const int cx = (int)locs[2 * plane], cy = (int)locs[2 * plane + 1];  // trunc toward zero (:130-131)
  const int cw = 2 * radius + 1;
  float acc = 0.f;
  for (int k = lane; k < cw * cw; k += 32) {
    const int y = cy + k / cw - radius, x = cx + k % cw - radius;
    if (y >= 0 && y < h && x >= 0 && x < w) acc += hp[(size_t)y * w + x];
  }
  acc = warp_sum(acc);
  if (lane == 0) out[plane] = acc;
}

}  // namespace lpb

namespace lpb {
// labeled keypoints that an augmentation moved out of the frame become NaN (both coordinates), so that their target
// plane is all-zero and the supervised losses skip them  (lightning_pose/data/datasets.py:496-508)
__global__ void keypoints_mask_oob_kernel(const float* __restrict__ kp, int64_t n, float height, float width,
                                          float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = kp[2 * i], y = kp[2 * i + 1];
  const bool oob = x < 0.f || y < 0.f || x >= width || y >= height;
  const float nanv = __int_as_float(0x7fc00000);
  out[2 * i] = oob ? nanv : x;
  out[2 * i + 1] = oob ? nanv : y;
}
}  // namespace lpb

extern "C" int lpb_keypoints_mask_oob(const float* keypoints, int64_t n_keypoints, float img_height, float img_width,
                                      float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && out && n_keypoints >= 0 && img_height > 0.f && img_width > 0.f, "keypoints_mask_oob: bad arguments");
  if (n_keypoints == 0) return LPB_OK;
  keypoints_mask_oob_kernel<<<(unsigned)((n_keypoints + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      keypoints, n_keypoints, img_height, img_width, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_generate_heatmaps(const float* keypoints, const int32_t* visibility, int64_t n_planes,
                                     float img_height, float img_width, int oh, int ow, float sigma, float* out,
                                     void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && out, "generate_heatmaps: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "generate_heatmaps: bad shape oh=%d ow=%d sigma=%f", oh, ow, sigma);
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "generate_heatmaps: bad n_planes");
  if (n_planes == 0) return LPB_OK;
  const size_t smem = (size_t)(oh + ow + 8) * sizeof(float);
  generate_heatmaps_kernel<<<(unsigned)n_planes, TGT_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, visibility, (float)((double)ow / (double)img_width), (float)((double)oh / (double)img_height), oh, ow,
      (float)(2.0 * (double)sigma * (double)sigma), out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_evaluate_heatmaps_at_location(const float* heatmaps, const float* locs, int64_t n_planes, int h,
                                                 int w, int radius, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && locs && out, "evaluate_heatmaps_at_location: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && radius >= 0 && radius <= 64, "evaluate_heatmaps_at_location: bad shape");
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 33), "evaluate_heatmaps_at_location: bad n_planes");
  if (n_planes == 0) return LPB_OK;
  const int wpb = 4;
  evaluate_at_location_kernel<<<(unsigned)((n_planes + wpb - 1) / wpb), wpb * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      heatmaps, locs, n_planes, h, w, radius, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_generate_heatmaps_bwd(const float* keypoints, const int32_t* visibility, const float* grad_out,
                                         int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                         float sigma, float* grad_keypoints, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && grad_out && grad_keypoints, "generate_heatmaps_bwd: null pointer");
  LPB_REQUIRE(oh >= 1 && ow >= 1 && oh + ow < 8000 && sigma > 0.f && img_height > 0.f && img_width > 0.f,
              "generate_heatmaps_bwd: bad shape");
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "generate_heatmaps_bwd: bad n_planes");
  if (n_planes == 0) return LPB_OK;
  const size_t smem = (size_t)(oh + ow + 16) * sizeof(float);
  generate_heatmaps_bwd_kernel<<<(unsigned)n_planes, TGT_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      keypoints, visibility, grad_out, (float)((double)ow / (double)img_width), (float)((double)oh / (double)img_height),
      oh, ow, (float)(2.0 * (double)sigma * (double)sigma), grad_keypoints);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
