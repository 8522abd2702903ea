// Crop-zoom inference (SURVEY 8f-4, bbox mode): detector keypoints -> per-frame boxes -> rolling-median smoothing ->
// per-frame crop + resize of the decoded frames, all on the device.
// References (lightning_pose, commit f54c477):
//   _calculate_bbox_size / _compute_bbox_df   utils/cropzoom.py:31-143    -> bboxes_kernel
//   smooth_bbox (rolling median)              utils/cropzoom.py:355-402   -> rolling_median_kernel
//   crop_and_resize_frames                    data/bboxes.py:291-343      -> crop_kernel
//   bbox-row cursor + last-row padding        data/video/dali.py:332-380, data/video/pynvvc.py:266-283
// The reference normalises every full-resolution frame to fp32, then loops over the frames in Python (one slice, one
// F.interpolate and one small host-built tensor per frame).  crop_kernel reads the uint8 surface directly, touches only
// the pixels its bilinear taps need, and normalises on the way out: one pass, no host sync, graph-capturable.
#include <cuda_bf16.h>

#include <cmath>
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {

// ---- crop + resize + normalise --------------------------------------------------------------------------------------
struct CropParams {
  const void* in;         // uint8 [F, H, W, 3] or fp32 [F, 3, H, W]
  const float* boxes;     // [n_boxes, 4] x, y, h, w
  const int64_t* cursor;  // device row cursor or NULL
  void* out;
  float* boxes_out;       // [F, 4] x1, y1, y2 - y1, x2 - x1
  int64_t n_boxes, row0;
  int F, H, W, OH, OW;
  float scale[3], shift[3];  // out = px * scale + shift (uint8 input only)
  // ragged arena (uint8 input only): frame f in slot f, its size from the video table at row *cursor + f
  const int64_t* videos;     // [n_videos][3]: first row, H, W
  int64_t slot_bytes;
  int n_videos;
};

// Python's int() of a float: truncation toward zero.  Clamped first so that the conversion is defined; far outside any
// frame either way.
__device__ __forceinline__ long long trunc_ll(float v) { return (long long)fminf(fmaxf(v, -1e15f), 1e15f); }

// Clamp of crop_and_resize_frames (data/bboxes.py:321-326) for frame f.  Two deliberate divergences, where the reference
// raises: an origin at or past the far edge is clamped to the last pixel (a one-pixel crop), and a row holding a NaN or
// an infinity is the whole frame.
// frame f of H x W pixels.
__device__ __forceinline__ void crop_box(const CropParams& P, int f, int H, int W, int& x1, int& y1, int& x2, int& y2) {
  int64_t r = (P.cursor ? *P.cursor : P.row0) + f;
  r = r < 0 ? 0 : (r > P.n_boxes - 1 ? P.n_boxes - 1 : r);  // past the end: the final row (dali.py:355-361)
  const float bx = P.boxes[r * 4 + 0], by = P.boxes[r * 4 + 1], bh = P.boxes[r * 4 + 2], bw = P.boxes[r * 4 + 3];
  if (!(isfinite(bx) && isfinite(by) && isfinite(bh) && isfinite(bw))) {
    x1 = 0, y1 = 0, x2 = W, y2 = H;
    return;
  }
  const long long xi = trunc_ll(bx), yi = trunc_ll(by);
  const long long xa = min(max(0LL, xi), (long long)W - 1), ya = min(max(0LL, yi), (long long)H - 1);
  x1 = (int)xa, y1 = (int)ya;
  x2 = (int)max(xa + 1, min((long long)W, xi + trunc_ll(bw)));  // far edge from the UNclamped origin
  y2 = (int)max(ya + 1, min((long long)H, yi + trunc_ll(bh)));
}

// channel c of pixel (y, x) of one H x W frame at img: fp32 [3, H, W] or uint8 [H, W, 3]
template <bool IN_F32>
__device__ __forceinline__ float load_px(const void* img, int H, int W, int c, int y, int x) {
  if (IN_F32) return static_cast<const float*>(img)[((size_t)c * H + y) * W + x];
  return (float)static_cast<const uint8_t*>(img)[((size_t)y * W + x) * 3 + c];
}

// grid (x-blocks, F): each block computes its frame's box, then strides over that frame's output pixels.  RAGGED: the
// frame is slot f of a uint8 arena and its size that of its video (ragged_video at row *cursor + f).
template <bool IN_F32, int LAYOUT, int FMT, bool RAGGED = false>
__global__ void __launch_bounds__(256) crop_kernel(const __grid_constant__ CropParams P) {
  const int f = blockIdx.y;
  int H = P.H, W = P.W;
  const void* img;
  if (RAGGED) {
    const int vid = ragged_video(P.videos, P.n_videos, *P.cursor + f);
    H = (int)P.videos[3 * vid + 1], W = (int)P.videos[3 * vid + 2];
    img = static_cast<const uint8_t*>(P.in) + (size_t)f * P.slot_bytes;
  } else if (IN_F32) {
    img = static_cast<const float*>(P.in) + (size_t)f * 3 * H * W;
  } else {
    img = static_cast<const uint8_t*>(P.in) + (size_t)f * H * W * 3;
  }
  int x1, y1, x2, y2;
  crop_box(P, f, H, W, x1, y1, x2, y2);
  const int ch = y2 - y1, cw = x2 - x1;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float* b = P.boxes_out + (size_t)f * 4;
    b[0] = (float)x1, b[1] = (float)y1, b[2] = (float)ch, b[3] = (float)cw;
  }
  // torch upsample_bilinear2d, align_corners=False, no scale factor: scale = in / out, src = max(scale (dst + 0.5) - 0.5, 0)
  const float ry = (float)ch / (float)P.OH, rx = (float)cw / (float)P.OW;
  const int npx = P.OH * P.OW;
  const size_t plane = (size_t)npx;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += gridDim.x * blockDim.x) {
    const int y = i / P.OW, x = i - y * P.OW;
    const float sy = fmaxf(__fsub_rn(__fmul_rn(ry, (float)y + 0.5f), 0.5f), 0.f);
    const float sx = fmaxf(__fsub_rn(__fmul_rn(rx, (float)x + 0.5f), 0.5f), 0.f);
    const int ya = min((int)sy, ch - 1), xa = min((int)sx, cw - 1);
    const int yb = ya + (ya < ch - 1), xb = xa + (xa < cw - 1);
    const float ly1 = sy - (float)ya, lx1 = sx - (float)xa, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float a = load_px<IN_F32>(img, H, W, c, y1 + ya, x1 + xa), b = load_px<IN_F32>(img, H, W, c, y1 + ya, x1 + xb);
      const float d = load_px<IN_F32>(img, H, W, c, y1 + yb, x1 + xa), e = load_px<IN_F32>(img, H, W, c, y1 + yb, x1 + xb);
      v[c] = __fadd_rn(__fmul_rn(ly0, __fadd_rn(__fmul_rn(lx0, a), __fmul_rn(lx1, b))),
                       __fmul_rn(ly1, __fadd_rn(__fmul_rn(lx0, d), __fmul_rn(lx1, e))));
      if (!IN_F32) v[c] = fmaf(v[c], P.scale[c], P.shift[c]);
    }
    if (LAYOUT == 0) {  // FCHW
      const size_t o = (size_t)f * 3 * plane + i;
#pragma unroll
      for (int c = 0; c < 3; ++c) store_fmt<FMT>(P.out, o + c * plane, v[c]);
    } else {  // FHWC
      const size_t o = ((size_t)f * plane + i) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) store_fmt<FMT>(P.out, o + c, v[c]);
    }
  }
}

// ---- boxes from keypoints ---------------------------------------------------------------------------------------------
struct BoxParams {
  const float* kp;
  float* out;
  int64_t n, row_stride;
  int point_stride, K, n_anchors, crop_h, crop_w;
  double ratio;  // > 0: crop_ratio mode; 0: fixed (crop_h, crop_w), already even
  int anchors[LPB_BBOX_MAX_ANCHORS];
};

// One thread per frame, fp64 throughout, in the reference's order: the centroid is summed in keypoint order (numpy's
// mean over axis 1 of a (frames, keypoints, 2) array), and the size's column 0 (h) is subtracted from x, column 1 (w)
// from y (cropzoom.py:135).
__global__ void __launch_bounds__(128) bboxes_kernel(const __grid_constant__ BoxParams P) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const float* row = P.kp + i * P.row_stride;
  const int na = P.n_anchors ? P.n_anchors : P.K;
  double sx = 0.0, sy = 0.0, mnx = INFINITY, mxx = -INFINITY, mny = INFINITY, mxy = -INFINITY;
  bool finite = true;
  for (int j = 0; j < na; ++j) {
    const int k = P.n_anchors ? P.anchors[j] : j;
    const double x = row[(int64_t)k * P.point_stride], y = row[(int64_t)k * P.point_stride + 1];
    finite &= isfinite(x) && isfinite(y);
    sx += x, sy += y;
    mnx = fmin(mnx, x), mxx = fmax(mxx, x), mny = fmin(mny, y), mxy = fmax(mxy, y);
  }
  float* o = P.out + i * 4;
  if (!finite) {  // the reference casts NaN to an undefined integer here: a documented divergence
    o[0] = o[1] = o[2] = o[3] = NAN;
    return;
  }
  long long h = P.crop_h, w = P.crop_w;
  if (P.ratio > 0.0) {
    long long s = (long long)ceil(fmax(mxx - mnx, mxy - mny) * P.ratio);
    s += s & 1;
    h = w = s;
  }
  const double cx = sx / na, cy = sy / na;
  o[0] = (float)(long long)(cx - (double)(h / 2));
  o[1] = (float)(long long)(cy - (double)(w / 2));
  o[2] = (float)h;
  o[3] = (float)w;
}

// ---- rolling median ---------------------------------------------------------------------------------------------------
// k-th smallest (0-based) of the non-NaN values in[lo..hi) of column c: the value whose rank range covers k.
__device__ __forceinline__ double kth_in_window(const float* in, int64_t lo, int64_t hi, int c, int k) {
  for (int64_t j = lo; j < hi; ++j) {
    const float v = in[j * 4 + c];
    if (isnan(v)) continue;
    int less = 0, equal = 0;
    for (int64_t t = lo; t < hi; ++t) {
      const float u = in[t * 4 + c];
      less += u < v;
      equal += u == v;
    }
    if (less <= k && k < less + equal) return (double)v;
  }
  return NAN;
}

// pandas rolling(window, center=True, min_periods=1).median() then .round(0): window [i + 1 + (w - 1) // 2 - w,
// i + 1 + (w - 1) // 2) clipped to the series, NaN skipped, the mean of the two middle values for an even count, round
// half to even.  A window with no value stays NaN.  One thread per (frame, column).
__global__ void __launch_bounds__(256) rolling_median_kernel(const float* __restrict__ in, int64_t n, int window,
                                                             float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * 4) return;
  const int64_t i = idx >> 2;
  const int c = (int)(idx & 3);
  const int64_t end = min(n, i + 1 + (window - 1) / 2), lo = max((int64_t)0, i + 1 + (window - 1) / 2 - window);
  int cnt = 0;
  for (int64_t j = lo; j < end; ++j) cnt += !isnan(in[j * 4 + c]);
  float r = NAN;
  if (cnt > 0) {
    const double m = (cnt & 1) ? kth_in_window(in, lo, end, c, cnt / 2)
                               : (kth_in_window(in, lo, end, c, cnt / 2 - 1) + kth_in_window(in, lo, end, c, cnt / 2)) / 2.0;
    r = (float)rint(m);
  }
  out[idx] = r;
}

}  // namespace lpb

extern "C" int lpb_frames_crop_normalize(const void* frames, int in_f32, int F, int H, int W, const float* boxes,
                                         int64_t n_boxes, const int64_t* cursor, int64_t row0, int out_h, int out_w,
                                         const float* mean3, const float* std3, int layout, int out_format, void* out,
                                         float* boxes_out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(frames && boxes && out && boxes_out && (in_f32 || (mean3 && std3)), "frames_crop_normalize: null pointer");
  LPB_REQUIRE(F >= 0 && F <= 65535 && H >= 1 && W >= 1 && out_h >= 1 && out_w >= 1 && (int64_t)out_h * out_w < (1LL << 31) &&
                  n_boxes >= 1 && row0 >= 0 && (layout == 0 || layout == 1),
              "frames_crop_normalize: bad shape/layout");
  LPB_REQUIRE(valid_out_format(out_format), "frames_crop_normalize: unknown output format %d", out_format);
  if (F == 0) return LPB_OK;
  CropParams p;
  p.in = frames, p.boxes = boxes, p.cursor = cursor, p.out = out, p.boxes_out = boxes_out;
  p.n_boxes = n_boxes, p.row0 = row0;
  p.F = F, p.H = H, p.W = W, p.OH = out_h, p.OW = out_w;
  p.videos = nullptr, p.slot_bytes = 0, p.n_videos = 0;
  for (int c = 0; c < 3; ++c) {  // mean3 / std3 are HOST arrays, as for lpb_frames_normalize
    p.scale[c] = 1.f, p.shift[c] = 0.f;
    if (in_f32) continue;
    LPB_REQUIRE(std3[c] > 0.f, "frames_crop_normalize: std must be positive");
    p.scale[c] = 1.0f / (255.0f * std3[c]);
    p.shift[c] = -mean3[c] / std3[c];
  }
  const int64_t px_blocks = ((int64_t)out_h * out_w + 255) / 256;
  dim3 grid((unsigned)(px_blocks < 64 ? px_blocks : 64), (unsigned)F);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  with_out_format(out_format, [&](auto fc) {
    constexpr int FMT = decltype(fc)::value;
    switch ((in_f32 ? 2 : 0) + layout) {
      case 0: crop_kernel<false, 0, FMT><<<grid, 256, 0, s>>>(p); break;
      case 1: crop_kernel<false, 1, FMT><<<grid, 256, 0, s>>>(p); break;
      case 2: crop_kernel<true, 0, FMT><<<grid, 256, 0, s>>>(p); break;
      default: crop_kernel<true, 1, FMT><<<grid, 256, 0, s>>>(p); break;
    }
  });
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_frames_crop_normalize_ragged(const uint8_t* arena, int64_t slot_bytes, int F, const int64_t* cursor,
                                                const int64_t* videos, const int64_t* videos_host, int n_videos,
                                                const float* boxes, int64_t n_boxes, int out_h, int out_w, const float* mean3,
                                                const float* std3, int layout, int out_format, void* out, float* boxes_out,
                                                void* stream) {
  using namespace lpb;
  LPB_REQUIRE(arena && cursor && videos && videos_host && boxes && mean3 && std3 && out && boxes_out,
              "frames_crop_normalize_ragged: null pointer");
  LPB_REQUIRE(out_h >= 1 && out_w >= 1 && (int64_t)out_h * out_w < (1LL << 31) && n_boxes >= 1 && (layout == 0 || layout == 1),
              "frames_crop_normalize_ragged: bad shape/layout");
  LPB_REQUIRE(valid_out_format(out_format), "frames_crop_normalize_ragged: unknown output format %d", out_format);
  LPB_TRY(check_ragged("frames_crop_normalize_ragged", arena, slot_bytes, F, videos, videos_host, n_videos));
  CropParams p;
  for (int c = 0; c < 3; ++c) {  // HOST arrays, as for lpb_frames_normalize
    LPB_REQUIRE(std3[c] > 0.f, "frames_crop_normalize_ragged: std must be positive");
    p.scale[c] = 1.0f / (255.0f * std3[c]);
    p.shift[c] = -mean3[c] / std3[c];
  }
  if (F == 0) return LPB_OK;
  p.in = arena, p.boxes = boxes, p.cursor = cursor, p.out = out, p.boxes_out = boxes_out;
  p.n_boxes = n_boxes, p.row0 = 0;
  p.F = F, p.H = 0, p.W = 0, p.OH = out_h, p.OW = out_w;
  p.videos = videos, p.slot_bytes = slot_bytes, p.n_videos = n_videos;
  const int64_t px_blocks = ((int64_t)out_h * out_w + 255) / 256;
  dim3 grid((unsigned)(px_blocks < 64 ? px_blocks : 64), (unsigned)F);  // the grid of lpb_frames_crop_normalize
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  with_out_format(out_format, [&](auto fc) {
    constexpr int FMT = decltype(fc)::value;
    if (layout == 0) crop_kernel<false, 0, FMT, true><<<grid, 256, 0, s>>>(p);
    else crop_kernel<false, 1, FMT, true><<<grid, 256, 0, s>>>(p);
  });
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_bboxes_from_keypoints(const float* keypoints, int64_t n, int K, int64_t row_stride, int point_stride,
                                         const int32_t* anchors, int n_anchors, double crop_ratio, int crop_height,
                                         int crop_width, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && out && (n_anchors == 0 || anchors), "bboxes_from_keypoints: null pointer");
  LPB_REQUIRE(n >= 0 && K >= 1 && point_stride >= 2 && row_stride >= (int64_t)K * point_stride && n_anchors >= 0 &&
                  n_anchors <= LPB_BBOX_MAX_ANCHORS,
              "bboxes_from_keypoints: bad shape");
  const bool ratio_mode = crop_ratio > 0.0, fixed_mode = crop_height > 0 && crop_width > 0;
  LPB_REQUIRE(ratio_mode != fixed_mode, "bboxes_from_keypoints: give either crop_ratio > 0 or crop_height, crop_width > 0, not both");
  BoxParams p;
  p.kp = keypoints, p.out = out, p.n = n, p.row_stride = row_stride, p.point_stride = point_stride, p.K = K;
  p.n_anchors = n_anchors;
  for (int j = 0; j < n_anchors; ++j) {  // HOST array
    LPB_REQUIRE(anchors[j] >= 0 && anchors[j] < K, "bboxes_from_keypoints: anchor index out of range");
    p.anchors[j] = anchors[j];
  }
  p.ratio = ratio_mode ? crop_ratio : 0.0;
  p.crop_h = ratio_mode ? 0 : crop_height + crop_height % 2;  // even sizes (cropzoom.py:124-126)
  p.crop_w = ratio_mode ? 0 : crop_width + crop_width % 2;
  if (n == 0) return LPB_OK;
  bboxes_kernel<<<(unsigned)((n + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_bboxes_rolling_median(const float* bboxes, int64_t n, int window, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(bboxes && out, "bboxes_rolling_median: null pointer");
  LPB_REQUIRE(bboxes != out, "bboxes_rolling_median: out must not alias the input");
  LPB_REQUIRE(n >= 0 && window >= 1, "bboxes_rolling_median: bad shape/window");
  if (n == 0) return LPB_OK;
  rolling_median_kernel<<<(unsigned)((n * 4 + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(bboxes, n, window, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
