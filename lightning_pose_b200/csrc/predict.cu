// Batched-inference plumbing (SURVEY 8f-1): decoded keypoints of one chunk -> rows of the preallocated (N, 3K)
// prediction table, on the device, at a device-resident row cursor, so the whole chunk (head -> decode -> remap ->
// table rows -> cursor += T) is one CUDA-graph replay with no host-side offset.
// Reference: PredictionHandler.unpack_preds / make_pred_arr_undo_resize  lightning_pose/utils/predictions.py:97-144,180-206
// (torch.vstack of per-batch tuples on the host, then numpy interleaving into bp_x, bp_y, bp_likelihood columns).
// Context models add HeatmapTrackerMHCRNN.predict_step  lightning_pose/models/heatmap_tracker_mhcrnn.py:180-229,
// PrepareDALI.num_iters  lightning_pose/data/video/dali.py:519-534 and fix_context_preds_confs  predictions.py:146-177.
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {

__global__ void pack_predictions_kernel(const float* __restrict__ kp, const float* __restrict__ conf, int n, int K,
                                        float* __restrict__ table, int64_t n_rows, const int64_t* __restrict__ cursor,
                                        int64_t row0) {
  const int64_t base = cursor ? *cursor : row0;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * K) return;
  const int f = i / K, k = i - f * K;
  const int64_t row = base + f;
  if (row < 0 || row >= n_rows) return;  // rows past the end of the video (last, partly filled chunk) are dropped
  float* dst = table + (row * K + k) * 3;
  dst[0] = kp[(size_t)f * 2 * K + 2 * k];
  dst[1] = kp[(size_t)f * 2 * K + 2 * k + 1];
  dst[2] = conf[(size_t)f * K + k];
}

__global__ void advance_cursor_kernel(int64_t* cursor, int64_t n) { *cursor += n; }

// ---- context (MHCRNN) models -------------------------------------------------------------------------------------
// Row r of the reference's final table holds the prediction of frame context_source_row(r) (see lpb200.h): its reader
// produces R = T * (ceil((N - S) / T) + 1) rows, S = T + 4 (R = N when T = 1: num_iters takes its step == 1 branch,
// one window per frame, dali.py:509-510), and fix_context_preds_confs shifts them by two and fills the edges.  Frames
// >= 2 only; every row has exactly one source frame.
__device__ __forceinline__ int64_t context_source_row(int64_t r, int64_t n, int64_t t) {
  const int64_t a = n - (t + 4);
  const int64_t r_rows = t == 1 ? n : t * ((a >= 0 ? (a + t - 1) / t : -((-a) / t)) + 1);
  if (r_rows >= n) return r < 2 ? 2 : (r > n - 3 ? n - 3 : r);
  return (r >= 2 && r <= r_rows - 1) ? r : 2;  // the tail repeats preds_combined[0] = pred(2) (predictions.py:163-170)
}

// one thread per (output frame, keypoint): output frame i of the call is video frame cursor - 2 + i
__global__ void pack_context_kernel(const float* __restrict__ kp_sf, const float* __restrict__ conf_sf,
                                    const float* __restrict__ kp_mf, const float* __restrict__ conf_mf, int n, int K,
                                    const float* __restrict__ bbox, float inv_mh, float inv_mw, float* __restrict__ table,
                                    int64_t n_rows, const int64_t* __restrict__ cursor, int64_t frame0, int64_t t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * K) return;
  const int o = i / K, k = i - o * K;
  const int64_t f = (cursor ? *cursor : frame0) - 2 + o;
  if (f < 2 || f > n_rows - 2) return;  // never the source of a row (halo frames, padding frames)
  // the candidates: the frame's own row and the rows the edge rules fill (0, 1 and the last four)
  const int64_t cand[7] = {f, 0, 1, n_rows - 4, n_rows - 3, n_rows - 2, n_rows - 1};
  bool any = false;
  for (int c = 0; c < 7; ++c) any |= cand[c] >= 0 && context_source_row(cand[c], n_rows, t) == f;
  if (!any) return;
  // the more confident head wins; NaN confidences keep the single-frame head (torch.gt, heatmap_tracker_mhcrnn.py:214-220)
  const float csf = conf_sf[(size_t)o * K + k], cmf = conf_mf[(size_t)o * K + k];
  const bool mf = cmf > csf;
  const float* src = mf ? kp_mf : kp_sf;
  const float x = src[(size_t)o * 2 * K + 2 * k], y = src[(size_t)o * 2 * K + 2 * k + 1];
  const float* bb = bbox + (size_t)o * 4;  // [x, y, h, w]; same operation order as remap_kernel (bboxes.py:94-97)
  const float fx = (x * inv_mw) * bb[3] + bb[0];
  const float fy = (y * inv_mh) * bb[2] + bb[1];
  const float fc = mf ? cmf : csf;
  for (int c = 0; c < 7; ++c) {
    const int64_t r = cand[c];
    if (r < 0 || context_source_row(r, n_rows, t) != f) continue;
    float* dst = table + (r * K + k) * 3;
    dst[0] = fx;
    dst[1] = fy;
    dst[2] = fc;
  }
}

}  // namespace lpb

extern "C" int lpb_pack_predictions(const float* keypoints, const float* confidences, int n_frames, int K, float* table,
                                    int64_t n_rows, int64_t* cursor, int64_t row0, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && confidences && table && n_frames >= 0 && K >= 1 && n_rows >= 0, "pack_predictions: bad arguments");
  if (n_frames == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int total = n_frames * K;
  pack_predictions_kernel<<<(total + 255) / 256, 256, 0, s>>>(keypoints, confidences, n_frames, K, table, n_rows, cursor, row0);
  if (cursor) advance_cursor_kernel<<<1, 1, 0, s>>>(cursor, n_frames);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_pack_context_predictions(const float* kp_sf, const float* conf_sf, const float* kp_mf,
                                            const float* conf_mf, int n_frames, int K, const float* bbox,
                                            float model_height, float model_width, float* table, int64_t n_rows,
                                            int64_t* cursor, int64_t frame0, int64_t step, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(kp_sf && conf_sf && kp_mf && conf_mf && bbox && table, "pack_context_predictions: null pointer");
  LPB_REQUIRE(n_frames >= 0 && K >= 1 && (int64_t)n_frames * K < (int64_t)1 << 31,
              "pack_context_predictions: bad shape n_frames=%d K=%d", n_frames, K);
  LPB_REQUIRE(n_rows >= 5, "pack_context_predictions: a context video needs at least 5 frames (got %lld)", (long long)n_rows);
  LPB_REQUIRE(step >= 1, "pack_context_predictions: step (sequence_length - 4) must be >= 1 (got %lld)", (long long)step);
  LPB_REQUIRE(model_height > 0.f && model_width > 0.f, "pack_context_predictions: bad model dims");
  LPB_REQUIRE(cursor || frame0 >= 0, "pack_context_predictions: frame0 must be >= 0");
  if (n_frames == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int total = n_frames * K;
  pack_context_kernel<<<(total + 255) / 256, 256, 0, s>>>(kp_sf, conf_sf, kp_mf, conf_mf, n_frames, K, bbox,
                                                          1.0f / model_height, 1.0f / model_width, table, n_rows,
                                                          cursor, frame0, step);
  if (cursor) advance_cursor_kernel<<<1, 1, 0, s>>>(cursor, n_frames);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
