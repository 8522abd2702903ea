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
__host__ __device__ __forceinline__ int64_t context_rows(int64_t n, int64_t t) {
  const int64_t a = n - (t + 4);
  return t == 1 ? n : t * ((a >= 0 ? (a + t - 1) / t : -((-a) / t)) + 1);
}

__device__ __forceinline__ int64_t context_source(int64_t r, int64_t n, int64_t r_rows) {
  if (r_rows >= n) return r < 2 ? 2 : (r > n - 3 ? n - 3 : r);
  return (r >= 2 && r <= r_rows - 1) ? r : 2;  // the tail repeats preds_combined[0] = pred(2) (predictions.py:163-170)
}

__device__ __forceinline__ int64_t context_source_row(int64_t r, int64_t n, int64_t t) {
  return context_source(r, n, context_rows(n, t));
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

// ---- context models over a list of videos ---------------------------------------------------------------------
// segments [S][3] = (row0, N, R) per video, back to back in the table.  The video holding global frame g: the last
// segment with row0 <= g (binary search; -1 before the first).
__device__ __forceinline__ int find_segment(const int64_t* __restrict__ seg, int n_seg, int64_t g) {
  int lo = 0, hi = n_seg;  // invariant: seg[lo - 1].row0 <= g < seg[hi].row0
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(seg + 3 * mid) <= g) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

// one thread per (output frame, keypoint): output frame i of the call is global frame g = cursor - 2 + i, frame
// f = g - row0 of its video.  Frames 0, 1, N - 1 (and N - 2 unless R = N - 1) own no row: their windows cross into a
// neighbouring video.  Every other frame goes to the rows of its own video that the one-video rule gives it.
__global__ void pack_context_segments_kernel(const float* __restrict__ kp_sf, const float* __restrict__ conf_sf,
                                             const float* __restrict__ kp_mf, const float* __restrict__ conf_mf, int n,
                                             int K, const float* __restrict__ bbox, float inv_mh, float inv_mw,
                                             float* __restrict__ table, int64_t n_rows, const int64_t* __restrict__ cursor,
                                             const int64_t* __restrict__ seg, int n_seg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * K) return;
  const int o = i / K, k = i - o * K;
  const int64_t g = *cursor - 2 + o;
  if (g < 0 || g >= n_rows) return;  // halo before the first video, padding after the last
  const int s = find_segment(seg, n_seg, g);
  const int64_t row0 = __ldg(seg + 3 * s), nv = __ldg(seg + 3 * s + 1), r_rows = __ldg(seg + 3 * s + 2);
  const int64_t f = g - row0;
  if (f < 2 || f > nv - 2) return;
  const int64_t cand[7] = {f, 0, 1, nv - 4, nv - 3, nv - 2, nv - 1};
  bool any = false;
  for (int c = 0; c < 7; ++c) any |= cand[c] >= 0 && context_source(cand[c], nv, r_rows) == f;
  if (!any) return;
  const float csf = conf_sf[(size_t)o * K + k], cmf = conf_mf[(size_t)o * K + k];
  const bool mf = cmf > csf;
  const float* src = mf ? kp_mf : kp_sf;
  const float x = src[(size_t)o * 2 * K + 2 * k], y = src[(size_t)o * 2 * K + 2 * k + 1];
  const float* bb = bbox + (size_t)o * 4;
  const float fx = (x * inv_mw) * bb[3] + bb[0];
  const float fy = (y * inv_mh) * bb[2] + bb[1];
  const float fc = mf ? cmf : csf;
  for (int c = 0; c < 7; ++c) {
    const int64_t r = cand[c];
    if (r < 0 || context_source(r, nv, r_rows) != f) continue;
    float* dst = table + ((row0 + r) * K + k) * 3;
    dst[0] = fx;
    dst[1] = fy;
    dst[2] = fc;
  }
}

// cursor += n, then the window table of the chunk that starts there: window i reads map rows i .. i + 4 (frames
// g - 2 .. g + 2, g = cursor - 2 + i), except that a video with R = N - 1 reads the map row step + 4 (the padding
// frame's) in place of frame N, the next video's first frame.  One block; every thread reads the cursor first.
__global__ void advance_cursor_windows_kernel(int64_t* cursor, int64_t n, int32_t* __restrict__ idx, int64_t step,
                                              const int64_t* __restrict__ seg, int n_seg, int64_t n_rows) {
  const int64_t c = *cursor + n;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < step; i += blockDim.x) {
    const int64_t g = c - 2 + i;
    bool pad = false;
    if (g >= 0 && g < n_rows) {
      const int s = find_segment(seg, n_seg, g);
      const int64_t nv = __ldg(seg + 3 * s + 1);
      pad = __ldg(seg + 3 * s + 2) == nv - 1 && g - __ldg(seg + 3 * s) == nv - 2;
    }
    for (int j = 0; j < 4; ++j) idx[i * 5 + j] = (int32_t)(i + j);
    idx[i * 5 + 4] = (int32_t)(pad ? step + 4 : i + 4);
  }
  if (threadIdx.x == 0) *cursor = c;
}

// ---- a live stream of one frame per call (FramePredictor.push_frame) ----------------------------------------------
// Model.predict_frame  lightning_pose/api/model.py:360-509 on frames t - 4 .. t, with each frame's maps, single-frame
// decode and box computed once and kept in a ring (see lpb200.h).  Slot s holds stream frame t with t mod 5 = s;
// count = the frames pushed so far.
__device__ __forceinline__ int ring_slot(int64_t t) {
  const int64_t s = t % LPB_CONTEXT_RING_SLOTS;
  return (int)(s < 0 ? s + LPB_CONTEXT_RING_SLOTS : s);
}

// grid-stride float4 copies of the frame's two maps into slot c mod 5; block 0 also stores the single-frame decode and
// the box, and writes the window [(c - 4) mod 5, ..., c mod 5]
__global__ void context_ring_push_kernel(const float4* __restrict__ wf, const float4* __restrict__ wb, int64_t map_vec,
                                         const float* __restrict__ kp_sf, const float* __restrict__ conf_sf,
                                         const float* __restrict__ bbox, int K, float4* __restrict__ ring_wf,
                                         float4* __restrict__ ring_wb, float* __restrict__ ring_kp,
                                         float* __restrict__ ring_conf, float* __restrict__ ring_box,
                                         const int64_t* __restrict__ count, int32_t* __restrict__ window) {
  const int64_t c = *count;
  const int s = ring_slot(c);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < map_vec; i += stride) {
    ring_wf[s * map_vec + i] = __ldg(wf + i);
    ring_wb[s * map_vec + i] = __ldg(wb + i);
  }
  if (blockIdx.x != 0) return;
  for (int i = threadIdx.x; i < 2 * K; i += blockDim.x) ring_kp[(size_t)s * 2 * K + i] = kp_sf[i];
  for (int i = threadIdx.x; i < K; i += blockDim.x) ring_conf[(size_t)s * K + i] = conf_sf[i];
  if (threadIdx.x < 4) ring_box[s * 4 + threadIdx.x] = bbox[threadIdx.x];
  if (threadIdx.x < LPB_CONTEXT_RING_SLOTS) window[threadIdx.x] = ring_slot(c - 4 + threadIdx.x);
}

// one block: frame c - 2's selection and remap (the rule and operation order of pack_context_kernel), then count += 1
__global__ void context_ring_select_kernel(const float* __restrict__ ring_kp, const float* __restrict__ ring_conf,
                                           const float* __restrict__ ring_box, const float* __restrict__ kp_mf,
                                           const float* __restrict__ conf_mf, int K, float inv_mh, float inv_mw,
                                           float* __restrict__ out, int64_t* count) {
  const int64_t c = *count;
  const int s = ring_slot(c - 2);
  const float* kp_sf = ring_kp + (size_t)s * 2 * K;
  const float* bb = ring_box + s * 4;  // [x, y, h, w] of frame c - 2
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float csf = ring_conf[(size_t)s * K + k], cmf = conf_mf[k];
    const bool mf = cmf > csf;  // a NaN keeps sf
    const float* src = mf ? kp_mf : kp_sf;
    const float x = src[2 * k], y = src[2 * k + 1];
    out[3 * k] = (x * inv_mw) * bb[3] + bb[0];
    out[3 * k + 1] = (y * inv_mh) * bb[2] + bb[1];
    out[3 * k + 2] = mf ? cmf : csf;
  }
  __syncthreads();  // every thread has read the count
  if (threadIdx.x == 0) *count = c + 1;
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

extern "C" int lpb_pack_context_predictions_segments(const float* kp_sf, const float* conf_sf, const float* kp_mf,
                                                     const float* conf_mf, int n_frames, int K, const float* bbox,
                                                     float model_height, float model_width, float* table, int64_t n_rows,
                                                     int64_t* cursor, const int64_t* segments,
                                                     const int64_t* segments_host, int n_segments, int64_t step,
                                                     int32_t* window_index, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(kp_sf && conf_sf && kp_mf && conf_mf && bbox && table && cursor && segments && segments_host,
              "pack_context_predictions_segments: null pointer");
  LPB_REQUIRE(aligned_to(kp_sf, 4) && aligned_to(conf_sf, 4) && aligned_to(kp_mf, 4) && aligned_to(conf_mf, 4) &&
                  aligned_to(bbox, 4) && aligned_to(table, 4) && aligned_to(cursor, 8) && aligned_to(segments, 8) &&
                  (!window_index || aligned_to(window_index, 4)),
              "pack_context_predictions_segments: misaligned pointer");
  LPB_REQUIRE(n_frames >= 0 && K >= 1 && (int64_t)n_frames * K < (int64_t)1 << 31,
              "pack_context_predictions_segments: bad shape n_frames=%d K=%d", n_frames, K);
  LPB_REQUIRE(step >= 1 && step + 4 < ((int64_t)1 << 31),
              "pack_context_predictions_segments: step (sequence_length - 4) must be >= 1 (got %lld)", (long long)step);
  LPB_REQUIRE(model_height > 0.f && model_width > 0.f, "pack_context_predictions_segments: bad model dims");
  LPB_REQUIRE(n_segments >= 1, "pack_context_predictions_segments: no segments (got %d)", n_segments);
  int64_t next = 0;
  for (int s = 0; s < n_segments; ++s) {
    const int64_t row0 = segments_host[3 * s], nv = segments_host[3 * s + 1], r_rows = segments_host[3 * s + 2];
    LPB_REQUIRE(nv >= 5, "pack_context_predictions_segments: video %d has %lld frames; a context video needs at least 5",
                s, (long long)nv);
    LPB_REQUIRE(row0 == next && nv <= n_rows - row0,
                "pack_context_predictions_segments: segment %d (row0 %lld, %lld frames) does not follow the previous "
                "one inside the %lld-row table", s, (long long)row0, (long long)nv, (long long)n_rows);
    LPB_REQUIRE(r_rows == context_rows(nv, step),
                "pack_context_predictions_segments: segment %d gives R = %lld; %lld frames at step %lld give %lld", s,
                (long long)r_rows, (long long)nv, (long long)step, (long long)context_rows(nv, step));
    next = row0 + nv;
  }
  LPB_REQUIRE(next == n_rows, "pack_context_predictions_segments: the segments cover %lld of the table's %lld rows",
              (long long)next, (long long)n_rows);
  if (n_frames == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int total = n_frames * K;
  pack_context_segments_kernel<<<(total + 255) / 256, 256, 0, s>>>(kp_sf, conf_sf, kp_mf, conf_mf, n_frames, K, bbox,
                                                                   1.0f / model_height, 1.0f / model_width, table,
                                                                   n_rows, cursor, segments, n_segments);
  if (window_index)
    advance_cursor_windows_kernel<<<1, 256, 0, s>>>(cursor, n_frames, window_index, step, segments, n_segments, n_rows);
  else
    advance_cursor_kernel<<<1, 1, 0, s>>>(cursor, n_frames);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_context_ring_push(const float* wf, const float* wb, const float* kp_sf, const float* conf_sf,
                                     const float* bbox, int K, int H, int W, float* ring_wf, float* ring_wb,
                                     float* ring_kp, float* ring_conf, float* ring_box, const int64_t* count,
                                     int32_t* window_index, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(wf && wb && kp_sf && conf_sf && bbox && ring_wf && ring_wb && ring_kp && ring_conf && ring_box && count &&
                  window_index,
              "context_ring_push: null pointer");
  LPB_REQUIRE(aligned_to(wf, 16) && aligned_to(wb, 16) && aligned_to(ring_wf, 16) && aligned_to(ring_wb, 16) &&
                  aligned_to(kp_sf, 4) && aligned_to(conf_sf, 4) && aligned_to(bbox, 4) && aligned_to(ring_kp, 4) &&
                  aligned_to(ring_conf, 4) && aligned_to(ring_box, 4) && aligned_to(count, 8) &&
                  aligned_to(window_index, 4),
              "context_ring_push: misaligned pointer (maps 16 bytes, count 8, the rest 4)");
  LPB_REQUIRE(K >= 1 && K <= LPB_CONTEXT_RING_MAX_K, "context_ring_push: bad K=%d (1 .. %d)", K, LPB_CONTEXT_RING_MAX_K);
  LPB_REQUIRE(H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0,
              "context_ring_push: maps must be (K, H, W) with even H, W >= 2 (got H=%d W=%d)", H, W);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t map_vec = (int64_t)K * H * W / 4;  // H, W even: a whole number of float4
  const int64_t blocks = (map_vec + 255) / 256;
  context_ring_push_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, s>>>(
      reinterpret_cast<const float4*>(wf), reinterpret_cast<const float4*>(wb), map_vec, kp_sf, conf_sf, bbox, K,
      reinterpret_cast<float4*>(ring_wf), reinterpret_cast<float4*>(ring_wb), ring_kp, ring_conf, ring_box, count,
      window_index);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_context_ring_select(const float* ring_kp, const float* ring_conf, const float* ring_box,
                                       const float* kp_mf, const float* conf_mf, int K, float model_height,
                                       float model_width, float* out, int64_t* count, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(ring_kp && ring_conf && ring_box && kp_mf && conf_mf && out && count, "context_ring_select: null pointer");
  LPB_REQUIRE(aligned_to(ring_kp, 4) && aligned_to(ring_conf, 4) && aligned_to(ring_box, 4) && aligned_to(kp_mf, 4) &&
                  aligned_to(conf_mf, 4) && aligned_to(out, 4) && aligned_to(count, 8),
              "context_ring_select: misaligned pointer (count 8 bytes, the rest 4)");
  LPB_REQUIRE(K >= 1 && K <= LPB_CONTEXT_RING_MAX_K, "context_ring_select: bad K=%d (1 .. %d)", K, LPB_CONTEXT_RING_MAX_K);
  LPB_REQUIRE(model_height > 0.f && model_width > 0.f, "context_ring_select: bad model dims");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  context_ring_select_kernel<<<1, 256, 0, s>>>(ring_kp, ring_conf, ring_box, kp_mf, conf_mf, K, 1.0f / model_height,
                                               1.0f / model_width, out, count);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
