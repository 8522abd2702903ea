/* lpb200 - C-ABI of the H100-native lightning-pose hot path (liblpb200.so, sm_90a only).
 *
 * Boundary contract
 *   - plain C: device pointers + sizes + a CUDA stream handle (cudaStream_t passed as void*);
 *     no torch / C++ types cross this boundary.
 *   - all tensor pointers are DEVICE pointers owned by the caller, contiguous, row-major, in the
 *     reference's own layouts (NCHW heatmaps / features, (N, 2K) keypoints [x0,y0,x1,y1,...]).
 *   - every call only enqueues work on `stream` (no host sync, CUDA-graph capturable once the
 *     per-shape tables exist: see lpb_decode_prepare); inputs are borrowed, nothing is retained.
 *   - return value: 0 = ok, <0 = error (LPB_ERR_*); lpb_last_error() gives the message for the
 *     calling thread.  There is NO CPU fallback anywhere behind this interface.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the
 * paninski-lab/lightning-pose tree, commit f54c477).
 */
#ifndef LPB200_H_
#define LPB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LPB_OK 0
#define LPB_ERR_INVALID (-1)
#define LPB_ERR_CUDA (-2)
#define LPB_ERR_UNSUPPORTED (-3)

/* heatmap loss kinds for lpb_heatmap_loss_* (lightning_pose/losses/losses.py:293-423) */
#define LPB_HM_MSE 0
#define LPB_HM_KL 1
#define LPB_HM_JS 2

/* library / build info -------------------------------------------------------------------- */
int lpb_version(void);                /* e.g. 100 = 0.1.0 */
const char* lpb_last_error(void);     /* message of the last failing call on this thread */
const char* lpb_build_arch(void);     /* "sm_90a" */

/* kernel-variant switches: a bring-up / profiling aid (A/B two implementations of the same stage on the same inputs);
 * every variant computes the same results.  lpb_get_tuning returns -1 for an unknown key. */
#define LPB_TUNE_K1A_ROW_TRANSPOSER 0   /* 1: row-per-lane operand transposer (coalesced saved-copy stores); 0 (default): 8x8 register blocks */
#define LPB_TUNE_SOFTMAX_EPILOGUE_V2 1  /* 1 (default): softmax epilogue with one vote per tile and hoisted addressing */
#define LPB_TUNE_WAIT_BACKOFF 2         /* 1 (default): idle warps back off between mbarrier polls */
#define LPB_TUNE_DECODE_RING 3          /* 1: soft-argmax planes staged once in shared memory by a bulk-copy ring; 0 (default): warp per plane from global */
#define LPB_TUNE_K1A_BULK_XS 4          /* 1: the saved operand copy leaves k1a by TMA bulk stores from the operand stage; 0 (default): producer stores */
#define LPB_TUNE_DECODE_L2_HINTS 5      /* 1 (default): L2 evict_last / evict_first hints on the decode's two sweeps of a plane */
#define LPB_TUNE_B3A_PREFETCH 6         /* 1 (default): b3a epilogue issues the next item's accumulator blocks before storing the current one */
#define LPB_TUNE_SOFTMAX_SPLIT 7         /* 1 (default): plane softmax as two launches parallel over (frame, band) when there are fewer frames than SMs, else one per-frame two-pass kernel; 0: never split; 2: always */
#define LPB_TUNE_DECODE_WARP_CTAS 8     /* > 0: resident CTAs per SM of the warp-per-plane decode are capped (fewer planes in flight than L2 holds); 0: no cap */
#define LPB_TUNE_DECODE_REVERSE 9       /* 1: the decode walks the planes last-to-first (the producer's most recent writes are still in L2) */
#define LPB_TUNE_B3A_TMA_STORE 10       /* 1 (default): b3a stages d features in shared memory and a TMA tensor store scatters them to NCHW; 0: direct 16-byte stores */
#define LPB_TUNE_WGRAD_SWAP 11          /* no effect in this build (accepted for compatibility): the weight gradient has one form */
#define LPB_TUNE_G2_PATCH 12            /* 1 (default): decode windows enter the gradient rows in a patch pass (one warp per plane) after a look-up-free streaming pass; 0: look-ups fused into the streaming pass */
#define LPB_TUNE_MMA_TILE_INNER 13      /* no effect in this build (accepted for compatibility): k1a has one MMA order */
#define LPB_TUNE_DECODE_HINTS 14        /* 1: the fused two-pass softmax emits per-plane decode hints (arg max + largest value outside its 32x32 box) and the decode skips its plane sweeps when they allow; 0 (default): hints never produced (measured: what the decode saves, the issue-bound softmax epilogue pays) */
#define LPB_TUNE_K1A_XS_COPY 15         /* k1a's saved operand copy: 2 (default): a dedicated extra warp sends each finished operand stage out with TMA bulk stores (the transposers store nothing); 1: streamed out of the finished stage by the transposer threads (whole sectors); 0: each transposer thread stores the rows it produced */
#define LPB_TUNE_COUNT 16
int lpb_set_tuning(int key, int value);
int lpb_get_tuning(int key);

/* ---- soft-argmax decode ---------------------------------------------------------------------
 * replaces run_subpixelmaxima / HeatmapHead.run_subpixelmaxima
 *   lightning_pose/models/heads/heatmap.py:103-144, :214-227
 * (upsample x ds [:86-100] -> spatial_softmax2d(T) -> spatial_expectation2d ->
 *  evaluate_heatmaps_at_location [lightning_pose/data/heatmaps.py:90-142] -> offset fix).
 *
 * heatmaps  [n_planes, h, w] fp32 (n_planes = batch * num_keypoints)
 * xy        [n_planes, 2]  (x, y) in model-pixel units, offset {0.5,1.5,2.5} already removed
 * conf      [n_planes]
 * stats     [n_planes, 8] or NULL: {shift M, sum S, xhat, yhat (field coords), A0, A1, B0, B1
 *           (evaluated coarse region)} - the residual lpb_decode_bwd needs.
 * ds in {1,2,3}.  Evaluation is exact up to a dropped softmax mass < 1e-12 (see DESIGN.md).
 */
int lpb_decode_prepare(int h, int w, int ds);
int lpb_decode_fwd(const float* heatmaps, int64_t n_planes, int h, int w, int ds, float temperature,
                   float* xy, float* conf, float* stats, void* stream);
/* lpb_decode_fwd with optional per-plane hints (16 bytes per plane: int32 arg-max row, int32 arg-max column, float32 bits of
 * the largest value outside the 32 x 32 box [row - 16, row + 15] x [col - 16, col + 15], int32 valid) as written by
 * lpb_head_fwd_bf16_hinted for the SAME heatmaps: planes whose outside bound is below the pruning threshold are decoded
 * from the window around the arg max alone (no sweep of the plane; identical candidate hull, identical results); planes
 * with valid = 0 and hints = NULL take the plain route.  No reference counterpart: the reference materialises the field. */
int lpb_decode_fwd_hinted(const float* heatmaps, int64_t n_planes, int h, int w, int ds, float temperature,
                          float* xy, float* conf, float* stats, const void* hints, void* stream);
/* d loss / d heatmaps given d loss / d xy (confidence carries no gradient: it only feeds `<`
 * comparisons, lightning_pose/losses/losses.py:636). grad_heatmaps [n_planes,h,w] is overwritten. */
int lpb_decode_bwd(const float* heatmaps, const float* stats, const float* grad_xy, int64_t n_planes,
                   int h, int w, int ds, float temperature, float* grad_heatmaps, void* stream);

/* sparse form of lpb_decode_bwd for the fused head backward: per plane a 32x32 window of d loss / d heatmap
 * (win [n_planes, 32, 32]) and meta [n_planes, 4] = {window row0, col0, flag, float bits of sum(win * heatmap)};
 * flag 0: zero gradient, 1: window valid, 2: the support does not fit a window -- that plane's dense
 * gradient is written to g_overflow [n_planes, h, w] instead (other planes of g_overflow are not touched).
 * queue: n_planes + 1 ints of scratch (work list of the overflow planes). */
int lpb_decode_bwd_windows(const float* heatmaps, const float* stats, const float* grad_xy, int64_t n_planes, int h,
                           int w, int ds, float temperature, float* win, int32_t* meta, float* g_overflow,
                           int32_t* queue, void* stream);

/* one materialised upsampling stage: drop-in for `upsample`
 *   lightning_pose/models/heads/heatmap.py:86-100 ; in [n_planes,h,w] -> out [n_planes,2h,2w] */
int lpb_upsample2x(const float* in, int64_t n_planes, int h, int w, float* out, void* stream);

/* ---- Gaussian target generation --------------------------------------------------------------
 * replaces generate_heatmaps  lightning_pose/data/heatmaps.py:11-87
 * keypoints [n_planes, 2] fp32 image pixels; visibility [n_planes] int32 {0,1,2} or NULL.
 * out [n_planes, oh, ow] fp32.
 */
int lpb_generate_heatmaps(const float* keypoints, const int32_t* visibility, int64_t n_planes,
                          float img_height, float img_width, int oh, int ow, float sigma, float* out,
                          void* stream);

/* the labeled-data rule that precedes target generation when targets are made on the GPU (SURVEY 8f-2): keypoints an
 * augmentation moved outside [0, width) x [0, height) become NaN in both coordinates
 *   lightning_pose/data/datasets.py:496-508 (HeatmapDataset.compute_heatmap).  keypoints, out: [n_keypoints, 2]
 * (may alias). */
int lpb_keypoints_mask_oob(const float* keypoints, int64_t n_keypoints, float img_height, float img_width, float* out,
                           void* stream);

/* gradient of lpb_generate_heatmaps wrt keypoints (keep_gradients=True, data/heatmaps.py:37-40);
 * grad_out [n_planes,oh,ow] -> grad_keypoints [n_planes,2] */
int lpb_generate_heatmaps_bwd(const float* keypoints, const int32_t* visibility, const float* grad_out,
                              int64_t n_planes, float img_height, float img_width, int oh, int ow, float sigma,
                              float* grad_keypoints, void* stream);

/* replaces evaluate_heatmaps_at_location  lightning_pose/data/heatmaps.py:90-142
 * heatmaps [n_planes,h,w], locs [n_planes,2] (x,y) -> out [n_planes]; radius = floor(sigma*num_stds) */
int lpb_evaluate_heatmaps_at_location(const float* heatmaps, const float* locs, int64_t n_planes, int h,
                                      int w, int radius, float* out, void* stream);

/* ---- heatmap head ----------------------------------------------------------------------------
 * replaces HeatmapHead.forward  lightning_pose/models/heads/heatmap.py:203-212
 * (PixelShuffle(2) -> ConvTranspose2d(k3,s2,p1,op1) x n_layers [:20-71] -> spatial_softmax2d(T=1)).
 *
 * features  [B, C, H, W]   fp32 (lpb_head_fwd_f32) or bf16 (lpb_head_fwd_bf16), NCHW contiguous
 * w1 [C/4, c1, 3, 3], b1 [c1]   first deconv (ConvTranspose2d layout, fp32 or bf16 to match)
 * w2 [c1, c2, 3, 3],  b2 [c2]   second deconv, or NULL/NULL for a one-layer head (then c2 = 0)
 * out [B, K, Ho, Wo] fp32 with K = c2 ? c2 : c1, Ho = 4H*(n_layers==2?2:1) ...
 * workspace: lpb_head_workspace_bytes() bytes of scratch (device), may be NULL if that is 0.
 */
int lpb_head_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes);
int lpb_head_fwd_f32(const float* features, int B, int C, int H, int W, const float* w1, const float* b1,
                     int c1, const float* w2, const float* b2, int c2, int final_softmax, float* out,
                     void* workspace, void* stream);

/* The same stack one layer at a time (any number of deconvs: n_layers = log2(stride) - downsample_factor - 1,
 * heads/heatmap.py:192-193), with its native backward -- the fp32 reference precision path trains through these.
 *   lpb_convt_fwd_f32   in [B, Cin(*4 if shuffle), Hi(/2), Wi(/2)] -> out [B, Cout, 2Hi, 2Wi]; shuffle != 0 folds
 *                       PixelShuffle(2) into the load (Hi, Wi are the conv-input = shuffled sizes)
 *   lpb_plane_softmax_f32  in-place spatial softmax (T = 1) of [n_planes, hw]
 *   lpb_convt_bwd_f32   autograd of lpb_convt_fwd_f32: grad_in (same shape as `in`, may be NULL), grad_w [Cin,Cout,3,3],
 *                       grad_bias [Cout] (may be NULL); all overwritten. */
int lpb_convt_fwd_f32(const float* in, int B, int Cin, int Hi, int Wi, int shuffle, const float* w, const float* bias,
                      int Cout, float* out, void* stream);
int lpb_plane_softmax_f32(float* x, int64_t n_planes, int hw, void* stream);
int lpb_convt_bwd_f32(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w,
                      int Cout, float* grad_in, float* grad_w, float* grad_bias, void* stream);

/* bf16 tensor-core path (tensor-core mma): features bf16 NCHW, fp32 master weights (rounded to bf16 on device, as
 * autocast does), fp32 accumulate, fp32 heatmaps.  One-deconv heads (ViT family, heads/heatmap.py:192-193: pass
 * w2 = b2 = NULL, c2 = 0) and two-deconv heads (ResNet family); C % 128 == 0, H*W % 8 == 0, c1, c2 <= 20 (c1 < 20 for
 * two deconvs).  Two kernel families serve it: whole-frame kernels for two-deconv heads on feature maps up to
 * 12x12 ("fast path"), and banded kernels for everything else (one-deconv heads, 16x16 / 24x24 ... maps).
 * lpb_head_bf16_plan reports which one a shape takes: plan[0] = 1 fast path, 0 banded (then saved_xs is REQUIRED by
 * lpb_head_fwd_bf16: it is the pixel-shuffled operand itself); LPB_ERR_UNSUPPORTED if neither fits. */
int lpb_head_bf16_plan(int C, int H, int W, int c1, int c2, int* plan);
int lpb_head_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes);
int lpb_head_fwd_bf16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                      const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                      void* workspace, void* stream);
/* lpb_head_fwd_bf16 that also fills `decode_hints` ([B * K] x 16 bytes, see lpb_decode_fwd_hinted; NULL = none) when the
 * head ends in the plane softmax: the softmax pass knows each plane's maximum and what lies outside the box around it. */
int lpb_head_fwd_bf16_hinted(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                             const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                             void* workspace, void* decode_hints, void* stream);
/* saved_xs: on the fast path NULL for inference; for training (and always on the banded path) a device buffer of lpb_head_bf16_saved_bytes() bytes; it
 * receives the pixel-shuffled features in the padded row layout the weight-gradient GEMM reads, and must stay
 * alive (together with `workspace`, which holds the activations between the two deconvs) until
 * lpb_head_bwd_bf16. */
int lpb_head_bf16_saved_bytes(int B, int C, int H, int W, size_t* bytes);

/* backward of lpb_head_fwd_bf16 (replaces autograd through heatmap.py:203-212 and, fused into its front end,
 * through spatial_softmax2d :211 and run_subpixelmaxima :103-144).  Kernels: gradient front end (G2 writer),
 * layer-2 wgrad, layer-2 dgrad, layer-1 wgrad, layer-1 dgrad + inverse PixelShuffle (all tensor-core).
 * The gradient w.r.t. the head OUTPUT [B, c2, 8H, 8W] is the sum of
 *   g_out        dense fp32 gradient (heatmap losses), or NULL
 *   win/win_meta/g_overflow   sparse soft-argmax gradient from lpb_decode_bwd_windows, or NULL/NULL/NULL
 * probs: the head output itself when the head ends in the spatial softmax (its backward is applied on the fly),
 *   NULL when the head returns logits.
 * dfeat [B, C, H, W] bf16 or NULL (frozen backbone); dw1 [C/4, c1, 3, 3], db1 [c1], dw2 [c1, c2, 3, 3],
 * db2 [c2] fp32 (overwritten).  One-deconv heads: w2 = dw2 = db2 = NULL, c2 = 0 (output [B, c1, 4H, 4W]).
 * Feature maps: H even, W in {4, 8, 12, 16, 24, 32}.  workspace: lpb_head_bwd_bf16_workspace_bytes(). */
int lpb_head_bwd_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes);
int lpb_head_bwd_bf16(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                      const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H,
                      int W, const float* w1, int c1, const float* w2, int c2, void* dfeat, float* dw1, float* db1,
                      float* dw2, float* db2, void* workspace, void* stream);

/* ---- coordinate remap -------------------------------------------------------------------------
 * replaces undo_affine_transform_batch + model_to_frame_batch
 *   lightning_pose/data/utils.py:142-234, lightning_pose/data/bboxes.py:74-105,222-288
 * keypoints_in [n, 2K]; transforms: NULL (identity) | [2,3] (per_frame=0) | [n,2,3] (per_frame=1)
 * | [V,2,3] with num_views=V>1 (per_frame=0, view-sliced); bbox [n_bbox, 4V] (x,y,h,w per view),
 * n_bbox == n or n + 4 (context batches use rows 2..n_bbox-3).  keypoints_out [n, 2K] (may alias in).
 */
int lpb_remap_keypoints(const float* keypoints_in, int64_t n, int K, const float* transforms,
                        int per_frame, int num_views, const float* bbox, int64_t n_bbox,
                        float model_height, float model_width, float* keypoints_out, void* stream);

/* gradient of lpb_remap_keypoints wrt keypoints_in (a linear map: transpose of the same transform) */
int lpb_remap_keypoints_bwd(const float* grad_out, int64_t n, int K, const float* transforms, int per_frame,
                            int num_views, const float* bbox, int64_t n_bbox, float model_height, float model_width,
                            float* grad_in, void* stream);

/* ---- MHCRNN context head (SURVEY 8a-17/18, 8f-3) ------------------------------------------------------------
 * replaces UpsamplingCRNN.forward  lightning_pose/models/heads/heatmap_mhcrnn.py:268-316  and
 * get_context_from_sequence  lightning_pose/models/base.py:159-196.
 * H_f / H_b (grouped Conv2d k2 s2 -> grouped ConvTranspose2d k2 s2, no nonlinearity) are 4x4 affine maps per keypoint
 * on 2x2 blocks:  lpb_crnn_prepare turns the four parameter tensors conv_w [K*F,1,2,2], conv_b [K*F], convt_w
 * [K*F,1,2,2], convt_b [K] into L [K,4,4], h [K,4];  lpb_crnn_prepare_bwd maps (dL, dh) back to their gradients.
 * lpb_crnn_combine_fwd: WF, WB [N, K, H, W] = W_f / W_b applied to each of N frames ONCE (head kernels), idx [M, 5] =
 * frame index of each context slot of each of M outputs (overlapping windows share frames: no 5x feature tiling)
 * -> out_logits [M, K, H, W] = (x_f + x_b) / 2 before the spatial softmax.  lpb_crnn_combine_bwd: its autograd
 * (dWF, dWB [N,K,H,W], dLf/dLb [K,4,4], dhf/dhb [K,4]; all overwritten).  M * K < 65536 per call.
 * lpb_context_gather: the materialised window tensor out[i][s] = seq[clamp(i + s - ctx/2)] for API parity
 * (n items of item_bytes, a multiple of 16). */
int lpb_crnn_prepare(const float* conv_w, const float* conv_b, const float* convt_w, const float* convt_b, int K, int F,
                     float* L, float* h, void* stream);
int lpb_crnn_prepare_bwd(const float* conv_w, const float* conv_b, const float* convt_w, const float* dL, const float* dh,
                         int K, int F, float* d_conv_w, float* d_conv_b, float* d_convt_w, float* d_convt_b, void* stream);
int lpb_crnn_combine_fwd(const float* WF, const float* WB, const int32_t* idx, int M, int N, int K, int H, int W,
                         const float* Lf, const float* hf, const float* Lb, const float* hb, float* out_logits, void* stream);
int lpb_crnn_combine_bwd(const float* WF, const float* WB, const int32_t* idx, const float* grad_logits, int M, int N, int K,
                         int H, int W, const float* Lf, const float* hf, const float* Lb, const float* hb, float* dWF,
                         float* dWB, float* dLf, float* dhf, float* dLb, float* dhb, void* stream);
int lpb_context_gather(const void* seq, int64_t n, int64_t item_bytes, int ctx, void* out, void* stream);

/* ---- video-ingest boundary (SURVEY 8f-4) ----------------------------------------------------------------
 * replaces the tail of the DALI pipeline  lightning_pose/data/video/dali.py:157-197
 *   fn.resize -> / 255 -> fn.crop_mirror_normalize(output_layout="FCHW", mean, std)
 * frames_u8 [F, H, W, 3] decoded RGB (device) -> out [F, 3, out_h, out_w] (layout 0, the reference's FCHW) or
 * [F, out_h, out_w, 3] (layout 1, channels-last), fp32 or bf16 (out_bf16).  mean3 / std3: HOST arrays of three floats
 * in (0, 1) units (ImageNet statistics, dali.py:44-45).  Resize (when out size != input size): bilinear, half-pixel
 * centres, no antialiasing. */
int lpb_frames_normalize(const uint8_t* frames_u8, int F, int H, int W, int out_h, int out_w, const float* mean3,
                         const float* std3, int layout, int out_bf16, void* out, void* stream);

/* ---- batched inference (SURVEY 8f-1) ------------------------------------------------------------------
 * replaces PredictionHandler.unpack_preds + make_pred_arr_undo_resize  lightning_pose/utils/predictions.py:97-144,180-206
 * keypoints [n_frames, 2K], confidences [n_frames, K] of one chunk -> rows [r, r + n_frames) of the prediction table
 * [n_rows, 3K] (columns bp0_x, bp0_y, bp0_likelihood, bp1_x, ...), r = *cursor (device int64, advanced by n_frames
 * afterwards, so a captured chunk graph needs no host-side offset) or row0 when cursor is NULL.  Rows >= n_rows
 * (padding frames of the last chunk) are dropped. */
int lpb_pack_predictions(const float* keypoints, const float* confidences, int n_frames, int K, float* table,
                         int64_t n_rows, int64_t* cursor, int64_t row0, void* stream);

/* ---- optimizer step (the tail of a training step) ---------------------------------------------------
 * replaces torch.optim.Adam / AdamW as configured by configure_optimizers  lightning_pose/models/base.py:458-477
 * (no amsgrad).  One launch over up to 16 fp32 tensors; params / grads / exp_avg / exp_avg_sq / numel are HOST arrays
 * of n_tensors device pointers / element counts.  step: device float, the number of steps taken so far (advanced by
 * the launch, so a captured graph replays correctly); block_counter: device uint32 initialised to 0.
 * lr_dev: optional device float overriding lr (learning-rate schedules under graph replay).
 * beta1 / beta2 are doubles: 1 - beta^t is evaluated in fp64 (fp32 loses five digits at beta2 = 0.999).
 * decoupled = 0: Adam (weight_decay is an L2 term added to the gradient), 1: AdamW. */
int lpb_adam_step(int n_tensors, float* const* params, const float* const* grads, float* const* exp_avg,
                  float* const* exp_avg_sq, const int64_t* numel, float* step, uint32_t* block_counter, float lr,
                  const float* lr_dev, double beta1, double beta2, float eps, float weight_decay, int decoupled,
                  void* stream);

/* backward of the head's final spatial softmax: grad_logits = p * (g - sum(g * p)) per plane
 * (reference: autograd of spatial_softmax2d, lightning_pose/models/heads/heatmap.py:211) */
int lpb_plane_softmax_bwd(const float* probs, const float* grad_probs, int64_t n_planes, int hw, float* grad_logits,
                          void* stream);

/* ---- heatmap losses ---------------------------------------------------------------------------
 * replaces HeatmapMSELoss / HeatmapKLLoss / HeatmapJSLoss (remove_nans + compute_loss + mean)
 *   lightning_pose/losses/losses.py:229-289, :314-335, :360-378, :404-423
 * targets/preds [n_planes, hw]; planes whose target is all-zero are dropped on device (no
 * boolean gather, no host sync).  out[0] = scalar loss, out[1] = number of kept planes.
 * workspace: n_planes * 2 floats {plane sum, kept flag}; the backward pass reads it again.
 */
int lpb_heatmap_loss_fwd(const float* targets, const float* preds, int64_t n_planes, int h, int w, int kind,
                         float* out, float* workspace, void* stream);
/* d loss/d preds (targets get no gradient); grad_out is the upstream scalar gradient (device ptr). */
int lpb_heatmap_loss_bwd(const float* targets, const float* preds, int64_t n_planes, int h, int w, int kind,
                         const float* workspace, const float* fwd_out, const float* grad_out, float* grad_preds,
                         void* stream);
/* fused target generation + MSE: targets never touch HBM (SURVEY 8(d) K3). */
int lpb_heatmap_mse_from_keypoints_fwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                       int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                       float sigma, float* out, float* workspace, void* stream);

int lpb_heatmap_mse_from_keypoints_bwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                       int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                       float sigma, const float* fwd_out, const float* grad_out, float* grad_preds,
                                       void* stream);

/* replaces TemporalHeatmapLoss.__call__  lightning_pose/losses/losses.py:793-854
 * heatmaps [T,K,h,w], confidences [T,K], eps [K]; kind LPB_HM_MSE | LPB_HM_KL; out[0] = scalar loss;
 * workspace (T-1)*K floats. */
int lpb_temporal_heatmap_loss_fwd(const float* heatmaps, const float* confidences, int64_t T, int K, int h, int w,
                                  int kind, const float* eps, float prob_threshold, float* out, float* workspace,
                                  void* stream);
/* autograd of the call above w.r.t. heatmaps (the reference trains through it: temporal_heatmap_mse / _kl are
 * unsupervised losses, losses/factory.py:73-91).  workspace = the forward's (per-pair differences); grad_out [1];
 * grad_heatmaps [T,K,h,w] is overwritten. */
int lpb_temporal_heatmap_loss_bwd(const float* heatmaps, const float* confidences, const float* workspace, int64_t T,
                                  int K, int h, int w, int kind, const float* eps, float prob_threshold,
                                  const float* grad_out, float* grad_heatmaps, void* stream);

/* ---- unsupervised losses on the (T, K, 2) keypoint tensor -------------------------------------
 * replaces TemporalLoss.__call__ and PCALoss.__call__ (+ KeypointPCA._format_data / reproject /
 * compute_reprojection_error)
 *   lightning_pose/losses/losses.py:548-573, :608-703; lightning_pose/utils/pca.py:97-190,266-309
 *
 * One launch evaluates every clip: keypoints [n_clips, T, 2K], confidences [n_clips, T, K] or NULL.
 * temporal: eps_k [K] (per-keypoint epsilon), prob_threshold.
 * pca (optional, may be NULL-disabled by n_obs_dims = 0):
 *   columns [D/2 ... ] see lpb_pca_desc.
 * out [n_clips, LPB_UNSUP_NOUT] = {temporal, pca_singleview, pca_multiview, 0}
 */
#define LPB_UNSUP_NOUT 4
typedef struct lpb_pca_desc {
  /* singleview: kp_index[i] for i < n_sel = selected keypoint ids; D = 2*n_sel.
   * multiview:  kp_index[v*n_sel + j] = keypoint id of body part j in view v; D = 2*n_views. */
  const int32_t* kp_index; /* device */
  int32_t n_sel;
  int32_t n_views;     /* 0 = singleview */
  int32_t centering;   /* singleview only: 0 none, 1 mean, 2 median (quantile 0.5) */
  int32_t n_components;
  const float* mean;   /* [D] device */
  const float* kept;   /* [n_components, D] device, rows = kept eigenvectors */
  float epsilon;
} lpb_pca_desc;

int lpb_unsup_losses_fwd(const float* keypoints, const float* confidences, int64_t n_clips, int T, int K,
                         const float* temporal_eps, float prob_threshold, int temporal_enabled,
                         const lpb_pca_desc* pca_singleview, const lpb_pca_desc* pca_multiview, float* out,
                         void* stream);
/* gradient wrt keypoints; grad_out [n_clips, LPB_UNSUP_NOUT] upstream per-loss gradients. */
int lpb_unsup_losses_bwd(const float* keypoints, const float* confidences, int64_t n_clips, int T, int K,
                         const float* temporal_eps, float prob_threshold, int temporal_enabled,
                         const lpb_pca_desc* pca_singleview, const lpb_pca_desc* pca_multiview,
                         const float* grad_out, float* grad_keypoints, void* stream);

/* ---- calibrated multi-view geometry (lightning-pose 3-D mode) ------------------------------------
 * Camera tensors per (batch, view), fp32, as the batch dict carries them: intrinsics [B, V, 3, 3], extrinsics
 * [B, V, 3, 4], dist [B, V, P] with P in {4, 5, 8, 12} (OpenCV order k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4; tilt, P = 14,
 * is rejected).  The distortion model reads fx, fy, cx, cy only.  Per-point geometry is evaluated in fp64.  Cameras
 * get no gradient.  Backward calls sum every input gradient in one thread in a fixed order (bit-reproducible) and give
 * NaN inputs a zero gradient.  2 <= V <= 64 for triangulation, 1 <= V <= 64 for projection.
 *
 * replaces project_camera_pairs_to_3d  lightning_pose/data/cameras.py:22-83
 *   points [B, V, K, 2] frame pixels -> out [B, V(V-1)/2, K, 3], pairs in itertools.combinations order; undistortion
 *   (kornia undistort_points, new_K = I, 5 iterations) then the DLT of each pair (smallest right singular vector,
 *   kornia triangulate_points / convert_points_from_homogeneous).  A keypoint NaN in either view gives a NaN triple. */
int lpb_triangulate_pairs_fwd(const float* points, const float* intrinsics, const float* extrinsics, const float* dist, int B,
                              int V, int K, int P, float* out, void* stream);
/* d loss / d points given d loss / d out (grad_out [B, V(V-1)/2, K, 3]); grad_points [B, V, K, 2] is overwritten. */
int lpb_triangulate_pairs_bwd(const float* points, const float* intrinsics, const float* extrinsics, const float* dist,
                              const float* grad_out, int B, int V, int K, int P, float* grad_points, void* stream);

/* replaces project_3d_to_2d  lightning_pose/data/cameras.py:86-171  (+ torch.mean(dim=1) before it and
 * frame_to_model_batch, lightning_pose/data/bboxes.py:194-219, after it, as the tracker chains them:
 * lightning_pose/models/heatmap_tracker_multiview.py:281-291)
 *   points3d [B, K, 3] (n_pairs = 0) or [B, n_pairs, K, 3] averaged over the pair axis first (NaN-propagating);
 *   out [B, V, K, 2]: pinhole projection with K E, then distortion for the (b, v) whose dist row is not all zero, then
 *   (bbox [B, 4V] of [x, y, h, w] per view, or NULL) frame -> model coordinates of a model_height x model_width input.
 *   A NaN point is NaN in every view. */
int lpb_project_points_fwd(const float* points3d, int n_pairs, const float* intrinsics, const float* extrinsics, const float* dist,
                           const float* bbox, float model_height, float model_width, int B, int V, int K, int P, float* out,
                           void* stream);
/* d loss / d points3d given d loss / d out; grad_points3d (the shape of points3d) is overwritten. */
int lpb_project_points_bwd(const float* points3d, int n_pairs, const float* intrinsics, const float* extrinsics, const float* dist,
                           const float* bbox, float model_height, float model_width, const float* grad_out, int B, int V, int K,
                           int P, float* grad_points3d, void* stream);

/* replaces frame_to_model_batch  lightning_pose/data/bboxes.py:194-219
 *   keypoints [B, V, K, 2] frame pixels -> out [B, V, K, 2]: ((x - bx) / bw * model_width, (y - by) / bh * model_height)
 *   with bbox [B, 4V] = [x, y, h, w] per view; grad != 0 applies the linear part only (the backward). */
int lpb_frame_to_model(const float* keypoints, int B, int V, int K, const float* bbox, float model_height, float model_width,
                       int grad, float* out, void* stream);

/* replaces PairwiseProjectionsLoss.__call__ (compute_loss + remove_nans + mean)  lightning_pose/losses/losses.py:1014-1126
 * targets [B, K, 3], preds [B, n_pairs, K, 3]: mean L2 distance over the (b, pair, k) with neither side NaN, 0 when
 * none is (no boolean gather, fixed-order reduction in one CTA).  out[0] = loss, out[1] = number of kept entries. */
int lpb_pairwise_projections_loss_fwd(const float* targets, const float* preds, int B, int n_pairs, int K, float* out, void* stream);
/* d loss / d preds (targets get no gradient); fwd_out = the forward's out, grad_out [1]; grad_preds is overwritten. */
int lpb_pairwise_projections_loss_bwd(const float* targets, const float* preds, int B, int n_pairs, int K, const float* fwd_out,
                                      const float* grad_out, float* grad_preds, void* stream);

/* ---- diagnostics ------------------------------------------------------------------------------
 * Tensor-core operand self-test (bring-up aid): one-CTA GEMM over operands in the library's row layout
 * [kchunk][row][8] bf16; mode 0 = K-major view, 1 = MN-major view; d [128][n] fp32.  col_off has no effect
 * (kept for ABI compatibility). */
int lpb_selftest_umma(const void* a, int kca, int rows_a, const void* b, int kcb, int rows_b, int mode, int n, int k,
                      int row_shift, int col_off, float* d, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LPB200_H_ */
