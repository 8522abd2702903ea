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

/* tuning switch: which form of the head's final plane softmax runs (both compute the same results).  lpb_set_tuning
 * returns LPB_ERR_INVALID and lpb_get_tuning -1 for any other key. */
#define LPB_TUNE_SOFTMAX_SPLIT 7  /* 1 (default): plane softmax as two launches parallel over (frame, band) when there are fewer frames than SMs, else one per-frame two-pass kernel; 0: never split; 2: always */
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
 * workspace lpb_decode_fwd_workspace_bytes(n_planes) bytes of device scratch, 4-byte aligned; NULL only when
 *           n_planes == 0.  Only the call's own kernels use it, so one buffer can serve every call on a stream.
 * ds in {1,2,3}.  Evaluation is exact up to a dropped softmax mass < 1e-12 (see DESIGN.md).
 */
int lpb_decode_prepare(int h, int w, int ds);
int lpb_decode_fwd_workspace_bytes(int64_t n_planes, size_t* bytes);
int lpb_decode_fwd(const float* heatmaps, int64_t n_planes, int h, int w, int ds, float temperature,
                   float* xy, float* conf, float* stats, void* workspace, void* stream);
/* lpb_decode_fwd on heatmaps whose per-band maxima the head's softmax wrote (lpb_head_fwd_bf16_band_max): the same
 * outputs, bit for bit, from fewer bytes.  band_max [n_planes][nbands][8] uint32, 4-byte aligned: the bits of the
 * largest value in each band's rows, in 8 slots whose maximum is the band's; heatmap rows [2 b band_rows,
 * 2 (b + 1) band_rows) form band b (lpb_head_band_max_dims).  Every value of a plane must be >= 0 or NaN, and the
 * largest of a band's slots must be the largest non-NaN value of its rows (the softmax writes exactly that).  Refused: nbands < 0, a
 * null or misaligned band_max with nbands > 0, an odd h, and band counts that do not cut h / 2 rows into bands of
 * band_rows.  nbands = 0 is lpb_decode_fwd. */
int lpb_decode_fwd_banded(const float* heatmaps, int64_t n_planes, int h, int w, int ds, float temperature,
                          const uint32_t* band_max, int band_rows, int nbands, float* xy, float* conf, float* stats,
                          void* workspace, void* stream);
/* d loss / d heatmaps given d loss / d xy (confidence carries no gradient: it only feeds `<`
 * comparisons, lightning_pose/losses/losses.py:636). grad_heatmaps [n_planes,h,w] is overwritten. */
int lpb_decode_bwd(const float* heatmaps, const float* stats, const float* grad_xy, int64_t n_planes,
                   int h, int w, int ds, float temperature, float* grad_heatmaps, void* stream);

/* Both decode backward entries are bit-reproducible: every element of grad_heatmaps / g_overflow is a sum in an order
 * fixed by the shapes and the inputs (no float atomics), so identical inputs give identical bits on the same device
 * model. */
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
 * keypoints [n_planes, 2] fp32 image pixels; visibility [n_planes] int32 or NULL (the reference's None: a NaN x or
 * a point outside [-1, size + 1] on the grid gives a zero plane).  With a visibility, 0 -> zero plane, 1 -> uniform
 * 1/(oh ow), 2 -> Gaussian (zero plane when NaN x / outside), any other value (3, -1, ...) -> the clamped Gaussian
 * (NaN plane for a NaN coordinate), as the reference's masks leave it.  The same rule holds for every entry that
 * takes a visibility (lpb_heatmap_mse_from_keypoints_*, lpb_mse_targets).
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
 * Every convolution runs on the tensor cores in 3xTF32 (fp32 accuracy); any Cin, Cout, Hi, Wi (even with shuffle).
 *   lpb_convt_fwd_f32   in [B, Cin(*4 if shuffle), Hi(/2), Wi(/2)] -> out [B, Cout, 2Hi, 2Wi]; shuffle != 0 folds
 *                       PixelShuffle(2) into the load (Hi, Wi are the conv-input = shuffled sizes).  shuffle =
 *                       LPB_SHUFFLE_NHWC: the same with `in` channels-last, [B, Hi/2, Wi/2, 4 Cin] in memory (and so
 *                       grad_in of lpb_convt_bwd_f32); results are bit-identical to LPB_SHUFFLE_NCHW (= 1) on the same
 *                       logical tensor.
 *   lpb_plane_softmax_f32  in-place spatial softmax (T = 1) of [n_planes, hw]
 *   lpb_convt_bwd_f32   autograd of lpb_convt_fwd_f32: grad_in (same shape as `in`, may be NULL), grad_w [Cin,Cout,3,3],
 *                       grad_bias [Cout] (may be NULL); all overwritten.  NOT bit-reproducible: grad_w and grad_bias are
 *                       summed over the K-split CTAs with float atomics, so their last bits can change from call to call.
 *   lpb_convt_bwd_f32_ws   the same gradients, bit-reproducible: each K-split CTA ("slot") stores its grad_w tile and
 *                       bias sums as a partial in `workspace`, and the slots are added in slot order.  The slot count
 *                       follows the device's SM count (at most 264), so the order -- and the bits -- are fixed per device
 *                       model and shape.  workspace: lpb_convt_bwd_f32_workspace_bytes(B, Cin, Hi, Wi, Cout) bytes (the
 *                       conv-input sizes, as above), 4-byte aligned; NULL only when that is 0.  workspace_bytes is its
 *                       size (LPB_ERR_INVALID if smaller, before anything is queued).  Only the call's own kernels use it. */
#define LPB_SHUFFLE_NONE 0
#define LPB_SHUFFLE_NCHW 1
#define LPB_SHUFFLE_NHWC 2
int lpb_convt_fwd_f32(const float* in, int B, int Cin, int Hi, int Wi, int shuffle, const float* w, const float* bias,
                      int Cout, float* out, void* stream);
int lpb_plane_softmax_f32(float* x, int64_t n_planes, int hw, void* stream);
int lpb_convt_bwd_f32(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w,
                      int Cout, float* grad_in, float* grad_w, float* grad_bias, void* stream);
int lpb_convt_bwd_f32_workspace_bytes(int B, int Cin, int Hi, int Wi, int Cout, size_t* bytes);
int lpb_convt_bwd_f32_ws(const float* in, const float* grad_out, int B, int Cin, int Hi, int Wi, int shuffle, const float* w,
                         int Cout, float* grad_in, float* grad_w, float* grad_bias, void* workspace, size_t workspace_bytes,
                         void* stream);

/* bf16 tensor-core path (tensor-core mma): features bf16 NCHW, fp32 master weights (rounded to bf16 on device, as
 * autocast does), fp32 accumulate, fp32 heatmaps.  One-deconv heads (ViT family, heads/heatmap.py:192-193: pass
 * w2 = b2 = NULL, c2 = 0) and two-deconv heads (ResNet family); C % 128 == 0, H*W % 8 == 0, and channel counts of
 *   narrow heads: c1, c2 <= 20 (c1 < 20 for two deconvs), or
 *   wide heads:   a last layer of 21 .. LPB_HEAD_MAX_CHANNELS channels (c1 > 20 for one deconv, c2 > 20 for two) and
 *                 1 <= c1 <= LPB_HEAD_MAX_CHANNELS in front of it.
 * The output channels of a wide layer are keypoint groups of 20, each one GEMM of a banded-kernel work item.
 * Two kernel families serve it: whole-frame kernels for narrow two-deconv heads on feature maps up to
 * 12x12 ("fast path"), and banded kernels for everything else (one-deconv heads, 16x16 / 24x24 ... maps, wide heads).
 * lpb_head_bf16_plan reports which one a shape takes: plan[0] = 1 fast path, 0 banded (then saved_xs is REQUIRED by
 * lpb_head_fwd_bf16: it is the pixel-shuffled operand itself); LPB_ERR_UNSUPPORTED if neither fits or the last layer
 * has more than LPB_HEAD_MAX_CHANNELS channels (the head then runs the fp32 kernels).  The cap is four keypoint groups:
 * the forward's registers and shared memory do not grow with the group count (a group is a work item), so it bounds the
 * workspace and the range the tests cover. */
#define LPB_HEAD_MAX_CHANNELS 80
int lpb_head_bf16_plan(int C, int H, int W, int c1, int c2, int* plan);
int lpb_head_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes);
int lpb_head_fwd_bf16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                      const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                      void* workspace, void* stream);
/* saved_xs: on the fast path NULL for inference; for training (and always on the banded path) a device buffer of lpb_head_bf16_saved_bytes() bytes; it
 * receives the pixel-shuffled features in the padded row layout the weight-gradient GEMM reads, and must stay
 * alive (together with `workspace`, which holds the activations between the two deconvs) until
 * lpb_head_bwd_bf16.  features, saved_xs and workspace must be 16-byte aligned, out 8-byte aligned (LPB_ERR_INVALID
 * otherwise, before anything is queued). */
int lpb_head_bf16_saved_bytes(int B, int C, int H, int W, size_t* bytes);

/* fp16 forward (inference under autocast(float16)): lpb_head_fwd_bf16 with fp16 features, the fp32 master weights and
 * the bias that rides on the constant-one channel rounded to fp16 on device (round-to-nearest-even, subnormals kept,
 * overflow to inf: torch's .half()), fp16 mid activations, fp32 accumulate, fp32 heatmaps.  Shapes, kernels and plan are
 * those of the bf16 forward, and the layouts are identical with 2-byte elements: size it with lpb_head_bf16_plan,
 * lpb_head_bf16_workspace_bytes and lpb_head_bf16_saved_bytes.  Same alignment rules.  There is no fp16 backward. */
int lpb_head_fwd_f16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                     const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                     void* workspace, void* stream);

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
 * Shapes: the forward's channel limits (narrow and wide heads), and feature maps with H even, W in {4, 8, 12, 16, 24, 32}; both entries return
 * LPB_ERR_UNSUPPORTED for any other shape, so lpb_head_bwd_bf16_workspace_bytes (which needs no GPU) tells whether a
 * head can train on this path.  workspace: lpb_head_bwd_bf16_workspace_bytes() bytes.  g_out, probs, win_meta,
 * g_overflow, saved_xs, fwd_workspace, dfeat and workspace must be 16-byte aligned (LPB_ERR_INVALID otherwise, before
 * anything is queued). */
int lpb_head_bwd_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes);
int lpb_head_bwd_bf16(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                      const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H,
                      int W, const float* w1, int c1, const float* w2, int c2, void* dfeat, float* dw1, float* db1,
                      float* dw2, float* db2, void* workspace, void* stream);

/* Channels-last features (torch.channels_last; a transformer encoder's tokens (B, H*W, C) viewed as (B, C, H, W)):
 * the same head on features whose memory is [B, H, W, C], read and, for d features, written where they lie -- no NCHW
 * copy on either side (the reference permutes the tokens, lightning_pose/models/heatmap_tracker_multiview.py forward_vit;
 * heads/heatmap.py:203-212 is the forward these stand for).  The _layout entries are the entries above with a
 * feature_layout argument, and LPB_FEATURES_NCHW makes them exactly those.  With LPB_FEATURES_NHWC:
 *   lpb_head_bf16_plan_layout   plan[0] = 0 for every shape: the banded kernels serve all of them, so saved_xs is always
 *                        REQUIRED by the forward (inference: scratch), and the NCHW shuffle stage's feature-map limit
 *                        does not apply.
 *   lpb_head_fwd_bf16_layout / lpb_head_fwd_f16_layout   features [B, H, W, C]; everything else as above.  saved_xs
 *                        receives byte for byte what the NCHW entry writes for the same logical tensor.
 *   lpb_head_bwd_bf16_workspace_bytes_layout   the NCHW shapes except W = 32 (LPB_ERR_UNSUPPORTED), same size.
 *   lpb_head_bwd_bf16_layout   dfeat [B, H, W, C] bf16; saved_xs / fwd_workspace from either forward layout.
 * lpb_head_bf16_workspace_bytes and lpb_head_bf16_saved_bytes do not depend on the layout and serve both.  Alignment:
 * the same buffers, 16 bytes. */
#define LPB_FEATURES_NCHW 0
#define LPB_FEATURES_NHWC 1
int lpb_head_bf16_plan_layout(int C, int H, int W, int c1, int c2, int feature_layout, int* plan);
int lpb_head_fwd_bf16_layout(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                             const float* w2, const float* b2, int c2, int final_softmax, int feature_layout, float* out,
                             void* saved_xs, void* workspace, void* stream);
int lpb_head_fwd_f16_layout(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                            const float* w2, const float* b2, int c2, int final_softmax, int feature_layout, float* out,
                            void* saved_xs, void* workspace, void* stream);
/* The forwards above with final_softmax = 1 that also write the per-band maxima of the heatmaps for
 * lpb_decode_fwd_banded: band_max [B][c_out][nbands][8] uint32 (4-byte aligned, REQUIRED), for an h x w heatmap
 * (h = 8 H, w = 8 W for two deconvs, 4 H / 4 W for one) band_rows and nbands from lpb_head_band_max_dims(h, w).
 * Slot [b][k][j][e] holds the bits of the largest value the softmax's epilogue warp e stored in rows
 * [2 j band_rows, 2 (j + 1) band_rows) of plane k (0 where it stored none).  The heatmaps are those of the plain
 * entries, bit for bit. */
int lpb_head_band_max_dims(int h, int w, int* band_rows, int* nbands);
int lpb_head_fwd_bf16_band_max(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                               const float* w2, const float* b2, int c2, int feature_layout, float* out,
                               uint32_t* band_max, void* saved_xs, void* workspace, void* stream);
int lpb_head_fwd_f16_band_max(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                              const float* w2, const float* b2, int c2, int feature_layout, float* out,
                              uint32_t* band_max, void* saved_xs, void* workspace, void* stream);
int lpb_head_bwd_bf16_workspace_bytes_layout(int B, int C, int H, int W, int c1, int c2, int feature_layout, size_t* bytes);
int lpb_head_bwd_bf16_layout(const float* g_out, const float* probs, const float* win, const int32_t* win_meta,
                             const float* g_overflow, const void* saved_xs, const void* fwd_workspace, int B, int C, int H,
                             int W, const float* w1, int c1, const float* w2, int c2, int feature_layout, void* dfeat,
                             float* dw1, float* db1, float* dw2, float* db2, void* workspace, void* stream);

/* Keypoint-target source of the head backward: the gradient of lpb_heatmap_mse_from_keypoints_fwd w.r.t. its preds
 * (which must be the head output, probs), rebuilt inside the backward's front end from the keypoints instead of read
 * from a dense g_out.  The per-pixel values are those lpb_heatmap_mse_from_keypoints_bwd writes, bit for bit; the
 * [n_planes, 8H, 8W] fp32 gradient never exists.  Fields are the arguments of the two loss entries (device pointers):
 * keypoints [B*C][2], visibility [B*C] or NULL (the rule of lpb_generate_heatmaps), fwd_out the forward's out (out[1] = kept planes), grad_out the scalar
 * upstream gradient. */
typedef struct lpb_mse_targets {
  const float* keypoints;
  const int32_t* visibility;
  float img_height, img_width, sigma;
  const float* fwd_out;
  const float* grad_out;
} lpb_mse_targets;
/* lpb_head_bwd_bf16_layout with a keypoint-target source: mse NULL makes it exactly that entry.  With mse, g_out must be
 * NULL (the targets stand for it), probs non-NULL, and the workspace is lpb_head_bwd_bf16_workspace_bytes_targets(...,
 * with_targets = 1) bytes (a per-plane row of target factors more); with_targets = 0 gives the _layout size. */
int lpb_head_bwd_bf16_workspace_bytes_targets(int B, int C, int H, int W, int c1, int c2, int feature_layout, int with_targets,
                                              size_t* bytes);
int lpb_head_bwd_bf16_targets(const float* g_out, const lpb_mse_targets* mse, const float* probs, const float* win,
                              const int32_t* win_meta, const float* g_overflow, const void* saved_xs, const void* fwd_workspace,
                              int B, int C, int H, int W, const float* w1, int c1, const float* w2, int c2, int feature_layout,
                              void* dfeat, float* dw1, float* db1, float* dw2, float* db2, void* workspace, void* stream);

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
 * (dWF, dWB [N,K,H,W], dLf/dLb [K,4,4], dhf/dhb [K,4]; all overwritten).  M * K < 65536 per call.  It sums with
 * float atomics and is NOT bit-reproducible.  lpb_crnn_combine_bwd_ws: the same gradients, bit-reproducible for any idx:
 * each element of dWF / dWB is one sum over the (window, slot) pairs that read its frame, window ascending then slot
 * (a pair list built on the device, no host sync), and dL / dh are per-CTA partials added in a fixed order.  workspace:
 * lpb_crnn_combine_bwd_workspace_bytes(M, N, K, H, W) bytes, 16-byte aligned, workspace_bytes its size (LPB_ERR_INVALID
 * if smaller or NULL, before anything is queued).
 * lpb_context_gather: the materialised window tensor out[i][s] = seq[clamp(i + s - ctx/2)] for API parity
 * (n items of item_bytes, a multiple of 16).  lpb_context_gather_bwd: its adjoint, d_seq [n, elems] = for each frame
 * the sum of the grad [n, ctx, elems] slots that read it (the repeated edge frames included), in a fixed order without
 * atomics; elements in the LPB_OUT_* format `format` (see the ingest entries below), summed in fp32. */
int lpb_crnn_prepare(const float* conv_w, const float* conv_b, const float* convt_w, const float* convt_b, int K, int F,
                     float* L, float* h, void* stream);
int lpb_crnn_prepare_bwd(const float* conv_w, const float* conv_b, const float* convt_w, const float* dL, const float* dh,
                         int K, int F, float* d_conv_w, float* d_conv_b, float* d_convt_w, float* d_convt_b, void* stream);
int lpb_crnn_combine_fwd(const float* WF, const float* WB, const int32_t* idx, int M, int N, int K, int H, int W,
                         const float* Lf, const float* hf, const float* Lb, const float* hb, float* out_logits, void* stream);
int lpb_crnn_combine_bwd(const float* WF, const float* WB, const int32_t* idx, const float* grad_logits, int M, int N, int K,
                         int H, int W, const float* Lf, const float* hf, const float* Lb, const float* hb, float* dWF,
                         float* dWB, float* dLf, float* dhf, float* dLb, float* dhb, void* stream);
int lpb_crnn_combine_bwd_workspace_bytes(int M, int N, int K, int H, int W, size_t* bytes);
int lpb_crnn_combine_bwd_ws(const float* WF, const float* WB, const int32_t* idx, const float* grad_logits, int M, int N, int K,
                            int H, int W, const float* Lf, const float* hf, const float* Lb, const float* hb, float* dWF,
                            float* dWB, float* dLf, float* dhf, float* dLb, float* dhb, void* workspace, size_t workspace_bytes,
                            void* stream);
int lpb_context_gather(const void* seq, int64_t n, int64_t item_bytes, int ctx, void* out, void* stream);
int lpb_context_gather_bwd(const void* grad, int64_t n, int64_t elems, int ctx, int format, void* d_seq, void* stream);

/* ---- video-ingest boundary (SURVEY 8f-4) ----------------------------------------------------------------
 * replaces the tail of the DALI pipeline  lightning_pose/data/video/dali.py:157-197
 *   fn.resize -> / 255 -> fn.crop_mirror_normalize(output_layout="FCHW", mean, std)
 * frames_u8 [F, H, W, 3] decoded RGB (device) -> out [F, 3, out_h, out_w] (layout 0, the reference's FCHW) or
 * [F, out_h, out_w, 3] (layout 1, channels-last), in the element type of out_format: LPB_OUT_F32, LPB_OUT_BF16 or
 * LPB_OUT_F16 (rounded to nearest even from the fp32 value, so bf16 / fp16 output is the fp32 output's .bfloat16() /
 * .half() bit for bit); any other code is LPB_ERR_INVALID.  mean3 / std3: HOST arrays of three floats in (0, 1) units
 * (ImageNet statistics, dali.py:44-45).  Resize (when out size != input size): bilinear, half-pixel centres, no
 * antialiasing. */
#define LPB_OUT_F32 0
#define LPB_OUT_BF16 1
#define LPB_OUT_F16 2
int lpb_frames_normalize(const uint8_t* frames_u8, int F, int H, int W, int out_h, int out_w, const float* mean3,
                         const float* std3, int layout, int out_format, void* out, void* stream);

/* ---- multi-view video ingest: every camera's frames in one launch -----------------------------------------------
 * replaces the multi-view tail of the DALI pipeline  lightning_pose/data/video/dali.py:301-330  (one reader per view,
 * each through fn.resize -> / 255 -> fn.crop_mirror_normalize as in lpb_frames_normalize, then the views stacked into
 * (seq, V, 3, H, W)).  frames_u8: HOST array of V device pointers, view v [F, H[v], W[v], 3] decoded RGB; H, W: HOST
 * arrays of V ints (views may differ in size).  out [F, V, 3, out_h, out_w] (layout 0) or [F, V, out_h, out_w, 3]
 * (layout 1), in the element type of out_format (as for lpb_frames_normalize): reshaped to [F * V, ...] it is the frame-major, view-minor batch the multi-view
 * trackers read.  Every output image is bit-identical to lpb_frames_normalize on that view alone (a view already at
 * out_h x out_w is copied and normalised without resampling).  1 <= V <= LPB_INGEST_MAX_VIEWS, F * V < 2^31; the
 * output may pass 2^31 elements.  F = 0 is a no-op. */
#define LPB_INGEST_MAX_VIEWS 16
int lpb_frames_normalize_views(const uint8_t* const* frames_u8, int V, int F, const int* H, const int* W, int out_h,
                               int out_w, const float* mean3, const float* std3, int layout, int out_format, void* out,
                               void* stream);

/* ---- augmented video ingest: the unlabeled branch's DALI augmentation ----------------------------------------
 * replaces  lightning_pose/data/video/dali.py:154-192  (training.imgaug "dlc" / "dlc-top-down") in front of the
 * normalisation of lpb_frames_normalize, one view, one draw per call.  Per frame of frames_u8 [F, H, W, 3]:
 *   1. resize to out_h x out_w exactly as lpb_frames_normalize (bilinear, half-pixel centres, no antialiasing);
 *   2. params (DEVICE, 6 floats, read at run time) = angle (degrees), sx, sy, brightness, contrast, factor;
 *   3. M = S_c R_c (fn.transforms.rotation(angle, center=c), then fn.transforms.scale(scale, center=c)) in (x, y):
 *      A = diag(sx, sy) [[cos, -sin], [sin, cos]], t = c - A c, c = (out_h / 2, out_w / 2) taken as (x, y), the
 *      reference's own centre (off the image centre when out_h != out_w);
 *   4. fn.warp_affine(matrix=M, inverse_map=False, fill_value=0): destination pixel (x, y) samples the resized image
 *      bilinearly at M^-1 (x + 0.5, y + 0.5) - 0.5; taps outside it read 0;
 *   5. fn.brightness_contrast: brightness * (0.5 + contrast * (v - 0.5)) on 0..255 values (float contrast centre);
 *   6. fn.noise.shot: Poisson(max(0, v / factor)) * factor, v when factor == 0; Philox4x32-10 keyed by *seed (DEVICE
 *      int64) and counted by (x, y, frame, channel): the noise does not depend on the launch shape;
 *   7. / 255 and mean3 / std3 (HOST arrays) to out, layout 0 [F, 3, out_h, out_w] or 1 [F, out_h, out_w, 3], fp32 or
 *      bf16 (out_bf16: LPB_OUT_F32 or LPB_OUT_BF16; this training-only entry refuses LPB_OUT_F16 with LPB_ERR_INVALID).
 * transform_out (DEVICE, 6 floats): M row-major [[a00, a01, t0], [a10, a11, t1]], the transform lpb_remap_keypoints
 * undoes.  Reading params and seed on the device lets draws made inside a captured graph take effect on replay.
 * F = 0 is a no-op. */
int lpb_frames_augment_normalize(const uint8_t* frames_u8, int F, int H, int W, int out_h, int out_w, const float* params,
                                 const int64_t* seed, const float* mean3, const float* std3, int layout, int out_bf16,
                                 void* out, float* transform_out, void* stream);

/* ---- single-frame ingest: crop, OpenCV resize and numpy normalisation, bit for bit --------------------------------
 * replaces the preprocessing of Model.predict_frame  lightning_pose/api/model.py:388-430 (a numpy-slice crop,
 * cv2.resize(..., INTER_LINEAR) on uint8, then (u8 / 255.0 - mean) / std in fp32 numpy), for all F frames in one launch.
 * frames_u8 [F, H, W, 3] RGB (device), F >= 1 (1 frame, or the 5 frames of a context window).
 * box: DEVICE int32 [x, y, w, h], read at run time (one captured graph serves every box), or NULL for the whole frame.
 * It is cut as frame[y:y+h, x:x+w]: the crop is actual_h = min(H, y + h) - y rows by actual_w = min(W, x + w) - x
 * columns.  The caller refuses what the reference refuses (x or y < 0, w or h <= 0, an empty crop); a box outside those
 * rules is clamped into the frame, never read out of bounds.
 * bbox_out (DEVICE, 4 floats): [x, y, actual_h, actual_w], or [0, 0, H, W] without a box: the bbox of
 * lpb_remap_keypoints that maps model pixels back to the frame.
 * Resize to out_h x out_w: OpenCV 4.x INTER_LINEAR on 8-bit images (imgproc resize.cpp, the fixed-point path).  Per
 * output axis, scale = 1.0 / ((double)dst / src), f = (float)((d + 0.5) * scale - 0.5) in double then rounded to
 * float, s = floor(f), f -= s, s0 = clamp(s, 0, src - 1), s1 = clamp(s + 1, 0, src - 1), a1 = rint(f * 2048),
 * a0 = rint((1 - f) * 2048); the vertical weights are NOT zeroed where a row index is clamped.  Per channel
 * S(y, x) = a0[x] img[y, x0] + a1[x] img[y, x1] (int32) and
 *   u = clamp((((b0 (S(y0) >> 4)) >> 16) + ((b1 (S(y1) >> 4)) >> 16) + 2) >> 2, 0, 255),
 * the rule of OpenCV's vectorised vertical pass, used for every pixel (its scalar tail, (b0 S0 + b1 S1 + 2^21) >> 22,
 * differs in the last bit on about 10 % of pixels; cv2.resize 4.13 matched the vector rule on every tested shape).
 * An exact 2x downscale equals OpenCV's INTER_AREA switch under this rule; out size == crop size copies the crop.
 * Normalisation: (u / 255.0f - mean) / std, three correctly rounded fp32 operations without contraction; mean3 / std3
 * HOST arrays of three floats.  out: layout 0 [F, 3, out_h, out_w] or 1 [F, out_h, out_w, 3], LPB_OUT_F32 / BF16 /
 * F16 (bf16 / fp16 are the fp32 value rounded to nearest even). */
int lpb_frames_crop_resize_cv2(const uint8_t* frames_u8, int F, int H, int W, const int32_t* box, int out_h, int out_w,
                               const float* mean3, const float* std3, int layout, int out_format, void* out,
                               float* bbox_out, void* stream);

/* ---- curriculum patch masking of multi-view transformer training ----------------------------------------------
 * replaces PatchMasker.apply_patch_masking  lightning_pose/callbacks.py:303-401  (the PatchMasking callback's
 * on_train_batch_start, :222-263).  Images (B, V, C, H, W) are cut into LPB_PATCH_SIZE x LPB_PATCH_SIZE patches,
 * P = (H / 16) * (W / 16) per view (integer division), patch p = (y / 16) * (W / 16) + x / 16; the H % 16 bottom rows
 * and W % 16 right columns belong to no patch and are never masked, as in the reference.
 *
 * lpb_patch_mask_select: one CTA per (example, view).  step: DEVICE int64, read at run time (a captured graph replays
 * with an advancing step).  The curriculum of callbacks.py:344-357, in fp64 without contractions, so that it equals
 * Python's float64 result bit for bit:
 *   ratio = 0 for step < init_step, else init_ratio + min((step - init_step) / (final_step - init_step), 1)
 *           * (final_ratio - init_ratio);   m = clamp(int(ratio * P), 0, P)  (int() truncates toward zero).
 * Each view masks exactly m of its P patches, a uniformly random subset: patch p gets a 52-bit Philox4x32-10 key,
 * keyed by patch_seed and counted by (p, view, example, step); the m smallest keys (ties by patch index) are masked.
 * The same (patch_seed, step, example, view) gives the same patches; this is not the reference's torch.randperm draw.
 * mask [B, V, P] fp32: 1 = kept, 0 = masked (the reference's patch_mask).  Requires final_step > init_step,
 * P <= LPB_PATCH_MAX, V <= 65535.  P = 0 or B * V = 0 is a no-op.
 *
 * lpb_patch_mask_apply: out[b, v, c, y, x] = mask[b, v, p(y, x)] != 0 ? images[b, v, c, y, x] : 0 for pixels inside a
 * patch, images[...] elsewhere; bits are copied, not converted.  images, out: contiguous [B, V, C, H, W] in the element
 * type of in_format, LPB_OUT_F32 or LPB_OUT_BF16 (anything else is LPB_ERR_INVALID); out must not alias images (the
 * reference clones).  Accesses are 16 bytes wide where the row length and both pointers allow it. */
#define LPB_PATCH_SIZE 16
#define LPB_PATCH_MAX 4096
int lpb_patch_mask_select(const int64_t* step, int B, int V, int H, int W, int64_t patch_seed, int64_t init_step,
                          int64_t final_step, double init_ratio, double final_ratio, float* mask, void* stream);
int lpb_patch_mask_apply(const void* images, int B, int V, int C, int H, int W, int in_format, const float* mask, void* out,
                         void* stream);

/* ---- crop-zoom inference (bbox mode of the video-ingest boundary) ------------------------------------------------
 * replaces crop_and_resize_frames  lightning_pose/data/bboxes.py:291-343  and the bbox-row slicing in front of it
 *   lightning_pose/data/video/dali.py:332-380, lightning_pose/data/video/pynvvc.py:266-283
 * Frame f uses box row r = min(row0 + f, n_boxes - 1) of boxes [n_boxes, 4] (x, y, h, w fp32), row0 = *cursor (device
 * int64, read, never advanced: lpb_pack_predictions advances it) or row0 when cursor is NULL; rows past the end repeat
 * the final row (the reference pads the last chunk with it).  Clamp as the reference does: x1 = max(0, (int)x),
 * x2 = max(x1 + 1, min(W, (int)x + (int)w)), likewise y with h, H ((int) truncates toward zero).  Where the reference
 * raises, this does not: an origin at or past the far edge is clamped to W - 1 / H - 1 (a one-pixel crop), and a row
 * holding a NaN or an infinity is the whole frame.  The crop is resized to out_h x out_w (bilinear, half-pixel centres,
 * no antialiasing).
 *   in_f32 = 0: frames uint8 [F, H, W, 3] decoded RGB, normalised with mean3 / std3 (HOST arrays, as for
 *               lpb_frames_normalize) on the way out;
 *   in_f32 = 1: frames fp32 [F, 3, H, W] already normalised (the reference function's own input); crop + resize only,
 *               mean3 / std3 ignored (may be NULL).
 * out: layout 0 [F, 3, out_h, out_w] or layout 1 [F, out_h, out_w, 3], in the element type of out_format (as for
 * lpb_frames_normalize).
 * boxes_out [F, 4]: the clamped boxes [x1, y1, y2 - y1, x2 - x1], the bbox that maps model coordinates back to the
 * frame (lpb_remap_keypoints).  F <= 65535. */
int lpb_frames_crop_normalize(const void* frames, int in_f32, int F, int H, int W, const float* boxes, int64_t n_boxes,
                              const int64_t* cursor, int64_t row0, int out_h, int out_w, const float* mean3,
                              const float* std3, int layout, int out_format, void* out, float* boxes_out, void* stream);

/* replaces _calculate_bbox_size + _compute_bbox_df  lightning_pose/utils/cropzoom.py:31-143
 * keypoints: frame n, keypoint k at keypoints[n * row_stride + k * point_stride] (x) and + 1 (y): point_stride 2 reads
 * (N, K, 2) keypoints, 3 reads a (N, 3K) prediction table (lpb_pack_predictions) in place.  anchors: HOST array of
 * n_anchors keypoint indices, summed in the order given (the reference's column order); n_anchors = 0: all K.
 * Exactly one mode: crop_ratio > 0 (size = ceil(crop_ratio * max(x span, y span)), bumped to even, for h and w) or
 * crop_height, crop_width > 0 (each bumped to even).  out [N, 4] fp32 x, y, h, w holding integers: top-left =
 * int64(centroid - size // 2) evaluated in fp64, with h subtracted from x and w from y as the reference does
 * (cropzoom.py:135).  A frame with a NaN or infinite anchor gets a NaN row. */
#define LPB_BBOX_MAX_ANCHORS 256
int lpb_bboxes_from_keypoints(const float* keypoints, int64_t n, int K, int64_t row_stride, int point_stride,
                              const int32_t* anchors, int n_anchors, double crop_ratio, int crop_height, int crop_width,
                              float* out, void* stream);

/* replaces the smoothing of smooth_bbox  lightning_pose/utils/cropzoom.py:355-402
 *   rolling(window, center=True, min_periods=1).median().round(0) of each column of bboxes [n, 4] -> out [n, 4]
 * (not aliasing bboxes): pandas' centred and end-truncated windows, NaN skipped, the mean of the two middle values for
 * an even count, round half to even; a window with no value gives NaN. */
int lpb_bboxes_rolling_median(const float* bboxes, int64_t n, int window, float* out, void* stream);

/* ---- batched inference (SURVEY 8f-1) ------------------------------------------------------------------
 * replaces PredictionHandler.unpack_preds + make_pred_arr_undo_resize  lightning_pose/utils/predictions.py:97-144,180-206
 * keypoints [n_frames, 2K], confidences [n_frames, K] of one chunk -> rows [r, r + n_frames) of the prediction table
 * [n_rows, 3K] (columns bp0_x, bp0_y, bp0_likelihood, bp1_x, ...), r = *cursor (device int64, advanced by n_frames
 * afterwards, so a captured chunk graph needs no host-side offset) or row0 when cursor is NULL.  Rows >= n_rows
 * (padding frames of the last chunk) are dropped. */
int lpb_pack_predictions(const float* keypoints, const float* confidences, int n_frames, int K, float* table,
                         int64_t n_rows, int64_t* cursor, int64_t row0, void* stream);

/* ---- batched inference with context (MHCRNN) models --------------------------------------------------------------
 * replaces the selection and model -> frame step of HeatmapTrackerMHCRNN.predict_step
 *   lightning_pose/models/heatmap_tracker_mhcrnn.py:180-229 (torch.gt(confidence_mf, confidence_sf) per keypoint, then
 *   model_to_frame_batch with the window's bbox rows [2:-2]), and the host stacking / shift of
 *   PredictionHandler.unpack_preds + fix_context_preds_confs  lightning_pose/utils/predictions.py:97-177 for a reader of
 *   windows of S = step + 4 frames with step S - 4  lightning_pose/data/video/dali.py:519-534, 600-619.
 * Output frame i of the call is video frame f = c - 2 + i, c = *cursor (device int64: frames fed before this call,
 * advanced by n_frames afterwards) or frame0 when cursor is NULL.  Its single-frame / multi-frame keypoints
 * kp_* [n_frames, 2K] (model pixels) and confidences conf_* [n_frames, K]: mf where conf_mf > conf_sf (a NaN keeps sf),
 * then x * (1 / model_width) * w + bbox_x, y * (1 / model_height) * h + bbox_y with bbox [n_frames, 4] (x, y, h, w)
 * the frame's own box (lpb_remap_keypoints' operation order).  The result goes to every row r of table [n_rows, 3K]
 * whose source is f.  With N = n_rows, T = step and R = T * (ceil((N - S) / T) + 1) the rows the reader produces
 * (R = N for T = 1, where num_iters reads one window per frame, dali.py:509-510):
 *   R >= N: row r <- frame clamp(r, 2, N - 3);
 *   R <  N: row r <- frame r for 2 <= r <= R - 1, every other row (0, 1 and the last N - R <= 4) <- frame 2 (the
 *           reference pads with preds_combined[0], predictions.py:163-170).
 * Once frames 0 .. N have been fed (ceil(N / T) chunks of T frames, the last one padded) the table is final.  Only when R = N - 1 does a
 * kept row (N - 2) depend on frame N, the padding of the last chunk.  N >= 5 (with fewer frames the reference has no
 * window).  No atomics: every row is written by the one thread of its source frame. */
int lpb_pack_context_predictions(const float* kp_sf, const float* conf_sf, const float* kp_mf, const float* conf_mf,
                                 int n_frames, int K, const float* bbox, float model_height, float model_width,
                                 float* table, int64_t n_rows, int64_t* cursor, int64_t frame0, int64_t step,
                                 void* stream);

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

/* fused target generation + HeatmapMSELoss / HeatmapKLLoss / HeatmapJSLoss (kind LPB_HM_*): replaces generate_heatmaps
 * on the labeled keypoints (lightning_pose/data/heatmaps.py:37-87, called at data/datasets.py:516) followed by the loss
 * (lightning_pose/losses/losses.py:229-289, :314-335, :338-378, :381-423).  No target plane is written.
 * keypoints [n_planes, 2] image pixels, visibility [n_planes] or null (the plane rule of lpb_generate_heatmaps); preds
 * [n_planes, oh, ow].  A plane whose target is all-zero is dropped without reading its prediction; uniform planes
 * (visibility 1) use 1/(oh*ow); NaN planes are kept, so the loss is NaN as in the reference.  KL and JS add 1e-10 to
 * both operands (:375-376, :420-421).  out[0] = mean over kept planes of the per-plane sum of terms, out[1] = the kept
 * count; out[0] is NaN when nothing is kept.  workspace: n_planes * 2 floats.
 * LPB_HM_MSE runs lpb_heatmap_mse_from_keypoints_fwd / _bwd (same bits, same refusals). */
int lpb_heatmap_loss_from_keypoints_fwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                        int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                        float sigma, int kind, float* out, float* workspace, void* stream);
/* d loss/d preds of the call above, written dense (zeros on dropped planes, and everywhere when nothing is kept);
 * fwd_out is its out, grad_out the upstream scalar gradient (device pointers). */
int lpb_heatmap_loss_from_keypoints_bwd(const float* keypoints, const int32_t* visibility, const float* preds,
                                        int64_t n_planes, float img_height, float img_width, int oh, int ow,
                                        float sigma, int kind, const float* fwd_out, const float* grad_out,
                                        float* grad_preds, void* stream);

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

/* ---- coordinate-regression models (csrc/regression.cu) -------------------------------------------
 * replaces LinearRegressionHead.forward  lightning_pose/models/heads/regression.py:29-43, with the backbone's avgpool in
 * front of it (lightning_pose/models/backbones/factory.py:324 keeps torchvision's pool for regression)
 *   features [B, C, H, W] in the LPB_OUT_* element format `format` (fp32, bf16 or fp16), layout LPB_FEATURES_NCHW or
 *   LPB_FEATURES_NHWC (channels-last, [B, H, W, C] in memory); weight [n_out, C] fp32, bias [n_out] fp32.
 *   pooled [B, C] fp32: the mean over the H W pixels, summed in fp32 in a fixed order (the backward reads it);
 *   out [B, n_out] fp32 = pooled weight^T + bias.  Each feature byte is read once.  With H = W = 1 this is the
 *   reference's head exactly (features.reshape(B, C), then nn.Linear). */
int lpb_regression_head_fwd(const void* features, int format, int layout, int B, int C, int H, int W, const float* weight,
                            const float* bias, int n_out, float* pooled, float* out, void* stream);
/* grad_out [B, n_out] fp32.  dweight [n_out, C] and dbias [n_out] (both or neither) are overwritten with fixed-order sums
 * over the frames (no float atomics: the same bits from run to run).  dfeatures (NULL: not wanted) is overwritten with
 * (grad_out weight) / (H W) broadcast over the pixels, in the format and layout of the features, each element written
 * once; it needs workspace, B x C floats of device scratch. */
int lpb_regression_head_bwd(const float* grad_out, const float* pooled, const float* weight, int format, int layout, int B, int C,
                            int H, int W, int n_out, void* dfeatures, float* dweight, float* dbias, float* workspace,
                            void* stream);

/* replaces RegressionMSELoss.__call__ and RegressionRMSELoss.__call__ (remove_nans + compute_loss + mean)
 *   lightning_pose/losses/losses.py:880-996
 * targets, preds [n] fp32 (the (B, 2K) keypoint tensors), one CTA, no host sync.  out[4] =
 *   {mse, kept, rmse, pairs}: mse = mean of (t - p)^2 over the entries whose target is not NaN (NaN when none is);
 *   rmse = the reference's diagnostic: the kept squared errors compacted in order, paired as (x, y) (so an entry with
 *   only x NaN shifts the pairing of every later one, as reshape(-1, 2) does there), mean over the pairs of
 *   sqrt(pair mean); NaN when no entry is kept or their number is odd (where the reference's reshape raises).
 *   kept / pairs are the counts, exact up to 2^24.  A NaN prediction at a kept entry makes both losses NaN. */
int lpb_regression_losses_fwd(const float* targets, const float* preds, int64_t n, float* out, void* stream);
/* d mse / d preds given grad_out [1] (the rmse is a diagnostic: it gets no gradient); fwd_out = the forward's out;
 * grad_preds [n] is overwritten, 0 at the dropped entries. */
int lpb_regression_losses_bwd(const float* targets, const float* preds, int64_t n, const float* fwd_out, const float* grad_out,
                              float* grad_preds, void* stream);

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
