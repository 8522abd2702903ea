// Shape-generic bf16 heatmap head on the tensor cores: any feature map, one- or two-deconv heads (ViT / ResNet families).
// Reference: lightning_pose/models/heads/heatmap.py:20-71 (layer stack; ViT stride 16 -> one deconv, :192-193),
// :203-212 (forward).
//
// head_bf16.cu keeps a whole frame's operands in shared memory and therefore stops at 12x12 feature maps.  Here a
// transposed convolution is a *banded* 4-shift GEMM on the padded row layout (row_layout.cuh):
//   rows_shuffle_kernel   features (NCHW bf16) -> pixel-shuffled rows X[b][kchunk][row][8]      (one pass, HBM-bound)
//   convt_rows_kernel     X rows --TMA bulk, one copy per K-chunk--> smem stages (K streamed 32 channels at a time)
//                         --mma.sync, 4 shifted views--> register accumulators (<= 2 M-tiles = one band of image rows)
//                         --epilogue--> bf16 rows of the next layer | fp32 planes | two-pass plane softmax
// The band height adapts to the image width (R = 256 / (Wi + 1) image rows), so the accumulators (48 registers per
// tile and thread) and shared memory never depend on the frame size.  The softmax is computed by recomputation as in
// head_bf16.cu: pass 0 streams every band once for the per-plane (max, sum), pass 1 re-issues the GEMM and writes the
// normalised planes -- the logits never touch HBM.
#include <cuda_bf16.h>

#include <cstdint>
#include <type_traits>

#include "../../include/lpb200.h"
#include "head_prep.cuh"
#include "head_rows.cuh"
#include "lpb_common.cuh"
#include "row_layout.cuh"
#include "mma_sm90.cuh"

namespace lpb {

// ---- PixelShuffle(2) + NCHW -> padded row layout ----------------------------------------------------------------
// one CTA per (frame, K-chunk of 8 shuffled channels = 32 source channels): the slab is read with 16-byte loads,
// transposed through shared memory and written as whole rows (pads included, so the buffer needs no clearing)
__global__ void __launch_bounds__(256) rows_shuffle_kernel(const __nv_bfloat16* __restrict__ feat, int C, int H, int W,
                                                           __nv_bfloat16* __restrict__ xs, RowLayout L) {
  extern __shared__ __align__(16) unsigned char smraw[];
  __nv_bfloat16* sl = reinterpret_cast<__nv_bfloat16*>(smraw);  // [32][H*W]
  const int HW = H * W, nkc = C / 32;
  const int b = blockIdx.x / nkc, kc = blockIdx.x - b * nkc;
  const uint4* src = reinterpret_cast<const uint4*>(feat + ((size_t)b * C + (size_t)kc * 32) * HW);
  for (int i = threadIdx.x; i < 32 * HW / 8; i += 256) reinterpret_cast<uint4*>(sl)[i] = __ldg(src + i);
  __syncthreads();
  __nv_bfloat16* dst = xs + ((size_t)b * nkc + kc) * (size_t)L.rows * 8;
  const int body1 = L.lead + L.Hi * L.Pp;
  for (int r = threadIdx.x; r < L.rows; r += 256) {
    uint4 o = make_uint4(0, 0, 0, 0);
    if (r >= L.lead && r < body1) {
      const int t = r - L.lead, m = t / L.Pp, n = t - m * L.Pp;
      if (n < L.Wi) {
        const int q = 2 * (m & 1) + (n & 1), pos = (m >> 1) * W + (n >> 1);
        uint32_t pk[4];
#pragma unroll
        for (int e2 = 0; e2 < 4; ++e2) {
          const uint32_t lo = *reinterpret_cast<const unsigned short*>(sl + (size_t)(8 * e2 + q) * HW + pos);
          const uint32_t hi = *reinterpret_cast<const unsigned short*>(sl + (size_t)(8 * e2 + 4 + q) * HW + pos);
          pk[e2] = lo | (hi << 16);
        }
        o = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      }
    }
    *reinterpret_cast<uint4*>(dst + (size_t)r * 8) = o;
  }
}

int launch_rows_shuffle(const __nv_bfloat16* feat, int B, int C, int H, int W, __nv_bfloat16* xs, cudaStream_t s) {
  const RowLayout L = make_row_layout(2 * H, 2 * W);
  const size_t smem = (size_t)32 * H * W * 2;
  LPB_REQUIRE(smem <= 200 * 1024, "head_fwd_bf16: feature map %dx%d too large for the shuffle stage", H, W);
  if (smem > 48 * 1024) LPB_CUDA(cudaFuncSetAttribute(rows_shuffle_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  rows_shuffle_kernel<<<(unsigned)(B * (C / 32)), 256, smem, s>>>(feat, C, H, W, xs, L);
  return LPB_OK;
}

// ---- banded transposed-convolution GEMM ---------------------------------------------------------------------------
constexpr int CR_THREADS = 320;  // warp 0 loader, warp 1 idle, warps 2-9 MMA + epilogue
constexpr int CR_EPI = 256;
constexpr int CR_TILES = 2;      // M-tiles per band: a warp's accumulators (CR_TILES x 32 rows x 48 columns) stay in registers
static_assert(CR_TILES * 128 == CR_BAND_ROWS, "head_rows.cuh sizes the per-band softmax statistics with CR_BAND_ROWS");
constexpr int CR_STAGES = 2;

// NPL: compile-time plane count (17 = the usual keypoint count) or 0 for a run-time count <= 20.
// The softmax modes' epilogue takes one warp vote per tile (instead of one per plane), keeps the running-max rescale out
// of the common path, fetches (shift, 1/sum) as one 8-byte shared load and advances the output pointer by addition.
// WIDE: the output channels are P.ngroups keypoint groups (head_prep.cuh) and a work item is (frame [, band], group): it
// stages its rows, runs the group's 80-column GEMM and finishes the group's planes (or its mid channels [20g, 20g + 20),
// written as 8-byte halves of the K-chunks, since two groups can share a chunk).  The per-warp accumulators are those of
// a single group; a band is staged once per group and re-read from L2.
template <int MODE, int NPL, bool WIDE = false>
__global__ void __launch_bounds__(CR_THREADS, 1) convt_rows_kernel(const __grid_constant__ ConvtRowsParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int Pp = P.L.Pp, Wi = P.L.Wi, Hi = P.L.Hi;
  const int a_bytes = 4 * P.rows_alloc * 16, stage_bytes = a_bytes + HEAD_BSTAGE_BYTES;
  float* stat = reinterpret_cast<float*>(smem + CR_STAGES * stage_bytes);  // [2][HEAD_CLS][8 warps]
  float* fin = stat + 2 * HEAD_CLS * 8;                                       // [HEAD_CLS][2] = (max * log2 e, 1 / sum)
  uint64_t* bars = reinterpret_cast<uint64_t*>(fin + 2 * HEAD_CLS);
  uint64_t* full = bars;       // [2]
  uint64_t* empty = bars + 2;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < CR_STAGES * stage_bytes / 16; i += CR_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int s = 0; s < CR_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CR_EPI / 32);  // one arrival per MMA warp
    }
    fence_mbar_init();
  }
  fence_proxy_async();
  __syncthreads();

  const int R = P.R, nbands = (Hi + R - 1) / R, nst = P.nst;
  const int npass = MODE == CONVT_ROWS_SOFTMAX ? 2 : 1;
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  // Work items.  The fused two-pass softmax needs a whole frame per CTA (its per-plane max / sum run over all bands);
  // every other mode -- including the two halves of the SPLIT softmax (P0: per-band partial (max, sum) to global
  // scratch; P1: normalise with the frame's merged statistics) -- is independent per (frame, band), so small batches
  // (inference chunks, ViT training batches) still fill the GPU and large ones balance to within one band.
  constexpr bool PER_BAND = MODE != CONVT_ROWS_SOFTMAX;
  const int ng = WIDE ? P.ngroups : 1;
  const int nitems = (PER_BAND ? P.B * nbands : P.B) * ng;  // wide: the groups of a (frame, band) are consecutive items
  const int bands_per_item = PER_BAND ? 1 : nbands;
  constexpr bool SOFTMAX = MODE == CONVT_ROWS_SOFTMAX || MODE == CONVT_ROWS_SOFTMAX_P0 || MODE == CONVT_ROWS_SOFTMAX_P1;

  if (warp == 0) {
    // ================= loader: one bulk copy per K-chunk (band rows + the halo row below) + the stage's weights ====
    // single-stage GEMMs (K = 32) of one group keep their weights resident: each ring slot receives them once
    int it = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x)
      for (int pass = 0; pass < npass; ++pass)
        for (int bi = 0; bi < bands_per_item; ++bi) {
          const int g = WIDE ? item % ng : 0, fi = WIDE ? item / ng : item;
          const int b = PER_BAND ? fi / nbands : fi, band = PER_BAND ? fi - b * nbands : bi;
          const int y0 = band * R, rb = min(R, Hi - y0);
          const uint32_t nbytes = (uint32_t)((rb + 1) * Pp * 16);
          for (int st = 0; st < nst; ++st, ++it) {
            const int s = it % CR_STAGES;
            mbar_wait_idle(&empty[s], ((it / CR_STAGES) & 1) ^ 1);
            unsigned char* As = smem + s * stage_bytes;
            const bool load_b = nst > 1 || it < CR_STAGES || ng > 1;
            if (lane == 0) {
              mbar_expect_tx(&full[s], 4 * nbytes + (load_b ? HEAD_BSTAGE_BYTES : 0));
              if (load_b)
                bulk_g2s(As + a_bytes, reinterpret_cast<const unsigned char*>(P.wpk) + (size_t)(g * nst + st) * HEAD_BSTAGE_BYTES, HEAD_BSTAGE_BYTES,
                         &full[s]);
            }
            __syncwarp();
            if (lane < 4)
              bulk_g2s(As + (size_t)lane * P.rows_alloc * 16,
                       P.X + (((size_t)b * 4 * nst + 4 * st + lane) * P.L.rows + P.L.lead + (size_t)y0 * Pp) * 8, nbytes, &full[s]);
          }
        }
  } else if (warp >= 2) {
    // ================= MMA + epilogue: row quarter q = warp % 4, output-row parity e = (warp - 2) / 4 ===============
    // classes (py = e, px = 0 | 1) = accumulator columns [40e, 40e + 40); the warp accumulates [32e, 32e + 48) over the
    // stages and reads them out in "lane = row" form
    const int q = warp & 3, e = (warp - 2) >> 2, ew = warp - 2;
    const float L2E = 1.4426950408889634f;
    const size_t plane_stride = (size_t)Ho * Wo;
    const bool use_bias = P.bias && (MODE == CONVT_ROWS_MID || MODE == CONVT_ROWS_PLANES);  // a per-plane constant does not change a softmax
    const uint32_t lbo_a = P.rows_alloc * 16, lbo_b = HEAD_NCOLS * 16;
    int it = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int g = WIDE ? item % ng : 0, fi = WIDE ? item / ng : item;
      const int b = PER_BAND ? fi / nbands : fi;
      const int o0 = HEAD_CLS * g;                                       // the group's first output channel
      const int ncls = NPL ? NPL : (WIDE ? min(HEAD_CLS, P.cout - o0) : P.cout);  // planes handled by the unrolled loops
      const float* bias = use_bias ? P.bias + o0 : nullptr;
      float mx[HEAD_CLS], sm[HEAD_CLS];
#pragma unroll
      for (int o = 0; o < HEAD_CLS; ++o) {
        mx[o] = -1.0e30f;
        sm[o] = 0.f;
      }
      if constexpr (MODE == CONVT_ROWS_SOFTMAX_P1) {
        // merge the frame's per-band partials (written by the P0 launch) into (shift, 1 / sum) per plane
        asm volatile("bar.sync 1, 256;" ::: "memory");  // previous item's readers of fin are done
        if (tid - 64 < ncls) {
          const int o = tid - 64;
          const float* pp = P.partials + (((size_t)b * ng + g) * nbands * HEAD_CLS + o) * 2;
          float M = -1.0e30f;
          for (int j = 0; j < nbands; ++j) M = fmaxf(M, pp[(size_t)j * HEAD_CLS * 2]);
          float S = 0.f;
          for (int j = 0; j < nbands; ++j) S += pp[(size_t)j * HEAD_CLS * 2 + 1] * fast_exp2((pp[(size_t)j * HEAD_CLS * 2] - M) * L2E);
          fin[2 * o] = M * L2E;
          fin[2 * o + 1] = 1.0f / S;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      for (int pass = 0; pass < npass; ++pass) {
        const bool write = MODE == CONVT_ROWS_SOFTMAX_P0 ? false : (pass == npass - 1);
        for (int bi = 0; bi < bands_per_item; ++bi) {
          const int band = PER_BAND ? fi - b * nbands : bi;
          const int y0 = band * R, rb = min(R, Hi - y0), tiles = (rb * Pp + 127) / 128;
          float acc[CR_TILES][2][6][4];
#pragma unroll
          for (int t = 0; t < CR_TILES; ++t) mma::zero(acc[t]);
          for (int st = 0; st < nst; ++st, ++it) {
            const int s = it % CR_STAGES;
            mbar_wait_idle(&full[s], (it / CR_STAGES) & 1);
            const uint32_t a0 = smem_u32(smem + s * stage_bytes), b0 = a0 + a_bytes;
            // only the n8 tiles (of the warp's six, from column 32e) that the epilogue reads -- [40e, 40e + 40) -- and that
            // hold real taps of the shift: 8 tile-steps for e = 0 (shifts with dm = 1 carry nothing for py = 0), 16 for e = 1.
            // The softmax forms with a run-time plane count issue all six tiles with one body for both parities: there,
            // two per-parity bodies raised ptxas's local-memory spills.
            if constexpr (SOFTMAX && NPL == 0) {
#pragma unroll
              for (int t = 0; t < CR_TILES; ++t) {
                if (t >= tiles) break;
#pragma unroll
                for (int sh = 0; sh < 4; ++sh) {
                  const int shift_rows = (sh >> 1) * Pp + (sh & 1);
#pragma unroll
                  for (int k16 = 0; k16 < 2; ++k16)
                    mma::kstep(acc[t], a0 + (2 * k16) * lbo_a + (t * 128 + 32 * q + shift_rows) * 16, lbo_a,
                               b0 + (sh * 4 + 2 * k16) * lbo_b + 32 * e * 16, lbo_b, lane);
                }
              }
            } else {
              auto band_mma = [&](auto ec) {
                constexpr int E = decltype(ec)::value;
#pragma unroll
                for (int t = 0; t < CR_TILES; ++t) {
                  if (t >= tiles) break;
                  mma::for_shifts([&](auto shc) {
                    constexpr int sh = decltype(shc)::value;
                    constexpr unsigned mask = (NZ_N8[sh] >> (4 * E)) & (E ? 0x3eu : 0x1fu);
                    const int shift_rows = (sh >> 1) * Pp + (sh & 1);
#pragma unroll
                    for (int k16 = 0; k16 < 2; ++k16)
                      mma::kstep_nz<mask>(acc[t], a0 + (2 * k16) * lbo_a + (t * 128 + 32 * q + shift_rows) * 16, lbo_a,
                                          b0 + (sh * 4 + 2 * k16) * lbo_b + 32 * E * 16, lbo_b, lane);
                  });
                }
              };
              if (e == 0) band_mma(std::integral_constant<int, 0>{});
              else band_mma(std::integral_constant<int, 1>{});
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
          }
#pragma unroll
          for (int t = 0; t < CR_TILES; ++t) {
            if (t >= tiles) break;
            float d[48];
#pragma unroll
            for (int nt = 0; nt < 6; ++nt) mma::rows8(acc[t], nt, &d[8 * nt], lane);
            const int row = t * 128 + 32 * q + lane;
            const int ml = row / Pp, n = row - ml * Pp;
            const bool valid = (ml < rb) && (n < Wi);
            const int y = 2 * (y0 + ml) + e, x = 2 * n;
            auto body = [&](auto ec) {
              constexpr int E = decltype(ec)::value;
              if constexpr (MODE == CONVT_ROWS_MID && WIDE) {
                // bf16 rows of the next layer, by 4-channel units (8-byte halves of a K-chunk): the group's five units
                // 5g .. 5g + 4, and the last group also the units past the groups up to the end of the last K-chunk.
                // Channel `cout` is the constant one, every other channel >= cout is 0.
                if (valid) {
                  const int u1 = g == ng - 1 ? 2 * P.mid_kc : 5 * g + 5;
#pragma unroll
                  for (int px = 0; px < 2; ++px) {
                    const size_t row2 = (size_t)P.Lout.lead + (size_t)y * P.Lout.Pp + x + px;
                    __nv_bfloat16* base = P.mid + ((size_t)b * P.mid_kc * P.Lout.rows + row2) * 8;
#pragma unroll
                    for (int i = 0; i < HEAD_CLS / 4; ++i) {
                      const int u = 5 * g + i;
                      uint32_t pk[2];
#pragma unroll
                      for (int e2 = 0; e2 < 2; ++e2) {
                        float f[2];
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                          const int cl = 4 * i + 2 * e2 + hh;  // compile-time channel within the group
                          const int ch = o0 + cl;
                          f[hh] = ch < P.cout ? d[8 * E + px * HEAD_CLS + cl] + (use_bias ? __ldg(bias + cl) : 0.f) : (ch == P.cout ? 1.0f : 0.f);
                        }
                        __nv_bfloat162 h2 = __floats2bfloat162_rn(f[0], f[1]);
                        pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
                      }
                      *reinterpret_cast<uint2*>(base + (size_t)(u >> 1) * P.Lout.rows * 8 + (u & 1) * 4) = make_uint2(pk[0], pk[1]);
                    }
                    for (int u = 5 * g + 5; u < u1; ++u) {
                      const int c0 = 4 * u;
                      const uint32_t one = 0x3f80u;  // bf16 1.0
                      const uint32_t lo = (c0 == P.cout ? one : 0u) | (c0 + 1 == P.cout ? one << 16 : 0u);
                      const uint32_t hi = (c0 + 2 == P.cout ? one : 0u) | (c0 + 3 == P.cout ? one << 16 : 0u);
                      *reinterpret_cast<uint2*>(base + (size_t)(u >> 1) * P.Lout.rows * 8 + (u & 1) * 4) = make_uint2(lo, hi);
                    }
                  }
                }
                return;
              } else if constexpr (MODE == CONVT_ROWS_MID) {
                // bf16 rows of the next layer: channel `cout` is the constant one (carries that layer's bias)
                if (valid) {
#pragma unroll
                  for (int px = 0; px < 2; ++px) {
                    const size_t row2 = (size_t)P.Lout.lead + (size_t)y * P.Lout.Pp + x + px;
#pragma unroll
                    for (int kc = 0; kc < 4; ++kc) {
                      uint32_t pk[4];
#pragma unroll
                      for (int e2 = 0; e2 < 4; ++e2) {
                        float f[2];
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                          const int ch = kc * 8 + 2 * e2 + hh;  // compile-time
                          float val = 0.f;
                          if (ch < HEAD_CLS) {
                            if (ch < P.cout) val = d[8 * E + px * HEAD_CLS + ch] + (use_bias ? __ldg(P.bias + ch) : 0.f);
                            else if (ch == P.cout) val = 1.0f;
                          } else if (ch == P.cout) {
                            val = 1.0f;
                          }
                          f[hh] = val;
                        }
                        __nv_bfloat162 h2 = __floats2bfloat162_rn(f[0], f[1]);
                        pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
                      }
                      *reinterpret_cast<uint4*>(P.mid + ((((size_t)b * 4 + kc) * P.Lout.rows + row2) * 8)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                    }
                  }
                }
                return;
              }
              float* dst = P.out + (((size_t)b * P.cout + o0) * Ho + y) * Wo + x;  // plane o0 + o adds o * Ho * Wo
              if constexpr (SOFTMAX) {
                if (!write) {
                  // ---- pass 0: per-thread online (max, sum) per plane; the rescale is rare after the first tiles ----
                  bool need = false;
#pragma unroll
                  for (int o = 0; o < HEAD_CLS; ++o) {
                    if (o >= ncls) break;
                    need |= fmaxf(d[8 * E + o], d[8 * E + HEAD_CLS + o]) > mx[o];
                  }
                  if (__any_sync(0xffffffffu, need && valid)) {
                    if (valid) {
#pragma unroll
                      for (int o = 0; o < HEAD_CLS; ++o) {
                        if (o >= ncls) break;
                        const float tm = fmaxf(d[8 * E + o], d[8 * E + HEAD_CLS + o]);
                        if (tm > mx[o]) {
                          sm[o] *= fast_exp2((mx[o] - tm) * L2E);
                          mx[o] = tm;
                        }
                      }
                    }
                  }
                  if (valid) {
#pragma unroll
                    for (int o = 0; o < HEAD_CLS; ++o) {
                      if (o >= ncls) break;
                      const float mL = mx[o] * L2E;
                      sm[o] += fast_exp2(fmaf(d[8 * E + o], L2E, -mL)) + fast_exp2(fmaf(d[8 * E + HEAD_CLS + o], L2E, -mL));
                    }
                  }
                } else if (valid) {
                  // ---- pass 1: normalise and store; (shift, 1 / sum) is one 8-byte shared load per plane ----
#pragma unroll
                  for (int o = 0; o < HEAD_CLS; ++o) {
                    if (o >= ncls) break;
                    const float2 f = reinterpret_cast<const float2*>(fin)[o];
                    const float p0 = fast_exp2(fmaf(d[8 * E + o], L2E, -f.x)) * f.y;
                    const float p1 = fast_exp2(fmaf(d[8 * E + HEAD_CLS + o], L2E, -f.x)) * f.y;
                    *reinterpret_cast<float2*>(dst) = make_float2(p0, p1);
                    dst += plane_stride;
                  }
                }
              } else {
                // CONVT_ROWS_PLANES: raw planes (+ bias)
#pragma unroll
                for (int o = 0; o < HEAD_CLS; ++o) {
                  if (o >= ncls) break;
                  const float bo = use_bias ? __ldg(bias + o) : 0.f;
                  const float l0 = d[8 * E + o] + bo, l1 = d[8 * E + HEAD_CLS + o] + bo;
                  if (valid) *reinterpret_cast<float2*>(dst + (size_t)o * plane_stride) = make_float2(l0, l1);
                }
              }
            };
            if (e == 0) body(std::integral_constant<int, 0>{});
            else body(std::integral_constant<int, 1>{});
          }
        }
        if ((npass == 2 && pass == 0) || MODE == CONVT_ROWS_SOFTMAX_P0) {
          // merge the online-softmax states: lanes -> warp (shuffles) -> 8 epilogue warps (smem)
#pragma unroll
          for (int o = 0; o < HEAD_CLS; ++o) {
            if (o >= ncls) break;
            const float M = warp_max(mx[o]);
            const float S = warp_sum(sm[o] * fast_exp2((mx[o] - M) * L2E));
            if (lane == 0) {
              stat[o * 8 + ew] = M;
              stat[(HEAD_CLS + o) * 8 + ew] = S;
            }
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (tid - 64 < ncls) {
            const int o = tid - 64;
            float M = stat[o * 8];
#pragma unroll
            for (int i = 1; i < 8; ++i) M = fmaxf(M, stat[o * 8 + i]);
            float S = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) S += stat[(HEAD_CLS + o) * 8 + i] * fast_exp2((stat[o * 8 + i] - M) * L2E);
            if constexpr (MODE == CONVT_ROWS_SOFTMAX_P0) {
              float* pp = P.partials + ((((size_t)b * ng + g) * nbands + (fi - b * nbands)) * HEAD_CLS + o) * 2;
              pp[0] = M;
              pp[1] = S;
            } else {
              fin[2 * o] = M * L2E;
              fin[2 * o + 1] = 1.0f / S;
            }
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
      }
    }
  }
}

int launch_convt_rows(ConvtRowsParams p, int sms, cudaStream_t s) {
  const int Pp = p.L.Pp;
  LPB_REQUIRE(Pp <= CR_TILES * 128, "head_fwd_bf16: image width %d too large for one band", p.L.Wi);
  LPB_REQUIRE(p.cout >= 1 && p.cout <= HEAD_MAX_CH, "head_fwd_bf16: %d output channels exceed %d", p.cout, HEAD_MAX_CH);
  LPB_REQUIRE(p.mode != CONVT_ROWS_MID || p.mid_kc >= 4 * head_mid_stages(p.cout), "head_fwd_bf16: mid activations of %d K-chunks", p.mid_kc);
  p.R = (CR_TILES * 128) / Pp;
  if (p.R > p.L.Hi) p.R = p.L.Hi;
  const int tiles = (p.R * Pp + 127) / 128;
  p.rows_alloc = (tiles * 128 + Pp + 1 + 7) & ~7;
  if (p.rows_alloc < (p.R + 1) * Pp + 8) p.rows_alloc = ((p.R + 1) * Pp + 8 + 7) & ~7;
  const size_t smem = (size_t)CR_STAGES * (4 * p.rows_alloc * 16 + HEAD_BSTAGE_BYTES) + (2 * HEAD_CLS * 8 + 2 * HEAD_CLS) * sizeof(float) + 64;
  LPB_REQUIRE(smem <= 113 * 1024, "head_fwd_bf16: band stages need %zu B shared memory", smem);
  const int nbands = (p.L.Hi + p.R - 1) / p.R;
  auto run = [&](auto kern, long long nitems) -> int {
    const int grid = (int)(nitems < sms ? nitems : sms);  // one CTA per SM: the accumulators take the register file
    LPB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, CR_THREADS, smem, s>>>(p);
    return LPB_OK;
  };
  // wide layers (more than 20 output channels; 20 or more for the first of two, whose mid activations then take more
  // than one K stage) run the keypoint-group instantiations
  const bool wide = p.cout > HEAD_CLS || (p.mode == CONVT_ROWS_MID && p.cout >= HEAD_CLS);
  p.ngroups = head_groups(p.cout);
  if (wide) {
    const long long per_group = (long long)p.B * nbands * p.ngroups;
    if (p.mode == CONVT_ROWS_MID) return run(convt_rows_kernel<CONVT_ROWS_MID, 0, true>, per_group);
    if (p.mode == CONVT_ROWS_PLANES) return run(convt_rows_kernel<CONVT_ROWS_PLANES, 0, true>, per_group);
    // the split / fused choice of the narrow heads below, counting (frame, group) items
    if (p.partials && (g_softmax_split == 2 || (g_softmax_split == 1 && (long long)p.B * p.ngroups < sms))) {
      const int rc = run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P0, 0, true>, per_group);
      if (rc != LPB_OK) return rc;
      return run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P1, 0, true>, per_group);
    }
    return run(convt_rows_kernel<CONVT_ROWS_SOFTMAX, 0, true>, (long long)p.B * p.ngroups);
  }
  const bool k17 = p.cout == 17;
  const long long per_band = (long long)p.B * nbands;
  if (p.mode == CONVT_ROWS_MID) return run(convt_rows_kernel<CONVT_ROWS_MID, 0>, per_band);
  if (p.mode == CONVT_ROWS_PLANES) return k17 ? run(convt_rows_kernel<CONVT_ROWS_PLANES, 17>, per_band) : run(convt_rows_kernel<CONVT_ROWS_PLANES, 0>, per_band);
  // split softmax (statistics launch + normalising launch, both parallel over (frame, band)) when one CTA per frame would
  // leave SMs idle (fewer frames than SMs); otherwise the single two-pass kernel is faster, because a frame's second pass
  // re-reads operands its first pass left in L2 (768-frame step 1.768 vs 1.802 ms; with the 256-frame labeled call fused
  // as well: step 1.565 vs 1.583 ms, forward-only 0.611 vs 0.635 ms).  Key value 2 forces the split.
  const int split_key = g_softmax_split;
  if (p.partials && (split_key == 2 || (split_key == 1 && p.B < sms))) {
    int rc = k17 ? run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P0, 17>, per_band) : run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P0, 0>, per_band);
    if (rc != LPB_OK) return rc;
    return k17 ? run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P1, 17>, per_band) : run(convt_rows_kernel<CONVT_ROWS_SOFTMAX_P1, 0>, per_band);
  }
  return k17 ? run(convt_rows_kernel<CONVT_ROWS_SOFTMAX, 17>, p.B) : run(convt_rows_kernel<CONVT_ROWS_SOFTMAX, 0>, p.B);
}

}  // namespace lpb
