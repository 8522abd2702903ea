// bf16 heatmap head on the tensor cores (mma.sync m16n8k16, fp32 accumulators in registers), two-deconv (ResNet-family)
// heads.
// Reference: lightning_pose/models/heads/heatmap.py:20-71 (layer stack), :203-212 (forward).
//
// Formulation ("4-shift GEMM").  A stride-2 3x3 transposed convolution in gather form:
//   out[o, 2m+py, 2n+px] = b[o] + sum_c sum_{(dm,dn) valid for (py,px)} in[c, m+dm, n+dn] * W[c, o, ky, kx]
//   with ky = (py==0 ? 1 : (dm ? 0 : 2)), kx likewise.
// Lay the input out pixel-major, A[row = m*(Wi+1) + n][c] with a zero column n = Wi and a zero row
// m = Hi; then the four (dm,dn) shifts are the SAME matrix read from a start address moved by
// (dm*(Wi+1) + dn) rows, and
//   D[row, cls*20 + o] = sum_shift A_shift[row, :] . B_shift[cls*20 + o, :]
// is an ordinary GEMM accumulated over 4 shifts x K.  D needs no col2im: row (m,n), class
// (py,px) IS output pixel (2m+py, 2n+px).  Operands use the K-major row layout (16-byte rows, linear
// in memory), so a row shift is just a different ldmatrix start address (mma_sm90.cuh).
//
//   k1a: features (NCHW bf16) --[PixelShuffle folded into a transposing producer]--> smem A stages
//        --mma.sync--> registers --epilogue(+bias, ->bf16)--> mid activations in the A layout (global)
//   k1b: mid (A layout, TMA bulk rows) --mma.sync--> registers --epilogue--> two-pass plane softmax
//        (pass 0: online max/sum, pass 1: recompute the cheap K=32 GEMM and write normalised fp32)
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

constexpr int HB_NCOLS = 80;         // 4 classes x 20 (>= 17 keypoints), multiple of 16
constexpr int HB_CLS = 20;
constexpr int HB_KSTAGE = 32;        // channels per pipeline stage (4 K-chunks of 8)
constexpr int HB_BSTAGE_BYTES = 4 * 4 * HB_NCOLS * 16;  // [shift][kchunk][80 rows][16 B]

struct HeadGeom {
  int Hi, Wi;       // conv input spatial size (after PixelShuffle for layer 1)
  int P;            // row pitch = Wi + 1 (zero column)
  int rows;         // Hi * P
  int tiles;        // ceil(rows / 128)
  int rows_alloc;   // smem rows per K-chunk (multiple of 8), covers tiles*128 + P + 1
};

__host__ inline HeadGeom make_geom(int Hi, int Wi) {
  HeadGeom g;
  g.Hi = Hi;
  g.Wi = Wi;
  g.P = Wi + 1;
  g.rows = Hi * g.P;
  g.tiles = (g.rows + 127) / 128;
  g.rows_alloc = (g.tiles * 128 + g.P + 1 + 7) & ~7;
  return g;
}

// ---- everything a head call prepares, in one launch (head_prep.cuh) -------------------------------------------
// forward packs: W[Cin][Cout][3][3] (fp32) -> B[stage][shift][kchunk][80][8] bf16; a non-null bias rides on input
// channel `Cin` (the constant-one channel of the mid activations; shift (0,0) only, which every output class uses once)
constexpr int PREP_GB_K = 80, PREP_GB_KC = 10, PREP_GB_CLS = 20;  // class-major K of the gradient operands (head_bwd_bf16.cu)

__global__ void __launch_bounds__(256) head_prep_kernel(const __grid_constant__ PrepJobs J) {
  const long long tid0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (!J.fpack[j].out) continue;
    const float* w = J.fpack[j].w;
    const float* bias = J.fpack[j].bias;
    const int Cin = J.fpack[j].Cin, Cout = J.fpack[j].Cout;
    const long long total = (long long)J.fpack[j].nstages * 4 * 4 * HB_NCOLS * 8;
    for (long long i = tid0; i < total; i += nthr) {
      const int e = (int)(i & 7);
      long long r = i >> 3;
      const int nrow = (int)(r % HB_NCOLS);
      r /= HB_NCOLS;
      const int kc = (int)(r & 3);
      r >>= 2;
      const int sh = (int)(r & 3);
      const int st = (int)(r >> 2);
      const int c = st * HB_KSTAGE + kc * 8 + e;
      const int cls = nrow / HB_CLS, o = nrow % HB_CLS;
      const int py = cls >> 1, px = cls & 1, dm = sh >> 1, dn = sh & 1;
      float v = 0.f;
      if (c < Cin && o < Cout && !(py == 0 && dm == 1) && !(px == 0 && dn == 1)) {
        const int ky = py == 0 ? 1 : (dm ? 0 : 2);
        const int kx = px == 0 ? 1 : (dn ? 0 : 2);
        v = w[((size_t)c * Cout + o) * 9 + ky * 3 + kx];
      } else if (bias && c == Cin && o < Cout && sh == 0) {
        v = bias[o];
      }
      J.fpack[j].out[i] = __float2bfloat16_rn(v);
    }
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (!J.dpack[j].out) continue;
    const float* w = J.dpack[j].w;
    const int Cin = J.dpack[j].Cin, Cout = J.dpack[j].Cout, rpt = J.dpack[j].rows_per_tile;
    const long long total = (long long)J.dpack[j].ntiles * 4 * PREP_GB_KC * rpt * 8;
    for (long long i = tid0; i < total; i += nthr) {
      const int e = (int)(i & 7);
      long long r = i >> 3;
      const int row = (int)(r % rpt);
      r /= rpt;
      const int kc = (int)(r % PREP_GB_KC);
      r /= PREP_GB_KC;
      const int sh = (int)(r & 3);
      const int tile = (int)(r >> 2);
      const int c = tile * rpt + row;
      const int k = kc * 8 + e;
      const int cls = k / PREP_GB_CLS, o = k % PREP_GB_CLS;
      const int py = cls >> 1, px = cls & 1, dm = sh >> 1, dn = sh & 1;
      float v = 0.f;
      if (c < Cin && o < Cout && !(py == 0 && dm == 1) && !(px == 0 && dn == 1)) {
        const int ky = py == 0 ? 1 : (dm ? 0 : 2);
        const int kx = px == 0 ? 1 : (dn ? 0 : 2);
        v = w[((size_t)c * Cout + o) * 9 + ky * 3 + kx];
      }
      J.dpack[j].out[i] = __float2bfloat16_rn(v);
    }
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (!J.pads[j].buf) continue;
    const RowLayout L = J.pads[j].L;
    const int body0 = L.lead, body1 = L.lead + L.Hi * L.Pp;
    const int npad = L.lead + (L.rows - body1) + L.Hi;
    const long long total = J.pads[j].nslabs * npad;
    for (long long i = tid0; i < total; i += nthr) {
      const long long slab = i / npad;
      const int e = (int)(i - slab * npad);
      int row;
      if (e < L.lead) row = e;
      else if (e < L.lead + (L.rows - body1)) row = body1 + (e - L.lead);
      else row = body0 + (e - L.lead - (L.rows - body1)) * L.Pp + L.Wi;
      *reinterpret_cast<uint4*>(J.pads[j].buf + ((size_t)slab * L.rows + row) * 8) = make_uint4(0, 0, 0, 0);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (!J.zero[j].p) continue;
    for (long long i = tid0; i < J.zero[j].n; i += nthr) J.zero[j].p[i] = 0.f;
  }
}

int launch_head_prep(const PrepJobs& jobs, cudaStream_t s) {
  head_prep_kernel<<<132 * 2, 256, 0, s>>>(jobs);  // two CTAs per SM of an H100 SXM
  return LPB_OK;
}

// =====================================================================================================
// k1a: PixelShuffle + first transposed convolution
// =====================================================================================================
// warps 0..TW-1 transposers, warps TW..TW+CW-1 MMA + epilogue, warp TW+CW TMA loader (+ warp TW+CW+1: saved-copy stores)
// A CTA works on (frame, tile group) items: the group's K1A_TPG M-tiles of 128 raster rows keep their fp32 accumulators in
// the MMA warps' registers across all channel stages (warp = one tile's 32-row quarter, 80 columns = 80 registers).
constexpr int K1A_TW = 4;                      // transposer warps
constexpr int K1A_TPG = 2;                     // M-tiles per item
constexpr int K1A_CW = 4 * K1A_TPG;            // MMA warps
constexpr int K1A_LOADER = K1A_TW + K1A_CW;
constexpr int K1A_THREADS = 32 * (K1A_TW + K1A_CW + 1);
constexpr int K1A_ASTAGES = 2;  // K-major operand stages (A + packed weights)
constexpr int K1A_RSTAGES = 2;  // raw NCHW stages filled by the TMA engine
constexpr int K1A_MAXPAD = 6;   // pad rows of the saved copy a transposer thread writes per stage (host falls back to head_prep beyond)

struct K1aParams {
  const __nv_bfloat16* feat;  // [B][C][H*W]
  const __nv_bfloat16* wpk;   // packed weights [nstages][HB_BSTAGE_BYTES]
  const float* bias;          // [c1]
  __nv_bfloat16* mid;         // [B][4][Lmid.rows][8]  padded row layout of the next layer's input (row_layout.cuh)
  __nv_bfloat16* xs;          // optional [B][C/32][Lxs.rows][8]: shuffled features in the padded row layout (weight gradient)
  RowLayout Lmid, Lxs;
  int B, C, HW, W;            // feature geometry (C = 4 * Cin)
  int c1, nstages;
  int row_transposer;         // 1: row-per-lane transposer (coalesced operand-copy stores); 0: 8x8 register-block transposer
  int backoff;                // idle warps sleep between barrier polls
  int xs_bulk;                // 1: the saved operand copy is written by TMA bulk stores straight from the operand stage
  int xs_pads;                // 1: the block transposers also write the saved copy's pad rows (else head_prep cleared them)
  int xs_copy;                // 1: the saved copy is streamed out of the finished operand stage by all transposer threads (coalesced)
  int ntg;                    // tile groups per frame (items per frame); only group 0 writes the saved copy
  HeadGeom g;
};

// XS (compile time, block transposers): 0 = no saved copy (inference); 1 = the run-time forms (direct stores with / without
// pad rows, bulk stores, the row-form transposer); 2 = copy-out of the finished operand stage.  Forms 0 and 2 carry none of
// form 1's per-task address arithmetic (it cost the hot loop predicated-off instructions and local-memory spills).
// 3 = a dedicated extra warp (block of K1A_THREADS + 32) sends each finished operand stage to the saved copy with TMA bulk
// stores: the transposers store nothing, and unlike the loader-issued bulk form (xs_bulk) nothing else waits on the stores.
template <int XS>
__global__ void __launch_bounds__(K1A_THREADS + 32, 1) k1a_shuffle_convt_kernel(const __grid_constant__ K1aParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const HeadGeom g = P.g;
  const int a_stage_bytes = 4 * g.rows_alloc * 16;
  const int stage_bytes = a_stage_bytes + HB_BSTAGE_BYTES;
  const int raw_bytes = 4 * HB_KSTAGE * P.HW * 2;  // 128 source channels of one stage, contiguous in NCHW
  unsigned char* stage_base = smem;
  unsigned char* raw_base = smem + K1A_ASTAGES * stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(raw_base + K1A_RSTAGES * raw_bytes);
  uint64_t* full = bars;                        // [2] operands ready (128 transposer arrivals + weight bytes)
  uint64_t* empty = bars + 2;                   // [2] MMAs reading the stage have completed
  uint64_t* raw_full = bars + 4;                // [2] TMA bytes landed
  uint64_t* raw_empty = bars + 6;               // [2] transposers are done with the raw stage
  unsigned char* zreg = reinterpret_cast<unsigned char*>(bars) + 128;  // 1 KB of zeros: source of the saved copy's lead rows
  const bool xs_bulk = P.xs && P.xs_bulk;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // zero the operand stages once: halo rows/columns are never written again
  for (int i = tid; i < K1A_ASTAGES * stage_bytes / 16; i += K1A_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  if (tid < 64) reinterpret_cast<uint4*>(zreg)[tid] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full[s], 32 * K1A_TW + 1);
      mbar_init(&empty[s], K1A_CW + ((xs_bulk || XS == 3) ? 1 : 0));  // the MMA warps have read the stage (+ the bulk stores of the saved copy have)
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], 32 * K1A_TW);
    }
    fence_mbar_init();
  }
  fence_proxy_async();  // generic-proxy zero fill -> visible to the async proxy (bulk stores of the saved copy)
  __syncthreads();

  const int rows_mid = P.Lmid.rows;
  const int nitems = P.B * P.ntg;
  int nmine = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) ++nmine;
  const int total_it = nmine * P.nstages;
  // item of pipeline iteration it: frame b, tile group tg (group 0 also writes the saved copy)
  auto item_of = [&](int it, int& b, int& tg) {
    const int item = blockIdx.x + (it / P.nstages) * gridDim.x;
    b = item / P.ntg;
    tg = item - b * P.ntg;
  };

  if (warp == K1A_LOADER) {
    // ================= TMA loader: raw feature slabs run ahead, weights follow the operand slots ====
    if (lane == 0) {
      auto issue_raw = [&](int it) {
        const int r = it % K1A_RSTAGES;
        mbar_wait(&raw_empty[r], ((it / K1A_RSTAGES) & 1) ^ 1);
        int b, tg;
        item_of(it, b, tg);
        const int st = it % P.nstages;
        mbar_expect_tx(&raw_full[r], (uint32_t)raw_bytes);
        bulk_g2s(raw_base + r * raw_bytes, P.feat + ((size_t)b * P.C + (size_t)st * 4 * HB_KSTAGE) * P.HW, (uint32_t)raw_bytes,
                 &raw_full[r]);
      };
      if (total_it > 0) issue_raw(0);
      for (int it = 0; it < total_it; ++it) {
        if (it + 1 < total_it) issue_raw(it + 1);
        const int s = it % K1A_ASTAGES, st = it % P.nstages;
        mbar_wait(&empty[s], ((it / K1A_ASTAGES) & 1) ^ 1);
        mbar_expect_tx(&full[s], HB_BSTAGE_BYTES);
        bulk_g2s(stage_base + s * stage_bytes + a_stage_bytes,
                 reinterpret_cast<const unsigned char*>(P.wpk) + (size_t)st * HB_BSTAGE_BYTES, HB_BSTAGE_BYTES, &full[s]);
        if (xs_bulk) {
          // The operand stage IS the saved copy's layout (row_layout.cuh): once the producers have filled it, each
          // K-chunk goes to global memory as two bulk stores (the zero lead rows, then raster + halo rows) -- fully
          // coalesced, asynchronous, and no store instruction on the producers' LSU path (their 16-byte stores at a
          // 256-byte stride were k1a's critical path in training).  The stage is released once the MMAs AND these
          // stores have read it.
          mbar_wait(&full[s], (it / K1A_ASTAGES) & 1);
          int b, tg;
          item_of(it, b, tg);
          if (tg == 0) {
            unsigned char* slab = reinterpret_cast<unsigned char*>(P.xs + ((size_t)b * P.nstages + st) * 4 * (size_t)P.Lxs.rows * 8);
            const unsigned char* As = stage_base + s * stage_bytes;
            const uint32_t lead_b = (uint32_t)P.Lxs.lead * 16, body_b = (uint32_t)(g.rows + g.P + 1) * 16;
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {
              unsigned char* dst = slab + (size_t)kc * P.Lxs.rows * 16;
              bulk_s2g(dst, zreg, lead_b);
              bulk_s2g(dst + lead_b, As + (size_t)kc * g.rows_alloc * 16, body_b);
            }
            bulk_commit_group();
            bulk_wait_group_read0();
          }
          mbar_arrive(&empty[s]);
        }
      }
      if (xs_bulk) bulk_wait_group0();  // the copies are in global memory before the kernel ends
    }
  } else if (warp < K1A_TW && P.row_transposer) {
    // ================= transposers, row form: lane = shuffled pixel n of one image row ==================
    // A warp takes (K-chunk kc, image row m) pairs; lane n gathers its 8 channels (source channels 4(8kc+e)+q, q =
    // 2(m&1) + (n&1), position (m>>1, n>>1)) with 2-byte shared loads -- conflict-free: even / odd lanes read two
    // channel rows 288 B apart -- and stores ONE 16-byte operand row.  Consecutive lanes write consecutive rows, so
    // both the shared-memory store and the global store of the saved copy are fully coalesced (the 8x8 register-block
    // form writes 16 bytes per lane at a 256-byte stride: 32 half-used sectors per store instruction, which made the
    // transposers' LSU time -- not the tensor core -- the critical path of a training forward).
    const int Hi = g.Hi, Wi = g.Wi, npair = 4 * Hi;
    for (int it = 0; it < total_it; ++it) {
      const int s = it % K1A_ASTAGES, r = it % K1A_RSTAGES;
      mbar_wait(&raw_full[r], (it / K1A_RSTAGES) & 1);
      mbar_wait(&empty[s], ((it / K1A_ASTAGES) & 1) ^ 1);
      unsigned char* As = stage_base + s * stage_bytes;
      unsigned char* xs_st = nullptr;
      if (P.xs && !xs_bulk) {
        int b, tg;
        item_of(it, b, tg);
        const int st = it % P.nstages;
        if (tg == 0) xs_st = reinterpret_cast<unsigned char*>(P.xs + ((size_t)b * P.nstages + st) * 4 * (size_t)P.Lxs.rows * 8);
      }
      const unsigned short* raw = reinterpret_cast<const unsigned short*>(raw_base + r * raw_bytes);
      for (int pr = warp; pr < npair; pr += K1A_TW) {
        const int kc = pr / Hi, m = pr - kc * Hi;
        const int chan0 = 32 * kc + 2 * (m & 1);  // source channel of e = 0, dj = 0
        for (int n = lane; n < Wi; n += 32) {
          const unsigned short* src = raw + (size_t)(chan0 + (n & 1)) * P.HW + (m >> 1) * P.W + (n >> 1);
          uint32_t pk[4];
#pragma unroll
          for (int e2 = 0; e2 < 4; ++e2) pk[e2] = (uint32_t)src[(size_t)(8 * e2) * P.HW] | ((uint32_t)src[(size_t)(8 * e2 + 4) * P.HW] << 16);
          const uint4 o = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          const int row = m * g.P + n;
          *reinterpret_cast<uint4*>(As + ((size_t)kc * g.rows_alloc + row) * 16) = o;
          if (xs_st) *reinterpret_cast<uint4*>(xs_st + ((size_t)kc * P.Lxs.rows + P.Lxs.lead + row) * 16) = o;
        }
      }
      fence_proxy_async();
      mbar_arrive(&full[s]);
      mbar_arrive(&raw_empty[r]);
    }
  } else if (warp < K1A_TW) {
    // ================= transposers: raw NCHW slab (smem) -> K-major rows, PixelShuffle folded in ======
    // A task is one 8x8 bf16 transpose: 8 channels x 8 consecutive spatial positions (one 16-byte chunk per channel)
    // of one sub-pixel class q -> 8 rows of 16 bytes.  Which tasks a thread owns, and where they read / write, is the
    // same for every stage, so the index arithmetic (divisions by runtime sizes) is done once, up front.
    const int nchunk = P.HW / 8;  // 16-byte chunks of 8 consecutive spatial positions per channel
    const int ntasks = 4 * 4 * nchunk;
    constexpr int MAXT = 3;
    uint32_t t_raw[MAXT], t_a[MAXT], t_x[MAXT];
    int t_wrap[MAXT];
    int nt = 0;
#pragma unroll
    for (int k = 0; k < MAXT; ++k) {
      const int task = tid + k * 32 * K1A_TW;
      t_raw[k] = t_a[k] = t_x[k] = 0;
      t_wrap[k] = 8;
      if (task < ntasks) {
        const int sc = task % nchunk, q = (task / nchunk) & 3, kc = task / (4 * nchunk);
        const int sp0 = sc * 8, i0 = sp0 / P.W, jc0 = sp0 - i0 * P.W;
        const int row0 = (2 * i0 + (q >> 1)) * g.P + 2 * jc0 + (q & 1);
        t_raw[k] = (uint32_t)(((4 * kc * 8 + q) * P.HW + sc * 8) * 2);
        t_a[k] = (uint32_t)((kc * g.rows_alloc + row0) * 16);
        if (XS == 1) t_x[k] = (uint32_t)((kc * P.Lxs.rows + P.Lxs.lead + row0) * 16);
        t_wrap[k] = P.W - jc0;  // position at which the image row wraps (W >= 8: at most once per task)
        nt = k + 1;
      }
    }
    const uint32_t chan_stride = (uint32_t)(4 * P.HW * 2);       // next shuffled channel e -> 4 source channels on
    const uint32_t wrap_jump = (uint32_t)((2 * g.P - 2 * P.W) * 16);  // extra bytes once the position wraps to row i + 1
    // The saved copy's pad rows (the zero column of every image row, the lead / trail rows) are written here as well, next
    // to the real rows that share their 32-byte sectors: a separate clearing pass over those scattered 16-byte pieces
    // cost 35 us per 512 frames in the preparation launch.  Per stage: 4 K-chunks x npad rows over the 128 transposer threads.
    constexpr int MAXP = K1A_MAXPAD;
    uint32_t t_pad[MAXP];
    int npd = 0;
    if (XS == 1) {
      const RowLayout L = P.Lxs;
      const int body1 = L.lead + L.Hi * L.Pp, ntail = L.rows - body1, npad = L.lead + ntail + L.Hi;
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        const int e = tid + k * 32 * K1A_TW;
        t_pad[k] = 0;
        if (e < 4 * npad) {
          const int kc = e / npad, i = e - kc * npad;
          const int row = i < L.lead ? i : (i < L.lead + ntail ? body1 + (i - L.lead) : L.lead + (i - L.lead - ntail) * L.Pp + L.Wi);
          t_pad[k] = (uint32_t)((kc * L.rows + row) * 16);
          npd = k + 1;
        }
      }
    }
    for (int it = 0; it < total_it; ++it) {
      const int s = it % K1A_ASTAGES, r = it % K1A_RSTAGES;
      mbar_wait(&raw_full[r], (it / K1A_RSTAGES) & 1);
      mbar_wait(&empty[s], ((it / K1A_ASTAGES) & 1) ^ 1);
      unsigned char* As = stage_base + s * stage_bytes;
      unsigned char* xs_st = nullptr;  // this (frame, stage)'s 4 K-chunks of the saved copy
      unsigned char* xs_cp = nullptr;  // copy-out form: the saved copy leaves through the operand stage (below)
      int b_it, tg_it;
      item_of(it, b_it, tg_it);
      if (XS != 0 && XS != 3 && P.xs && !xs_bulk && tg_it == 0) {
        const int st = it % P.nstages;
        unsigned char* slab = reinterpret_cast<unsigned char*>(P.xs + ((size_t)b_it * P.nstages + st) * 4 * (size_t)P.Lxs.rows * 8);
        if (XS == 2) xs_cp = slab;
        else xs_st = slab;
      }
      const unsigned char* raw = raw_base + r * raw_bytes;
#pragma unroll
      for (int k = 0; k < MAXT; ++k) {
        if (k >= nt) break;
        uint4 v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = *reinterpret_cast<const uint4*>(raw + t_raw[k] + e * chan_stride);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t wj[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) wj[e] = j == 0 ? v[e].x : (j == 1 ? v[e].y : (j == 2 ? v[e].z : v[e].w));
#pragma unroll
          for (int hl = 0; hl < 2; ++hl) {
            const uint32_t sel = hl ? 0x7632u : 0x5410u;
            uint4 o;
            o.x = __byte_perm(wj[0], wj[1], sel);
            o.y = __byte_perm(wj[2], wj[3], sel);
            o.z = __byte_perm(wj[4], wj[5], sel);
            o.w = __byte_perm(wj[6], wj[7], sel);
            const int pos = 2 * j + hl;  // position within the task: spatial index sc*8 + pos
            const uint32_t delta = (uint32_t)(pos * 32) + (pos >= t_wrap[k] ? wrap_jump : 0u);
            *reinterpret_cast<uint4*>(As + t_a[k] + delta) = o;
            if (XS == 1 && xs_st) *reinterpret_cast<uint4*>(xs_st + t_x[k] + delta) = o;
          }
        }
      }
      if (XS == 1 && xs_st && P.xs_pads) {
#pragma unroll
        for (int k = 0; k < MAXP; ++k)
          if (k < npd) *reinterpret_cast<uint4*>(xs_st + t_pad[k]) = make_uint4(0, 0, 0, 0);
      }
      fence_proxy_async();
      mbar_arrive(&full[s]);
      mbar_arrive(&raw_empty[r]);
      if (xs_cp) {
        // Saved copy, copy-out form: the operand stage IS the copy's row layout (halo rows and zero columns included), so
        // once all four transposer warps have written it, the 128 threads stream it out with consecutive 16-byte rows per
        // lane -- every store instruction fills 16 whole sectors.  (The direct form stores each 16-byte row from the thread
        // that transposed it: 32 half-used sectors per instruction, every sector written twice -- the transposers' LSU
        // time was k1a's bound in training.)  The MMAs read the stage meanwhile; it is rewritten two stages later, after
        // this loop's next barrier.
        asm volatile("bar.sync 2, %0;" ::"n"(32 * K1A_TW) : "memory");
        const int lead = P.Lxs.lead, nrows = P.Lxs.rows, nbody = nrows - lead;
        constexpr int NT = 32 * K1A_TW, UB = 6;  // UB independent shared loads in flight per thread, then UB stores
#pragma unroll 1
        for (int kc = 0; kc < 4; ++kc) {
          const unsigned char* srcp = As + (size_t)kc * g.rows_alloc * 16;
          unsigned char* dstp = xs_cp + (size_t)kc * nrows * 16;
          if (tid < lead) *reinterpret_cast<uint4*>(dstp + (size_t)tid * 16) = make_uint4(0, 0, 0, 0);  // lead <= 128 rows (host)
          dstp += (size_t)lead * 16;
#pragma unroll 1
          for (int r0 = tid; r0 < nbody; r0 += UB * NT) {
            uint4 v[UB];
#pragma unroll
            for (int u = 0; u < UB; ++u)
              if (r0 + u * NT < nbody) v[u] = *reinterpret_cast<const uint4*>(srcp + (size_t)(r0 + u * NT) * 16);
#pragma unroll
            for (int u = 0; u < UB; ++u)
              if (r0 + u * NT < nbody) *reinterpret_cast<uint4*>(dstp + (size_t)(r0 + u * NT) * 16) = v[u];
          }
        }
      }
    }
  } else if (XS == 3 && warp == K1A_LOADER + 1) {
    // ================= store warp: finished operand stage -> saved copy, by TMA bulk stores =========================
    if (lane == 0) {
      const uint32_t lead_b = (uint32_t)P.Lxs.lead * 16, body_b = (uint32_t)(g.rows + g.P + 1) * 16;
      for (int it = 0; it < total_it; ++it) {
        const int s = it % K1A_ASTAGES, st = it % P.nstages;
        mbar_wait(&full[s], (it / K1A_ASTAGES) & 1);
        int b, tg;
        item_of(it, b, tg);
        if (tg == 0) {
          unsigned char* slab = reinterpret_cast<unsigned char*>(P.xs + ((size_t)b * P.nstages + st) * 4 * (size_t)P.Lxs.rows * 8);
          const unsigned char* As = stage_base + s * stage_bytes;
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) {
            unsigned char* dst = slab + (size_t)kc * P.Lxs.rows * 16;
            bulk_s2g(dst, zreg, lead_b);
            bulk_s2g(dst + lead_b, As + (size_t)kc * g.rows_alloc * 16, body_b);
          }
          bulk_commit_group();
          bulk_wait_group_read0();
        }
        mbar_arrive(&empty[s]);
      }
      bulk_wait_group0();  // the copies are in global memory before the kernel ends
    }
  } else if (warp < K1A_LOADER) {
    // ================= MMA warps: tile t = tg * K1A_TPG + tt, accumulator rows [32 q, 32 q + 32) of it, all 80 columns ====
    // epilogue: (+bias) -> bf16 -> mid activations (A layout); channel c1 of the mid activations is the constant 1 (lets
    // the next layer fold its bias into the GEMM)
    const int cw = warp - K1A_TW, q = cw & 3, tt = cw >> 2;
    const uint32_t lbo_a = g.rows_alloc * 16, lbo_b = HB_NCOLS * 16;
    int it = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int b = item / P.ntg, t = (item - b * P.ntg) * K1A_TPG + tt;
      const bool active = t < g.tiles;
      float acc[2][HB_NCOLS / 8][4];
      mma::zero(acc);
      for (int st = 0; st < P.nstages; ++st, ++it) {
        const int s = it % K1A_ASTAGES;
        mbar_wait(&full[s], (it / K1A_ASTAGES) & 1);
        if (active) {
          const uint32_t a0 = smem_u32(stage_base + s * stage_bytes);
          const uint32_t b0 = a0 + a_stage_bytes;
#pragma unroll
          for (int sh = 0; sh < 4; ++sh) {
            const int shift_rows = (sh >> 1) * g.P + (sh & 1);
#pragma unroll
            for (int k16 = 0; k16 < 2; ++k16)
              mma::kstep(acc, a0 + (2 * k16) * lbo_a + (t * 128 + 32 * q + shift_rows) * 16, lbo_a, b0 + (sh * 4 + 2 * k16) * lbo_b, lbo_b, lane);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
      }
      if (!active) continue;
      float d[HB_NCOLS];
#pragma unroll
      for (int nt = 0; nt < HB_NCOLS / 8; ++nt) mma::rows8(acc, nt, &d[nt * 8], lane);
      {
        const int row = t * 128 + 32 * q + lane;
        const int m = row / g.P, n = row - m * g.P;
        if (m < g.Hi && n < g.Wi) {
#pragma unroll
          for (int cls = 0; cls < 4; ++cls) {
            const int y = 2 * m + (cls >> 1), x = 2 * n + (cls & 1);
            const size_t row2 = (size_t)P.Lmid.lead + (size_t)y * P.Lmid.Pp + x;
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
                  if (ch < HB_CLS) {
                    if (ch < P.c1) val = d[cls * HB_CLS + ch] + __ldg(P.bias + ch);
                    else if (ch == P.c1) val = 1.0f;
                  } else if (ch == P.c1) {
                    val = 1.0f;
                  }
                  f[hh] = val;
                }
                __nv_bfloat162 h2 = __floats2bfloat162_rn(f[0], f[1]);
                pk[e2] = *reinterpret_cast<uint32_t*>(&h2);
              }
              *reinterpret_cast<uint4*>(P.mid + ((((size_t)b * 4 + kc) * rows_mid + row2) * 8)) =
                  make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
          }
        }
      }
    }
  }
}

// =====================================================================================================
// k1b: second transposed convolution + plane softmax (two CTAs per SM, half a frame resident at a time)
// =====================================================================================================
// warp 0 loader, warp 1 idle, warps 2-9 MMA + epilogue: row quarter q = warp % 4 of each 128-row M-tile,
// output-row parity e = (warp - 2) / 4 (classes 2e, 2e+1 = accumulator columns [40e, 40e+40)).  The whole K (4 shifts x
// 32 channels) of a half frame is resident, so a warp computes each 16-column block of its rows when its epilogue needs it.
constexpr int K1B_THREADS = 320;
constexpr int K1B_EPI = 256;    // epilogue threads

struct K1bParams {
  const __nv_bfloat16* mid;   // [B][4][L.rows][8] padded row layout
  RowLayout L;
  const __nv_bfloat16* wpk;   // packed weights, one stage (K = 32); bias folded into channel c1
  float* out;                 // [B][c2][2Hi][2Wi]
  int B, c2, final_softmax;
  int Hh;                     // image rows per half (Hi / 2)
  HeadGeom g;                 // geometry of one half: Hi = Hh, rows_alloc covers Hh + 1 rows
};

__global__ void __launch_bounds__(K1B_THREADS, 2) k1b_convt_softmax_kernel(const __grid_constant__ K1bParams P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const HeadGeom g = P.g;
  const int a_bytes = 4 * g.rows_alloc * 16;
  unsigned char* As = smem;
  unsigned char* Bs = smem + a_bytes;
  float* stat = reinterpret_cast<float*>(Bs + HB_BSTAGE_BYTES);  // [2][HB_CLS][8 warps]
  float* fin = stat + 2 * HB_CLS * 8;                            // [2][HB_CLS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(fin + 2 * HB_CLS + 8);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + 1;
  uint64_t* b_full = bars + 2;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < a_bytes / 16; i += K1B_THREADS) reinterpret_cast<uint4*>(As)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    mbar_init(a_full, 1);
    mbar_init(a_empty, K1B_EPI / 32);
    mbar_init(b_full, 1);
    fence_mbar_init();
  }
  fence_proxy_async();
  __syncthreads();

  const int Hi = 2 * P.Hh, Wi = g.Wi;        // full conv-input image
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const int npix = Hi * Wi;
  const int npass = P.final_softmax ? 2 : 1;
  const int nphase = 2 * npass;  // (pass, half)

  if (warp == 0) {
    // ================= loader =================
    if (lane == 0) {
      mbar_expect_tx(b_full, HB_BSTAGE_BYTES);
      bulk_g2s(Bs, P.wpk, HB_BSTAGE_BYTES, b_full);
    }
    int ph = 0;
    for (int b = blockIdx.x; b < P.B; b += gridDim.x) {
      for (int phase = 0; phase < nphase; ++phase, ++ph) {
        const int hf = phase & 1;
        mbar_wait(a_empty, (ph & 1) ^ 1);
        // one contiguous copy per K-chunk: Hh image rows + the halo row below, zero column included
        const uint32_t nbytes = (uint32_t)((P.Hh + 1) * g.P * 16);
        if (lane < 4) {
          if (lane == 0) mbar_expect_tx(a_full, 4 * nbytes);
          __syncwarp(0xf);
          bulk_g2s(As + (size_t)lane * g.rows_alloc * 16,
                   P.mid + (((size_t)b * 4 + lane) * P.L.rows + P.L.lead + (size_t)hf * P.Hh * g.P) * 8, nbytes, a_full);
        }
      }
    }
  } else if (warp >= 2) {
    // ================= epilogue =================
    const int q = warp & 3, e = (warp - 2) >> 2;
    const int ew = warp - 2;  // 0..7
    const float L2E = 1.4426950408889634f;
    const size_t plane_stride = (size_t)Ho * Wo;
    const uint32_t lbo_a = g.rows_alloc * 16, lbo_b = HB_NCOLS * 16;
    const uint32_t a0 = smem_u32(As), b0 = smem_u32(Bs);
    mbar_wait(b_full, 0);
    int ph = 0;
    for (int b = blockIdx.x; b < P.B; b += gridDim.x) {
      float mx[HB_CLS], sm[HB_CLS];
#pragma unroll
      for (int o = 0; o < HB_CLS; ++o) {
        mx[o] = -3.0e38f;
        sm[o] = 0.f;
      }
      for (int phase = 0; phase < nphase; ++phase) {
        const int hf = phase & 1;
        const bool write = (phase >= nphase - 2);
        mbar_wait(a_full, ph & 1);
        {
          for (int t = 0; t < g.tiles; ++t) {
            // columns [40e, 40e+40) = classes (py = e, px = 0|1) of this tile; computed in 16-column blocks [32e, 32e+48)
            // and picked with compile-time register indices
            float d[48];
#pragma unroll
            for (int cc = 0; cc < 3; ++cc) {
              float acc[2][2][4];
              mma::zero(acc);
#pragma unroll
              for (int sh = 0; sh < 4; ++sh) {
                const int shift_rows = (sh >> 1) * g.P + (sh & 1);
#pragma unroll
                for (int k16 = 0; k16 < 2; ++k16)
                  mma::kstep(acc, a0 + (2 * k16) * lbo_a + (t * 128 + 32 * q + shift_rows) * 16, lbo_a,
                             b0 + (sh * 4 + 2 * k16) * lbo_b + (32 * e + 16 * cc) * 16, lbo_b, lane);
              }
              mma::rows8(acc, 0, &d[cc * 16], lane);
              mma::rows8(acc, 1, &d[cc * 16 + 8], lane);
            }
            const int row = t * 128 + 32 * q + lane;
            const int ml = row / g.P, n = row - ml * g.P;
            const bool valid = (ml < P.Hh) && (n < Wi);
            const int m = hf * P.Hh + ml;
            float* dst = P.out + ((size_t)b * P.c2 * Ho + 2 * m + e) * Wo + 2 * n;  // plane o adds o * Ho * Wo
            auto planes = [&](auto ec) {  // compile-time class offset: no per-value selects
              constexpr int E = decltype(ec)::value;
#pragma unroll
              for (int o = 0; o < HB_CLS; ++o) {
                if (o >= P.c2) break;
                const float l0 = d[8 * E + o], l1 = d[8 * E + HB_CLS + o];
                if (!write) {
                  const float mm = valid ? fmaxf(l0, l1) : -3.0e38f;
                  if (__any_sync(0xffffffffu, mm > mx[o])) {
                    const float mn = fmaxf(mx[o], mm);
                    sm[o] *= fast_exp2((mx[o] - mn) * L2E);
                    mx[o] = mn;
                  }
                  if (valid) {
                    const float mL = mx[o] * L2E;
                    sm[o] += fast_exp2(fmaf(l0, L2E, -mL)) + fast_exp2(fmaf(l1, L2E, -mL));
                  }
                } else if (valid) {
                  float p0 = l0, p1 = l1;
                  if (P.final_softmax) {
                    const float mL = fin[o], inv = fin[HB_CLS + o];
                    p0 = fast_exp2(fmaf(l0, L2E, -mL)) * inv;
                    p1 = fast_exp2(fmaf(l1, L2E, -mL)) * inv;
                  }
                  *reinterpret_cast<float2*>(dst + (size_t)o * plane_stride) = make_float2(p0, p1);
                }
              }
            };
            if (e == 0) planes(std::integral_constant<int, 0>{});
            else planes(std::integral_constant<int, 1>{});
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(a_empty);  // this warp's reads of the half are done
          ++ph;
        }
        if (P.final_softmax && phase == 1) {
          // merge the online-softmax states: lanes -> warp (shuffles) -> 8 epilogue warps (smem)
#pragma unroll
          for (int o = 0; o < HB_CLS; ++o) {
            if (o >= P.c2) break;
            const float M = warp_max(mx[o]);
            const float S = warp_sum(sm[o] * fast_exp2((mx[o] - M) * L2E));
            if (lane == 0) {
              stat[o * 8 + ew] = M;
              stat[(HB_CLS + o) * 8 + ew] = S;
            }
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (tid - 64 < P.c2) {
            const int o = tid - 64;
            float M = stat[o * 8];
#pragma unroll
            for (int i = 1; i < 8; ++i) M = fmaxf(M, stat[o * 8 + i]);
            float S = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) S += stat[(HB_CLS + o) * 8 + i] * fast_exp2((stat[o * 8 + i] - M) * L2E);
            fin[o] = M * L2E;
            fin[HB_CLS + o] = 1.0f / S;
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
      }
    }
  }
}

static size_t k1a_smem_bytes(const HeadGeom& g, int HW) {
  return (size_t)K1A_ASTAGES * (4 * g.rows_alloc * 16 + HB_BSTAGE_BYTES) + (size_t)K1A_RSTAGES * 4 * HB_KSTAGE * HW * 2 + 128 + 1024;
}
static size_t k1b_smem_bytes(const HeadGeom& g) {
  return (size_t)4 * g.rows_alloc * 16 + HB_BSTAGE_BYTES + (2 * HB_CLS * 8 + 2 * HB_CLS + 8) * sizeof(float) + 64;
}

// geometry of one half image (Hh rows + 1 halo row) of the second layer
__host__ inline HeadGeom make_half_geom(int Hh, int Wi) {
  HeadGeom g = make_geom(Hh, Wi);
  g.rows_alloc = (g.tiles * 128 + g.P + 1 + 7) & ~7;
  if (g.rows_alloc < (Hh + 1) * g.P + 8) g.rows_alloc = ((Hh + 1) * g.P + 8 + 7) & ~7;
  return g;
}

}  // namespace lpb

// ---- which kernels serve a shape ---------------------------------------------------------------------------
// fast path (k1a + k1b): two-deconv heads whose whole frame fits the shared-memory tiling above;
// generic path (head_rows_bf16.cu): everything else -- one-deconv heads, larger feature maps.
static bool head_fast_path(int C, int H, int W, int c2, int max_smem) {
  using namespace lpb;
  if (c2 <= 0) return false;
  if (!((W >= 7 || W == 4 || W == 6) && H * W <= 192 && W <= 31)) return false;  // W <= 31: the saved copy's lead rows fit the 1 KB zero source
  const HeadGeom g1 = make_geom(2 * H, 2 * W), g2 = make_half_geom(2 * H, 4 * W);
  return (int64_t)k1a_smem_bytes(g1, H * W) <= max_smem && (int64_t)k1b_smem_bytes(g2) <= max_smem;
}

static int device_limits(int* max_smem, int* sms) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    *max_smem = 227 * 1024;  // sm_90a (also what a CPU-only caller sizing buffers should assume)
    *sms = 132;
  }
  return 0;
}

// plan[0] = 1: fast path (saved_xs optional: training only); 0: generic path (saved_xs REQUIRED: it is the operand)
extern "C" int lpb_head_bf16_plan(int C, int H, int W, int c1, int c2, int* plan) {
  using namespace lpb;
  LPB_REQUIRE(plan, "head_bf16_plan: null pointer");
  LPB_REQUIRE(C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && (H * W) % 8 == 0 && c1 >= 1 && c2 >= 0, "head_bf16_plan: bad shape");
  LPB_REQUIRE(c2 == 0 ? c1 <= HB_CLS : (c1 < HB_CLS && c2 <= HB_CLS), "head_bf16_plan: channel counts %d/%d exceed %d", c1, c2, HB_CLS);
  int max_smem, sms;
  device_limits(&max_smem, &sms);
  plan[0] = head_fast_path(C, H, W, c2, max_smem) ? 1 : 0;
  if (!plan[0] && ((size_t)32 * H * W * 2 > 200 * 1024 || (c2 > 0 ? 4 : 2) * W + 1 > CR_BAND_ROWS)) {
    set_error("head_bf16_plan: feature map %dx%d too large for this build", H, W);
    return LPB_ERR_UNSUPPORTED;
  }
  return LPB_OK;
}

// workspace layout: [packed w1][packed w2][mid activations (padded row layout; two-deconv heads only)]
extern "C" int lpb_head_bf16_saved_bytes(int B, int C, int H, int W, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes && B >= 0 && C >= 32 && C % 32 == 0 && H >= 1 && W >= 1, "head_bf16_saved_bytes: bad arguments");
  *bytes = (size_t)B * (C / 32) * make_row_layout(2 * H, 2 * W).rows * 16;
  return LPB_OK;
}

extern "C" int lpb_head_bf16_workspace_bytes(int B, int C, int H, int W, int c1, int c2, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "head_bf16_workspace_bytes: null pointer");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 0, "head_bf16_workspace_bytes: bad shape");
  const size_t w1 = (size_t)(C / 4 / HB_KSTAGE) * HB_BSTAGE_BYTES, w2 = HB_BSTAGE_BYTES;
  const size_t mid = c2 > 0 ? (size_t)B * 4 * make_row_layout(4 * H, 4 * W).rows * 16 : 0;
  // + the split softmax's per-band statistics of the LAST layer
  const size_t part = c2 > 0 ? convt_rows_partials_bytes(B, 4 * H, 4 * W) : convt_rows_partials_bytes(B, 2 * H, 2 * W);
  *bytes = w1 + w2 + mid + ((part + 255) & ~(size_t)255);
  return LPB_OK;
}

extern "C" int lpb_head_fwd_bf16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                 const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                                 void* workspace, void* stream) {
  return lpb_head_fwd_bf16_hinted(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, out, saved_xs, workspace, nullptr, stream);
}

extern "C" int lpb_head_fwd_bf16_hinted(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                        const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                                        void* workspace, void* decode_hints, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(features && w1 && b1 && out && workspace, "head_fwd_bf16: null pointer");
  LPB_REQUIRE(c2 == 0 || (w2 && b2), "head_fwd_bf16: a two-deconv head needs w2 and b2");
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1, "head_fwd_bf16: bad feature shape C=%d H=%d W=%d", C, H, W);
  LPB_REQUIRE((H * W) % 8 == 0, "head_fwd_bf16: H*W must be a multiple of 8 (got %d)", H * W);
  LPB_REQUIRE(c2 == 0 ? (c1 >= 1 && c1 <= HB_CLS) : (c1 >= 1 && c1 < HB_CLS && c2 >= 1 && c2 <= HB_CLS),
              "head_fwd_bf16: channel counts %d/%d exceed %d", c1, c2, HB_CLS);
  if (B == 0) return LPB_OK;
  int max_smem = 0, sms = 0;
  device_limits(&max_smem, &sms);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // decode hints are produced by the fused two-pass softmax of the banded kernel only (launch_convt_rows marks them invalid
  // on its other routes); the routes that never reach it do so here
  if (decode_hints && (!final_softmax || !g_tuning[LPB_TUNE_SOFTMAX_EPILOGUE_V2]))
    LPB_CUDA(cudaMemsetAsync(decode_hints, 0, (size_t)16 * B * (c2 > 0 ? c2 : c1), s));
  const int nst = C / 4 / HB_KSTAGE;
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const RowLayout Lxs = make_row_layout(2 * H, 2 * W), Lmid = make_row_layout(4 * H, 4 * W);
  __nv_bfloat16* wp1 = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* wp2 = reinterpret_cast<__nv_bfloat16*>(ws + (size_t)nst * HB_BSTAGE_BYTES);
  __nv_bfloat16* mid = reinterpret_cast<__nv_bfloat16*>(ws + (size_t)(nst + 1) * HB_BSTAGE_BYTES);
  float* partials = reinterpret_cast<float*>(ws + (size_t)(nst + 1) * HB_BSTAGE_BYTES + (c2 > 0 ? (size_t)B * 4 * Lmid.rows * 16 : 0));
  const bool fast = head_fast_path(C, H, W, c2, max_smem);
  // k1a's block transposers write the saved copy's pad rows themselves when a thread's share fits its registers
  const int xs_npad = Lxs.lead + (Lxs.rows - (Lxs.lead + Lxs.Hi * Lxs.Pp)) + Lxs.Hi;
  const bool k1a_pads = fast && !g_tuning[LPB_TUNE_K1A_ROW_TRANSPOSER] && !g_tuning[LPB_TUNE_K1A_BULK_XS] && 4 * xs_npad <= K1A_MAXPAD * 32 * K1A_TW;
  {
    // one launch: both operand packs + the pad rows of the fresh row-layout buffers
    PrepJobs jobs{};
    jobs.fpack[0] = {w1, nullptr, C / 4, c1, nst, wp1};
    // layer 2: bias rides on the constant-one channel c1 of the mid activations (only needed without softmax:
    // a per-plane constant does not change a softmax)
    if (c2 > 0) {
      jobs.fpack[1] = {w2, final_softmax ? nullptr : b2, c1, c2, 1, wp2};
      jobs.pads[0] = {mid, Lmid, (long long)B * 4};
    }
    // (the block transposer of k1a writes the saved copy's pads itself; the row-form variant does not)
    if (fast && saved_xs && !g_tuning[LPB_TUNE_K1A_BULK_XS] && !k1a_pads) jobs.pads[1] = {static_cast<__nv_bfloat16*>(saved_xs), Lxs, (long long)B * (C / 32)};  // (the banded path's shuffle kernel writes its own pads)
    launch_head_prep(jobs, s);
  }
  if (!fast) {
    // ---- generic path: shuffle rows -> banded GEMM(s) ----
    LPB_REQUIRE(saved_xs, "head_fwd_bf16: this shape takes the banded kernels (lpb_head_bf16_plan = 0): pass the "
                          "lpb_head_bf16_saved_bytes() buffer as saved_xs");
    __nv_bfloat16* xs = static_cast<__nv_bfloat16*>(saved_xs);
    int rc = launch_rows_shuffle(static_cast<const __nv_bfloat16*>(features), B, C, H, W, xs, s);
    if (rc != LPB_OK) return rc;
    ConvtRowsParams p{};
    p.X = xs;
    p.L = Lxs;
    p.wpk = wp1;
    p.bias = b1;
    p.nst = nst;
    p.B = B;
    p.cout = c1;
    p.out = out;
    p.partials = partials;
    if (c2 == 0) {
      p.hints = final_softmax ? static_cast<int4*>(decode_hints) : nullptr;
      p.mode = final_softmax ? CONVT_ROWS_SOFTMAX : CONVT_ROWS_PLANES;
      rc = launch_convt_rows(p, sms, s);
      if (rc != LPB_OK) return rc;
    } else {
      p.mode = CONVT_ROWS_MID;
      p.mid = mid;
      p.Lout = Lmid;
      rc = launch_convt_rows(p, sms, s);
      if (rc != LPB_OK) return rc;
      ConvtRowsParams p2{};
      p2.X = mid;
      p2.L = Lmid;
      p2.wpk = wp2;
      p2.bias = nullptr;  // folded into the GEMM through the ones channel (see the pack above)
      p2.nst = 1;
      p2.B = B;
      p2.cout = c2;
      p2.out = out;
      p2.partials = partials;
      p2.hints = final_softmax ? static_cast<int4*>(decode_hints) : nullptr;
      p2.mode = final_softmax ? CONVT_ROWS_SOFTMAX : CONVT_ROWS_PLANES;
      rc = launch_convt_rows(p2, sms, s);
      if (rc != LPB_OK) return rc;
    }
    LPB_CUDA(cudaGetLastError());
    return LPB_OK;
  }
  const HeadGeom g1 = make_geom(2 * H, 2 * W), g2 = make_half_geom(2 * H, 4 * W);  // layer 2: 4H rows in two halves
  const size_t s1 = k1a_smem_bytes(g1, H * W), s2 = k1b_smem_bytes(g2);
  K1aParams pa;
  pa.feat = static_cast<const __nv_bfloat16*>(features);
  pa.wpk = wp1;
  pa.bias = b1;
  pa.mid = mid;
  pa.xs = static_cast<__nv_bfloat16*>(saved_xs);
  pa.Lmid = Lmid;
  pa.Lxs = Lxs;
  pa.B = B;
  pa.C = C;
  pa.HW = H * W;
  pa.W = W;
  pa.c1 = c1;
  pa.nstages = nst;
  pa.row_transposer = g_tuning[LPB_TUNE_K1A_ROW_TRANSPOSER];
  pa.backoff = g_tuning[LPB_TUNE_WAIT_BACKOFF];
  pa.xs_bulk = g_tuning[LPB_TUNE_K1A_BULK_XS];
  pa.xs_copy = (g_tuning[LPB_TUNE_K1A_XS_COPY] && !pa.row_transposer && !pa.xs_bulk) ? 1 : 0;
  pa.xs_pads = k1a_pads ? 1 : 0;
  pa.g = g1;
  pa.ntg = (g1.tiles + K1A_TPG - 1) / K1A_TPG;
  {
    // compile-time form of the saved copy (see the kernel): none / run-time forms / copy-out
    if (pa.xs_copy && Lxs.lead > 32 * K1A_TW) pa.xs_copy = 0;
    const int form = (!pa.xs || pa.row_transposer || pa.xs_bulk) ? (pa.xs || pa.row_transposer ? 1 : 0) : (g_tuning[LPB_TUNE_K1A_XS_COPY] == 2 ? 3 : (pa.xs_copy ? 2 : 1));
    auto kern = form == 0 ? k1a_shuffle_convt_kernel<0> : (form == 1 ? k1a_shuffle_convt_kernel<1> : (form == 2 ? k1a_shuffle_convt_kernel<2> : k1a_shuffle_convt_kernel<3>));
    LPB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s1));
    const int items = B * pa.ntg;
    kern<<<items < sms ? items : sms, K1A_THREADS + (form == 3 ? 32 : 0), s1, s>>>(pa);
  }
  if (g_tuning[LPB_TUNE_SOFTMAX_EPILOGUE_V2]) {
    // layer 2 on the banded kernel (head_rows_bf16.cu): same GEMM, leaner softmax epilogue
    ConvtRowsParams p2{};
    p2.X = mid;
    p2.L = Lmid;
    p2.wpk = wp2;
    p2.bias = nullptr;  // folded into the GEMM through the ones channel
    p2.nst = 1;
    p2.B = B;
    p2.cout = c2;
    p2.out = out;
    p2.partials = partials;
    p2.hints = final_softmax ? static_cast<int4*>(decode_hints) : nullptr;
    p2.mode = final_softmax ? CONVT_ROWS_SOFTMAX : CONVT_ROWS_PLANES;
    const int rc = launch_convt_rows(p2, sms, s);
    if (rc != LPB_OK) return rc;
    LPB_CUDA(cudaGetLastError());
    return LPB_OK;
  }
  K1bParams pb;
  pb.mid = mid;
  pb.L = Lmid;
  pb.wpk = wp2;
  pb.out = out;
  pb.B = B;
  pb.c2 = c2;
  pb.final_softmax = final_softmax;
  pb.Hh = 2 * H;
  pb.g = g2;
  LPB_CUDA(cudaFuncSetAttribute(k1b_convt_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s2));
  const int grid2 = B < 2 * sms ? B : 2 * sms;
  k1b_convt_softmax_kernel<<<grid2, K1B_THREADS, s2, s>>>(pb);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
