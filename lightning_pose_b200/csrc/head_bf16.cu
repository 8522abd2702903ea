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
//   layer 2: mid activations --banded kernel (head_rows_bf16.cu)--> planes or two-pass plane softmax
#include <cuda_bf16.h>

#include <cstdint>
#include <type_traits>

#include "../../include/lpb200.h"
#include "head_prep.cuh"
#include "head_rows.cuh"
#include "lpb_common.cuh"
#include "row_layout.cuh"
#include "mma_sm90.cuh"
#include "tensor_map.cuh"

namespace lpb {

// ---- everything a head call prepares, in one launch (head_prep.cuh) -------------------------------------------
// forward packs: W[Cin][Cout][3][3] (fp32) -> B[group][stage][shift][kchunk][80][8] of operand type T (output channel
// o = HEAD_CLS * group + column % HEAD_CLS); a non-null bias rides on input channel `Cin` (the constant-one channel of the
// mid activations; shift (0,0) only, which every output class uses once) and is rounded to T like the weights
template <typename T>
__global__ void __launch_bounds__(256) head_prep_kernel(const __grid_constant__ PrepJobs J) {
  const long long tid0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, nthr = (long long)gridDim.x * blockDim.x;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    if (!J.fpack[j].out) continue;
    const float* w = J.fpack[j].w;
    const float* bias = J.fpack[j].bias;
    const int Cin = J.fpack[j].Cin, Cout = J.fpack[j].Cout, nst = J.fpack[j].nstages;
    const long long total = (long long)J.fpack[j].ngroups * nst * 4 * 4 * HEAD_NCOLS * 8;
    for (long long i = tid0; i < total; i += nthr) {
      const int e = (int)(i & 7);
      long long r = i >> 3;
      const int nrow = (int)(r % HEAD_NCOLS);
      r /= HEAD_NCOLS;
      const int kc = (int)(r & 3);
      r >>= 2;
      const int sh = (int)(r & 3);
      r >>= 2;
      const int st = (int)(r % nst), grp = (int)(r / nst);
      const int c = st * HEAD_KSTAGE + kc * 8 + e;
      const int cls = nrow / HEAD_CLS, o = grp * HEAD_CLS + nrow % HEAD_CLS;
      const int py = cls >> 1, px = cls & 1, dm = sh >> 1, dn = sh & 1;
      float v = 0.f;
      if (c < Cin && o < Cout && tap_nonzero(cls, sh)) {
        const int ky = py == 0 ? 1 : (dm ? 0 : 2);
        const int kx = px == 0 ? 1 : (dn ? 0 : 2);
        v = w[((size_t)c * Cout + o) * 9 + ky * 3 + kx];
      } else if (bias && c == Cin && o < Cout && sh == 0) {
        v = bias[o];
      }
      static_cast<T*>(J.fpack[j].out)[i] = Operand<T>::from(v);
    }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    if (!J.dpack[j].out) continue;
    const float* w = J.dpack[j].w;
    const int Cin = J.dpack[j].Cin, Cout = J.dpack[j].Cout, rpt = J.dpack[j].rows_per_tile, tch = J.dpack[j].tile_ch;
    const int ntiles = J.dpack[j].ntiles;
    const long long total = (long long)J.dpack[j].kgroups * ntiles * 4 * HEAD_KC * rpt * 8;
    for (long long i = tid0; i < total; i += nthr) {
      const int e = (int)(i & 7);
      long long r = i >> 3;
      const int row = (int)(r % rpt);
      r /= rpt;
      const int kc = (int)(r % HEAD_KC);
      r /= HEAD_KC;
      const int sh = (int)(r & 3);
      r >>= 2;
      const int tile = (int)(r % ntiles), kg = (int)(r / ntiles);
      const int c = tile * tch + row;
      const int k = kc * 8 + e;
      const int cls = k / HEAD_CLS, o = kg * HEAD_CLS + k % HEAD_CLS;
      const int py = cls >> 1, px = cls & 1, dm = sh >> 1, dn = sh & 1;
      float v = 0.f;
      if (row < tch && c < Cin && o < Cout && tap_nonzero(cls, sh)) {
        const int ky = py == 0 ? 1 : (dm ? 0 : 2);
        const int kx = px == 0 ? 1 : (dn ? 0 : 2);
        v = w[((size_t)c * Cout + o) * 9 + ky * 3 + kx];
      }
      J.dpack[j].out[i] = __float2bfloat16_rn(v);
    }
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
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
      *reinterpret_cast<uint4*>(static_cast<unsigned char*>(J.pads[j].buf) + ((size_t)slab * L.rows + row) * 16) = make_uint4(0, 0, 0, 0);
    }
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    if (!J.zero[j].p) continue;
    for (long long i = tid0; i < J.zero[j].n; i += nthr) J.zero[j].p[i] = 0.f;
  }
}

template <typename T>
int launch_head_prep(const PrepJobs& jobs, int sms, cudaStream_t s) {
  head_prep_kernel<T><<<2 * sms, 256, 0, s>>>(jobs);  // two CTAs per SM
  return LPB_OK;
}
template int launch_head_prep<__nv_bfloat16>(const PrepJobs&, int, cudaStream_t);
template int launch_head_prep<__half>(const PrepJobs&, int, cudaStream_t);

// =====================================================================================================
// k1a: PixelShuffle + first transposed convolution
// =====================================================================================================
// A CTA works on (frame, band) items.  A band is a run of feature rows (two shuffled image rows each); the G bands of a
// frame are as equal as possible, and G is the smallest count whose largest band fits the MMA warps' registers: each of
// the K1A_CW MMA warps keeps up to K1A_MT m16 row tiles x 80 columns of fp32 accumulators across all channel stages.
// Per 128-channel stage an item stages only its band's feature rows plus the halo row below (the next band's first row;
// the tensor map's zero fill past the frame's bottom edge), and the saved copy's rows are written by the item that holds
// them.  16 warps = 4 warpgroups, 128 registers per thread at launch, rebalanced with setmaxnreg:
//   warpgroup 0     transposers: raw NCHW rows -> K-major operand rows, PixelShuffle folded in
//   warpgroups 1-2  MMA warps + epilogue
//   warpgroup 3     warp 12 TMA loader, warp 13 saved-copy stores (training form), warps 14-15 exit
constexpr int K1A_TW = 4;                                // transposer warps
constexpr int K1A_CW = 8;                                // MMA warps
constexpr int K1A_MT = 3;                                // m16 row tiles per MMA warp at most (120 accumulators)
constexpr int K1A_BAND_ROWS = 16 * K1A_MT * K1A_CW;      // raster rows (incl. zero columns) of the largest band
constexpr int K1A_LOADER = K1A_TW + K1A_CW;              // warp 12; warp 13 stores the saved copy
constexpr int K1A_THREADS = 512;
constexpr int K1A_STAGES = 2;                            // operand stages (A + packed weights), and as many raw stages
constexpr int K1A_PROD_REGS = 80, K1A_MMA_REGS = 176;    // setmaxnreg: 128 x (2 x 80 + 2 x 176) = 64 K registers
constexpr int K1A_ZROWS = 72;                            // zero rows: source of the saved copy's lead / trail rows (<= 71 for W <= 31)

struct K1aGeom {
  int H, W;            // feature map
  int Wi, P;           // shuffled image width, operand row pitch Wi + 1 (zero column)
  int G;               // bands per frame (0: no split fits, the shape takes the banded generic path)
  int a, ubase, urem;  // band i = ubase + (i < urem) units of a feature rows (the last band clipped at H)
  int nbmax;           // feature rows of the largest band
  int nfs;             // feature rows staged per item: the largest band + the halo row (G > 1)
  int box;             // raw elements per channel staged per item: nfs * W rounded up to 8 (a 16-byte TMA box row)
  int rows_alloc;      // operand rows per K-chunk (multiple of 8)
};

__host__ inline K1aGeom make_k1a_geom(int H, int W) {
  K1aGeom k;
  k.H = H;
  k.W = W;
  k.Wi = 2 * W;
  k.P = 2 * W + 1;
  // A band starts at a feature row f0 whose first element f0 * W is a multiple of 8: the TMA box's start is then 16-byte
  // aligned (a start at any other element raises an illegal-instruction error on the H100).  So bands are made of units
  // of a = 8 / gcd(W, 8) feature rows, as equal as possible, and G is the smallest count whose largest band fits.
  k.a = 8 / ((W & -W) < 8 ? (W & -W) : 8);
  const int nu = (H + k.a - 1) / k.a;
  k.G = 0;
  for (int g = 1; g <= nu; ++g) {
    const int units = (nu + g - 1) / g, nb = units * k.a < H ? units * k.a : H;
    if (2 * nb * k.P <= K1A_BAND_ROWS) {
      k.G = g;
      break;
    }
  }
  if (k.G == 0) return k;
  k.ubase = nu / k.G;
  k.urem = nu % k.G;
  const int nbmax = (k.ubase + (k.urem > 0)) * k.a < H ? (k.ubase + (k.urem > 0)) * k.a : H;
  k.nbmax = nbmax;
  // one band: the frame's bottom edge is the halo, zero from the stages' one-time clear, so the box never reaches past
  // the tensor (H * W is a multiple of 8: box <= H * W)
  k.nfs = nbmax + (k.G > 1 ? 1 : 0);
  k.box = (k.nfs * W + 7) & ~7;
  // the MMAs read the band's m16 tiles shifted by up to P + 1 rows; the transposers write nfs feature rows
  const int mma_rows = (2 * nbmax * k.P + 15) / 16 * 16 + k.P + 1, tr_rows = 2 * k.nfs * k.P;
  k.rows_alloc = ((mma_rows > tr_rows ? mma_rows : tr_rows) + 7) & ~7;
  return k;
}

// T: the operand element type (head_prep.cuh Operand) of the features, the packed weights and the mid activations
template <typename T>
struct K1aParams {
  CUtensorMap feat;           // features [B * C][H * W] of type T, box {k.box, 128}: one stage's channels of an item's rows
  const T* wpk;               // packed weights [nstages][HEAD_BSTAGE_BYTES]
  const float* bias;          // [c1]
  T* mid;                     // [B][4][Lmid.rows][8]  padded row layout of the next layer's input (row_layout.cuh)
  T* xs;                      // [B][C/32][Lxs.rows][8] (training form): shuffled features in the padded row layout
  RowLayout Lmid, Lxs;
  int B, C;                   // feature batch and channels (C = 4 * Cin)
  int c1, nstages;
  K1aGeom k;
};

// item -> frame b, first feature row f0 and feature-row count nb of its band
__device__ __forceinline__ void k1a_band(const K1aGeom& k, int item, int& b, int& f0, int& nb) {
  b = item / k.G;
  const int band = item - b * k.G;
  f0 = k.a * (band * k.ubase + min(band, k.urem));
  nb = min(k.a * (k.ubase + (band < k.urem ? 1 : 0)), k.H - f0);
}

// One MMA warp's share of every item of its CTA: m16 tiles [m0, m0 + MT) of the band raster, all 80 columns, accumulated
// over the item's stages; then + bias -> T -> mid activations.  Per accumulator element
// the MMA sequence is stages, then shifts, then k16, then the shift's non-zero n8 tiles.
template <int MT, typename T>
__device__ __forceinline__ void k1a_mma_warp(const K1aParams<T>& P, unsigned char* stage_base, int stage_bytes, int a_stage_bytes,
                                             uint64_t* full, uint64_t* empty, int m0, int lane) {
  const K1aGeom& k = P.k;
  const uint32_t lbo_a = k.rows_alloc * 16, lbo_b = HEAD_NCOLS * 16;
  const int nitems = P.B * k.G;
  int it0 = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x, it0 += P.nstages) {
    int b, f0, nb;
    k1a_band(k, item, b, f0, nb);
    float acc[MT > 0 ? MT : 1][HEAD_NCOLS / 8][4];
    mma::zero(acc);
    for (int st = 0; st < P.nstages; ++st) {
      const int it = it0 + st, s = it % K1A_STAGES;
      mbar_wait(&full[s], (it / K1A_STAGES) & 1);
      if constexpr (MT > 0) {
        const uint32_t a0 = smem_u32(stage_base + s * stage_bytes);
        const uint32_t b0 = a0 + a_stage_bytes;
        mma::for_shifts([&](auto shc) {  // only the n8 tiles with real taps of the shift (24 of 40)
          constexpr int sh = decltype(shc)::value;
          const int shift_rows = (sh >> 1) * k.P + (sh & 1);
#pragma unroll
          for (int k16 = 0; k16 < 2; ++k16)
            mma::kstep_nz<NZ_N8[sh], T>(acc, a0 + (2 * k16) * lbo_a + (16 * m0 + shift_rows) * 16, lbo_a, b0 + (sh * 4 + 2 * k16) * lbo_b, lbo_b, lane);
        });
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    if constexpr (MT > 0) {
      // epilogue, 32 rows (two m16 tiles) at a time: (+bias) -> T -> mid activations (A layout); channel c1 of the mid
      // activations is the constant 1 (lets the next layer fold its bias into the GEMM)
      const int rows_mid = P.Lmid.rows;
      static_for<0, (MT + 1) / 2>([&](auto pc) {
        constexpr int M0 = 2 * decltype(pc)::value;
        float d[HEAD_NCOLS];
#pragma unroll
        for (int nt = 0; nt < HEAD_NCOLS / 8; ++nt) mma::rows8_at<M0>(acc, nt, &d[nt * 8], lane);
        const int row = 16 * (m0 + M0) + lane;  // band raster row
        const int ml = row / k.P, n = row - ml * k.P;
        if ((M0 + 1 < MT || lane < 16) && ml < 2 * nb && n < k.Wi) {
          const int m = 2 * f0 + ml;
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
                  if (ch < HEAD_CLS) {
                    if (ch < P.c1) val = d[cls * HEAD_CLS + ch] + __ldg(P.bias + ch);
                    else if (ch == P.c1) val = 1.0f;
                  } else if (ch == P.c1) {
                    val = 1.0f;
                  }
                  f[hh] = val;
                }
                pk[e2] = Operand<T>::pack2(f[0], f[1]);
              }
              *reinterpret_cast<uint4*>(P.mid + ((((size_t)b * 4 + kc) * rows_mid + row2) * 8)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
            }
          }
        }
      });
    }
  }
}

// XS = 1: training form, warp 13 writes the saved operand copy; XS = 0: inference.  T: the operand element type.
template <typename T, int XS>
__global__ void __launch_bounds__(K1A_THREADS, 1) k1a_shuffle_convt_kernel(const __grid_constant__ K1aParams<T> P) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const K1aGeom& k = P.k;
  const int a_stage_bytes = 4 * k.rows_alloc * 16;
  const int stage_bytes = a_stage_bytes + HEAD_BSTAGE_BYTES;
  const int raw_bytes = 4 * HEAD_KSTAGE * k.box * 2;  // 128 source channels x the item's staged positions
  unsigned char* stage_base = smem;
  unsigned char* raw_base = smem + K1A_STAGES * stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(raw_base + K1A_STAGES * raw_bytes);
  uint64_t* full = bars;                         // operands ready (128 transposer arrivals + weight bytes)
  uint64_t* empty = bars + K1A_STAGES;           // the MMA warps (+ the saved-copy stores) have read the stage
  uint64_t* raw_full = bars + 2 * K1A_STAGES;    // TMA bytes landed
  uint64_t* raw_empty = bars + 3 * K1A_STAGES;   // the transposers are done with the raw stage
  unsigned char* zrows = reinterpret_cast<unsigned char*>(bars) + 128;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // zero the operand stages once: zero columns and rows past the staged ones are never written again
  for (int i = tid; i < K1A_STAGES * stage_bytes / 16; i += K1A_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  for (int i = tid; i < K1A_ZROWS; i += K1A_THREADS) reinterpret_cast<uint4*>(zrows)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int s = 0; s < K1A_STAGES; ++s) {
      mbar_init(&full[s], 32 * K1A_TW + 1);
      mbar_init(&empty[s], K1A_CW + XS);
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], 32 * K1A_TW);
    }
    fence_mbar_init();
  }
  fence_proxy_async();  // generic-proxy zero fill -> visible to the async proxy (bulk stores of the saved copy)
  __syncthreads();

  const int nitems = P.B * k.G;
  const int nmine = (nitems - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int total_it = nmine * P.nstages;
  const int item_base = blockIdx.x;
  auto item_of = [&](int it) { return item_base + (it / P.nstages) * (int)gridDim.x; };

  const int wg = warp >> 2;
  if (wg == 1 || wg == 2) {
    setmaxnreg_inc<K1A_MMA_REGS>();
    // ================= MMA warps: m16 tiles dealt contiguously and evenly (warps w and w + 4 share an SM sub-partition's
    // tensor pipe, and warp w gets a tile more than warp w + 4 only when the others do).  The tiles of the LARGEST band are
    // dealt for every item, so each warp has one tile count for the whole launch; a smaller band's extra rows are staged
    // (feature rows past the band, or zeros) and their accumulator rows are not written.  =================
    const int cw = warp - K1A_TW;
    const int t16 = (2 * k.nbmax * k.P + 15) / 16, base = t16 / K1A_CW, extra = t16 - base * K1A_CW;
    const int cnt = base + (cw < extra ? 1 : 0), m0 = cw * base + min(cw, extra);
    if (cnt == 3) k1a_mma_warp<3>(P, stage_base, stage_bytes, a_stage_bytes, full, empty, m0, lane);
    else if (cnt == 2) k1a_mma_warp<2>(P, stage_base, stage_bytes, a_stage_bytes, full, empty, m0, lane);
    else if (cnt == 1) k1a_mma_warp<1>(P, stage_base, stage_bytes, a_stage_bytes, full, empty, m0, lane);
    else k1a_mma_warp<0>(P, stage_base, stage_bytes, a_stage_bytes, full, empty, m0, lane);
    return;
  }
  setmaxnreg_dec<K1A_PROD_REGS>();
  if (wg == 0) {
    // ================= transposers: raw NCHW rows (smem) -> K-major operand rows, PixelShuffle folded in ======
    // A task is one 8x8 bf16 transpose: 8 channels x 8 consecutive staged positions (one 16-byte chunk per channel) of
    // one sub-pixel class q -> 8 operand rows of 16 bytes.  Staged position p = (feature row - f0) * W + j is operand row
    // (2 (p / W) + (q >> 1)) * P + 2 (p % W) + (q & 1).  Which tasks a thread owns, and where they read / write, is the
    // same for every stage and item, so the index arithmetic is done once, up front.
    const int nchunk = k.box / 8;
    const int ntasks = 4 * 4 * nchunk;
    const int npos = k.nfs * k.W;  // positions past it (the box's rounding) are not operand rows
    constexpr int MAXT = 2;        // box <= 128 (make_k1a_geom: nfs * W <= 127), so <= 256 tasks over 128 threads
    uint32_t t_raw[MAXT], t_a[MAXT];
    int t_wrap[MAXT], t_lim[MAXT];
    int nt = 0;
#pragma unroll
    for (int kk = 0; kk < MAXT; ++kk) {
      const int task = tid + kk * 32 * K1A_TW;
      t_raw[kk] = t_a[kk] = 0;
      t_wrap[kk] = t_lim[kk] = 8;
      if (task < ntasks) {
        const int sc = task % nchunk, q = (task / nchunk) & 3, kc = task / (4 * nchunk);
        const int sp0 = sc * 8, i0 = sp0 / k.W, jc0 = sp0 - i0 * k.W;
        const int row0 = (2 * i0 + (q >> 1)) * k.P + 2 * jc0 + (q & 1);
        t_raw[kk] = (uint32_t)(((4 * kc * 8 + q) * k.box + sp0) * 2);
        t_a[kk] = (uint32_t)((kc * k.rows_alloc + row0) * 16);
        t_wrap[kk] = k.W - jc0;  // position at which the image row wraps (W >= 4: at most once per task)
        t_lim[kk] = npos - sp0;
        nt = kk + 1;
      }
    }
    const uint32_t chan_stride = (uint32_t)(4 * k.box * 2);          // next shuffled channel e -> 4 source channels on
    const uint32_t wrap_jump = (uint32_t)((2 * k.P - 2 * k.W) * 16);  // extra bytes once the position wraps to row i + 1
    for (int it = 0; it < total_it; ++it) {
      const int s = it % K1A_STAGES;
      mbar_wait(&raw_full[s], (it / K1A_STAGES) & 1);
      mbar_wait(&empty[s], ((it / K1A_STAGES) & 1) ^ 1);
      unsigned char* As = stage_base + s * stage_bytes;
      const unsigned char* raw = raw_base + s * raw_bytes;
#pragma unroll
      for (int kk = 0; kk < MAXT; ++kk) {
        if (kk >= nt) break;
        uint4 v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = *reinterpret_cast<const uint4*>(raw + t_raw[kk] + e * chan_stride);
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
            const int pos = 2 * j + hl;  // position within the task: staged position sc*8 + pos
            const uint32_t delta = (uint32_t)(pos * 32) + (pos >= t_wrap[kk] ? wrap_jump : 0u);
            if (pos < t_lim[kk]) *reinterpret_cast<uint4*>(As + t_a[kk] + delta) = o;
          }
        }
      }
      fence_proxy_async();  // the saved-copy bulk stores read the stage through the async proxy
      mbar_arrive(&full[s]);
      mbar_arrive(&raw_empty[s]);
    }
  } else if (warp == K1A_LOADER) {
    // ================= TMA loader: raw feature rows run one stage ahead, weights follow the operand slots ====
    if (lane == 0) {
      auto issue_raw = [&](int it) {
        const int r = it % K1A_STAGES;
        mbar_wait(&raw_empty[r], ((it / K1A_STAGES) & 1) ^ 1);
        int b, f0, nb;
        k1a_band(k, item_of(it), b, f0, nb);
        const int st = it % P.nstages;
        mbar_expect_tx(&raw_full[r], (uint32_t)raw_bytes);  // out-of-range elements (past the frame) land as zeros
        tma_load_2d(raw_base + r * raw_bytes, &P.feat, f0 * k.W, b * P.C + st * 4 * HEAD_KSTAGE, &raw_full[r]);
      };
      if (total_it > 0) issue_raw(0);
      for (int it = 0; it < total_it; ++it) {
        if (it + 1 < total_it) issue_raw(it + 1);
        const int s = it % K1A_STAGES, st = it % P.nstages;
        mbar_wait(&empty[s], ((it / K1A_STAGES) & 1) ^ 1);
        mbar_expect_tx(&full[s], HEAD_BSTAGE_BYTES);
        bulk_g2s(stage_base + s * stage_bytes + a_stage_bytes,
                 reinterpret_cast<const unsigned char*>(P.wpk) + (size_t)st * HEAD_BSTAGE_BYTES, HEAD_BSTAGE_BYTES, &full[s]);
      }
    }
  } else if (XS && warp == K1A_LOADER + 1) {
    // ================= store warp: the finished operand stage -> the saved copy, by TMA bulk stores =================
    // The operand stage IS the saved copy's row layout (row_layout.cuh), zero columns included: per K-chunk, the band's
    // image rows are one contiguous store.  The first band also writes the lead rows, the last band the trail rows, so
    // every row of the copy is written exactly once.
    if (lane == 0) {
      const int lead = P.Lxs.lead, trail = P.Lxs.rows - lead - P.Lxs.Hi * P.Lxs.Pp;
      for (int it = 0; it < total_it; ++it) {
        const int s = it % K1A_STAGES, st = it % P.nstages;
        mbar_wait(&full[s], (it / K1A_STAGES) & 1);
        int b, f0, nb;
        k1a_band(k, item_of(it), b, f0, nb);
        unsigned char* slab = reinterpret_cast<unsigned char*>(P.xs + ((size_t)b * P.nstages + st) * 4 * (size_t)P.Lxs.rows * 8);
        const unsigned char* As = stage_base + s * stage_bytes;
        const uint32_t body_b = (uint32_t)(2 * nb * k.P) * 16;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          unsigned char* dst = slab + (size_t)kc * P.Lxs.rows * 16;
          if (f0 == 0) bulk_s2g(dst, zrows, (uint32_t)lead * 16);
          bulk_s2g(dst + (size_t)(lead + 2 * f0 * k.P) * 16, As + (size_t)kc * k.rows_alloc * 16, body_b);
          if (f0 + nb == k.H) bulk_s2g(dst + (size_t)(P.Lxs.rows - trail) * 16, zrows, (uint32_t)trail * 16);
        }
        bulk_commit_group();
        bulk_wait_group_read0();
        mbar_arrive(&empty[s]);
      }
      bulk_wait_group0();  // the copies are in global memory before the kernel ends
    }
  }
}

static size_t k1a_smem_bytes(const K1aGeom& k) {
  return (size_t)K1A_STAGES * (4 * k.rows_alloc * 16 + HEAD_BSTAGE_BYTES) + (size_t)K1A_STAGES * 4 * HEAD_KSTAGE * k.box * 2 + 128 + K1A_ZROWS * 16;
}

// features [B][C][HW] of type T viewed as [B * C][HW]; box = {box_px positions, 128 channels}, box_px <= HW (make_k1a_geom)
template <typename T>
static bool make_feat_tensor_map(CUtensorMap* tm, const void* feat, int B, int C, int HW, int box_px) {
  const TensorMapEncodeFn encode = tensor_map_encoder();
  if (!encode || (HW * 2) % 16 != 0 || (box_px * 2) % 16 != 0 || box_px > 256 || box_px > HW) return false;
  const cuuint64_t gdim[2] = {(cuuint64_t)HW, (cuuint64_t)B * C};
  const cuuint64_t gstride[1] = {(cuuint64_t)HW * 2};  // bytes, dim 1
  const cuuint32_t box[2] = {(cuuint32_t)box_px, 4 * HEAD_KSTAGE};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dtype = std::is_same_v<T, __half> ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  return encode(tm, dtype, 2, const_cast<void*>(feat), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
}  // namespace lpb

// ---- which kernels serve a shape ---------------------------------------------------------------------------
// fast path (k1a, then layer 2 on the banded kernel): two-deconv heads whose bands fit the shared-memory tiling above;
// generic path (head_rows_bf16.cu): everything else -- one-deconv heads, larger feature maps.
static bool head_fast_path(int C, int H, int W, int c2, int max_smem) {
  using namespace lpb;
  if (c2 <= 0) return false;
  // W <= 31: the saved copy's lead / trail rows fit the K1A_ZROWS zero source, and a band's staged rows one TMA box
  if (!((W >= 7 || W == 4 || W == 6) && H * W <= 192 && W <= 31)) return false;
  const K1aGeom k1 = make_k1a_geom(H, W);
  return k1.G > 0 && (int64_t)k1a_smem_bytes(k1) <= max_smem;
}

static_assert(lpb::HEAD_MAX_CH == LPB_HEAD_MAX_CHANNELS, "the cap lpb200.h states is the keypoint groups' (head_prep.cuh)");

// plan[0] = 1: fast path (saved_xs optional: training only); 0: generic path (saved_xs REQUIRED: it is the operand).
// Wide heads (more than HEAD_CLS keypoints, head_prep.cuh) always take the generic path.
// Channels-last features always take the banded kernels: k1a's TMA loader and transposer warps read NCHW slabs, while
// rows_shuffle_nhwc_kernel needs no shared memory, so the shuffle stage's feature-map limit does not apply either.
extern "C" int lpb_head_bf16_plan_layout(int C, int H, int W, int c1, int c2, int feature_layout, int* plan) {
  using namespace lpb;
  LPB_REQUIRE(plan, "head_bf16_plan: null pointer");
  LPB_REQUIRE(feature_layout == LPB_FEATURES_NCHW || feature_layout == LPB_FEATURES_NHWC, "head_bf16_plan: unknown feature layout %d", feature_layout);
  const bool nhwc = feature_layout == LPB_FEATURES_NHWC;
  LPB_REQUIRE(C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && (H * W) % 8 == 0 && c1 >= 1 && c2 >= 0, "head_bf16_plan: bad shape");
  if ((c2 > 0 ? c2 : c1) > HEAD_CLS && !head_wide(c1, c2)) {
    set_error("head_bf16_plan: channel counts %d/%d exceed the keypoint groups of this build (%d channels per layer)", c1, c2, HEAD_MAX_CH);
    return LPB_ERR_UNSUPPORTED;
  }
  LPB_REQUIRE(head_narrow(c1, c2) || head_wide(c1, c2), "head_bf16_plan: channel counts %d/%d exceed %d", c1, c2, HEAD_CLS);
  plan[0] = !nhwc && !head_wide(c1, c2) && head_fast_path(C, H, W, c2, planning_limits().max_smem) ? 1 : 0;
  if (!plan[0] && ((!nhwc && rows_shuffle_smem_bytes(H, W) > HEAD_FEATURE_SMEM_BUDGET) || (c2 > 0 ? 4 : 2) * W + 1 > CR_BAND_ROWS)) {
    set_error("head_bf16_plan: feature map %dx%d too large for this build", H, W);
    return LPB_ERR_UNSUPPORTED;
  }
  return LPB_OK;
}

extern "C" int lpb_head_bf16_plan(int C, int H, int W, int c1, int c2, int* plan) {
  return lpb_head_bf16_plan_layout(C, H, W, c1, c2, LPB_FEATURES_NCHW, plan);
}

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
  *bytes = head_fwd_layout(B, C, H, W, c1, c2).total;
  return LPB_OK;
}

// lpb_head_fwd_bf16 (T = __nv_bfloat16) and lpb_head_fwd_f16 (T = __half), and lpb_head3_fwd (c3 > 0): one plan, one
// workspace layout, one kernel sequence; T is the element type of the features, the packed weights and the mid
// activations.  A three-deconv head is the two-deconv sequence with its layer 2 writing mid activations (mid2) instead
// of planes, and a third banded launch over mid2 for the planes or the softmax.
template <typename T>
static int head_fwd(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1, const float* w2,
                    const float* b2, int c2, int final_softmax, int feature_layout, float* out, void* saved_xs, void* workspace,
                    void* stream, uint32_t* band_max = nullptr, const float* w3 = nullptr, const float* b3 = nullptr, int c3 = 0) {
  using namespace lpb;
  const char* name = head_fwd_name<T>;
  LPB_REQUIRE(feature_layout == LPB_FEATURES_NCHW || feature_layout == LPB_FEATURES_NHWC, "%s: unknown feature layout %d", name, feature_layout);
  const bool nhwc = feature_layout == LPB_FEATURES_NHWC, three = c3 > 0;
  LPB_REQUIRE(features && w1 && b1 && out && workspace, "%s: null pointer", name);
  LPB_REQUIRE(c2 == 0 || (w2 && b2), "%s: a two-deconv head needs w2 and b2", name);
  LPB_REQUIRE(!three || (c2 > 0 && w3 && b3), "%s: a three-deconv head needs w2, b2, w3 and b3", name);
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1, "%s: bad feature shape C=%d H=%d W=%d", name, C, H, W);
  LPB_REQUIRE((H * W) % 8 == 0, "%s: H*W must be a multiple of 8 (got %d)", name, H * W);
  LPB_REQUIRE(head_narrow(c1, c2) || head_wide(c1, c2), "%s: channel counts %d/%d outside this build's set (lpb200.h)", name, c1, c2);
  // features: TMA or uint4 loads; saved_xs, workspace: bulk copies and uint4 stores; out: float2 stores
  LPB_REQUIRE(aligned_to(features, 16), "%s: features must be 16-byte aligned", name);
  LPB_REQUIRE(aligned_to(saved_xs, 16), "%s: saved_xs must be 16-byte aligned", name);
  LPB_REQUIRE(aligned_to(workspace, 16), "%s: workspace must be 16-byte aligned", name);
  LPB_REQUIRE(aligned_to(out, 8), "%s: out must be 8-byte aligned", name);
  LPB_REQUIRE(aligned_to(band_max, 4), "%s: band_max must be 4-byte aligned", name);
  if (B == 0) return LPB_OK;
  DeviceLimits dev;
  LPB_TRY(device_limits(&dev));
  const int sms = dev.sms;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool fast = !nhwc && !head_wide(c1, c2) && head_fast_path(C, H, W, c2, dev.max_smem);
  const K1aGeom k1 = make_k1a_geom(H, W);
  // k1a's feature tensor map, encoded before anything is queued, so a failure leaves the stream untouched.  The plan stays
  // a function of the shape (CPU-only callers size buffers with it); every driver that runs sm_90a code has the encoder,
  // and the features' alignment was checked with the arguments.
  CUtensorMap feat_map;
  if (fast && !make_feat_tensor_map<T>(&feat_map, features, B, C, H * W, k1.box)) {
    set_error("%s: cannot encode the feature tensor map", name);
    return LPB_ERR_INVALID;
  }
  const int nst = C / 4 / HEAD_KSTAGE, nst2 = head_mid_stages(c1), nst3 = three ? head_mid_stages(c2) : 0;
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const RowLayout Lxs = make_row_layout(2 * H, 2 * W), Lmid = make_row_layout(4 * H, 4 * W), Lmid2 = make_row_layout(8 * H, 8 * W);
  const HeadFwdLayout wl = head_fwd_layout(B, C, H, W, c1, c2, c3);
  T* wp1 = reinterpret_cast<T*>(ws + wl.w1);
  T* wp2 = reinterpret_cast<T*>(ws + wl.w2);
  T* wp3 = reinterpret_cast<T*>(ws + wl.w3);
  T* mid = reinterpret_cast<T*>(ws + wl.mid);
  T* mid2 = reinterpret_cast<T*>(ws + wl.mid2);
  float* partials = reinterpret_cast<float*>(ws + wl.partials);
  {
    // one launch: both operand packs + the pad rows of the fresh row-layout buffers (k1a writes every row of the saved
    // copy itself; the banded path's shuffle kernel writes its own pads)
    PrepJobs jobs{};
    jobs.fpack[0] = {w1, nullptr, C / 4, c1, nst, head_groups(c1), wp1};
    // layer 2: bias rides on the constant-one channel c1 of the mid activations (only needed without softmax:
    // a per-plane constant does not change a softmax)
    if (c2 > 0) {
      jobs.fpack[1] = {w2, final_softmax && !three ? nullptr : b2, c1, c2, nst2, head_groups(c2), wp2};
      jobs.pads[0] = {mid, Lmid, (long long)B * 4 * nst2};
    }
    if (three) {  // layer 3 likewise, its bias on the constant-one channel c2 of mid2
      jobs.fpack[2] = {w3, final_softmax ? nullptr : b3, c2, c3, nst3, 1, wp3};
      jobs.pads[1] = {mid2, Lmid2, (long long)B * 4 * nst3};
    }
    launch_head_prep<T>(jobs, sms, s);
  }
  if (!fast) {
    // ---- generic path: shuffle rows -> banded GEMM(s) ----
    LPB_REQUIRE(saved_xs, "%s: this shape takes the banded kernels (lpb_head_bf16_plan = 0): pass the "
                          "lpb_head_bf16_saved_bytes() buffer as saved_xs", name);
    T* xs = static_cast<T*>(saved_xs);
    int rc = nhwc ? launch_rows_shuffle_nhwc(static_cast<const T*>(features), B, C, H, W, xs, s)
                  : launch_rows_shuffle(static_cast<const T*>(features), B, C, H, W, xs, s);
    if (rc != LPB_OK) return rc;
    ConvtRowsParams<T> p{};
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
      p.mode = final_softmax ? CONVT_ROWS_SOFTMAX : CONVT_ROWS_PLANES;
      p.band_max = final_softmax ? band_max : nullptr;
      rc = launch_convt_rows(p, sms, s);
      if (rc != LPB_OK) return rc;
      LPB_CUDA(cudaGetLastError());
      return LPB_OK;
    }
    p.mode = CONVT_ROWS_MID;
    p.mid = mid;
    p.Lout = Lmid;
    p.mid_kc = 4 * nst2;
    rc = launch_convt_rows(p, sms, s);
    if (rc != LPB_OK) return rc;
  } else {
    const size_t s1 = k1a_smem_bytes(k1);
    K1aParams<T> pa{};
    pa.feat = feat_map;
    pa.wpk = wp1;
    pa.bias = b1;
    pa.mid = mid;
    pa.xs = static_cast<T*>(saved_xs);
    pa.Lmid = Lmid;
    pa.Lxs = Lxs;
    pa.B = B;
    pa.C = C;
    pa.c1 = c1;
    pa.nstages = nst;
    pa.k = k1;
    auto kern = saved_xs ? k1a_shuffle_convt_kernel<T, 1> : k1a_shuffle_convt_kernel<T, 0>;
    LPB_TRY(set_dynamic_smem(kern, s1, name));
    // items are dealt round-robin (item = blockIdx.x + k gridDim.x), so with G = 2 and an even grid (132 SMs) a CTA always
    // takes the same band, and likewise with G = 3 and a grid divisible by 3: bands of equal size keep the CTAs even.
    // Unequal bands (H % G != 0, e.g. 16 x 12 features: 6 / 5 / 5 rows) leave the CTAs of the larger bands one row pair
    // more per item.
    const int items = B * k1.G;
    kern<<<items < sms ? items : sms, K1A_THREADS, s1, s>>>(pa);
  }
  // ---- the layers after the first, on both paths: the banded kernel over the mid activations; the bias is folded into
  // the GEMM through the ones channel (see the packs above).  `next` null: the head's last layer (planes or softmax);
  // otherwise the layer writes the next one's mid activations.
  auto banded_layer = [&](const T* X, RowLayout L, const T* wpk, int nstg, int cout, T* next, RowLayout Lnext, int next_kc) {
    ConvtRowsParams<T> p{};
    p.X = X;
    p.L = L;
    p.wpk = wpk;
    p.bias = nullptr;
    p.nst = nstg;
    p.B = B;
    p.cout = cout;
    p.out = out;
    p.partials = partials;
    if (next) {
      p.mode = CONVT_ROWS_MID;
      p.mid = next;
      p.Lout = Lnext;
      p.mid_kc = next_kc;
    } else {
      p.mode = final_softmax ? CONVT_ROWS_SOFTMAX : CONVT_ROWS_PLANES;
      p.band_max = final_softmax ? band_max : nullptr;
    }
    return launch_convt_rows(p, sms, s);
  };
  int rc = three ? banded_layer(mid, Lmid, wp2, nst2, c2, mid2, Lmid2, 4 * nst3) : banded_layer(mid, Lmid, wp2, nst2, c2, nullptr, RowLayout{}, 0);
  if (rc != LPB_OK) return rc;
  if (three) {
    rc = banded_layer(mid2, Lmid2, wp3, nst3, c3, nullptr, RowLayout{}, 0);
    if (rc != LPB_OK) return rc;
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_head_fwd_bf16_layout(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                        const float* w2, const float* b2, int c2, int final_softmax, int feature_layout, float* out,
                                        void* saved_xs, void* workspace, void* stream) {
  return head_fwd<__nv_bfloat16>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, feature_layout, out, saved_xs, workspace, stream);
}

extern "C" int lpb_head_fwd_f16_layout(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                       const float* w2, const float* b2, int c2, int final_softmax, int feature_layout, float* out,
                                       void* saved_xs, void* workspace, void* stream) {
  return head_fwd<__half>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, feature_layout, out, saved_xs, workspace, stream);
}

extern "C" int lpb_head_band_max_dims(int h, int w, int* band_rows, int* nbands) {
  using namespace lpb;
  LPB_REQUIRE(band_rows && nbands, "head_band_max_dims: null pointer");
  LPB_REQUIRE(h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0, "head_band_max_dims: bad heatmap size %dx%d", h, w);
  // launch_convt_rows' cut of the softmax layer's (h / 2) x (w / 2) input
  const int Hi = h / 2, Wi = w / 2;
  int R = CR_BAND_ROWS / (Wi + 1);
  R = R > Hi ? Hi : (R < 1 ? 1 : R);
  *band_rows = R;
  *nbands = convt_rows_bands(Hi, Wi);
  return LPB_OK;
}

extern "C" int lpb_head_fwd_bf16_band_max(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                          const float* w2, const float* b2, int c2, int feature_layout, float* out,
                                          uint32_t* band_max, void* saved_xs, void* workspace, void* stream) {
  LPB_REQUIRE(band_max, "head_fwd_bf16: null band_max");
  return head_fwd<__nv_bfloat16>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, 1, feature_layout, out, saved_xs, workspace, stream, band_max);
}

extern "C" int lpb_head_fwd_f16_band_max(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                         const float* w2, const float* b2, int c2, int feature_layout, float* out,
                                         uint32_t* band_max, void* saved_xs, void* workspace, void* stream) {
  LPB_REQUIRE(band_max, "head_fwd_f16: null band_max");
  return head_fwd<__half>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, 1, feature_layout, out, saved_xs, workspace, stream, band_max);
}

extern "C" int lpb_head_fwd_bf16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                 const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                                 void* workspace, void* stream) {
  return lpb_head_fwd_bf16_layout(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, LPB_FEATURES_NCHW, out, saved_xs, workspace, stream);
}

extern "C" int lpb_head_fwd_f16(const void* features, int B, int C, int H, int W, const float* w1, const float* b1, int c1,
                                const float* w2, const float* b2, int c2, int final_softmax, float* out, void* saved_xs,
                                void* workspace, void* stream) {
  return lpb_head_fwd_f16_layout(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, LPB_FEATURES_NCHW, out, saved_xs, workspace, stream);
}

// ---- three-deconv heads (lpb200.h lpb_head3_fwd; the size query is with the backward's, head_bwd_bf16.cu) -------------
extern "C" int lpb_head3_fwd(const void* features, int operand, int feature_layout, int B, int C, int H, int W, const float* w1,
                             const float* b1, int c1, const float* w2, const float* b2, int c2, const float* w3, const float* b3, int c3,
                             int final_softmax, float* out, uint32_t* band_max, void* saved_xs, void* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(operand == LPB_OUT_BF16 || operand == LPB_OUT_F16, "head3_fwd: operand type %d is neither LPB_OUT_BF16 nor LPB_OUT_F16", operand);
  LPB_REQUIRE(feature_layout == LPB_FEATURES_NCHW || feature_layout == LPB_FEATURES_NHWC, "head3_fwd: unknown feature layout %d", feature_layout);
  LPB_REQUIRE(B >= 0 && C >= 128 && C % 128 == 0 && H >= 1 && W >= 1 && c1 >= 1 && c2 >= 1 && c3 >= 1, "head3_fwd: bad shape");
  LPB_REQUIRE(!band_max || final_softmax, "head3_fwd: band maxima are written by the softmax; final_softmax must be 1");
  const char* why = nullptr;
  if (!head3_covered(H, W, c1, c2, c3, false, &why)) {
    set_error("head3_fwd: %dx%d features, channels %d/%d/%d: %s", H, W, c1, c2, c3, why);
    return LPB_ERR_UNSUPPORTED;
  }
  int plan = 0;
  LPB_TRY(lpb_head_bf16_plan_layout(C, H, W, c1, c2, feature_layout, &plan));
  LPB_REQUIRE(plan || saved_xs, "head3_fwd: this shape takes the banded kernels (lpb_head3_query plan = 0): pass saved_xs");
  if (operand == LPB_OUT_F16)
    return head_fwd<__half>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, feature_layout, out, saved_xs, workspace, stream,
                            band_max, w3, b3, c3);
  return head_fwd<__nv_bfloat16>(features, B, C, H, W, w1, b1, c1, w2, b2, c2, final_softmax, feature_layout, out, saved_xs, workspace,
                                 stream, band_max, w3, b3, c3);
}
