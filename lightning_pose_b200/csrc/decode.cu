// Soft-argmax decode: heatmaps (n_planes, h, w) -> (x, y, confidence) per plane.
//
// Reference semantics (lightning_pose/models/heads/heatmap.py:103-144, data/heatmaps.py:90-142):
//   field = upsample^ds(h)  (each stage: 2x bicubic + zero-padded 5x5 binomial blur, :86-100)
//   p = softmax(T * field) over the whole (h*2^ds, w*2^ds) field
//   (x, y) = sum p * (col, row);  conf = sum of the 5x5 window of p around (trunc y, trunc x)
//   (x, y) -= {0.5, 1.5, 2.5}
//
// Design (DESIGN.md "K2"): the 4x-upsampled field is never materialised: field = U_H h U_W^T is evaluated separably in
// registers (horizontal pass from shared memory, vertical pass on a sliding register window with the phase-periodic
// interior weights in the constant bank).
// Forward: one warp per plane (decode_fwd_warp_kernel) bounds the coarse box that can hold softmax mass > exp(-40)
// relative to the peak (rigorous bound |field| <= lip * max|h| over the tap footprint) with two sweeps of the plane, and
// evaluates only that box, from a 32 x 32 window in shared memory.  The planes whose box does not fit the window
// (diffuse / multi-modal: freshly initialised networks), NaN planes and T <= 0 are queued for decode_fwd_kernel, which
// stages each queued plane into shared memory once (TMA row copies into a zero-padded tile, or plain loads), splits it
// over several CTAs and evaluates all of it.
// Backward: the same split, a 32 x 32 window per plane (decode_bwd_window_kernel) or the whole plane (decode_bwd_kernel).
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"
#include "upsample_tables.cuh"

namespace lpb {

constexpr int DEC_THREADS = 256;
constexpr int DEC_WARPS = DEC_THREADS / 32;
constexpr float DEC_CUT = 40.0f;  // dropped pixels have weight < exp(-40) = 4e-18 of the peak pixel
constexpr int DEC_MAX_PARTS = 16;  // CTAs a queued (dense) plane can be split over
constexpr int DEC_CONF_R = 2;     // floor(1.25 * 2), lightning_pose/data/heatmaps.py:111

// What the forward and backward kernels share: the planes, their upsampling tables and the tap constants (decode_geom).
template <int DS>
struct DecodeGeom {
  static constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1;
  const float* heat;
  const float* tabH;  // [h*F][W] vertical-axis window weights
  const float* tabW;  // [w*F][W] horizontal-axis window weights
  int h, w, pitch, padl;  // a plane's zero-padded shared-memory tile: row pitch, first plane column (floats)
  int bulk;           // w % 4 == 0 and heat 16-byte aligned: TMA row copies, 16-byte loads
  int64_t n_planes;
  float T;
  float lipw;         // max row sum of |horizontal taps|
  float wabs[W];      // max over rows / phases of |vertical tap| per offset (row pruning of the window kernels)
  float2 phase2[F / 2][W];  // vertical taps of the interior rows' phases 2q, 2q+1: packed-pair constant-bank operands
};

template <int DS>
struct DecodeParams : DecodeGeom<DS> {
  float* xy;
  float* conf;
  float* stats;
  float lip, offset;
  int* queue;         // {count, plane ids ...}: the planes the warp kernel leaves for the CTA kernel
  int* qcounter;      // [n_planes] arrival counters (zeroed) and
  float* qscratch;    // [n_planes][DEC_MAX_PARTS][4] partial softmax states of a plane split over several CTAs
};

__host__ __device__ inline int dec_padl(int R) { return (R + 3) & ~3; }
__host__ __device__ inline int dec_pitch(int w, int R) { return (dec_padl(R) + w + R + 3) & ~3; }

template <int W>
__device__ __forceinline__ float dot_w(const float* __restrict__ p, const float (&wc)[W]) {
  float r = 0.f;
#pragma unroll
  for (int t = 0; t < W; ++t) r = fmaf(wc[t], p[t], r);
  return r;
}

// exact field value at fine pixel (i, j) (W*W taps)
template <int DS>
__device__ float eval_point(const float* tile, int pitch, int padl, const float* __restrict__ tabH,
                            const float* __restrict__ tabW, int i, int j) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1;
  const float* base = tile + (i / F) * pitch + padl + (j / F - R);  // row index (a - R) + R = a
  float acc = 0.f;
#pragma unroll 1
  for (int t = 0; t < W; ++t) {
    const float* row = base + t * pitch;
    float r = 0.f;
#pragma unroll
    for (int u = 0; u < W; ++u) r = fmaf(__ldg(tabW + j * W + u), row[u], r);
    acc = fmaf(__ldg(tabH + i * W + t), r, acc);
  }
  return acc;
}

// exact field values at npts fine pixels (scratch: npts * W floats), spread over the CTA: thread (pt, t) evaluates one horizontal tap row, the W rows
// of a point meet in shared memory.  (One thread per point walked W x W dependent table loads: ~3 us per call.)
// Returns the value of point `tid` for tid < npts; contains a __syncthreads().
template <int DS, class CoordFn>
__device__ __forceinline__ float eval_points_cta(const float* tile, int pitch, int padl, const float* __restrict__ tabH,
                                                 const float* __restrict__ tabW, int npts, CoordFn coord, float* scratch, int tid) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1;
  for (int idx = tid; idx < npts * W; idx += DEC_THREADS) {
    const int pt = idx / W, t = idx - pt * W;
    int i = 0, j = 0;
    float val = 0.f;
    if (coord(pt, i, j)) {
      const float* row = tile + (i / F + t) * pitch + padl + (j / F - R);
      float r = 0.f;
#pragma unroll
      for (int u = 0; u < W; ++u) r = fmaf(__ldg(tabW + j * W + u), row[u], r);
      val = __ldg(tabH + i * W + t) * r;
    }
    scratch[idx] = val;
  }
  __syncthreads();
  float out = 0.f;
  if (tid < npts) {
#pragma unroll
    for (int t = 0; t < W; ++t) out += scratch[tid * W + t];
  }
  return out;
}

// one coarse row of the vertical pass: F fine values from the W-row window `t`, as F/2 packed pairs of phases
// (fma.rn.f32x2: the same fp32 roundings as the scalar chain, half the issue slots)
template <int DS>
__device__ __forceinline__ void column_pass(const DecodeGeom<DS>& P, int a, int h, const float* t, f32x2* v2) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1, HP = F / 2;
  if (a >= R && a <= h - 1 - R) {  // interior: phase-periodic weights are kernel-parameter constants (uniform registers)
#pragma unroll
    for (int q = 0; q < HP; ++q) {
      f32x2 r = pack2(0.f, 0.f);
#pragma unroll
      for (int k = 0; k < W; ++k) r = fma2(pack2(P.phase2[q][k].x, P.phase2[q][k].y), dup2(t[k]), r);
      v2[q] = r;
    }
  } else {  // border rows: per-row table (edge-clamped bicubic taps, zero-padded blur)
    const float* __restrict__ tr = P.tabH + (size_t)a * F * W;
#pragma unroll
    for (int q = 0; q < HP; ++q) {
      f32x2 r = pack2(0.f, 0.f);
#pragma unroll
      for (int k = 0; k < W; ++k) r = fma2(pack2(__ldg(tr + (2 * q) * W + k), __ldg(tr + (2 * q + 1) * W + k)), dup2(t[k]), r);
      v2[q] = r;
    }
  }
}

// online-softmax update of one lane's column with the F fine values of one coarse row (yrow = fine row index of phase 0):
//   s += sum_p e_p,  sy += sum_p (yrow + p) e_p,  e_p = 2^((v_p - m) c);  m is raised (and s, sy rescaled) warp-wide
template <int DS>
__device__ __forceinline__ void softmax_row(const f32x2* v2, float yrow, float c, float kill, float& m, float& mc, float& s_it,
                                            float& sy_it) {
  constexpr int HP = (1 << DS) / 2;
  float vm = -3.0e38f;
#pragma unroll
  for (int q = 0; q < HP; ++q) {
    float lo, hi;
    unpack2(v2[q], lo, hi);
    vm = fmaxf(vm, fmaxf(lo, hi));
  }
  vm += kill;
  if (__any_sync(0xffffffffu, vm > m)) {
    const float mn = fmaxf(m, vm);
    const float sc = fast_exp2((m - mn) * c);
    s_it *= sc;
    sy_it *= sc;
    m = mn;
    mc = mn * c;
  }
  const f32x2 c2 = dup2(c), nmc2 = dup2(-mc), kill2 = dup2(kill);
  f32x2 rs2 = pack2(0.f, 0.f), pw2 = pack2(0.f, 0.f);
#pragma unroll
  for (int q = 0; q < HP; ++q) {
    float x0, x1;
    unpack2(add2(fma2(v2[q], c2, nmc2), kill2), x0, x1);
    const f32x2 e2 = pack2(fast_exp2(x0), fast_exp2(x1));
    rs2 = add2(rs2, e2);
    pw2 = fma2(e2, pack2((float)(2 * q), (float)(2 * q + 1)), pw2);
  }
  float r0, r1, p0, p1;
  unpack2(rs2, r0, r1);
  unpack2(pw2, p0, p1);
  const float rs = r0 + r1;
  s_it += rs;
  sy_it = fmaf(yrow, rs, sy_it) + (p0 + p1);
}

// One strip of the forward evaluation: the lane's fine column over coarse rows [r0, r1).  `base` points at the lane's first
// horizontal tap in the tile row of coarse row r0 - R ("window row" 0); window row k is `base + k * pitch`.
// The horizontal pass of W + 1 window rows lives in a ROTATING register window of packed pairs (no shifting moves): two
// coarse rows are evaluated per step and the two window rows they free are refilled by one paired horizontal pass
// (fma.rn.f32x2 over two tile rows).  In the round-2 capture of the dense kernel the shifting moves and their integer
// bookkeeping were 40 % of the loop's instructions.
template <int DS>
__device__ __forceinline__ void fwd_strip(const DecodeGeom<DS>& P, const float* base, int pitch, const float (&wc)[2 * (DS + 2) + 1],
                                          int r0, int r1, float c, float kill, float& m, float& mc, float& s_it, float& sy_it) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1, NS = W + 1, NP2 = NS / 2, HP = F / 2;
  const int h = P.h, nrows = r1 - r0, kmax = nrows - 1 + 2 * R;  // last window row a valid coarse row uses
  auto hpair = [&](int k) -> f32x2 {  // horizontal pass of window rows k, k+1 (clamped to the rows that exist)
    const float* ra = base + min(k, kmax) * pitch;
    const float* rb = base + min(k + 1, kmax) * pitch;
    f32x2 acc = pack2(0.f, 0.f);
#pragma unroll
    for (int u = 0; u < W; ++u) acc = fma2(dup2(wc[u]), pack2(ra[u], rb[u]), acc);
    return acc;
  };
  f32x2 win[NP2];  // window rows la .. la+W; row la+j sits in slot (2i + j) % NS of pair-step i
#pragma unroll
  for (int i = 0; i < NP2; ++i) win[i] = hpair(2 * i);
  for (int la0 = 0; la0 < nrows; la0 += NS) {
    static_for<0, NP2>([&](auto ic) {
      constexpr int i = decltype(ic)::value;
      const int la = la0 + 2 * i;
      if (la >= nrows) return;  // warp-uniform
      float sl[NS];
#pragma unroll
      for (int j = 0; j < NP2; ++j) unpack2(win[j], sl[2 * j], sl[2 * j + 1]);
      f32x2 v2[HP];
      {
        float t[W];
#pragma unroll
        for (int k = 0; k < W; ++k) t[k] = sl[(2 * i + k) % NS];
        column_pass<DS>(P, r0 + la, h, t, v2);
        softmax_row<DS>(v2, (float)((r0 + la) * F), c, kill, m, mc, s_it, sy_it);
      }
      if (la + 1 < nrows) {
        float t[W];
#pragma unroll
        for (int k = 0; k < W; ++k) t[k] = sl[(2 * i + 1 + k) % NS];
        column_pass<DS>(P, r0 + la + 1, h, t, v2);
        softmax_row<DS>(v2, (float)((r0 + la + 1) * F), c, kill, m, mc, s_it, sy_it);
      }
      win[i] = hpair(la + NS);  // window rows la+W+1, la+W+2 take the slots of la, la+1
    });
  }
}

// Shared memory the CTA kernel requests beyond its tile, in floats.  The kernel uses less; the request keeps the size it
// had when the kernel also pruned planes itself, because the request sets how many CTAs are resident, and with that over
// how many CTAs each queued plane is split and in which order its partial sums are added.
constexpr int DEC_FWD_SCRATCH = 880;

// The planes the warp kernel queued, evaluated whole.  A queued plane is split over NP CTAs (a call queues few planes,
// which alone would leave most SMs idle): its work items -- (32-fine-column strip, row segment) pairs -- are dealt
// round-robin over the parts, the parts' online-softmax states meet in global scratch, and the last CTA to arrive merges
// them and finishes the plane.  The CTAs are persistent over the (plane, part) pairs.
template <int DS>
__global__ void __launch_bounds__(DEC_THREADS, DS == 3 ? 2 : 4) decode_fwd_kernel(const __grid_constant__ DecodeParams<DS> P) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1, CW = 2 * DEC_CONF_R + 1;
  static_assert(4 * DEC_WARPS + 3 + CW * CW * W <= DEC_FWD_SCRATCH, "decode_fwd_kernel: scratch exceeds the request");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int h = P.h, w = P.w, pitch = P.pitch, padl = P.padl;
  float* tile = reinterpret_cast<float*>(smem_raw);  // (h + 2R) x pitch; logical (a,b) at [(a+R)*pitch + padl + b]
  float* red = tile + (h + 2 * R) * pitch;           // [DEC_WARPS][4] per-warp softmax states
  uint64_t* bar = reinterpret_cast<uint64_t*>(red + 4 * DEC_WARPS);
  int* arrival = reinterpret_cast<int*>(bar + 1);       // this CTA's place among the parts of its plane
  float* evs = reinterpret_cast<float*>(arrival + 1);  // CW * CW * W floats: tap rows of eval_points_cta
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- once per CTA: barrier + zero halo (the CTA is persistent; only the interior is rewritten) ----
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  for (int r = warp; r < h + 2 * R; r += DEC_WARPS) {
    float* row = tile + r * pitch;
    if (r < R || r >= h + R) {
      for (int b = lane; b < pitch; b += 32) row[b] = 0.f;
    } else {
      for (int b = lane; b < padl; b += 32) row[b] = 0.f;
      for (int b = padl + w + lane; b < pitch; b += 32) row[b] = 0.f;
    }
  }
  __syncthreads();

  uint32_t tma_phase = 0;
  const int qcount = P.queue[0];
  const int NP = qcount > 0 ? min(DEC_MAX_PARTS, max(1, (int)gridDim.x / qcount)) : 1;
  const size_t nwork = (size_t)qcount * NP;
  for (size_t work = blockIdx.x; work < nwork; work += gridDim.x) {
  const size_t slot = work / NP;
  const int part = (int)(work - slot * NP);
  const size_t plane = (size_t)P.queue[1 + slot];
  const float* __restrict__ src = P.heat + plane * (size_t)h * w;

  // ---- stage the plane: TMA bulk row copies into the zero-padded tile, or plain loads ------------
  if (P.bulk) {
    if (warp == 0) {
      if (lane == 0) mbar_expect_tx(bar, (uint32_t)(h * w * 4));
      __syncwarp();
      for (int a = lane; a < h; a += 32)
        bulk_g2s(tile + (a + R) * pitch + padl, src + (size_t)a * w, (uint32_t)(w * 4), bar);
      mbar_wait(bar, tma_phase);  // one warp polls; the bytes are in shared memory once the phase flips
    }
    tma_phase ^= 1;
  } else {
    for (int r = warp; r < h; r += DEC_WARPS) {
      const float* g = src + (size_t)r * w;
      float* row = tile + (r + R) * pitch + padl;
      for (int b = lane; b < w; b += 32) row[b] = __ldg(g + b);
    }
  }
  __syncthreads();

  // ---- the items of this part: a per-lane online softmax over the whole plane, from a low finite maximum ----------
  // a strip's rows [0, h) are cut into nseg segments of seglen rows: at most 48 rows, and short enough that all the warps
  // of all NP CTAs have an item (a queued plane's latency matters, not throughput).  These are the same for every plane,
  // but computed outside the plane loop they took uniform registers that the interior tap constants of column_pass need:
  // at ds = 2 the constants were then reloaded inside the strip loop, and flat planes decoded about 4 % slower.
  const int nstrips = (w * F + 31) >> 5;  // <= 32 (checked on the host)
  const int per_strip = max(1, (NP * DEC_WARPS) / nstrips);
  const int seg_cap = min(48, max(8, (h + per_strip - 1) / per_strip));
  const int nseg = (h + seg_cap - 1) / seg_cap, seglen = (h + nseg - 1) / nseg, nitems = nstrips * nseg;
  const float c = P.T * 1.4426950408889634f;
  float M = -1.0e30f, S = 0.f, SX = 0.f, SY = 0.f;
  for (int itw = warp;; itw += DEC_WARPS) {
    const int item = itw * NP + part;
    if (item >= nitems) break;
    const int sl = item / nseg;  // strip index
    const int r0 = (item - sl * nseg) * seglen, r1 = min(r0 + seglen, h);
    if (r0 >= r1) continue;
    const int jf = sl * 32 + lane;
    const bool ok = jf < w * F;
    const int jc = ok ? jf : (w * F - 1);
    float wc[W];
#pragma unroll
    for (int t = 0; t < W; ++t) wc[t] = __ldg(P.tabW + jc * W + t);
    const float* colbase = tile + padl + (jc / F - R);  // add (a + R) * pitch for coarse row a
    float m = M, mc = M * c, s_it = 0.f, sy_it = 0.f;
    const float kill = ok ? 0.f : -3.0e38f;
    fwd_strip<DS>(P, colbase + r0 * pitch, pitch, wc, r0, r1, c, kill, m, mc, s_it, sy_it);
    {  // fold the item into the lane's running state
      const float Mn = fmaxf(M, m);
      const float a1 = fast_exp2((M - Mn) * c), a2 = fast_exp2((m - Mn) * c);
      S = fmaf(s_it, a2, S * a1);
      SX = fmaf((float)jf * s_it, a2, SX * a1);
      SY = fmaf(sy_it, a2, SY * a1);
      M = Mn;
    }
  }

  // ---- merge the per-lane online-softmax states ----------------------------------------------------
  {
    const float Mw = warp_max(M);
    const float sc = fast_exp2((M - Mw) * c);
    S = warp_sum(S * sc);
    SX = warp_sum(SX * sc);
    SY = warp_sum(SY * sc);
    if (lane == 0) {
      red[4 * warp + 0] = Mw;
      red[4 * warp + 1] = S;
      red[4 * warp + 2] = SX;
      red[4 * warp + 3] = SY;
    }
  }
  __syncthreads();
  M = red[0];
#pragma unroll
  for (int k = 1; k < DEC_WARPS; ++k) M = fmaxf(M, red[4 * k]);
  S = 0.f;
  SX = 0.f;
  SY = 0.f;
#pragma unroll
  for (int k = 0; k < DEC_WARPS; ++k) {
    const float sc = fast_exp2((red[4 * k] - M) * c);
    S = fmaf(red[4 * k + 1], sc, S);
    SX = fmaf(red[4 * k + 2], sc, SX);
    SY = fmaf(red[4 * k + 3], sc, SY);
  }
  bool finisher = true;
  if (NP > 1) {  // cross-CTA merge of the parts of this plane
    float* part_state = P.qscratch + (slot * DEC_MAX_PARTS + part) * 4;
    if (tid == 0) {
      part_state[0] = M;
      part_state[1] = S;
      part_state[2] = SX;
      part_state[3] = SY;
      __threadfence();
      *arrival = atomicAdd(P.qcounter + slot, 1);
    }
    __syncthreads();
    finisher = *arrival == NP - 1;
    if (finisher) {
      __threadfence();
      const volatile float* ps = P.qscratch + slot * DEC_MAX_PARTS * 4;
      M = ps[0];
      for (int k = 1; k < NP; ++k) M = fmaxf(M, ps[4 * k]);
      S = 0.f;
      SX = 0.f;
      SY = 0.f;
      for (int k = 0; k < NP; ++k) {
        const float sc = fast_exp2((ps[4 * k] - M) * c);
        S = fmaf(ps[4 * k + 1], sc, S);
        SX = fmaf(ps[4 * k + 2], sc, SX);
        SY = fmaf(ps[4 * k + 3], sc, SY);
      }
    }
  }
  if (finisher) {
  const float xhat = SX / S, yhat = SY / S;

  // ---- confidence: softmax mass of the (2r+1)^2 window around (trunc y, trunc x) -----------------
  float cw = 0.f;
  {
    auto wcoord = [&](int pt, int& i, int& j) {
      i = (int)yhat + pt / CW - DEC_CONF_R;
      j = (int)xhat + pt % CW - DEC_CONF_R;
      return i >= 0 && i < h * F && j >= 0 && j < w * F;
    };
    const float v = eval_points_cta<DS>(tile, pitch, padl, P.tabH, P.tabW, CW * CW, wcoord, evs, tid);
    int i, j;
    if (tid < CW * CW && wcoord(tid, i, j)) cw = fast_exp2((v - M) * c) / S;
  }
  cw = warp_sum(cw);  // CW*CW = 25 <= 32: all in warp 0
  if (tid == 0) {
    P.xy[2 * plane + 0] = xhat - P.offset;
    P.xy[2 * plane + 1] = yhat - P.offset;
    P.conf[plane] = cw;
    if (P.stats) {  // the evaluated box is the whole plane
      float* st = P.stats + 8 * plane;
      st[0] = M;
      st[1] = S;
      st[2] = xhat;
      st[3] = yhat;
      st[4] = 0.f;
      st[5] = (float)(h - 1);
      st[6] = 0.f;
      st[7] = (float)(w - 1);
    }
  }
  }  // finisher
  __syncthreads();  // every read of the tile / scratch is done before the next plane is staged
  }  // persistent plane loop
}

// ------------------------------------------------------------------------------------------------
// Warp-per-plane forward, run on every plane.  One warp owns a plane end to end and only warp-level primitives are used
// (a CTA per plane synchronised eight warps five times per plane, and more than half of its stall samples were at
// those barriers):
//   pass 1  stream the plane in 4-column groups, arg max |h|
//   window  32x32 coarse pixels around the arg max -> shared memory; m_lb = exact field on the arg max's F x F block
//   pass 2  stream the plane again (L2), hull of the candidates |h| >= theta
//   window  re-centred on the hull +- R; rows pruned with the tap-decay bound; separable evaluation of the strips
//           with a per-lane online softmax; exact 5x5 confidence window
// Planes whose hull does not fit a window (diffuse / multi-modal), NaN planes and T <= 0 are appended to the queue of
// decode_fwd_kernel.
// BULK (w % 4 == 0, plane 16-byte aligned): a group is one 16-byte load.  Otherwise it is four scalar loads, columns >= w
// read as 0: the same groups in the same order with the same tie-breaks, so an aligned and a misaligned copy of the same
// planes decode to the same bits.
constexpr int DECW_WIN = 32, DECW_WP = 33;

template <int DS>
__device__ float eval_point_win(const float* tile, int r0w, int c0w, const float* __restrict__ tabH,
                                const float* __restrict__ tabW, int i, int j) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1;
  const float* base = tile + (i / F - R - r0w) * DECW_WP + (j / F - R - c0w);
  float acc = 0.f;
#pragma unroll 1
  for (int t = 0; t < W; ++t) {
    const float* row = base + t * DECW_WP;
    float r = 0.f;
#pragma unroll
    for (int u = 0; u < W; ++u) r = fmaf(__ldg(tabW + j * W + u), row[u], r);
    acc = fmaf(__ldg(tabH + i * W + t), r, acc);
  }
  return acc;
}

__device__ __forceinline__ void load_window(float* tile, const float* __restrict__ src, int h, int w, int r0w, int c0w, int lane) {
  const int x = c0w + lane;
  const bool xin = x >= 0 && x < w;
#pragma unroll 8
  for (int r = 0; r < DECW_WIN; ++r) {
    const int y = r0w + r;
    tile[r * DECW_WP + lane] = (xin && y >= 0 && y < h) ? __ldg(src + (size_t)y * w + x) : 0.f;
  }
}

// One plane, one warp; `src` is the plane in global memory (read-only path, three sweeps of it).
template <int DS, bool BULK>
__device__ void decode_plane_warp(const DecodeParams<DS>& P, long long plane, const float* __restrict__ src, float* tile,
                                  int* __restrict__ queue, int lane) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1;
  const int h = P.h, w = P.w, w4 = BULK ? w >> 2 : (w + 3) >> 2, n4 = h * w4;
  const float4* __restrict__ src4 = reinterpret_cast<const float4*>(src);
  // L2 residency hints: the arg-max sweep asks L2 to KEEP the plane (evict_last), the hull sweep that follows re-reads it
  // from L2 and releases it (evict_first) -- without them the second sweep misses L2 (measured DRAM traffic 2.05x the
  // plane bytes: the kernel ran at ~80 % of HBM peak on twice the necessary bytes)
  uint64_t pol_keep, pol_drop;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_keep));
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_drop));
  auto ld4 = [&](int idx) -> float4 {  // 4-column group idx = a * w4 + g
    if constexpr (BULK) {
      return __ldg(src4 + idx);
    } else {
      const int a = idx / w4, b = 4 * (idx - a * w4);
      const float* p = src + (size_t)a * w + b;
      return make_float4(__ldg(p), b + 1 < w ? __ldg(p + 1) : 0.f, b + 2 < w ? __ldg(p + 2) : 0.f, b + 3 < w ? __ldg(p + 3) : 0.f);
    }
  };
  auto ld4h = [&](int idx, uint64_t pol) -> float4 {  // the same, with the L2 hint where the load is one instruction
    if constexpr (BULK) {
      float4 v;
      asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(src4 + idx), "l"(pol));
      return v;
    } else {
      return ld4(idx);
    }
  };
  auto to_queue = [&]() {
    if (lane == 0) queue[1 + atomicAdd(queue, 1)] = (int)plane;
  };

  // ---- pass 1: arg max of |h| ----------------------------------------------------------------------------
  float best = -1.f;
  int bidx = 0;
#pragma unroll 8
  for (int idx = lane; idx < n4; idx += 32) {
    const float4 x = ld4h(idx, pol_keep);
    const float m4 = fmaxf(fmaxf(fabsf(x.x), fabsf(x.y)), fmaxf(fabsf(x.z), fabsf(x.w)));
    if (m4 > best) {
      best = m4;
      bidx = idx;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (ob > best || (ob == best && oi < bidx)) {
      best = ob;
      bidx = oi;
    }
  }
  if (!(best >= 0.f) || !(P.T > 0.f)) {  // NaN plane or no temperature: the CTA kernel's whole-plane evaluation
    to_queue();
    return;
  }
  const int besta = bidx / w4;
  int bestb = (bidx - besta * w4) * 4;
  {
    const float4 x = ld4(bidx);
    bestb += (fabsf(x.x) == best) ? 0 : ((fabsf(x.y) == best) ? 1 : ((fabsf(x.z) == best) ? 2 : 3));
    if constexpr (!BULK) bestb = min(bestb, w - 1);
  }
  // ---- lower bound of the field maximum: exact values on the arg max's F x F block ---------------------
  int r0w = besta - DECW_WIN / 2, c0w = bestb - DECW_WIN / 2;
  load_window(tile, src, h, w, r0w, c0w, lane);
  __syncwarp();
  float lb = -3.0e38f;
  if (lane < F * F) lb = eval_point_win<DS>(tile, r0w, c0w, P.tabH, P.tabW, besta * F + lane / F, bestb * F + lane % F);
  const float mlb = warp_max(lb);
  const float thr = mlb - DEC_CUT / P.T;
  const float theta = thr / P.lip;

  // ---- pass 2: hull of the candidates (|h| >= theta), 4-column granularity ---------------------------------
  int amin = h, amax = -1, bmin = w, bmax = -1;
  {
    int a = 0, g = lane;  // idx = a * w4 + g
    while (g >= w4) {
      g -= w4;
      ++a;
    }
#pragma unroll 4
    for (int idx = lane; idx < n4; idx += 32) {
      const float4 x = ld4h(idx, pol_drop);
      const bool c = (fabsf(x.x) >= theta) || (fabsf(x.y) >= theta) || (fabsf(x.z) >= theta) || (fabsf(x.w) >= theta);
      if (c) {
        amin = min(amin, a);
        amax = max(amax, a);
        bmin = min(bmin, 4 * g);
        bmax = max(bmax, min(4 * g + 3, w - 1));
      }
      g += 32;
      while (g >= w4) {
        g -= w4;
        ++a;
      }
    }
  }
  amin = warp_min_i(amin);
  amax = warp_max_i(amax);
  bmin = warp_min_i(bmin);
  bmax = warp_max_i(bmax);
  const int A0 = max(amin - R, 0), A1 = min(amax + R, h - 1);
  const int B0 = max(bmin - R, 0), B1 = min(bmax + R, w - 1);
  const int nrows = A1 - A0 + 1, ncols = B1 - B0 + 1;
  // one spare row / column on each side: the confidence window may step one coarse pixel outside the box
  if (amax < 0 || nrows > DECW_WIN - 2 * R - 2 || ncols > DECW_WIN - 2 * R - 2) {
    to_queue();
    return;
  }
  r0w = A0 - R - 1;
  c0w = B0 - R - 1;
  __syncwarp();
  load_window(tile, src, h, w, r0w, c0w, lane);
  __syncwarp();

  // ---- rows that can carry weight (tap-decay bound, see decode_bwd_window_kernel); lane r owns window row r ----
  int ra0 = A0, ra1 = A1;
  {
    float rmx = 0.f;
#pragma unroll 8
    for (int cc = 0; cc < DECW_WIN; ++cc) rmx = fmaxf(rmx, fabsf(tile[lane * DECW_WP + cc]));
    float bnd = 0.f;
#pragma unroll
    for (int t = 0; t < W; ++t) {
      const int sl = lane - R + t;
      const float v = __shfl_sync(0xffffffffu, rmx, sl & 31);
      if ((unsigned)sl < (unsigned)DECW_WIN) bnd = fmaf(P.wabs[t], v, bnd);
    }
    const int arow = r0w + lane;  // coarse row of window row `lane`
    const unsigned am = __ballot_sync(0xffffffffu, arow >= A0 && arow <= A1 && bnd * P.lipw >= thr);
    if (am) {
      ra0 = r0w + (__ffs(am) - 1);
      ra1 = r0w + (31 - __clz(am));
    }
  }

  // ---- strips of 32 fine columns over rows [ra0, ra1]: separable evaluation + per-lane online softmax -------
  const float c = P.T * 1.4426950408889634f;
  float M = mlb, S = 0.f, SX = 0.f, SY = 0.f;
  const int J0 = B0 * F, J1 = (B1 + 1) * F;
  for (int jf0 = J0; jf0 < J1; jf0 += 32) {
    const int jf = jf0 + lane;
    const bool ok = jf < J1;
    const int jc = ok ? jf : (J1 - 1);
    float wc[W];
#pragma unroll
    for (int t = 0; t < W; ++t) wc[t] = __ldg(P.tabW + jc * W + t);
    const float* colbase = tile + (jc / F - R - c0w);  // add (a - R - r0w + t) * WP for coarse row a - R + t
    const int tr0 = ra0 - R - r0w;
    float m = M, mc = M * c, s_it = 0.f, sy_it = 0.f;
    const float kill = ok ? 0.f : -3.0e38f;
    // a window holds a handful of rows: the shifting register window (small code, 64 registers) beats the rotating
    // one of fwd_strip here (measured: 0.185 vs 0.201 ms per 768 frames; the dense CTA kernel is the other way round)
    float tmp[W];
#pragma unroll
    for (int t = 0; t < W; ++t) tmp[t] = dot_w<W>(colbase + (tr0 + t) * DECW_WP, wc);
    float yrow = (float)(ra0 * F);
    for (int a = ra0; a <= ra1; ++a, yrow += (float)F) {
      f32x2 v2[F / 2];
      column_pass<DS>(P, a, h, tmp, v2);
      softmax_row<DS>(v2, yrow, c, kill, m, mc, s_it, sy_it);
      if (a < ra1) {
#pragma unroll
        for (int t = 0; t < W - 1; ++t) tmp[t] = tmp[t + 1];
        tmp[W - 1] = dot_w<W>(colbase + (tr0 + (a - ra0) + 1 + 2 * R) * DECW_WP, wc);
      }
    }
    {
      const float Mn = fmaxf(M, m);
      const float a1 = fast_exp2((M - Mn) * c), a2 = fast_exp2((m - Mn) * c);
      S = fmaf(s_it, a2, S * a1);
      SX = fmaf((float)jf * s_it, a2, SX * a1);
      SY = fmaf(sy_it, a2, SY * a1);
      M = Mn;
    }
  }
  {
    const float Mw = warp_max(M);
    const float sc = fast_exp2((M - Mw) * c);
    S = warp_sum(S * sc);
    SX = warp_sum(SX * sc);
    SY = warp_sum(SY * sc);
    M = Mw;
  }
  const float xhat = SX / S, yhat = SY / S;

  // ---- confidence: softmax mass of the (2r+1)^2 window around (trunc y, trunc x) -----------------
  constexpr int CW = 2 * DEC_CONF_R + 1;
  float cw = 0.f;
  if (lane < CW * CW) {
    const int i = (int)yhat + lane / CW - DEC_CONF_R;
    const int j = (int)xhat + lane % CW - DEC_CONF_R;
    const int tr = i / F - R - r0w, tc = j / F - R - c0w;  // footprint inside the window by construction; guard anyway
    if (i >= 0 && i < h * F && j >= 0 && j < w * F && tr >= 0 && tr + W <= DECW_WIN && tc >= 0 && tc + W <= DECW_WIN) {
      const float v = eval_point_win<DS>(tile, r0w, c0w, P.tabH, P.tabW, i, j);
      cw = fast_exp2((v - M) * c) / S;
    }
  }
  cw = warp_sum(cw);
  if (lane == 0) {
    P.xy[2 * plane + 0] = xhat - P.offset;
    P.xy[2 * plane + 1] = yhat - P.offset;
    P.conf[plane] = cw;
    if (P.stats) {
      float* st = P.stats + 8 * plane;
      st[0] = M;
      st[1] = S;
      st[2] = xhat;
      st[3] = yhat;
      st[4] = (float)A0;
      st[5] = (float)A1;
      st[6] = (float)B0;
      st[7] = (float)B1;
    }
  }
}

template <int DS, bool BULK>
__global__ void __launch_bounds__(128) decode_fwd_warp_kernel(const __grid_constant__ DecodeParams<DS> P) {
  __shared__ float tile_s[4][DECW_WIN * DECW_WP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int plane = blockIdx.x * 4 + warp;  // n_planes < 2^31 (lpb_decode_fwd); the queue holds int plane ids as well
  if (plane >= P.n_planes) return;
  decode_plane_warp<DS, BULK>(P, plane, P.heat + (size_t)plane * P.h * P.w, tile_s[warp], P.queue, lane);
}

// d loss / d h = U_H^T G U_W with G[i,j] = T * p[i,j] * ((j - xhat) gx + (i - yhat) gy), p the
// temperature softmax.  G is non-negligible only inside the box saved by the forward pass; each warp
// recomputes the field on its strip exactly as the forward does and scatters G through the same taps
// into a zero-initialised smem gradient plane, which is then written out with coalesced stores.
template <int DS>
struct DecodeBwdParams : DecodeGeom<DS> {
  const float* stats;
  const float* gxy;
  float* gheat;
  const int* queue;      // optional {count, plane ids...}: dense fallback units of the window path
};

// Transposed horizontal pass for one coarse row of one 32-fine-column strip: out[oc] = sum_jj gv[jj] * tabW[jj][oc - jj/F]
// over the strip's fine columns jj, for the NOUT = 32/F + W - 1 coarse columns the strip touches.  Every lane drops its
// gv = (U_H^T G)[row][jj] into a 32-float row buffer in shared memory; the output columns then GATHER: lane (oc, part) reads
// 16 consecutive values (four 16-byte loads) and multiplies them with weights it fetched once per strip (`ScatterPlan`),
// the two parts of a column meet in one shuffle, and the row costs ONE shared-memory update per output column.  (The
// first version reduced the F lanes of a coarse column with shuffles, tap by tap: 27 shuffles + 36 adds per row, the
// largest share of the backward's instructions in the round-2 capture.)
template <int DS>
struct ScatterPlan {
  static constexpr int F = 1 << DS, W = 2 * (DS + 2) + 1, NG = 32 / F, NOUT = NG + W - 1, SPLIT = NOUT <= 16 ? 2 : 1;
  float wt[16];  // weight of fine column jstart + i for this lane's output column (0 outside the band / the strip)
  int oc, jstart;
  bool writer;
  __device__ __forceinline__ void init(const DecodeGeom<DS>& g, int jf0, int J1, int lane) {
    const int part = SPLIT == 2 ? (lane & 1) : 0;
    oc = SPLIT == 2 ? (lane >> 1) : lane;
    if (SPLIT == 2) {
      jstart = 16 * part;
    } else {
      int js = ((oc - (W - 1)) * F) & ~3;
      jstart = js < 0 ? 0 : (js > 16 ? 16 : js);
    }
    writer = oc < NOUT && part == 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int jj = jstart + i, u = oc - jj / F;
      wt[i] = (oc < NOUT && u >= 0 && u < W && jf0 + jj < J1) ? __ldg(g.tabW + (size_t)(jf0 + jj) * W + u) : 0.f;
    }
  }
};

template <int DS>
__device__ __forceinline__ void scatter_row(float* grow0, float gv, const ScatterPlan<DS>& sp, float* srow, int lane, int maxcols) {
  srow[lane] = gv;
  __syncwarp();
  const float4* s4 = reinterpret_cast<const float4*>(srow + sp.jstart);
  f32x2 acc2 = pack2(0.f, 0.f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 x = s4[i];
    acc2 = fma2(pack2(x.x, x.y), pack2(sp.wt[4 * i], sp.wt[4 * i + 1]), acc2);
    acc2 = fma2(pack2(x.z, x.w), pack2(sp.wt[4 * i + 2], sp.wt[4 * i + 3]), acc2);
  }
  float lo, hi;
  unpack2(acc2, lo, hi);
  float acc = lo + hi;
  if (ScatterPlan<DS>::SPLIT == 2) acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (sp.writer && sp.oc < maxcols && acc != 0.f) grow0[sp.oc] += acc;
}

// One strip (32 fine columns starting at fine column jf0, a multiple of F) over coarse rows [r0, r1): evaluates the
// softmax weights of the fine field and accumulates U_H^T G U_W into gt.  `tile` / `gt` are addressed as
// row * pitch + column with (trow0, tcol0) the tile coordinates of coarse row r0 - R and of coarse column jf0/F - R.
template <int DS>
__device__ __forceinline__ void decode_bwd_strip(const DecodeGeom<DS>& P, const float* tile, float* gt, int pitch,
                                                 int trow0, int tcol0, int maxcols, int jf0, int J1, int r0, int r1, float M,
                                                 float c, float kscale, float xhat, float yhat, float gx, float gy, int lane,
                                                 float* srow) {
  constexpr int F = 1 << DS, R = DS + 2, W = 2 * R + 1, HP = F / 2;
  const int h = P.h;
  const int jf = jf0 + lane;
  const bool ok = jf < J1;
  const int jc = ok ? jf : (J1 - 1);
  float wc[W];
#pragma unroll
  for (int t = 0; t < W; ++t) wc[t] = __ldg(P.tabW + jc * W + t);
  const float* colbase = tile + tcol0 + (jc / F - jf0 / F);
  ScatterPlan<DS> sp;
  sp.init(P, jf0, J1, lane);
  // Register windows over the W coarse rows a-R .. a+R that the fine rows of coarse row a touch.  They are ROTATED, not
  // shifted: the row loop is unrolled W times and in its `rot`-th copy tap t lives in slot (t + rot) % W, so advancing a
  // row costs no register moves.  The F phases are processed as pairs (packed fp32, lpb_common.cuh): `gacc[slot]` holds
  // the even-phase sum in its low half and the odd-phase sum in its high half.
  float tmp[W];   // horizontal pass of h
  f32x2 gacc[W];  // vertical-transpose accumulators: sum_i wr[i][t] * G[i][j]
#pragma unroll
  for (int t = 0; t < W; ++t) {
    tmp[t] = dot_w<W>(colbase + (trow0 + t) * pitch, wc);
    gacc[t] = pack2(0.f, 0.f);
  }
  const f32x2 ks2 = dup2(ok ? kscale : 0.f), c2 = dup2(c), nM2 = dup2(-M), nyh2 = dup2(-yhat), gx2 = dup2(gx), gy2 = dup2(gy);
  const f32x2 dx2 = dup2((float)jf - xhat);
  const int nrows = r1 - r0, nemit = nrows + W - 1;  // the last W-1 emissions flush the partial rows r1-R .. r1+R-1
  for (int la0 = 0; la0 < nemit; la0 += W) {
    static_for<0, W>([&](auto rot_c) {
      constexpr int rot = decltype(rot_c)::value;
      const int la = la0 + rot;
      if (la >= nemit) return;  // warp-uniform
      if (la < nrows) {
        const int a = r0 + la;
        const float af = (float)(a * F);
        // one pair of phases (2q, 2q+1) with vertical taps w(t) = {wr[2q][t], wr[2q+1][t]}
        auto phase_pair = [&](int q, auto&& w) {
          f32x2 v2 = pack2(0.f, 0.f);
#pragma unroll
          for (int t = 0; t < W; ++t) v2 = fma2(w(t), dup2(tmp[(t + rot) % W]), v2);
          float e0, e1;
          unpack2(mul2(add2(v2, nM2), c2), e0, e1);
          const f32x2 pr2 = pack2(fast_exp2(e0), fast_exp2(e1));
          const f32x2 y2 = add2(pack2(af + (float)(2 * q), af + (float)(2 * q + 1)), nyh2);
          const f32x2 lin2 = fma2(dx2, gx2, mul2(y2, gy2));
          const f32x2 g2 = mul2(mul2(ks2, pr2), lin2);
#pragma unroll
          for (int t = 0; t < W; ++t) gacc[(t + rot) % W] = fma2(w(t), g2, gacc[(t + rot) % W]);
        };
        if (a >= R && a <= h - 1 - R) {  // interior: phase-periodic weights are kernel-parameter constants
#pragma unroll
          for (int q = 0; q < HP; ++q) phase_pair(q, [&](int t) { return pack2(P.phase2[q][t].x, P.phase2[q][t].y); });
        } else {  // border rows: per-row table
          const float* __restrict__ tr = P.tabH + (size_t)a * F * W;
#pragma unroll
          for (int q = 0; q < HP; ++q) {
            f32x2 wr[W];
#pragma unroll
            for (int t = 0; t < W; ++t) wr[t] = pack2(__ldg(tr + (2 * q) * W + t), __ldg(tr + (2 * q + 1) * W + t));
            phase_pair(q, [&](int t) { return wr[t]; });
          }
        }
      }
      // coarse row r0 + la - R is complete for this lane's column
      float lo, hi;
      unpack2(gacc[rot], lo, hi);
      scatter_row<DS>(gt + (trow0 + la) * pitch + tcol0, lo + hi, sp, srow + 32 * (la & 1), lane, maxcols);
      gacc[rot] = pack2(0.f, 0.f);
      tmp[rot] = (la + 1 < nrows) ? dot_w<W>(colbase + (trow0 + la + 1 + 2 * R) * pitch, wc) : 0.f;
    });
  }
}

// Dense form: one CTA per plane (grid = n_planes), or -- queue mode -- per (plane, row segment) unit of the planes
// the window kernel could not take.  Every gradient element is a sum in a fixed order, with no atomics, so this gradient
// (and the windows' overflow planes, which it writes) has the same bits from call to call:
//   * inside a CTA, the work items (32-column strip, row group) run in phases of a barrier each, and the items of one
//     phase touch disjoint gradient elements; so each element receives its items' adds in phase order;
//   * a queue-mode segment owns a band of gradient rows, evaluates the R coarse rows either side of the band as well
//     (the rows whose taps reach it), and stores only its band: one writer per element, no scratch.
constexpr int DEC_BWD_SEGS = 8;

template <int DS>
__global__ void __launch_bounds__(DEC_THREADS) decode_bwd_kernel(const __grid_constant__ DecodeBwdParams<DS> P) {
  constexpr int F = 1 << DS, R = DS + 2;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int h = P.h, w = P.w, pitch = P.pitch, padl = P.padl;
  const int tile_floats = (h + 2 * R) * pitch;
  float* tile = reinterpret_cast<float*>(smem_raw);
  float* gtile = tile + tile_floats;  // same padded geometry, accumulates U_H^T G U_W
  float* srows = gtile + tile_floats;  // [DEC_WARPS][2][32] row buffers of the transposed horizontal pass
  uint64_t* bar = reinterpret_cast<uint64_t*>(srows + DEC_WARPS * 64);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (P.bulk) {
    if (tid == 0) {
      mbar_init(bar, 1);
      fence_mbar_init();
    }
    __syncthreads();
  }
  uint32_t phase = 0;
  // queue mode: a few left-over planes are split into row segments so that every resident CTA has work; when the queue
  // alone fills the grid (flat heatmaps of a freshly initialised network: every plane is dense) a unit is a whole plane
  const int nseg = P.queue ? max(1, min(DEC_BWD_SEGS, (int)gridDim.x / max(P.queue[0], 1))) : 1;
  const long long nunits = P.queue ? (long long)P.queue[0] * nseg : P.n_planes;
  for (long long unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
    const size_t plane = P.queue ? (size_t)P.queue[1 + unit / nseg] : (size_t)unit;
    const float* st = P.stats + 8 * plane;
    const float M = st[0], S = st[1], xhat = st[2], yhat = st[3];
    const int A0 = (int)st[4], A1 = (int)st[5], B0 = (int)st[6], B1 = (int)st[7];
    const float gx = P.gxy[2 * plane], gy = P.gxy[2 * plane + 1];
    const int nrows = A1 - A0 + 1;
    int own0 = 0, own1 = h;          // gradient rows this unit stores
    int useg0 = A0, useg1 = A1 + 1;  // coarse rows it evaluates
    if (nseg > 1) {  // segment k owns the rows from the start of its share of [A0, A1] to the next share's start
      const int sg = (nrows + nseg - 1) / nseg, k = (int)(unit % nseg);
      if (k * sg >= nrows) continue;  // uniform per CTA; an empty share owns no rows (nor does a plane with none)
      own0 = k == 0 ? 0 : A0 + k * sg;
      own1 = (k + 1) * sg >= nrows ? h : A0 + (k + 1) * sg;
      useg0 = max(A0, own0 - R);
      useg1 = min(A1 + 1, own1 + R);
    }
    const float* __restrict__ src = P.heat + plane * (size_t)h * w;
    if (P.bulk) {
      if (warp == 0) {
        if (lane == 0) mbar_expect_tx(bar, (uint32_t)(h * w * 4));
        __syncwarp();
        for (int a = lane; a < h; a += 32)
          bulk_g2s(tile + (a + R) * pitch + padl, src + (size_t)a * w, (uint32_t)(w * 4), bar);
      }
    }
    for (int i = tid; i < tile_floats; i += DEC_THREADS) gtile[i] = 0.f;
    for (int r = warp; r < h + 2 * R; r += DEC_WARPS) {
      float* row = tile + r * pitch;
      if (r < R || r >= h + R) {
        for (int b = lane; b < pitch; b += 32) row[b] = 0.f;
      } else {
        for (int b = lane; b < padl; b += 32) row[b] = 0.f;
        for (int b = padl + w + lane; b < pitch; b += 32) row[b] = 0.f;
        if (!P.bulk) {
          const float* g = src + (size_t)(r - R) * w;
          for (int b = lane; b < w; b += 32) row[padl + b] = __ldg(g + b);
        }
      }
    }
    if (P.bulk) {
      mbar_wait(bar, phase);
      phase ^= 1;
    }
    __syncthreads();

    const float c = P.T * 1.4426950408889634f;
    const float kscale = P.T / S;
    if (gx != 0.f || gy != 0.f) {
      const int J0 = B0 * F, J1 = (B1 + 1) * F;
      const int nstrips = (J1 - J0 + 31) >> 5;
      const int urows = useg1 - useg0;
      // Items (strip, row group): a strip adds into 32/F + 2R coarse columns, 32/F apart, so strips NCS apart are
      // disjoint; a group of sg rows adds into sg + 2R rows, so groups ncg apart are.  Phase (cs, cg) runs the strips
      // cs (mod NCS) of the groups cg (mod ncg), and a barrier ends it.  The rows are split into G groups so that all
      // warps have items, at the least cost over the phases.
      constexpr int NG = 32 / F, NCS = (NG + 2 * R + NG - 1) / NG;
      auto ncolours = [&](int g, int sg) { return min(g, 1 + (2 * R + sg - 1) / sg); };
      auto phase_items = [&](int n, int nc, int c) { return (n - c + nc - 1) / nc; };
      int G = 1, seg = urows, ncg = 1;
      {
        int bestcost = 0x7fffffff;
        for (int g = 1; g <= 8; ++g) {
          const int sg = (urows + g - 1) / g, nc = ncolours(g, sg);
          int rounds = 0;
          for (int cs = 0; cs < NCS; ++cs)
            for (int cg = 0; cg < nc; ++cg) rounds += (phase_items(nstrips, NCS, cs) * phase_items(g, nc, cg) + DEC_WARPS - 1) / DEC_WARPS;
          const int cost = rounds * (sg + 2 * R);
          if (cost < bestcost) {
            bestcost = cost;
            G = g;
            seg = sg;
            ncg = nc;
          }
        }
      }
      for (int cs = 0; cs < NCS; ++cs)
        for (int cg = 0; cg < ncg; ++cg) {
          const int ns = phase_items(nstrips, NCS, cs), nitems = ns * phase_items(G, ncg, cg);
          for (int item = warp; item < nitems; item += DEC_WARPS) {
            const int sidx = cs + NCS * (item % ns), g = cg + ncg * (item / ns);
            const int r0 = useg0 + g * seg, r1 = min(r0 + seg, useg1);
            if (r0 >= r1) continue;
            const int jf0 = J0 + sidx * 32;
            const int tcol0 = padl + (jf0 / F - R);
            decode_bwd_strip<DS>(P, tile, gtile, pitch, r0, tcol0, pitch - tcol0, jf0, J1, r0, r1, M, c, kscale, xhat, yhat, gx, gy, lane,
                                 srows + warp * 64);
          }
          __syncthreads();
        }
    }
    __syncthreads();
    float* __restrict__ dst = P.gheat + plane * (size_t)h * w;
    for (int a = own0 + warp; a < own1; a += DEC_WARPS) {
      const float* row = gtile + (a + R) * pitch + padl;
      for (int b = lane; b < w; b += 32) dst[(size_t)a * w + b] = row[b];
    }
    __syncthreads();  // tile / gtile are reused by the next unit
  }
}

// ------------------------------------------------------------------------------------------------
// Sparse form of the decode backward.  With T = 1000 the softmax weights vanish a few fine pixels away from
// the peak, so d loss / d heatmap is supported on the forward pass's candidate box dilated by the R-tap halo:
// a window of at most DEC_WIN x DEC_WIN coarse pixels instead of the whole plane.  One warp per plane loads that
// window straight from global memory, runs the same transpose-of-the-upsample accumulation as decode_bwd_kernel
// and emits   win[plane][32][32], meta[plane] = {row0, col0, flag, bits(sum(win * heat))}
// flag 0: zero gradient, 1: window valid, 2: the box does not fit: the plane is queued for decode_bwd_kernel's
// queue mode and its dense gradient (cleared here) goes to P.gheat.
constexpr int DEC_WIN = 32, DEC_WP = 33;

template <int DS>
__global__ void __launch_bounds__(128) decode_bwd_window_kernel(const __grid_constant__ DecodeBwdParams<DS> P, float* __restrict__ win,
                                                                int* __restrict__ meta, int* __restrict__ queue) {
  constexpr int F = 1 << DS, R = DS + 2;
  __shared__ float tile_s[4][DEC_WIN * DEC_WP];
  __shared__ float g_s[4][DEC_WIN * DEC_WP];
  __shared__ __align__(16) float srow_s[4][64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long plane = (long long)blockIdx.x * 4 + warp;
  if (plane >= P.n_planes) return;
  const int h = P.h, w = P.w;
  const float gx = P.gxy[2 * plane], gy = P.gxy[2 * plane + 1];
  int4* mout = reinterpret_cast<int4*>(meta) + plane;
  if (gx == 0.f && gy == 0.f) {
    if (lane == 0) *mout = make_int4(0, 0, 0, 0);
    return;
  }
  const float* st = P.stats + 8 * plane;
  const float M = st[0], S = st[1], xhat = st[2], yhat = st[3];
  const int A0 = (int)st[4], A1 = (int)st[5], B0 = (int)st[6], B1 = (int)st[7];
  const int nrows = A1 - A0 + 1, ncols = B1 - B0 + 1;
  if (nrows > DEC_WIN - 2 * R || ncols > DEC_WIN - 2 * R || nrows < 1 || ncols < 1) {
    if (lane == 0) {
      *mout = make_int4(0, 0, 2, 0);
      queue[1 + atomicAdd(queue, 1)] = (int)plane;
    }
    float* dst = P.gheat + (size_t)plane * h * w;
    for (int i = lane; i < h * w; i += 32) dst[i] = 0.f;
    return;
  }
  float* tile = tile_s[warp];
  float* gt = g_s[warp];
  const int r0w = A0 - R, c0w = B0 - R;
  const float* __restrict__ src = P.heat + (size_t)plane * h * w;
  {
    const int x = c0w + lane;
    const bool xin = x >= 0 && x < w;
#pragma unroll 8
    for (int r = 0; r < DEC_WIN; ++r) {
      const int y = r0w + r;
      tile[r * DEC_WP + lane] = (xin && y >= 0 && y < h) ? __ldg(src + (size_t)y * w + x) : 0.f;
      gt[r * DEC_WP + lane] = 0.f;
    }
  }
  __syncwarp();
  // Tighten the row range.  The forward's box is "a candidate within R samples" (global Lipschitz bound); with the
  // window in shared memory the decay of the taps can be used: for a fine pixel in coarse row a,
  //   |field| <= lipW * sum_t wabs[t] * rowmax[a - R + t]      (rowmax over the window's columns = the strips' footprint)
  // and rows whose bound is below M - CUT/T carry weight < exp(-CUT) of the peak.  Lane r owns window row r.
  int ra0 = A0, ra1 = A1;
  if (P.T > 0.f) {
    float rmx = 0.f;
#pragma unroll 8
    for (int cc = 0; cc < DEC_WIN; ++cc) rmx = fmaxf(rmx, fabsf(tile[lane * DEC_WP + cc]));
    float bnd = 0.f;
#pragma unroll
    for (int t = 0; t < 2 * R + 1; ++t) {
      const int src = lane - R + t;
      const float v = __shfl_sync(0xffffffffu, rmx, src & 31);
      if ((unsigned)src < (unsigned)DEC_WIN) bnd = fmaf(P.wabs[t], v, bnd);
    }
    const bool act = lane >= R && lane < R + nrows && bnd * P.lipw >= M - DEC_CUT / P.T;
    const unsigned am = __ballot_sync(0xffffffffu, act);
    if (am) {
      ra0 = A0 + (__ffs(am) - 1 - R);
      ra1 = A0 + (31 - __clz(am) - R);
    }
  }
  const float c = P.T * 1.4426950408889634f;
  const float kscale = P.T / S;
  const int J0 = B0 * F, J1 = (B1 + 1) * F;
  const int nstrips = (J1 - J0 + 31) >> 5;
  for (int sidx = 0; sidx < nstrips; ++sidx) {
    const int jf0 = J0 + sidx * 32;
    const int tcol0 = jf0 / F - B0;  // window column of coarse column jf0/F - R
    decode_bwd_strip<DS>(P, tile, gt, DEC_WP, ra0 - A0, tcol0, DEC_WIN - tcol0, jf0, J1, ra0, ra1 + 1, M, c, kscale, xhat, yhat, gx,
                                gy, lane, srow_s[warp]);
    __syncwarp();
  }
  float dot = 0.f;
  float* wout = win + (size_t)plane * (DEC_WIN * DEC_WIN);
#pragma unroll 8
  for (int r = 0; r < DEC_WIN; ++r) {
    const float g = gt[r * DEC_WP + lane];
    dot = fmaf(g, tile[r * DEC_WP + lane], dot);
    wout[r * DEC_WIN + lane] = g;
  }
  dot = warp_sum(dot);
  if (lane == 0) *mout = make_int4(r0w, c0w, 1, __float_as_int(dot));
}

// One materialised upsampling stage (drop-in for `upsample`, lightning_pose/models/heads/heatmap.py:86-100).
// Not on the fused path (the decode never materialises the field); kept for API completeness.
__global__ void __launch_bounds__(DEC_THREADS) upsample2x_kernel(const float* __restrict__ in, int h, int w, int pitch,
                                                                 int padl, const float* __restrict__ tabH,
                                                                 const float* __restrict__ tabW, float* __restrict__ out) {
  constexpr int R = 3;
  extern __shared__ __align__(16) float ups_tile[];
  const size_t plane = blockIdx.x;
  const float* __restrict__ src = in + plane * (size_t)h * w;
  for (int i = threadIdx.x; i < (h + 2 * R) * pitch; i += DEC_THREADS) {
    const int r = i / pitch - R, c = i % pitch - padl;
    ups_tile[i] = (r >= 0 && r < h && c >= 0 && c < w) ? __ldg(src + (size_t)r * w + c) : 0.f;
  }
  __syncthreads();
  float* __restrict__ dst = out + plane * (size_t)(4 * h * w);
  for (int o = threadIdx.x; o < 4 * h * w; o += DEC_THREADS) {
    const int i = o / (2 * w), j = o - i * (2 * w);
    dst[o] = eval_point<1>(ups_tile, pitch, padl, tabH, tabW, i, j);
  }
}

// ------------------------------------------------------------------------------------------------
// Fills what both directions share.  lip (forward): Lipschitz bound of the 2-D upsampling.
template <int DS>
static int decode_geom(DecodeGeom<DS>& g, const float* heat, int64_t n_planes, int h, int w, float T, float* lip = nullptr) {
  using G = UpsampleGeom<DS>;
  const DeviceTable* th = get_device_table(h, DS);
  const DeviceTable* tw = get_device_table(w, DS);
  if (!th || !tw) return LPB_ERR_INVALID;
  g.heat = heat;
  g.tabH = th->win;
  g.tabW = tw->win;
  g.h = h;
  g.w = w;
  g.padl = dec_padl(G::R);
  g.pitch = dec_pitch(w, G::R);
  g.bulk = ((w % 4) == 0 && aligned_to(heat, 16)) ? 1 : 0;
  g.n_planes = n_planes;
  g.T = T;
  g.lipw = tw->host.lip;
  for (int t = 0; t < G::W; ++t) {
    float m = 0.f;
    for (size_t i = 0; i < (size_t)h * G::F; ++i) m = std::fmax(m, std::fabs(th->host.win[i * G::W + t]));
    g.wabs[t] = m * (1.0f + 1e-6f);
  }
  for (int q = 0; q < G::F / 2; ++q)
    for (int t = 0; t < G::W; ++t)
      g.phase2[q][t] = make_float2(th->host.phase[(size_t)(2 * q) * G::W + t], th->host.phase[(size_t)(2 * q + 1) * G::W + t]);
  if (lip) *lip = th->host.lip * tw->host.lip;
  return LPB_OK;
}

// forward workspace: {queue count, queued plane ids}[1 + n] and arrival counters[n] (ints, zeroed by every call), then the
// partial softmax states of split planes, float[n][DEC_MAX_PARTS][4]
static size_t decode_fwd_workspace_bytes(int64_t n_planes) {
  return sizeof(int) * (size_t)(2 * n_planes + 1) + sizeof(float) * (size_t)n_planes * DEC_MAX_PARTS * 4;
}

template <int DS>
static int launch_decode_fwd(const float* heat, int64_t n_planes, int h, int w, float T, float* xy, float* conf,
                             float* stats, void* workspace, cudaStream_t stream) {
  using G = UpsampleGeom<DS>;
  DecodeParams<DS> P;
  DeviceLimits dev;
  LPB_TRY(decode_geom<DS>(P, heat, n_planes, h, w, T, &P.lip));
  LPB_TRY(device_limits(&dev));
  P.xy = xy;
  P.conf = conf;
  P.stats = stats;
  P.offset = (DS == 1) ? 0.5f : (DS == 2 ? 1.5f : 2.5f);  // lightning_pose/models/heads/heatmap.py:131-136
  P.queue = static_cast<int*>(workspace);
  P.qcounter = P.queue + 1 + n_planes;
  P.qscratch = reinterpret_cast<float*>(P.queue + 1 + 2 * n_planes);
  const size_t smem = ((size_t)(h + 2 * G::R) * P.pitch + DEC_FWD_SCRATCH) * sizeof(float) + 16;
  LPB_TRY(set_dynamic_smem(decode_fwd_kernel<DS>, smem, "decode_fwd"));
  int per_sm = 0;
  LPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_fwd_kernel<DS>, DEC_THREADS, smem));
  const int64_t resident = (int64_t)dev.sms * (per_sm > 0 ? per_sm : 1);  // persistent CTAs: one wave
  // warp per plane first; what it cannot take (diffuse / multi-modal / NaN planes) is queued for the CTA kernel
  LPB_CUDA(cudaMemsetAsync(P.queue, 0, sizeof(int) * (size_t)(2 * n_planes + 1), stream));
  const unsigned wgrid = (unsigned)((n_planes + 3) / 4);
  if (P.bulk) decode_fwd_warp_kernel<DS, true><<<wgrid, 128, 0, stream>>>(P);
  else decode_fwd_warp_kernel<DS, false><<<wgrid, 128, 0, stream>>>(P);
  decode_fwd_kernel<DS><<<(unsigned)(n_planes < resident ? n_planes : resident), DEC_THREADS, smem, stream>>>(P);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

template <int DS>
static int launch_decode_bwd(const float* heat, const float* stats, const float* gxy, int64_t n_planes, int h, int w,
                             float T, float* gheat, cudaStream_t stream, float* win = nullptr, int* meta = nullptr,
                             int* queue = nullptr) {
  using G = UpsampleGeom<DS>;
  DecodeBwdParams<DS> P;
  DeviceLimits dev;
  LPB_TRY(decode_geom<DS>(P, heat, n_planes, h, w, T));
  LPB_TRY(device_limits(&dev));
  P.stats = stats;
  P.gxy = gxy;
  P.gheat = gheat;
  P.queue = queue;
  if (win) {  // sparse windows first; the dense kernel below then only runs the planes they queued
    LPB_CUDA(cudaMemsetAsync(queue, 0, sizeof(int), stream));
    decode_bwd_window_kernel<DS><<<(unsigned)((n_planes + 3) / 4), 128, 0, stream>>>(P, win, meta, queue);
  }
  const size_t smem = ((size_t)2 * (h + 2 * G::R) * P.pitch + DEC_WARPS * 64) * sizeof(float) + 16;
  LPB_TRY(set_dynamic_smem(decode_bwd_kernel<DS>, smem, "decode_bwd"));
  unsigned grid = (unsigned)n_planes;
  if (queue && grid > (unsigned)(2 * dev.sms)) grid = (unsigned)(2 * dev.sms);  // queue mode: one wave of resident CTAs
  decode_bwd_kernel<DS><<<grid, DEC_THREADS, smem, stream>>>(P);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

}  // namespace lpb

extern "C" int lpb_decode_prepare(int h, int w, int ds) {
  using namespace lpb;
  LPB_REQUIRE(h >= 1 && w >= 1 && ds >= 1 && ds <= 3, "decode_prepare: bad shape h=%d w=%d ds=%d", h, w, ds);
  if (!get_device_table(h, ds) || !get_device_table(w, ds)) return LPB_ERR_INVALID;
  return LPB_OK;
}

extern "C" int lpb_decode_fwd_workspace_bytes(int64_t n_planes, size_t* bytes) {
  using namespace lpb;
  LPB_REQUIRE(bytes, "decode_fwd_workspace_bytes: null pointer");
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "decode_fwd_workspace_bytes: bad n_planes");
  *bytes = decode_fwd_workspace_bytes(n_planes);
  return LPB_OK;
}

extern "C" int lpb_decode_fwd(const float* heatmaps, int64_t n_planes, int h, int w, int ds, float temperature,
                              float* xy, float* conf, float* stats, void* workspace, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && xy && conf, "decode_fwd: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && ds >= 1 && ds <= 3, "decode_fwd: bad shape h=%d w=%d ds=%d", h, w, ds);
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "decode_fwd: bad n_planes");
  LPB_REQUIRE(workspace || n_planes == 0, "decode_fwd: null workspace");
  LPB_REQUIRE(aligned_to(workspace, 4), "decode_fwd: workspace must be 4-byte aligned");
  if (((int64_t)w << ds) > 1024 || w > 256) {
    lpb::set_error("decode_fwd: heatmap width %d (x%d) exceeds this build's 1024-column field limit", w, 1 << ds);
    return LPB_ERR_UNSUPPORTED;
  }
  if (n_planes == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (ds) {
    case 1: return launch_decode_fwd<1>(heatmaps, n_planes, h, w, temperature, xy, conf, stats, workspace, s);
    case 2: return launch_decode_fwd<2>(heatmaps, n_planes, h, w, temperature, xy, conf, stats, workspace, s);
    default: return launch_decode_fwd<3>(heatmaps, n_planes, h, w, temperature, xy, conf, stats, workspace, s);
  }
}

extern "C" int lpb_decode_bwd(const float* heatmaps, const float* stats, const float* grad_xy, int64_t n_planes, int h,
                              int w, int ds, float temperature, float* grad_heatmaps, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && stats && grad_xy && grad_heatmaps, "decode_bwd: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && ds >= 1 && ds <= 3, "decode_bwd: bad shape h=%d w=%d ds=%d", h, w, ds);
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "decode_bwd: bad n_planes");
  if (n_planes == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (ds) {
    case 1: return launch_decode_bwd<1>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, grad_heatmaps, s);
    case 2: return launch_decode_bwd<2>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, grad_heatmaps, s);
    default: return launch_decode_bwd<3>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, grad_heatmaps, s);
  }
}

extern "C" int lpb_decode_bwd_windows(const float* heatmaps, const float* stats, const float* grad_xy, int64_t n_planes, int h,
                                      int w, int ds, float temperature, float* win, int32_t* meta, float* g_overflow,
                                      int32_t* queue, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(heatmaps && stats && grad_xy && win && meta && g_overflow && queue, "decode_bwd_windows: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && ds >= 1 && ds <= 3, "decode_bwd_windows: bad shape h=%d w=%d ds=%d", h, w, ds);
  LPB_REQUIRE(n_planes >= 0 && n_planes < (1ll << 31), "decode_bwd_windows: bad n_planes");
  if (n_planes == 0) return LPB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (ds) {
    case 1: return launch_decode_bwd<1>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, g_overflow, s, win, meta, queue);
    case 2: return launch_decode_bwd<2>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, g_overflow, s, win, meta, queue);
    default: return launch_decode_bwd<3>(heatmaps, stats, grad_xy, n_planes, h, w, temperature, g_overflow, s, win, meta, queue);
  }
}

extern "C" int lpb_upsample2x(const float* in, int64_t n_planes, int h, int w, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(in && out, "upsample2x: null pointer");
  LPB_REQUIRE(h >= 1 && w >= 1 && n_planes >= 0 && n_planes < (1ll << 31), "upsample2x: bad shape");
  if (n_planes == 0) return LPB_OK;
  const DeviceTable* th = get_device_table(h, 1);
  const DeviceTable* tw = get_device_table(w, 1);
  if (!th || !tw) return LPB_ERR_INVALID;
  const int padl = dec_padl(3), pitch = dec_pitch(w, 3);
  const size_t smem = (size_t)(h + 6) * pitch * sizeof(float);
  LPB_TRY(set_dynamic_smem(upsample2x_kernel, smem, "upsample2x"));
  upsample2x_kernel<<<(unsigned)n_planes, DEC_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(in, h, w, pitch, padl,
                                                                                                 th->win, tw->win, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
