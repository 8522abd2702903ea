// Coordinate-regression models: the pooled linear head (forward, both gradients) and the regression losses.
//
// Head: features (B, C, h, w) in bf16 / fp16 / fp32, NCHW or channels-last -> pooled (B, C) fp32, the mean over the h w
// pixels summed in a fixed order -> out = pooled W^T + b, (B, N) fp32.  Each feature byte is read once.  The backward
// writes dW and db as fixed-order sums over the batch (one thread owns one output, no float atomics), and d features
// = (g W) / (h w) broadcast over the pixels, written once in the dtype and layout of the features.
//
// Losses: the mean of (t - p)^2 over the non-NaN target entries, and the RMSE diagnostic of the reference, which
// compacts the kept entries before pairing them as (x, y): one CTA walks the entries in order with a block scan, so the
// pairing is the reference's and every sum has one order.
#include <cub/block/block_scan.cuh>

#include "lpb_common.cuh"

namespace lpb {
namespace {

template <typename T>
__device__ __forceinline__ float to_f32(T v) {
  if constexpr (std::is_same_v<T, __nv_bfloat16>) return __bfloat162float(v);
  else if constexpr (std::is_same_v<T, __half>) return __half2float(v);
  else return v;
}
template <typename T>
__device__ __forceinline__ T from_f32(float v) {
  if constexpr (std::is_same_v<T, __nv_bfloat16>) return __float2bfloat16_rn(v);
  else if constexpr (std::is_same_v<T, __half>) return __float2half_rn(v);
  else return v;
}
template <typename T, int V>
struct alignas(sizeof(T) * V) Pack {
  T v[V];
};

// frames are the grid's y axis, looped past the 65535 limit
constexpr int MAX_GRID_Y = 65535;
inline unsigned grid_y(int B) { return (unsigned)(B < MAX_GRID_Y ? B : MAX_GRID_Y); }
inline unsigned n_blocks(int64_t n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

// ---- pooling ----------------------------------------------------------------------------------------------------------
// Channels-last features (and any layout at h w = 1): one thread per (frame, V channels), pixels added in order.
constexpr int POOL_THREADS = 256;
template <typename T, int V>
__global__ void __launch_bounds__(POOL_THREADS) pool_channels_kernel(const T* __restrict__ x, int B, int C, int hw,
                                                                     float* __restrict__ pooled) {
  const int g = blockIdx.x * POOL_THREADS + threadIdx.x;
  if (g * V >= C) return;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const T* src = x + (size_t)b * hw * C + (size_t)g * V;
    float s[V];
#pragma unroll
    for (int j = 0; j < V; ++j) s[j] = 0.f;
#pragma unroll 4
    for (int p = 0; p < hw; ++p) {
      const Pack<T, V> q = *reinterpret_cast<const Pack<T, V>*>(src + (size_t)p * C);
#pragma unroll
      for (int j = 0; j < V; ++j) s[j] += to_f32(q.v[j]);
    }
#pragma unroll
    for (int j = 0; j < V; ++j) pooled[(size_t)b * C + g * V + j] = s[j] / (float)hw;
  }
}

// NCHW features with h w > 1: one warp per (frame, channel) row, ROWS rows per warp with their loads in flight together;
// lane l adds vectors l, l + 32, ... in order, then a fixed butterfly adds the lanes.
constexpr int ROWS_PER_WARP = 4, ROW_WARPS = 8;
template <typename T, int V>
__global__ void __launch_bounds__(ROW_WARPS * 32) pool_rows_kernel(const T* __restrict__ x, int B, int C, int hw,
                                                                   float* __restrict__ pooled) {
  const int lane = threadIdx.x & 31;
  const int c0 = (blockIdx.x * ROW_WARPS + (threadIdx.x >> 5)) * ROWS_PER_WARP;
  const int vecs = hw / V;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    float s[ROWS_PER_WARP];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
      s[r] = 0.f;
      if (c0 + r >= C) continue;
      const T* row = x + ((size_t)b * C + c0 + r) * hw;
      for (int i = lane; i < vecs; i += 32) {
        const Pack<T, V> q = *reinterpret_cast<const Pack<T, V>*>(row + (size_t)i * V);
#pragma unroll
        for (int j = 0; j < V; ++j) s[r] += to_f32(q.v[j]);
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
      const float t = warp_sum(s[r]);
      if (lane == 0 && c0 + r < C) pooled[(size_t)b * C + c0 + r] = t / (float)hw;
    }
  }
}

// ---- out = pooled W^T + b -----------------------------------------------------------------------------------------------
// A CTA owns 16 frames x 32 outputs; the channel sum runs in 32-wide steps, in order.
constexpr int LIN_BM = 16, LIN_BN = 32, LIN_BK = 32;
__global__ void __launch_bounds__(256) linear_fwd_kernel(const float* __restrict__ pooled, const float* __restrict__ w,
                                                         const float* __restrict__ bias, int B, int C, int N, float* __restrict__ out) {
  __shared__ float ps[LIN_BM][LIN_BK + 1], ws[LIN_BN][LIN_BK + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // output n0 + tx, frames b0 + ty and b0 + ty + 8
  const int b0 = blockIdx.x * LIN_BM, n0 = blockIdx.y * LIN_BN;
  float acc[2] = {0.f, 0.f};
  for (int k0 = 0; k0 < C; k0 += LIN_BK) {
    for (int i = threadIdx.x; i < LIN_BM * LIN_BK; i += 256) {
      const int r = i / LIN_BK, k = i % LIN_BK;
      ps[r][k] = (b0 + r < B && k0 + k < C) ? pooled[(size_t)(b0 + r) * C + k0 + k] : 0.f;
    }
    for (int i = threadIdx.x; i < LIN_BN * LIN_BK; i += 256) {
      const int r = i / LIN_BK, k = i % LIN_BK;
      ws[r][k] = (n0 + r < N && k0 + k < C) ? w[(size_t)(n0 + r) * C + k0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < LIN_BK; ++k) {
      const float wv = ws[tx][k];
      acc[0] = fmaf(ps[ty][k], wv, acc[0]);
      acc[1] = fmaf(ps[ty + 8][k], wv, acc[1]);
    }
    __syncthreads();
  }
  const int n = n0 + tx;
  if (n >= N) return;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int b = b0 + ty + 8 * i;
    if (b < B) out[(size_t)b * N + n] = acc[i] + bias[n];
  }
}

// ---- out[r, c] = scale * sum_s A(s, r) X[s, c], s in order --------------------------------------------------------------
// dW: s = frame, r = output (A = g, X = pooled), with column C of X read as ones: that column is db.
// d pooled: s = output, r = frame (A = g^T, X = W), scale 1 / (h w).
// A thread owns one column c and GR consecutive rows; A is staged through shared memory SCHUNK values of s at a time.
constexpr int CG_THREADS = 128, CG_ROWS = 8, CG_SCHUNK = 256;
__global__ void __launch_bounds__(CG_THREADS) colsum_kernel(const float* __restrict__ a, int64_t a_s, int64_t a_r, int S, int R,
                                                            const float* __restrict__ x, int C, int ones_col, float scale,
                                                            float* __restrict__ out, float* __restrict__ out_ones) {
  __shared__ float4 at[CG_SCHUNK][CG_ROWS / 4];
  const int r0 = blockIdx.x * CG_ROWS, c = blockIdx.y * CG_THREADS + threadIdx.x;
  const int ncol = C + ones_col;
  float acc[CG_ROWS];
#pragma unroll
  for (int j = 0; j < CG_ROWS; ++j) acc[j] = 0.f;
  for (int s0 = 0; s0 < S; s0 += CG_SCHUNK) {
    const int ns = S - s0 < CG_SCHUNK ? S - s0 : CG_SCHUNK;
    float* atf = reinterpret_cast<float*>(at);
    for (int i = threadIdx.x; i < CG_SCHUNK * CG_ROWS; i += CG_THREADS) {
      const int s = i / CG_ROWS, j = i % CG_ROWS;
      atf[i] = (s < ns && r0 + j < R) ? a[(s0 + s) * a_s + (int64_t)(r0 + j) * a_r] : 0.f;
    }
    __syncthreads();
    if (c < ncol) {
      for (int s = 0; s < ns; ++s) {
        const float xv = c < C ? x[(size_t)(s0 + s) * C + c] : 1.f;
        const float4 lo = at[s][0], hi = at[s][1];
        acc[0] = fmaf(lo.x, xv, acc[0]);
        acc[1] = fmaf(lo.y, xv, acc[1]);
        acc[2] = fmaf(lo.z, xv, acc[2]);
        acc[3] = fmaf(lo.w, xv, acc[3]);
        acc[4] = fmaf(hi.x, xv, acc[4]);
        acc[5] = fmaf(hi.y, xv, acc[5]);
        acc[6] = fmaf(hi.z, xv, acc[6]);
        acc[7] = fmaf(hi.w, xv, acc[7]);
      }
    }
    __syncthreads();
  }
  if (c >= ncol) return;
#pragma unroll
  for (int j = 0; j < CG_ROWS; ++j) {
    if (r0 + j >= R) break;
    if (c < C) out[(size_t)(r0 + j) * C + c] = acc[j] * scale;
    else out_ones[r0 + j] = acc[j] * scale;
  }
}

// ---- d features: d pooled (already / h w) broadcast over the pixels, V elements per store ------------------------------
template <typename T, int V, bool NHWC>
__global__ void __launch_bounds__(POOL_THREADS) broadcast_kernel(const float* __restrict__ dpool, int B, int C, int hw, T* __restrict__ dx) {
  const int per_frame = C * hw;
  const int e = (blockIdx.x * POOL_THREADS + threadIdx.x) * V;
  if (e >= per_frame) return;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float* dp = dpool + (size_t)b * C;
    Pack<T, V> q;
    if constexpr (NHWC) {
      const int c = e % C;  // V | C: the pack's channels are c .. c + V - 1
#pragma unroll
      for (int j = 0; j < V; ++j) q.v[j] = from_f32<T>(dp[c + j]);
    } else {
      const T v = from_f32<T>(dp[e / hw]);  // V | h w: the pack lies in one row
#pragma unroll
      for (int j = 0; j < V; ++j) q.v[j] = v;
    }
    *reinterpret_cast<Pack<T, V>*>(dx + (size_t)b * per_frame + e) = q;
  }
}

// ---- losses -------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
constexpr int RL_THREADS = 512;
__global__ void __launch_bounds__(RL_THREADS) regression_losses_fwd_kernel(const float* __restrict__ targ, const float* __restrict__ pred,
                                                                           int64_t n, float* __restrict__ out) {
  using Scan = cub::BlockScan<int, RL_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ float buf[RL_THREADS + 1];  // this chunk's kept squared errors, compacted, after the previous chunk's unpaired one
  __shared__ float carry;
  __shared__ double red[2][RL_THREADS / 32];
  const int tid = threadIdx.x;
  double sq = 0.0, root = 0.0;  // this thread's share of sum (t - p)^2 and of sum sqrt(pair mean)
  int64_t kept = 0;             // kept entries before the current chunk (the same in every thread)
  for (int64_t e0 = 0; e0 < n; e0 += RL_THREADS) {
    const int64_t e = e0 + tid;
    bool keep = false;
    float d2 = 0.f;
    if (e < n) {
      const float t = targ[e];
      keep = t == t;
      const float d = t - pred[e];
      d2 = d * d;
    }
    if (keep) sq += (double)d2;
    int rank, count;
    Scan(scan_tmp).ExclusiveSum(keep ? 1 : 0, rank, count);
    const int off = (int)(kept & 1);
    if (keep) buf[off + rank] = d2;
    if (off && tid == 0) buf[0] = carry;
    __syncthreads();
    const int m = off + count;
    if (tid < m / 2) root += (double)sqrtf((buf[2 * tid] + buf[2 * tid + 1]) / 2.f);
    if ((m & 1) && tid == 0) carry = buf[m - 1];
    kept += count;
    __syncthreads();
  }
  sq = warp_sum_d(sq);
  root = warp_sum_d(root);
  if ((tid & 31) == 0) red[0][tid >> 5] = sq, red[1][tid >> 5] = root;
  __syncthreads();
  if (tid == 0) {
    double s0 = 0.0, s1 = 0.0;
    for (int w = 0; w < RL_THREADS / 32; ++w) s0 += red[0][w], s1 += red[1][w];
    const int64_t pairs = kept / 2;
    out[0] = kept > 0 ? (float)(s0 / (double)kept) : __int_as_float(0x7fc00000);
    out[1] = (float)kept;
    out[2] = (kept > 0 && !(kept & 1)) ? (float)(s1 / (double)pairs) : __int_as_float(0x7fc00000);
    out[3] = (float)pairs;
  }
}

__global__ void __launch_bounds__(256) regression_losses_bwd_kernel(const float* __restrict__ targ, const float* __restrict__ pred, int64_t n,
                                                                    const float* __restrict__ fwd_out, const float* __restrict__ grad_out,
                                                                    float* __restrict__ grad_pred) {
  const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= n) return;
  const float t = targ[e], kept = fwd_out[1];
  grad_pred[e] = (t == t && kept > 0.f) ? grad_out[0] * 2.f * (pred[e] - t) / kept : 0.f;
}

// ---- launchers ----------------------------------------------------------------------------------------------------------
bool valid_format(int fmt) { return fmt == LPB_OUT_F32 || fmt == LPB_OUT_BF16 || fmt == LPB_OUT_F16; }
size_t format_bytes(int fmt) { return fmt == LPB_OUT_F32 ? 4 : 2; }

template <typename F>
void with_type(int fmt, F&& f) {
  if (fmt == LPB_OUT_BF16) f(__nv_bfloat16{});
  else if (fmt == LPB_OUT_F16) f(__half{});
  else f(float{});
}

// the 16-byte vector width for elements of this type, or 1 when the pointer or the contiguous run `run` does not allow it
template <typename T>
int vec_width(const void* p, int run) {
  constexpr int V = 16 / sizeof(T);
  return aligned_to(p, 16) && run % V == 0 ? V : 1;
}

template <typename T>
void launch_pool(const void* features, int layout, int B, int C, int hw, float* pooled, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  const T* x = static_cast<const T*>(features);
  if (layout == LPB_FEATURES_NHWC || hw == 1) {
    const bool vec = vec_width<T>(features, C) == V;
    const dim3 grid(n_blocks(C / (vec ? V : 1), POOL_THREADS), grid_y(B));
    if (vec) pool_channels_kernel<T, V><<<grid, POOL_THREADS, 0, s>>>(x, B, C, hw, pooled);
    else pool_channels_kernel<T, 1><<<grid, POOL_THREADS, 0, s>>>(x, B, C, hw, pooled);
  } else {
    const dim3 grid(n_blocks(C, ROW_WARPS * ROWS_PER_WARP), grid_y(B));
    if (vec_width<T>(features, hw) == V) pool_rows_kernel<T, V><<<grid, ROW_WARPS * 32, 0, s>>>(x, B, C, hw, pooled);
    else pool_rows_kernel<T, 1><<<grid, ROW_WARPS * 32, 0, s>>>(x, B, C, hw, pooled);
  }
}

template <typename T>
void launch_broadcast(const float* dpool, int layout, int B, int C, int hw, void* dfeat, cudaStream_t s) {
  constexpr int V = 16 / sizeof(T);
  T* dx = static_cast<T*>(dfeat);
  const bool nhwc = layout == LPB_FEATURES_NHWC || hw == 1;
  const bool vec = vec_width<T>(dfeat, nhwc ? C : hw) == V;
  const dim3 grid(n_blocks((int64_t)C * hw / (vec ? V : 1), POOL_THREADS), grid_y(B));
  if (nhwc) {
    if (vec) broadcast_kernel<T, V, true><<<grid, POOL_THREADS, 0, s>>>(dpool, B, C, hw, dx);
    else broadcast_kernel<T, 1, true><<<grid, POOL_THREADS, 0, s>>>(dpool, B, C, hw, dx);
  } else {
    if (vec) broadcast_kernel<T, V, false><<<grid, POOL_THREADS, 0, s>>>(dpool, B, C, hw, dx);
    else broadcast_kernel<T, 1, false><<<grid, POOL_THREADS, 0, s>>>(dpool, B, C, hw, dx);
  }
}

int check_head_shape(const char* entry, int format, int layout, int B, int C, int H, int W, int n_out) {
  LPB_REQUIRE(valid_format(format), "%s: unknown feature format %d", entry, format);
  LPB_REQUIRE(layout == LPB_FEATURES_NCHW || layout == LPB_FEATURES_NHWC, "%s: unknown feature layout %d", entry, layout);
  LPB_REQUIRE(B >= 0 && C >= 1 && H >= 1 && W >= 1 && n_out >= 1 && (int64_t)C * H * W <= INT32_MAX, "%s: bad shape", entry);
  return LPB_OK;
}

}  // namespace
}  // namespace lpb

extern "C" int lpb_regression_head_fwd(const void* features, int format, int layout, int B, int C, int H, int W, const float* weight,
                                       const float* bias, int n_out, float* pooled, float* out, void* stream) {
  using namespace lpb;
  LPB_TRY(check_head_shape("regression_head_fwd", format, layout, B, C, H, W, n_out));
  if (B == 0) return LPB_OK;
  LPB_REQUIRE(features && weight && bias && pooled && out, "regression_head_fwd: null pointer");
  LPB_REQUIRE(aligned_to(features, format_bytes(format)), "regression_head_fwd: features must be %d-byte aligned", (int)format_bytes(format));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  with_type(format, [&](auto t) { launch_pool<decltype(t)>(features, layout, B, C, H * W, pooled, s); });
  linear_fwd_kernel<<<dim3(n_blocks(B, LIN_BM), n_blocks(n_out, LIN_BN)), 256, 0, s>>>(pooled, weight, bias, B, C, n_out, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_regression_head_bwd(const float* grad_out, const float* pooled, const float* weight, int format, int layout, int B,
                                       int C, int H, int W, int n_out, void* dfeatures, float* dweight, float* dbias, float* workspace,
                                       void* stream) {
  using namespace lpb;
  LPB_TRY(check_head_shape("regression_head_bwd", format, layout, B, C, H, W, n_out));
  LPB_REQUIRE(!dweight == !dbias, "regression_head_bwd: dweight and dbias are given together");
  LPB_REQUIRE(grad_out && pooled && weight, "regression_head_bwd: null pointer");
  LPB_REQUIRE(!dfeatures || workspace, "regression_head_bwd: d features need a workspace of B x C floats");
  LPB_REQUIRE(aligned_to(dfeatures, format_bytes(format)), "regression_head_bwd: dfeatures must be %d-byte aligned", (int)format_bytes(format));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dweight) {  // over the frames; B = 0 gives zeros
    colsum_kernel<<<dim3(n_blocks(n_out, CG_ROWS), n_blocks(C + 1, CG_THREADS)), CG_THREADS, 0, s>>>(
        grad_out, n_out, 1, B, n_out, pooled, C, 1, 1.f, dweight, dbias);
    LPB_CUDA(cudaGetLastError());
  }
  if (dfeatures && B > 0) {
    colsum_kernel<<<dim3(n_blocks(B, CG_ROWS), n_blocks(C, CG_THREADS)), CG_THREADS, 0, s>>>(
        grad_out, 1, n_out, n_out, B, weight, C, 0, 1.f / (float)(H * W), workspace, nullptr);
    with_type(format, [&](auto t) { launch_broadcast<decltype(t)>(workspace, layout, B, C, H * W, dfeatures, s); });
    LPB_CUDA(cudaGetLastError());
  }
  return LPB_OK;
}

extern "C" int lpb_regression_losses_fwd(const float* targets, const float* preds, int64_t n, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(n >= 0, "regression_losses_fwd: bad shape");
  LPB_REQUIRE(out && (n == 0 || (targets && preds)), "regression_losses_fwd: null pointer");  // n = 0: NaN, 0, NaN, 0
  regression_losses_fwd_kernel<<<1, RL_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(targets, preds, n, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_regression_losses_bwd(const float* targets, const float* preds, int64_t n, const float* fwd_out, const float* grad_out,
                                         float* grad_preds, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(n >= 0, "regression_losses_bwd: bad shape");
  if (n == 0) return LPB_OK;
  LPB_REQUIRE(targets && preds && fwd_out && grad_out && grad_preds, "regression_losses_bwd: null pointer");
  regression_losses_bwd_kernel<<<n_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(targets, preds, n, fwd_out, grad_out,
                                                                                                 grad_preds);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
