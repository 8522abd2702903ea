// Curriculum patch masking of multi-view transformer training (include/lpb200.h, lpb_patch_mask_*).
// Reference: PatchMasker.apply_patch_masking  lightning_pose/callbacks.py:303-401, which builds a torch.Generator and
// runs one randperm per (example, view) and zeroes the chosen patches one slice at a time from Python.  Here:
//   select  one CTA per (example, view): the curriculum's patch count m from the device step, one Philox key per patch,
//           a shared-memory bitonic sort of the keys, the m smallest masked -> mask [B, V, P] fp32;
//   apply   one grid over every image plane: 16-byte loads and stores, one mask lookup per vector.
#include <cuda_bf16.h>

#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {

constexpr int kSelectThreads = 512;
constexpr int kPatchIndexBits = 12;  // LPB_PATCH_MAX = 2^12: a key's low bits hold its patch index
static_assert(LPB_PATCH_MAX == 1 << kPatchIndexBits, "patch index field");

// m = int(ratio * P) of callbacks.py:344-357, every operation rounded as Python's float64 rounds it (no FMA contraction).
// (step - init_step) and (final_step - init_step) are exact in fp64 below 2^53, and IEEE division of the two is Python's
// correctly rounded int / int.
__device__ __forceinline__ int patches_to_mask(int64_t step, int64_t init_step, int64_t final_step, double r0, double r1, int P) {
  if (step < init_step) return 0;  // ratio 0.0
  const double progress = fmin(__ddiv_rn((double)(step - init_step), (double)(final_step - init_step)), 1.0);
  const double ratio = __dadd_rn(r0, __dmul_rn(progress, __dsub_rn(r1, r0)));
  const double x = __dmul_rn(ratio, (double)P);
  if (!(x > 0.0)) return 0;  // int() of a negative ratio: the reference masks nothing (patches_to_mask_per_view <= 0)
  return x >= (double)P ? P : (int)x;  // randperm(P)[:m] with m > P is every patch
}

struct SelectParams {
  const int64_t* step;
  float* mask;
  int V, P, pad;  // pad: P rounded up to a power of two (the sort's length)
  uint2 key;      // patch_seed
  int64_t init_step, final_step;
  double r0, r1;
};

__global__ void __launch_bounds__(kSelectThreads) patch_select_kernel(const __grid_constant__ SelectParams p) {
  __shared__ uint64_t s_key[LPB_PATCH_MAX];
  __shared__ uint8_t s_keep[LPB_PATCH_MAX];
  const int bv = blockIdx.x, b = bv / p.V, v = bv % p.V;
  const int64_t step = *p.step;
  const int m = patches_to_mask(step, p.init_step, p.final_step, p.r0, p.r1, p.P);
  float* row = p.mask + (size_t)bv * p.P;
  if (m == 0 || m == p.P) {  // no draw needed (block-uniform branch)
    for (int i = threadIdx.x; i < p.P; i += blockDim.x) row[i] = m == 0 ? 1.f : 0.f;
    return;
  }
  // key = 52 random bits above the patch index: distinct keys, and equal random parts order by index
  const uint4 base = make_uint4(0u, (uint32_t)v << 16, (uint32_t)b, 0u);
  for (int i = threadIdx.x; i < p.pad; i += blockDim.x) {
    uint64_t k = ~0ull;
    if (i < p.P) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)i | base.y, base.z, (uint32_t)step, (uint32_t)((uint64_t)step >> 32)), p.key);
      k = ((((uint64_t)r.x << 32) | r.y) << kPatchIndexBits) | (uint64_t)i;
      s_keep[i] = 1;
    }
    s_key[i] = k;
  }
  __syncthreads();
  // bitonic sort, ascending, of pad keys (pad <= 4096: at most 78 compare-exchange stages)
  for (int k = 2; k <= p.pad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < (p.pad >> 1); i += blockDim.x) {
        const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo + j;
        const uint64_t a = s_key[lo], c = s_key[hi];
        if ((a > c) == ((lo & k) == 0)) s_key[lo] = c, s_key[hi] = a;
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < m; i += blockDim.x) s_keep[s_key[i] & (LPB_PATCH_MAX - 1)] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < p.P; i += blockDim.x) row[i] = s_keep[i] ? 1.f : 0.f;
}

struct ApplyParams {
  const void* in;
  void* out;
  const float* mask;
  int64_t planes;  // B * V * C
  int C, H, W, PH, PW;
};

// VT: the access type (16, 8, 4 or 2 bytes), E elements of ELEM bytes each.  W * ELEM % sizeof(VT) == 0, so a vector
// never crosses a row, and E divides 16, so it never crosses a patch column or the unmasked right margin.
template <typename VT, int ELEM>
__global__ void __launch_bounds__(256) patch_apply_kernel(const __grid_constant__ ApplyParams p) {
  constexpr int E = (int)sizeof(VT) / ELEM;
  const int hw = p.H * p.W, n = hw / E, W = p.W;
  const int ymax = p.PH * LPB_PATCH_SIZE, xmax = p.PW * LPB_PATCH_SIZE;
  for (int64_t plane = blockIdx.y; plane < p.planes; plane += gridDim.y) {
    const float* mrow = p.mask + (plane / p.C) * (int64_t)p.PH * p.PW;
    const VT* src = reinterpret_cast<const VT*>(static_cast<const char*>(p.in) + plane * hw * ELEM);
    VT* dst = reinterpret_cast<VT*>(static_cast<char*>(p.out) + plane * hw * ELEM);
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
      const int e = j * E, y = e / W, x = e - y * W;
      const bool keep = y >= ymax || x >= xmax || mrow[(y >> 4) * p.PW + (x >> 4)] != 0.f;
      VT val = __ldcs(src + j);
      if (!keep) val = VT{};
      __stcs(dst + j, val);
    }
  }
}

// __ldcs / __stcs have no 2-byte overload: a plain access there
template <>
__global__ void __launch_bounds__(256) patch_apply_kernel<uint16_t, 2>(const __grid_constant__ ApplyParams p) {
  const int hw = p.H * p.W, W = p.W;
  const int ymax = p.PH * LPB_PATCH_SIZE, xmax = p.PW * LPB_PATCH_SIZE;
  for (int64_t plane = blockIdx.y; plane < p.planes; plane += gridDim.y) {
    const float* mrow = p.mask + (plane / p.C) * (int64_t)p.PH * p.PW;
    const uint16_t* src = static_cast<const uint16_t*>(p.in) + plane * hw;
    uint16_t* dst = static_cast<uint16_t*>(p.out) + plane * hw;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < hw; j += gridDim.x * blockDim.x) {
      const int y = j / W, x = j - y * W;
      const bool keep = y >= ymax || x >= xmax || mrow[(y >> 4) * p.PW + (x >> 4)] != 0.f;
      dst[j] = keep ? src[j] : (uint16_t)0;
    }
  }
}

template <typename VT, int ELEM>
void launch_apply(const ApplyParams& p, cudaStream_t s) {
  constexpr int E = (int)sizeof(VT) / ELEM;
  const int64_t n = (int64_t)p.H * p.W / E;
  // about 16 CTAs of 256 threads per SM of an H100 SXM over the whole batch, at least one per plane
  const int64_t want = (n + 255) / 256, planes_y = p.planes < 65535 ? p.planes : 65535;
  int64_t bx = (132 * 16 + planes_y - 1) / planes_y;
  if (bx > want) bx = want;
  if (bx < 1) bx = 1;
  patch_apply_kernel<VT, ELEM><<<dim3((unsigned)bx, (unsigned)planes_y), 256, 0, s>>>(p);
}

}  // namespace lpb

extern "C" int lpb_patch_mask_select(const int64_t* step, int B, int V, int H, int W, int64_t patch_seed, int64_t init_step,
                                     int64_t final_step, double init_ratio, double final_ratio, float* mask, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(step && mask, "patch_mask_select: null pointer");
  LPB_REQUIRE(B >= 0 && V >= 0 && H >= 0 && W >= 0, "patch_mask_select: bad shape");
  LPB_REQUIRE(V <= 65535 && (int64_t)B * V <= INT32_MAX, "patch_mask_select: bad shape (V <= 65535, B * V < 2^31)");
  const int64_t P = (int64_t)(H / LPB_PATCH_SIZE) * (W / LPB_PATCH_SIZE);
  LPB_REQUIRE(P <= LPB_PATCH_MAX, "patch_mask_select: %lld patches per view; at most %d (%d x %d patches)", (long long)P,
              LPB_PATCH_MAX, LPB_PATCH_SIZE, LPB_PATCH_SIZE);
  LPB_REQUIRE(final_step > init_step, "patch_mask_select: final_step (%lld) must be greater than init_step (%lld)",
              (long long)final_step, (long long)init_step);
  LPB_REQUIRE(init_ratio == init_ratio && final_ratio == final_ratio, "patch_mask_select: NaN ratio");
  if (P == 0 || B == 0 || V == 0) return LPB_OK;
  SelectParams p;
  p.step = step;
  p.mask = mask;
  p.V = V, p.P = (int)P;
  p.pad = 1;
  while (p.pad < p.P) p.pad <<= 1;
  p.key = make_uint2((uint32_t)(uint64_t)patch_seed, (uint32_t)((uint64_t)patch_seed >> 32));
  p.init_step = init_step, p.final_step = final_step;
  p.r0 = init_ratio, p.r1 = final_ratio;
  patch_select_kernel<<<B * V, kSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_patch_mask_apply(const void* images, int B, int V, int C, int H, int W, int in_format, const float* mask,
                                    void* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(images && out, "patch_mask_apply: null pointer");
  LPB_REQUIRE(B >= 0 && V >= 0 && C >= 0 && H >= 0 && W >= 0, "patch_mask_apply: bad shape");
  LPB_REQUIRE((int64_t)H * W <= INT32_MAX, "patch_mask_apply: bad shape (H * W < 2^31)");
  LPB_REQUIRE(in_format == LPB_OUT_F32 || in_format == LPB_OUT_BF16, "patch_mask_apply: format %d (0 = fp32, 1 = bf16)", in_format);
  const int PH = H / LPB_PATCH_SIZE, PW = W / LPB_PATCH_SIZE;
  LPB_REQUIRE((int64_t)PH * PW <= LPB_PATCH_MAX, "patch_mask_apply: %lld patches per view; at most %d", (long long)PH * PW, LPB_PATCH_MAX);
  LPB_REQUIRE(mask || PH * PW == 0, "patch_mask_apply: null pointer");
  const int64_t planes = (int64_t)B * V * C;
  const int elem = in_format == LPB_OUT_F32 ? 4 : 2;
  const int64_t bytes = planes * H * W * elem;
  const char *a = static_cast<const char*>(images), *o = static_cast<const char*>(out);
  LPB_REQUIRE(a + bytes <= o || o + bytes <= a, "patch_mask_apply: out must not alias images");
  if (planes == 0 || H == 0 || W == 0) return LPB_OK;
  ApplyParams p;
  p.in = images, p.out = out, p.mask = mask;
  p.planes = planes;
  p.C = C, p.H = H, p.W = W, p.PH = PH, p.PW = PW;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t row = (int64_t)W * elem;  // widest access that divides a row and both pointers
  auto fits = [&](int v) { return row % v == 0 && aligned_to(images, v) && aligned_to(out, v); };
  if (elem == 4) {
    if (fits(16)) launch_apply<uint4, 4>(p, s);
    else if (fits(8)) launch_apply<uint2, 4>(p, s);
    else launch_apply<uint32_t, 4>(p, s);
  } else {
    if (fits(16)) launch_apply<uint4, 2>(p, s);
    else if (fits(8)) launch_apply<uint2, 2>(p, s);
    else if (fits(4)) launch_apply<uint32_t, 2>(p, s);
    else launch_apply<uint16_t, 2>(p, s);
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
