// Video-ingest boundary (SURVEY 8f-4): decoded RGB surfaces -> the normalised frame tensor of an UnlabeledBatchDict.
// Reference: the tail of the DALI pipeline  lightning_pose/data/video/dali.py:157-197
//   fn.resize(video, size=resize_dims) -> video / 255.0 -> fn.crop_mirror_normalize(output_layout="FCHW", mean, std)
// fused into one pass: uint8 [F, H, W, 3] (what NVDEC + colour conversion, or any reader, leaves on the device) is read
// once (3 B / pixel) and written once, in the layout / precision the consumer wants:
//   FCHW fp32 (the reference's layout), FCHW bf16, or FHWC (channels-last) bf16 for tensor-core backbone tiles.
// Resize is the plain bilinear filter with half-pixel centres (torch's align_corners=False, no antialiasing).
// HBM-bound: no shared memory staging needed (every input byte is used by at most 4 neighbouring outputs: L1/L2).
#include <cuda_bf16.h>

#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {

struct IngestParams {
  const uint8_t* in;
  void* out;
  int F, H, W, OH, OW;
  float scale[3], shift[3];  // out = px * scale + shift  (scale = 1 / (255 std), shift = -mean / std)
  float ry, rx;              // H / OH, W / OW
};

// Pixel (y, x) of the resized image: 3 channels in 0..255.  RESIZE = false reads the source pixel itself.
template <bool RESIZE>
__device__ __forceinline__ void resized_pixel(const uint8_t* img, int H, int W, float ry, float rx, int y, int x, float v[3]) {
  if (RESIZE) {
    const float sy = fmaxf((y + 0.5f) * ry - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * rx - 0.5f, 0.f);
    const int y0 = min((int)sy, H - 1), x0 = min((int)sx, W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float wy = sy - (float)y0, wx = sx - (float)x0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float a = img[((size_t)y0 * W + x0) * 3 + c], b = img[((size_t)y0 * W + x1) * 3 + c];
      const float d = img[((size_t)y1 * W + x0) * 3 + c], e = img[((size_t)y1 * W + x1) * 3 + c];
      const float top = a + wx * (b - a), bot = d + wx * (e - d);
      v[c] = top + wy * (bot - top);
    }
  } else {
    const uint8_t* px = img + ((size_t)y * W + x) * 3;
    v[0] = px[0], v[1] = px[1], v[2] = px[2];
  }
}

// Normalised output pixel (f, y, x) in the FCHW (LAYOUT 0) or FHWC (LAYOUT 1) layout, fp32 or bf16.
template <int LAYOUT, bool BF16>
__device__ __forceinline__ void store_pixel(void* out, int OH, int OW, int f, int y, int x, const float v[3]) {
  const size_t plane = (size_t)OH * OW;
  if (LAYOUT == 0) {  // FCHW
    const size_t o = (size_t)f * 3 * plane + (size_t)y * OW + x;
    if (BF16) {
      __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(out);
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[o + c * plane] = __float2bfloat16_rn(v[c]);
    } else {
      float* dst = static_cast<float*>(out);
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[o + c * plane] = v[c];
    }
  } else {  // FHWC
    const size_t o = ((size_t)f * plane + (size_t)y * OW + x) * 3;
    if (BF16) {
      __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(out);
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[o + c] = __float2bfloat16_rn(v[c]);
    } else {
      float* dst = static_cast<float*>(out);
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[o + c] = v[c];
    }
  }
}

template <int LAYOUT, bool BF16, bool RESIZE>
__global__ void __launch_bounds__(256) ingest_kernel(const __grid_constant__ IngestParams P) {
  const int64_t total = (int64_t)P.F * P.OH * P.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % P.OW);
    const int64_t r = i / P.OW;
    const int y = (int)(r % P.OH), f = (int)(r / P.OH);
    float v[3];
    resized_pixel<RESIZE>(P.in + (size_t)f * P.H * P.W * 3, P.H, P.W, P.ry, P.rx, y, x, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = fmaf(v[c], P.scale[c], P.shift[c]);
    store_pixel<LAYOUT, BF16>(P.out, P.OH, P.OW, f, y, x, v);
  }
}

// ---- augmented ingest: the DALI video augmentation of dali.py:156-178 ---------------------------------------------
// Per output pixel (f, y, x) of one view, with M = [A | t] the rotate-scale matrix (source -> destination, (x, y)):
//   warp     the resized image sampled bilinearly at  M^-1 (x + 0.5, y + 0.5) - 0.5, taps outside it read 0.
//            DALI's warp_affine docs: pixel centres at half-integer coordinates, and "fill_value: value used to fill
//            areas that are outside the source image".  Each tap is the resize sample of resized_pixel, evaluated on
//            the fly from the uint8 frame (4 source pixels per tap, byte loads through L1): no intermediate image.
//   bc       brightness * (0.5 + contrast * (in - 0.5)): DALI's brightness_contrast docs give contrast_center = half
//            the input type's range, and 0.5 for float input, which is what the reader hands it (normalized=False,
//            dtype=FLOAT: values 0..255).  No clamping for float.
//   shot     Poisson(max(0, in / factor)) * factor (DALI's noise.shot docs); in when factor == 0.
//   /255 + normalise, as ingest_kernel.
// Parameters are read from device memory (params: angle in degrees, sx, sy, brightness, contrast, factor; seed), so
// draws made inside a captured graph take effect on replay.
struct AugmentParams {
  const uint8_t* in;
  void* out;
  const float* params;
  const int64_t* seed;
  float* transform_out;
  int F, H, W, OH, OW;
  float scale[3], shift[3];
  float ry, rx;
};

// Philox4x32-10 (Salmon et al., SC'11): a counter-based generator, so a draw depends only on (key, counter).
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const uint32_t lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u, key.y += 0xBB67AE85u;
  }
  return ctr;
}

__device__ __forceinline__ float open_uniform(uint32_t r) { return ((float)(r >> 8) + 0.5f) * (1.0f / 16777216.0f); }  // (0, 1)

// log k! for k < 16; above, Stirling's series to 1 / (360 k^3) (truncation error < 1e-12 at k = 16).
__constant__ float c_log_factorial[16] = {0.f, 0.f, 0.69314718f, 1.7917595f, 3.1780538f, 4.7874917f, 6.5792512f, 8.5251614f,
                                          10.604603f, 12.801827f, 15.104413f, 17.502308f, 19.987214f, 22.552164f, 25.191221f, 27.899271f};

// log of the Poisson pmf at integer k >= 0, lam >= 10, in fp32 without the cancellation of -lam + k log lam - log k!:
// for k >= 16 it is -lam ((1 + d) log1p(d) - d) - log(2 pi k) / 2 - 1 / (12 k) + 1 / (360 k^3), d = (k - lam) / lam,
// whose absolute error grows like eps sqrt(lam) (6e-6 at lam = 1e4), not like eps lam.
__device__ __forceinline__ float poisson_log_pmf(float k, float lam) {
  if (k < 16.f) return k * __logf(lam) - lam - c_log_factorial[(int)k];
  const float d = (k - lam) / lam, ik = 1.f / k;
  return -lam * fmaf(1.f + d, log1pf(d), -d) - 0.5f * __logf(6.2831853f * k) - ik * fmaf(-ik * ik, 1.f / 360.f, 1.f / 12.f);
}

// Exact Poisson(lam) sample, expected cost bounded in lam.  lam < 10: inversion by sequential search (at most
// lam + 1 steps on average).  lam >= 10: PTRS, the transformed rejection of Hormann (1993), acceptance >= 0.87 at
// lam = 10 and rising, with poisson_log_pmf for the exact test.  k is an fp32 integer: exact below 2^24, and for larger
// lam its rounding stays far below the sample's spread sqrt(lam).  Draws come from the counter sequence (ctr.w counts
// blocks of four), so the result depends only on (key, ctr).
__device__ float poisson_sample(float lam, uint4 ctr, uint2 key) {
  if (!(lam > 0.f)) return 0.f;
  if (lam < 10.f) {
    const float u = open_uniform(philox4x32_10(ctr, key).x);
    float p = __expf(-lam), cdf = p;
    int k = 0;
    // stops where the pmf no longer moves the fp32 cdf: a u above the rounded total lands in the far tail
    while (u > cdf && p > cdf * 5.9604645e-8f) {
      ++k;
      p *= lam / (float)k;
      cdf += p;
    }
    return (float)k;
  }
  const float slam = sqrtf(lam);
  const float b = 0.931f + 2.53f * slam, a = -0.059f + 0.02483f * b;
  const float inv_alpha = 1.1239f + 1.1328f / (b - 3.4f), vr = 0.9277f - 3.6224f / (b - 2.f);
  for (;; ++ctr.w) {
    const uint4 r = philox4x32_10(ctr, key);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float U = open_uniform(h ? r.z : r.x) - 0.5f, V = open_uniform(h ? r.w : r.y);
      const float us = 0.5f - fabsf(U);
      const float k = floorf((2.f * a / us + b) * U + lam + 0.43f);
      if (us >= 0.07f && V <= vr) return k;
      if (k < 0.f || (us < 0.013f && V > us)) continue;
      if (__logf(V * inv_alpha / (a / (us * us) + b)) <= poisson_log_pmf(k, lam)) return k;
    }
  }
}

template <int LAYOUT, bool BF16, bool RESIZE>
__global__ void __launch_bounds__(256) augment_kernel(const __grid_constant__ AugmentParams P) {
  __shared__ float s_map[6];    // inverse map with the half-pixel shifts folded in: src = B (x, y) + d
  __shared__ float s_photo[3];  // brightness, contrast, factor
  __shared__ uint2 s_key;
  if (threadIdx.x == 0) {
    const double deg = P.params[0], sx = P.params[1], sy = P.params[2];
    // fn.transforms.rotation(angle, center=c) then fn.transforms.scale(scale, center=c): M = S_c R_c,
    // A = diag(sx, sy) R(angle), t = c - A c, with c = (OH / 2, OW / 2) taken as (x, y) as the reference passes it
    const double th = deg * 0.017453292519943295, cs = cos(th), sn = sin(th);
    const double a00 = sx * cs, a01 = -sx * sn, a10 = sy * sn, a11 = sy * cs;
    const double cx = 0.5 * P.OH, cy = 0.5 * P.OW;
    const double t0 = cx - (a00 * cx + a01 * cy), t1 = cy - (a10 * cx + a11 * cy);
    const double det = a00 * a11 - a01 * a10;
    const double b00 = a11 / det, b01 = -a01 / det, b10 = -a10 / det, b11 = a00 / det;
    // src = A^-1 (dst + 0.5 - t) - 0.5
    const double u0 = 0.5 - t0, u1 = 0.5 - t1;
    s_map[0] = (float)b00, s_map[1] = (float)b01, s_map[2] = (float)(b00 * u0 + b01 * u1 - 0.5);
    s_map[3] = (float)b10, s_map[4] = (float)b11, s_map[5] = (float)(b10 * u0 + b11 * u1 - 0.5);
    s_photo[0] = P.params[3], s_photo[1] = P.params[4], s_photo[2] = P.params[5];
    const uint64_t seed = (uint64_t)*P.seed;
    s_key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    if (blockIdx.x == 0) {
      P.transform_out[0] = (float)a00, P.transform_out[1] = (float)a01, P.transform_out[2] = (float)t0;
      P.transform_out[3] = (float)a10, P.transform_out[4] = (float)a11, P.transform_out[5] = (float)t1;
    }
  }
  __syncthreads();
  const float m00 = s_map[0], m01 = s_map[1], m02 = s_map[2], m10 = s_map[3], m11 = s_map[4], m12 = s_map[5];
  const float bright = s_photo[0], contrast = s_photo[1], factor = s_photo[2];
  const uint2 key = s_key;
  const int64_t total = (int64_t)P.F * P.OH * P.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % P.OW);
    const int64_t r = i / P.OW;
    const int y = (int)(r % P.OH), f = (int)(r / P.OH);
    const uint8_t* img = P.in + (size_t)f * P.H * P.W * 3;
    const float u = fmaf(m00, (float)x, fmaf(m01, (float)y, m02)), w = fmaf(m10, (float)x, fmaf(m11, (float)y, m12));
    const float fu = floorf(u), fw = floorf(w);
    const float wx = u - fu, wy = w - fw;
    float v[3] = {0.f, 0.f, 0.f};
    if (fu >= -1.f && fu < (float)P.OW && fw >= -1.f && fw < (float)P.OH) {  // else all four taps are fill (or NaN)
      const int x0 = (int)fu, y0 = (int)fw;
#pragma unroll
      for (int tap = 0; tap < 4; ++tap) {
        const int tx = x0 + (tap & 1), ty = y0 + (tap >> 1);
        if (tx < 0 || tx >= P.OW || ty < 0 || ty >= P.OH) continue;
        const float wt = ((tap & 1) ? wx : 1.f - wx) * ((tap >> 1) ? wy : 1.f - wy);
        float s[3];
        resized_pixel<RESIZE>(img, P.H, P.W, P.ry, P.rx, ty, tx, s);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = fmaf(wt, s[c], v[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float q = bright * fmaf(contrast, v[c] - 0.5f, 0.5f);
      if (factor != 0.f)
        q = poisson_sample(fmaxf(q / factor, 0.f), make_uint4((uint32_t)x, (uint32_t)y, (uint32_t)f, (uint32_t)c << 24), key) * factor;
      v[c] = fmaf(q, P.scale[c], P.shift[c]);
    }
    store_pixel<LAYOUT, BF16>(P.out, P.OH, P.OW, f, y, x, v);
  }
}

}  // namespace lpb

extern "C" int lpb_frames_normalize(const uint8_t* frames_u8, int F, int H, int W, int out_h, int out_w, const float* mean3,
                                    const float* std3, int layout, int out_bf16, void* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(frames_u8 && mean3 && std3 && out, "frames_normalize: null pointer");
  LPB_REQUIRE(F >= 0 && H >= 1 && W >= 1 && out_h >= 1 && out_w >= 1 && (layout == 0 || layout == 1), "frames_normalize: bad shape/layout");
  if (F == 0) return LPB_OK;
  IngestParams p;
  p.in = frames_u8;
  p.out = out;
  p.F = F, p.H = H, p.W = W, p.OH = out_h, p.OW = out_w;
  for (int c = 0; c < 3; ++c) {  // mean3 / std3 are HOST arrays (three floats of configuration, dali.py:44-45)
    LPB_REQUIRE(std3[c] > 0.f, "frames_normalize: std must be positive");
    p.scale[c] = 1.0f / (255.0f * std3[c]);
    p.shift[c] = -mean3[c] / std3[c];
  }
  p.ry = (float)H / (float)out_h;
  p.rx = (float)W / (float)out_w;
  const bool resize = (out_h != H) || (out_w != W);
  const int64_t total = (int64_t)F * out_h * out_w;
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;  // 32 CTAs per SM of an H100 SXM
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int key = layout * 4 + (out_bf16 ? 2 : 0) + (resize ? 1 : 0);
  switch (key) {
    case 0: ingest_kernel<0, false, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 1: ingest_kernel<0, false, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 2: ingest_kernel<0, true, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 3: ingest_kernel<0, true, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 4: ingest_kernel<1, false, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 5: ingest_kernel<1, false, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 6: ingest_kernel<1, true, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    default: ingest_kernel<1, true, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_frames_augment_normalize(const uint8_t* frames_u8, int F, int H, int W, int out_h, int out_w,
                                            const float* params, const int64_t* seed, const float* mean3, const float* std3,
                                            int layout, int out_bf16, void* out, float* transform_out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(frames_u8 && params && seed && mean3 && std3 && out && transform_out, "frames_augment_normalize: null pointer");
  LPB_REQUIRE(F >= 0 && H >= 1 && W >= 1 && out_h >= 1 && out_w >= 1 && (layout == 0 || layout == 1),
              "frames_augment_normalize: bad shape/layout");
  LPB_REQUIRE(F <= 16777215 && out_h <= 16777215 && out_w <= 16777215, "frames_augment_normalize: shape too large");
  if (F == 0) return LPB_OK;
  AugmentParams p;
  p.in = frames_u8;
  p.out = out;
  p.params = params;
  p.seed = seed;
  p.transform_out = transform_out;
  p.F = F, p.H = H, p.W = W, p.OH = out_h, p.OW = out_w;
  for (int c = 0; c < 3; ++c) {
    LPB_REQUIRE(std3[c] > 0.f, "frames_augment_normalize: std must be positive");
    p.scale[c] = 1.0f / (255.0f * std3[c]);
    p.shift[c] = -mean3[c] / std3[c];
  }
  p.ry = (float)H / (float)out_h;
  p.rx = (float)W / (float)out_w;
  const bool resize = (out_h != H) || (out_w != W);
  const int64_t total = (int64_t)F * out_h * out_w;
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int key = layout * 4 + (out_bf16 ? 2 : 0) + (resize ? 1 : 0);
  switch (key) {
    case 0: augment_kernel<0, false, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 1: augment_kernel<0, false, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 2: augment_kernel<0, true, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 3: augment_kernel<0, true, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 4: augment_kernel<1, false, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 5: augment_kernel<1, false, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    case 6: augment_kernel<1, true, false><<<(unsigned)blocks, 256, 0, s>>>(p); break;
    default: augment_kernel<1, true, true><<<(unsigned)blocks, 256, 0, s>>>(p); break;
  }
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
