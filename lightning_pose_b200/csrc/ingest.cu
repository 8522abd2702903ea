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

template <int LAYOUT, bool BF16, bool RESIZE>
__global__ void __launch_bounds__(256) ingest_kernel(const __grid_constant__ IngestParams P) {
  const int64_t total = (int64_t)P.F * P.OH * P.OW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % P.OW);
    const int64_t r = i / P.OW;
    const int y = (int)(r % P.OH), f = (int)(r / P.OH);
    float v[3];
    const uint8_t* img = P.in + (size_t)f * P.H * P.W * 3;
    if (RESIZE) {
      const float sy = fmaxf((y + 0.5f) * P.ry - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * P.rx - 0.5f, 0.f);
      const int y0 = min((int)sy, P.H - 1), x0 = min((int)sx, P.W - 1);
      const int y1 = min(y0 + 1, P.H - 1), x1 = min(x0 + 1, P.W - 1);
      const float wy = sy - (float)y0, wx = sx - (float)x0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float a = img[((size_t)y0 * P.W + x0) * 3 + c], b = img[((size_t)y0 * P.W + x1) * 3 + c];
        const float d = img[((size_t)y1 * P.W + x0) * 3 + c], e = img[((size_t)y1 * P.W + x1) * 3 + c];
        const float top = a + wx * (b - a), bot = d + wx * (e - d);
        v[c] = top + wy * (bot - top);
      }
    } else {
      const uint8_t* px = img + ((size_t)y * P.W + x) * 3;
      v[0] = px[0], v[1] = px[1], v[2] = px[2];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = fmaf(v[c], P.scale[c], P.shift[c]);
    const size_t plane = (size_t)P.OH * P.OW;
    if (LAYOUT == 0) {  // FCHW
      const size_t o = (size_t)f * 3 * plane + (size_t)y * P.OW + x;
      if (BF16) {
        __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(P.out);
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[o + c * plane] = __float2bfloat16_rn(v[c]);
      } else {
        float* dst = static_cast<float*>(P.out);
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[o + c * plane] = v[c];
      }
    } else {  // FHWC
      const size_t o = ((size_t)f * plane + (size_t)y * P.OW + x) * 3;
      if (BF16) {
        __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(P.out);
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[o + c] = __float2bfloat16_rn(v[c]);
      } else {
        float* dst = static_cast<float*>(P.out);
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[o + c] = v[c];
      }
    }
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
