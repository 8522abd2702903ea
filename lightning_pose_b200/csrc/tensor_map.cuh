// The driver's tensor-map encoder (cuTensorMapEncodeTiled), looked up once through cudaGetDriverEntryPoint: the library
// needs no link-time dependency on libcuda.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

namespace lpb {

typedef CUresult (*TensorMapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// null when the driver has no encoder (every caller then has to take a route without a tensor map)
inline TensorMapEncodeFn tensor_map_encoder() {
  static const TensorMapEncodeFn encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess;
    (void)cudaGetLastError();
    return ok ? reinterpret_cast<TensorMapEncodeFn>(fn) : nullptr;
  }();
  return encode;
}

}  // namespace lpb
