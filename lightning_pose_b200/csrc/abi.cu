// Library-level C-ABI entry points (version / error string), and the device queries and shared-memory launch rule every
// entry shares (lpb_common.cuh).
#include <map>
#include <mutex>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {
const char* last_error_cstr();
}

extern "C" int lpb_version(void) { return 200; }
extern "C" const char* lpb_last_error(void) { return lpb::last_error_cstr(); }
extern "C" const char* lpb_build_arch(void) { return "sm_90a"; }

// Tuning switch (see include/lpb200.h).  Process-global, read at launch time only.
namespace lpb {
int g_softmax_split = 1;
}
extern "C" int lpb_set_tuning(int key, int value) {
  if (key != LPB_TUNE_SOFTMAX_SPLIT) return LPB_ERR_INVALID;
  lpb::g_softmax_split = value;
  return LPB_OK;
}
extern "C" int lpb_get_tuning(int key) { return key == LPB_TUNE_SOFTMAX_SPLIT ? lpb::g_softmax_split : -1; }

namespace lpb {

int device_limits(DeviceLimits* d) {
  static std::mutex mu;
  static std::map<int, DeviceLimits> cache;
  int dev = 0;
  LPB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(dev);
  if (it == cache.end()) {
    DeviceLimits q{};
    LPB_CUDA(cudaDeviceGetAttribute(&q.sms, cudaDevAttrMultiProcessorCount, dev));
    LPB_CUDA(cudaDeviceGetAttribute(&q.max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    it = cache.emplace(dev, q).first;
  }
  *d = it->second;
  return LPB_OK;
}

DeviceLimits planning_limits() {
  DeviceLimits d;
  if (device_limits(&d) == LPB_OK) return d;
  (void)cudaGetLastError();
  return DeviceLimits{132, 227 * 1024};
}

int smem_refused(cudaError_t e, const char* entry, size_t bytes) {
  if (e != cudaErrorInvalidValue) return cuda_fail(e, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)", __FILE__, __LINE__);
  (void)cudaGetLastError();
  set_error("%s: needs %zu B of dynamic shared memory, more than this device allows beside the kernel's static memory", entry, bytes);
  return LPB_ERR_UNSUPPORTED;
}

}  // namespace lpb
