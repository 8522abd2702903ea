// Library-level C-ABI entry points (version / error string).
#include "../../include/lpb200.h"

namespace lpb {
const char* last_error_cstr();
}

extern "C" int lpb_version(void) { return 100; }
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
