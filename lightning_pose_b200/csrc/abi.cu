// Library-level C-ABI entry points (version / error string).
#include "../../include/lpb200.h"

namespace lpb {
const char* last_error_cstr();
}

extern "C" int lpb_version(void) { return 100; }
extern "C" const char* lpb_last_error(void) { return lpb::last_error_cstr(); }
extern "C" const char* lpb_build_arch(void) { return "sm_90a"; }

// Kernel-variant switches (profiling / bring-up aid; defaults are the measured-best variants).  Process-global, read at
// launch time only.
namespace lpb {
int g_tuning[LPB_TUNE_COUNT] = {
    0,  // LPB_TUNE_K1A_ROW_TRANSPOSER (measured: 2x the instructions of the block form, slower)
    1,  // LPB_TUNE_SOFTMAX_EPILOGUE_V2
    1,  // LPB_TUNE_WAIT_BACKOFF
    0,  // LPB_TUNE_DECODE_RING (measured: 1.0x DRAM traffic but too few resident warps: 2x slower at 96x96)
    0,  // LPB_TUNE_K1A_BULK_XS (measured: 268 vs 223 us per 512 frames: the loader's wait on the filled stage costs more than the producers' stores)
    1,  // LPB_TUNE_DECODE_L2_HINTS
    1,  // LPB_TUNE_B3A_PREFETCH
    1,  // LPB_TUNE_SOFTMAX_SPLIT
    0,  // LPB_TUNE_DECODE_WARP_CTAS
    0,  // LPB_TUNE_DECODE_REVERSE
    1,  // LPB_TUNE_B3A_TMA_STORE
    2,  // LPB_TUNE_WGRAD_SWAP (no effect)
    1,  // LPB_TUNE_G2_PATCH
    1,  // LPB_TUNE_MMA_TILE_INNER (no effect)
    0,  // LPB_TUNE_DECODE_HINTS (measured: decode 118 -> 52 us per 512 frames, but the bound costs the softmax epilogue +80 us: net zero)
    2,  // LPB_TUNE_K1A_XS_COPY (2: a dedicated warp sends the finished stage to the saved copy with TMA bulk stores)
};
}
extern "C" int lpb_set_tuning(int key, int value) {
  if (key < 0 || key >= LPB_TUNE_COUNT) return LPB_ERR_INVALID;
  lpb::g_tuning[key] = value;
  return LPB_OK;
}
extern "C" int lpb_get_tuning(int key) { return (key < 0 || key >= LPB_TUNE_COUNT) ? -1 : lpb::g_tuning[key]; }
