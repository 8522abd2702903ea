// The padded "row layout" every tensor-core kernel of the head exchanges through global memory:
//   X[b][kchunk][row][8] bf16,  row = lead + y * (Wi + 1) + n
// i.e. the image raster with one zero column per image row plus `lead` zero rows before and after.  It is
// byte-for-byte the operand image the kernels keep in shared memory (zero column = horizontal halo, lead /
// trail rows = vertical halo), so any run of image rows -- halo included -- is ONE contiguous bulk copy per
// K-chunk instead of one copy per image row (the TMA unit spends ~50 cycles per copy, whatever its size).
// Producers write only real pixels; the head's preparation launch (head_prep.cuh) clears the pads of fresh buffers.
#pragma once
#include <cuda_bf16.h>

#include <cstddef>
#include <cstdint>

namespace lpb {

struct RowLayout {
  int Hi, Wi, Pp;  // Pp = Wi + 1
  int lead;        // zero rows before (and at least as many after) the raster = Pp + 1
  int rows;        // rows per K-chunk including pads (multiple of 8)
};

__host__ __device__ inline RowLayout make_row_layout(int Hi, int Wi) {
  RowLayout L;
  L.Hi = Hi;
  L.Wi = Wi;
  L.Pp = Wi + 1;
  L.lead = L.Pp + 1;
  L.rows = (Hi * L.Pp + 2 * L.lead + 7) & ~7;
  return L;
}

}  // namespace lpb
