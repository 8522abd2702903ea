// Fixed-order sums of per-CTA gradient partials.  A kernel that would otherwise add its share of a gradient into global
// memory with float atomics writes it as a partial instead (one slot per CTA or CTA group, one writer per element), and
// reduce_partials adds the slots in slot order.  The result is then the same bits from run to run, whatever the order the
// CTAs ran in.  Used by the bf16 head backward, the fp32 head's weight gradient and the context head's combine backward.
#pragma once

#include <cstdint>
#include <type_traits>

#include "lpb_common.cuh"

namespace lpb {

__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// out[i] = sum_{p < nparts} sum_{j < NSUB} part[p * stride + j * n + i], in that order (i < n), with plain fp32 adds: the
// same result bit for bit as one thread adding the partials one after another.  Partial q = p * NSUB + j is a row of n
// floats.  A CTA owns TILE consecutive outputs and has TILE owner threads, then RP_COPIERS copy threads.  The copiers
// copy chunks of ROWS = RP_CHUNK / TILE partial rows of the tile into a ring of RP_STAGES shared-memory stages (up to
// RP_STAGES - 1 chunks in flight); owner t adds column t of each chunk in order.  Only the adds are serial: the copies of
// the next chunks are in flight while they run, issuing them takes no owner's time, and a full chunk's adds are unrolled
// with compile-time offsets, so the owner's loads run ahead of its add chain.
constexpr int RP_COPIERS = 256, RP_CHUNK = 2048, RP_STAGES = 6;  // 6 stages x 8 KB: 48 KB of shared memory at most
template <int NSUB, int TILE>
__global__ void __launch_bounds__(TILE + RP_COPIERS) reduce_partials_kernel(const float* __restrict__ part, int nparts, size_t stride, int n,
                                                                            float* __restrict__ out) {
  constexpr int ROWS = RP_CHUNK / TILE;
  extern __shared__ float rp_buf[];  // [stage][row][TILE]
  const int nq = nparts * NSUB, nchunk = (nq + ROWS - 1) / ROWS;
  const int tid = threadIdx.x, u = tid - TILE;  // u >= 0: copier u
  // copy k of a chunk by copier u: row u / TILE + k * (RP_COPIERS / TILE), column u % TILE -> stage element u + k * RP_COPIERS
  const int i = blockIdx.x * TILE + (u >= 0 ? u : tid) % TILE, r0 = u / TILE;
  auto issue = [&](int c) {
    if (c < nchunk && i < n) {
      float* dst = rp_buf + (c % RP_STAGES) * RP_CHUNK + u;
#pragma unroll
      for (int k = 0; k < RP_CHUNK / RP_COPIERS; ++k) {
        const int q = c * ROWS + r0 + k * (RP_COPIERS / TILE);
        if (q < nq) cp_async4(dst + k * RP_COPIERS, part + (size_t)(q / NSUB) * stride + (size_t)(q % NSUB) * n + i);
      }
    }
    cp_async_commit();  // (an empty group past the last chunk keeps the wait count below uniform)
  };
  if (u >= 0)
    for (int c = 0; c < RP_STAGES - 1; ++c) issue(c);
  float s = 0.f;
  for (int c = 0; c < nchunk; ++c) {
    if (u >= 0) cp_async_wait<RP_STAGES - 2>();  // this copier's copies of chunk c have landed
    __syncthreads();                             // every copier's have, and the owners are done with chunk c - 1
    if (u >= 0) {
      issue(c + RP_STAGES - 1);
    } else {
      const float* src = rp_buf + (c % RP_STAGES) * RP_CHUNK + tid;
      const int nr = nq - c * ROWS;
      if (nr >= ROWS) {
#pragma unroll
        for (int r = 0; r < ROWS; ++r) s += src[r * TILE];
      } else {
        for (int r = 0; r < nr; ++r) s += src[r * TILE];
      }
    }
  }
  if (u < 0 && i < n) out[i] = s;
}
template <int NSUB>
static void reduce_partials(const float* part, int nparts, size_t stride, int n, float* out, int sms, cudaStream_t s) {
  auto launch = [&](auto tile) {
    constexpr int TILE = decltype(tile)::value, ROWS = RP_CHUNK / TILE;
    const int nchunk = (nparts * NSUB + ROWS - 1) / ROWS;
    const size_t smem = (size_t)(nchunk < RP_STAGES ? nchunk : RP_STAGES) * RP_CHUNK * sizeof(float);
    reduce_partials_kernel<NSUB, TILE><<<(n + TILE - 1) / TILE, TILE + RP_COPIERS, smem, s>>>(part, nparts, stride, n, out);
  };
  // 256-wide tiles (1 KB partial rows) while they still give every SM a CTA; 32-wide ones for the small sums
  if ((n + 255) / 256 >= sms) launch(std::integral_constant<int, 256>{});
  else launch(std::integral_constant<int, 32>{});
}

}  // namespace lpb
