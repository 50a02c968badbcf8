// detsum.cuh — deterministic cross-CTA sums.  A float atomicAdd per CTA adds the CTAs' partial sums in whatever order
// they finish, so a BatchNorm statistic or a weight gradient could differ from run to run in its last bits, and Adam's
// early, sign-like updates turn such bits into visibly different weights.  Instead every CTA stores its partial
// vector into its own row of a workspace (plain stores), and det_finish_kernel, launched right behind on the same
// stream, adds the rows in a fixed order:  out[(i / inner) * out_stride + i % inner] += sum_r ws[r * row_stride + i].
// Each translation unit owns its workspaces (static __device__ arrays), so launches of one stream never share one.
#pragma once
#include "host_common.h"

namespace mcb {

// The fixed order (it decides the last bits of every statistic and weight gradient, so it never changes): 32 partial
// sums p_l = ((0 + row l) + row l + 32) + ..., combined as a butterfly, p_l += p_{l+o} for o = 16, 8, 4, 2, 1; the
// result is p_0.  Two layouts compute exactly this:
//  - more than 32 rows (a persistent producer's 132 CTAs, channel_reduce's 4 per SM): one warp per output element,
//    lane l adds rows l, l + 32, ... and the butterfly is a shuffle; few elements still spread over many CTAs;
//  - at most 32 rows (split-K weight gradients: a few splits of up to millions of elements): one thread per output
//    element holds all 32 partial sums; consecutive threads read consecutive elements of a row (coalesced), and the
//    grid is one CTA per 256 elements instead of one per 8, whose launch alone took longer than the sums.
constexpr int kDetFinishThreads = 256;

inline bool det_finish_per_thread(int rows) { return rows <= 32; }

inline dim3 det_finish_grid(long n, int rows) {
  const long per_cta = det_finish_per_thread(rows) ? kDetFinishThreads : kDetFinishThreads / 32;
  return dim3((unsigned)((n + per_cta - 1) / per_cta));
}

template <typename T>
__device__ __forceinline__ void det_finish_body(const T* __restrict__ ws, int rows, long row_stride, long n, long inner,
                                                T* __restrict__ out, long out_stride) {
  if (rows <= 32) {   // det_finish_per_thread
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    T p[32];
#pragma unroll
    for (int l = 0; l < 32; ++l) p[l] = l < rows ? T(0) + ws[(long)l * row_stride + i] : T(0);
#pragma unroll
    for (int l = 0; l < 16; ++l) p[l] += p[l + 16];
#pragma unroll
    for (int l = 0; l < 8; ++l) p[l] += p[l + 8];
#pragma unroll
    for (int l = 0; l < 4; ++l) p[l] += p[l + 4];
    p[0] += p[2];
    p[1] += p[3];
    out[(i / inner) * out_stride + i % inner] += p[0] + p[1];
    return;
  }
  const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  T t = 0;
  for (int r = lane; r < rows; r += 32) t += ws[(long)r * row_stride + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (lane == 0) out[(i / inner) * out_stride + i % inner] += t;
}

}  // namespace mcb

// Defines a workspace WS of CAP elements of type T in this translation unit and FINISH, its finishing kernel.
#define MCB_DET_WORKSPACE(T, WS, CAP, FINISH)                                                                      \
  static __device__ T WS[CAP];                                                                                    \
  __global__ void __launch_bounds__(mcb::kDetFinishThreads)                                                       \
      FINISH(long ws_off, int rows, long row_stride, long n, long inner, T* out, long out_stride) {               \
    mcb::det_finish_body<T>(WS + ws_off, rows, row_stride, n, inner, out, out_stride);                            \
  }
