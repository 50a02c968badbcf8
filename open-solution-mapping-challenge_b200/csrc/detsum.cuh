// detsum.cuh — deterministic cross-CTA sums.  A float atomicAdd per CTA adds the CTAs' partial sums in whatever order
// they finish, so a BatchNorm statistic or a weight gradient could differ from run to run in its last bits, and Adam's
// early, sign-like updates turn such bits into visibly different weights.  Instead every CTA stores its partial
// vector into its own row of a workspace (plain stores), and det_finish_kernel, launched right behind on the same
// stream, adds the rows in a fixed order:  out[(i / inner) * out_stride + i % inner] += sum_r ws[r * row_stride + i].
// Each translation unit owns its workspaces (static __device__ arrays), so launches of one stream never share one.
#pragma once
#include "host_common.h"

namespace mcb {

// one warp per output element: lane l adds rows l, l + 32, ... in order, then a fixed butterfly combines the lanes
template <typename T>
__device__ __forceinline__ void det_finish_body(const T* __restrict__ ws, int rows, long row_stride, long n, long inner,
                                                T* __restrict__ out, long out_stride) {
  const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  T t = 0;
  for (int r = lane; r < rows; r += 32) t += ws[(long)r * row_stride + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (lane == 0) out[(i / inner) * out_stride + i % inner] += t;
}

constexpr int kDetFinishThreads = 256;  // 8 output elements per block

inline dim3 det_finish_grid(long n) { return dim3((unsigned)((n + 7) / 8)); }

}  // namespace mcb

// Defines a workspace WS of CAP elements of type T in this translation unit and FINISH, its finishing kernel.
#define MCB_DET_WORKSPACE(T, WS, CAP, FINISH)                                                                      \
  static __device__ T WS[CAP];                                                                                    \
  __global__ void __launch_bounds__(mcb::kDetFinishThreads)                                                       \
      FINISH(long ws_off, int rows, long row_stride, long n, long inner, T* out, long out_stride) {               \
    mcb::det_finish_body<T>(WS + ws_off, rows, row_stride, n, inner, out, out_stride);                            \
  }
