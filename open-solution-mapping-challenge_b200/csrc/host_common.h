// host_common.h — host-side helpers shared by every translation unit of libmcb200.so:
// thread-local error string (mcb_last_error), CUDA error checks, TMA tensor-map encoding through the
// driver entry point (no link-time libcuda dependency, so the library loads on a GPU-less box).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#define MCB_OK 0
#define MCB_ERR_INVALID (-1)
#define MCB_ERR_CUDA (-2)
#define MCB_ERR_UNSUPPORTED (-3)

namespace mcb {

char* err_buf();  // thread-local, 512 bytes
int fail(int code, const char* fmt, ...);

#define MCB_CHECK_CUDA(expr)                                                                         \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return mcb::fail(MCB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)

#define MCB_REQUIRE(cond, ...)                                 \
  do {                                                         \
    if (!(cond)) return mcb::fail(MCB_ERR_INVALID, __VA_ARGS__); \
  } while (0)

#define MCB_LAUNCH_CHECK() MCB_CHECK_CUDA(cudaPeekAtLastError())

// Encode a tiled bf16/fp32 tensor map.  dims/strides innermost first; strides in BYTES for dims 1..rank-1.
// swizzle_bytes: 0 (none), 32, 64 or 128.  Returns MCB_OK or sets the error string.
int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

// NHWC bf16 tensor viewed as (C, W, H, N); optional 2x2 parity sub-grid (stride 2 view): py/px in {0,1}, or -1 for
// the plain view.  box = (box_c, bw, bh, bn).
int encode_nhwc_view(CUtensorMap* out, const void* base, int N, int H, int W, int C, int c_off, int c_len, int py,
                     int px, int box_c, int bw, int bh, int bn, int swizzle_bytes);

int num_sms();

}  // namespace mcb
