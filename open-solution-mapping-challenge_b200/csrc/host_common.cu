// host_common.cu — error string, driver entry point lookup, tensor-map encoding.
#include "host_common.h"
#include <string.h>
#include <mutex>

namespace mcb {

static thread_local char g_err[512] = {0};

char* err_buf() { return g_err; }

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int encode_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return fail(MCB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(MCB_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u] sw %d base %p",
                (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, swizzle_bytes, base);
  }
  return MCB_OK;
}

int encode_nhwc_view(CUtensorMap* out, const void* base, int N, int H, int W, int C, int c_off, int c_len, int py,
                     int px, int box_c, int bw, int bh, int bn, int swizzle_bytes) {
  const uint64_t es = 2;  // bf16
  const char* b = static_cast<const char*>(base) + (uint64_t)c_off * es;
  uint64_t dims[4], str[3];
  if (py < 0) {
    dims[0] = c_len; dims[1] = W; dims[2] = H; dims[3] = N;
    str[0] = (uint64_t)C * es; str[1] = (uint64_t)W * C * es; str[2] = (uint64_t)H * W * C * es;
  } else {
    // rows py, py+2, ... and columns px, px+2, ...
    int Wv = (W - px + 1) / 2, Hv = (H - py + 1) / 2;
    b += ((uint64_t)py * W + px) * C * es;
    dims[0] = c_len; dims[1] = Wv; dims[2] = Hv; dims[3] = N;
    str[0] = 2ull * C * es; str[1] = 2ull * W * C * es; str[2] = (uint64_t)H * W * C * es;
  }
  uint32_t box[4] = {(uint32_t)box_c, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
  return encode_tmap(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, b, dims, str, box, swizzle_bytes);
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace mcb

extern "C" const char* mcb_last_error(void) { return mcb::err_buf(); }
extern "C" int mcb_version(void) { return 101; }

// zero-fill of accumulation buffers (gradient arena, BatchNorm statistic sums, loss sums) as a memset node on the caller's
// stream -- captured into the step's graphs like any launch; no library kernel involved
extern "C" int mcb_zero_bytes(void* p, size_t bytes, void* stream) {
  if (!p || bytes == 0) return MCB_OK;
  MCB_CHECK_CUDA(cudaMemsetAsync(p, 0, bytes, static_cast<cudaStream_t>(stream)));
  return MCB_OK;
}
