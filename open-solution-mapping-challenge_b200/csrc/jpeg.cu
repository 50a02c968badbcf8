// jpeg.cu — baseline / extended sequential Huffman JPEG decoded on the device, bit-exact to libjpeg-turbo as Pillow
// runs it (islow IDCT, fancy upsampling, JFIF YCbCr -> RGB).  The host (mcb200.jpeg) parses the markers, removes the
// byte stuffing, splits the entropy data at its restart markers and builds the Huffman lookup tables; see
// include/mcb200.h for the table layouts.  Three launches per batch, no allocation, no synchronisation.
#include <algorithm>

#include "host_common.h"
#include "../../include/mcb200.h"

namespace mcb {
namespace {

constexpr int kLookahead = 9;
constexpr int kHuffWords = (1 << kLookahead) + 18 + 18 + 256;
constexpr int kMaxcode = 1 << kLookahead, kValoff = kMaxcode + 18, kVals = kValoff + 18;
constexpr int kComp0 = 6, kImageWords = kComp0 + 3 * 10, kSegWords = 5;

__constant__ unsigned char kZigzag[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Bit reader over one segment.  acc holds the next bits MSB-first; bits past the segment's end read as zero but are
// never consumed: `avail` counts the real ones, and consuming more than it is the truncation error.
struct Bits {
  const uint8_t* p;
  int left;           // segment bytes not yet in acc
  unsigned long long acc;
  int avail;          // real bits in acc
  __device__ void fill() {
    while (avail <= 56 && left > 0) {
      acc |= (unsigned long long)__ldg(p++) << (56 - avail);
      avail += 8;
      --left;
    }
  }
  __device__ bool skip(int n) {
    if (n > avail) return false;
    acc <<= n;
    avail -= n;
    return true;
  }
};

// one Huffman symbol; returns -1 (data ends) or -2 (no such code)
__device__ __forceinline__ int huff_decode(Bits& b, const int* t) {
  b.fill();
  const int e = t[(int)(b.acc >> (64 - kLookahead))];
  if (e) return b.skip(e >> 8) ? (e & 0xFF) : -1;
  for (int len = kLookahead + 1; len <= 16; ++len) {
    const int code = (int)(b.acc >> (64 - len));
    if (code <= t[kMaxcode + len]) {
      if (!b.skip(len)) return -1;
      return t[kVals + t[kValoff + len] + code];
    }
  }
  return -2;
}

// s raw bits, sign-extended as T.81 EXTEND; false when the data ends
__device__ __forceinline__ bool receive_extend(Bits& b, int s, int& v) {
  if (s == 0) { v = 0; return true; }
  b.fill();
  if (s > b.avail) return false;
  const int r = (int)(b.acc >> (64 - s));
  b.skip(s);
  v = r < (1 << (s - 1)) ? r - (1 << s) + 1 : r;
  return true;
}

// One thread per independent segment (an image, or one restart interval of it): DC predictors start at 0, so no
// thread waits on another.  One CTA per image: its Huffman tables are staged in shared memory and its threads take the
// image's segments in turn.  Blocks are zeroed and their non-zero coefficients scattered in natural order.
__global__ void __launch_bounds__(32) jpeg_entropy_kernel(const uint8_t* __restrict__ data, const int* __restrict__ segs,
                                                           const int* __restrict__ images,
                                                           const int* __restrict__ huff, int16_t* __restrict__ coef,
                                                           int* __restrict__ status) {
  __shared__ int tab[8 * kHuffWords];
  const int img = blockIdx.x;
  const int* im = images + (long)img * kImageWords;
  const int ncomp = im[0], mcux = im[1], seg0 = im[4], nseg = im[5];
  for (int i = threadIdx.x; i < 8 * kHuffWords; i += blockDim.x) tab[i] = __ldg(huff + (long)img * 8 * kHuffWords + i);
  __syncthreads();
  for (int s = seg0 + threadIdx.x; s < seg0 + nseg; s += blockDim.x) {
    const int* sg = segs + (long)s * kSegWords;
    const int first = sg[3], count = sg[4];
    Bits b{data + sg[1], sg[2], 0ull, 0};
    int pred[3] = {0, 0, 0};
    int err = 0;
    for (int m = first; m < first + count && !err; ++m) {
      const int my = m / mcux, mx = m - my * mcux;
      for (int c = 0; c < ncomp && !err; ++c) {
        const int* cp = im + kComp0 + 10 * c;
        const int ch = cp[0], cv = cp[1], bw = cp[2];
        const int* dc = tab + (cp[7] - img * 8) * kHuffWords;
        const int* ac = tab + (cp[8] - img * 8) * kHuffWords;
        for (int v = 0; v < cv && !err; ++v) {
          for (int h = 0; h < ch && !err; ++h) {
            int16_t* blk = coef + ((long)cp[4] + (long)(my * cv + v) * bw + mx * ch + h) * 64;
            uint4* b4 = reinterpret_cast<uint4*>(blk);
#pragma unroll
            for (int i = 0; i < 8; ++i) b4[i] = make_uint4(0, 0, 0, 0);
            int sym = huff_decode(b, dc), val;
            if (sym < 0) { err = sym == -1 ? 1 : 2; break; }
            if (!receive_extend(b, sym, val)) { err = 1; break; }
            pred[c] += val;
            blk[0] = (int16_t)pred[c];
            for (int k = 1; k < 64;) {
              sym = huff_decode(b, ac);
              if (sym < 0) { err = sym == -1 ? 1 : 2; break; }
              const int r = sym >> 4, sz = sym & 15;
              if (sz) {
                k += r;
                if (k > 63) { err = 3; break; }
                if (!receive_extend(b, sz, val)) { err = 1; break; }
                blk[kZigzag[k]] = (int16_t)val;
                ++k;
              } else if (r == 15) {
                k += 16;
              } else {
                break;
              }
            }
          }
        }
      }
    }
    if (err) atomicMax(status + img, err);
  }
}

// libjpeg's jpeg_idct_islow constants (CONST_BITS 13)
constexpr long long F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633,
                    F1_501 = 12299, F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;
constexpr int kConstBits = 13, kPass1Bits = 2;

// one 1-D islow pass on in[0..7] (stride-free), results before descaling in out[0..7]
__device__ __forceinline__ void idct_1d(const long long* in, long long* out) {
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * F0_541;
  long long tmp2 = z1 + z3 * -F1_847;
  long long tmp3 = z1 + z2 * F0_765;
  z2 = in[0];
  z3 = in[4];
  long long tmp0 = (z2 + z3) * (1LL << kConstBits);
  long long tmp1 = (z2 - z3) * (1LL << kConstBits);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F1_175;
  tmp0 *= F0_298;
  tmp1 *= F2_053;
  tmp2 *= F3_072;
  tmp3 *= F1_501;
  z1 *= -F0_899;
  z2 *= -F2_562;
  z3 = z3 * -F1_961 + z5;
  z4 = z4 * -F0_390 + z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3;
  out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2;
  out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1;
  out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0;
  out[4] = tmp13 - tmp0;
}

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// the sample limit as Pillow's libjpeg-turbo applies it on x86: its AVX2 islow IDCT packs the descaled result with
// signed saturation and adds 128, so a value outside [-128, 127] saturates (the C code's range-limit table would wrap
// values beyond +-512; the two agree inside that)
__device__ __forceinline__ uint8_t range_limit(int x) { return (uint8_t)(min(max(x, -128), 127) + 128); }

// One thread per 8x8 block: dequantise (the table entry as libjpeg's 16-bit multiplier), columns, int32 workspace,
// rows, saturation to the sample range.  Blocks of one image are contiguous from its first component's offset.
__global__ void __launch_bounds__(128) jpeg_idct_kernel(const int16_t* __restrict__ coef, const int* __restrict__ qt,
                                                         const int* __restrict__ images, int n, int n_blocks,
                                                         uint8_t* __restrict__ planes) {
  const int blk = blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= n_blocks) return;
  int lo = 0, hi = n - 1;                         // last image whose first block <= blk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(images + (long)mid * kImageWords + kComp0 + 4) <= blk) lo = mid; else hi = mid - 1;
  }
  const int* im = images + (long)lo * kImageWords;
  int c = 0;
  for (int k = 1; k < __ldg(im); ++k)
    if (__ldg(im + kComp0 + 4 + 10 * k) <= blk) c = k;
  const int* q = qt + ((long)lo * 3 + c) * 64;
  int16_t x[64];
  const uint4* src = reinterpret_cast<const uint4*>(coef + (long)blk * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(x + 8 * i) = __ldg(src + i);
  int ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    long long in[8], out[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) in[r] = (long long)((int)x[r * 8 + col] * (int)(int16_t)__ldg(q + r * 8 + col));
    idct_1d(in, out);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (int)descale(out[r], kConstBits - kPass1Bits);
  }
  uint32_t packed[16];
#pragma unroll
  for (int row = 0; row < 8; ++row) {
    long long in[8], out[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) in[k] = ws[row * 8 + k];
    idct_1d(in, out);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t w = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        w |= (uint32_t)range_limit((int)descale(out[h * 4 + k], kConstBits + kPass1Bits + 3)) << (8 * k);
      packed[row * 2 + h] = w;
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(planes + (long)blk * 64);
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
}

// sample (y, x) of a component stored as 8x8 blocks, bw blocks per row
__device__ __forceinline__ int sample(const uint8_t* __restrict__ p, int bw, int y, int x) {
  return __ldg(p + ((long)(y >> 3) * bw + (x >> 3)) * 64 + (y & 7) * 8 + (x & 7));
}

// libjpeg-turbo's upsampled value of one component at output pixel (y, x).  Neighbour samples are clamped into the
// component's downsampled size (jdmainct.c's context rows replicate the first and last rows; jdsample.c's first and
// last columns reduce to the same formula), so padding-block samples are never read.
__device__ __forceinline__ int upsampled(const uint8_t* __restrict__ p, const int* __restrict__ cp, int rx, int ry,
                                         int y, int x) {
  const int bw = cp[2], cw = cp[5], ch = cp[6];
  if (rx == 1 && ry == 1) return sample(p, bw, y, x);
  const int i = ry == 2 ? y >> 1 : y;
  const int j = rx == 2 ? x >> 1 : x;
  if (rx == 2 && cw <= 2) return sample(p, bw, i, j);     // jdsample.c: box filter for a component <= 2 wide
  const int ni = ry == 2 ? min(max((y & 1) ? i + 1 : i - 1, 0), ch - 1) : i;
  if (rx == 1)                                             // h1v2: +1 for the upper output row, +2 for the lower
    return (3 * sample(p, bw, i, j) + sample(p, bw, ni, j) + 1 + (y & 1)) >> 2;
  const int nj = min(max((x & 1) ? j + 1 : j - 1, 0), cw - 1);
  if (ry == 1)                                             // h2v1: +1 even, +2 odd output column
    return (3 * sample(p, bw, i, j) + sample(p, bw, i, nj) + 1 + (x & 1)) >> 2;
  const int s0 = 3 * sample(p, bw, i, j) + sample(p, bw, ni, j);  // h2v2: column sums, then +8 even, +7 odd
  const int s1 = 3 * sample(p, bw, i, nj) + sample(p, bw, ni, nj);
  return (3 * s0 + s1 + 8 - (x & 1)) >> 4;
}

// One thread per output pixel: upsample every component, then jdcolor.c's ycc_rgb_convert with the host-built tables
// (Cr->R, Cb->B, Cr->G, Cb->G at SCALEBITS 16); a grayscale image is replicated to three bands.
__global__ void __launch_bounds__(256) jpeg_upsample_rgb_kernel(const uint8_t* __restrict__ planes,
                                                                 const int* __restrict__ images,
                                                                 const int* __restrict__ tables, int h, int w,
                                                                 uint8_t* __restrict__ out) {
  const int img = blockIdx.y;
  const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long)h * w) return;
  const int y = (int)(pix / w), x = (int)(pix - (long)y * w);
  const int* gi = images + (long)img * kImageWords;
  const int ncomp = __ldg(gi), hmax = __ldg(gi + 2), vmax = __ldg(gi + 3);
  int v[3] = {0, 0, 0};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c >= ncomp) break;
    int cp[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) cp[k] = __ldg(gi + kComp0 + 10 * c + k);
    v[c] = upsampled(planes + (long)cp[4] * 64, cp, hmax / cp[0], vmax / cp[1], y, x);
  }
  uint8_t* o = out + ((long)img * h * w + pix) * 3;
  if (ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)v[0];
    return;
  }
  const int yy = v[0], cb = v[1], cr = v[2];
  const int r = yy + __ldg(tables + cr);
  const int g = yy + ((__ldg(tables + 768 + cb) + __ldg(tables + 512 + cr)) >> 16);
  const int b = yy + __ldg(tables + 256 + cb);
  o[0] = (uint8_t)min(max(r, 0), 255);
  o[1] = (uint8_t)min(max(g, 0), 255);
  o[2] = (uint8_t)min(max(b, 0), 255);
}

}  // namespace
}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int mcb_jpeg_entropy_decode(const uint8_t* data, const int* segments, int nseg, const int* images,
                                       const int* huff, int n, int16_t* coef, int* status, void* stream) {
  MCB_REQUIRE(data && segments && images && huff && coef && status, "jpeg_entropy_decode: null pointer");
  MCB_REQUIRE(nseg > 0 && n > 0, "jpeg_entropy_decode: %d segments, %d images", nseg, n);
  MCB_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int) * (size_t)n, ST));
  jpeg_entropy_kernel<<<n, 32, 0, ST>>>(data, segments, images, huff, coef, status);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_jpeg_idct(const int16_t* coef, const int* qt, const int* images, int n, int n_blocks,
                             uint8_t* planes, void* stream) {
  MCB_REQUIRE(coef && qt && images && planes, "jpeg_idct: null pointer");
  MCB_REQUIRE(n > 0 && n_blocks > 0, "jpeg_idct: %d images, %d blocks", n, n_blocks);
  jpeg_idct_kernel<<<(n_blocks + 127) / 128, 128, 0, ST>>>(coef, qt, images, n, n_blocks, planes);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_jpeg_upsample_rgb(const uint8_t* planes, const int* images, const int* tables, int n, int h, int w,
                                     uint8_t* out, void* stream) {
  MCB_REQUIRE(planes && images && tables && out, "jpeg_upsample_rgb: null pointer");
  MCB_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0, "jpeg_upsample_rgb: bad shape (n %d, %dx%d)", n, h, w);
  const long hw = (long)h * w;
  jpeg_upsample_rgb_kernel<<<dim3((unsigned)((hw + 255) / 256), n), 256, 0, ST>>>(planes, images, tables, h, w, out);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
