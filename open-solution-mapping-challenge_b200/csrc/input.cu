// input.cu — the input side of the path (SURVEY.md 8f-4), the step right before the network:
//   * image tile -> network input: replicate / reflect-101 padding (src/augmentation.py:40-86, cv2.copyMakeBorder) +
//     torchvision ToTensor + Normalize (src/loaders.py:232-247, 311-317), uint8 HWC -> fp32 NCHW, bit-exact;
//   * offline target preparation (src/preparation.py:151-195): per-instance exact Euclidean distance transforms reduced
//     to the two nearest buildings per pixel (update_distances + clean_distances), and the component-size map
//     (get_size_matrix);
//   * the target tensor the distance-weighted loss consumes (src/loaders.py:141-171: uint16 / uint8 casts, sqrt of the
//     size map, to_monochrome) as one pass.
// Integer / byte work bound by HBM (pad + normalise, target assembly) or by shared-memory min-reductions (distance
// transform); no tensor cores.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>
#include <cuda_fp16.h>

namespace mcb {

// ------------------------------------------------------------------------------------------ pad + ToTensor + Normalize
// out[n][c][y][x] = ((float)img[n][sy][sx][c] / 255 - mean[c]) / std[c], every operation an IEEE fp32 round-to-nearest
// (torchvision: img.to(float32).div(255); tensor.sub_(mean).div_(std) with fp32 mean / std)
__device__ __forceinline__ int pad_src(int i, int n, int mode) {
  if (i < 0) return mode == 0 ? 0 : -i;                 // replicate | reflect-101 (cv2.BORDER_REFLECT_101)
  if (i >= n) return mode == 0 ? n - 1 : 2 * n - 2 - i;
  return i;
}
__global__ void pad_normalize_kernel(const uint8_t* __restrict__ img, float* __restrict__ out, int H, int W, int ph, int pw,
                                     int mode, float m0, float m1, float m2, float s0, float s1, float s2) {
  const int n = blockIdx.y;
  const int Ho = H + 2 * ph, Wo = W + 2 * pw;
  const long plane = (long)Ho * Wo;
  const uint8_t* src = img + (long)n * H * W * 3;
  float* dst = out + (long)n * 3 * plane;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < plane; q += (long)gridDim.x * blockDim.x) {
    const int y = q / Wo, x = q % Wo;
    const int sy = pad_src(y - ph, H, mode), sx = pad_src(x - pw, W, mode);
    const uint8_t* p = src + ((long)sy * W + sx) * 3;
    dst[q] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)p[0], 255.f), m0), s0);
    dst[plane + q] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)p[1], 255.f), m1), s1);
    dst[2 * plane + q] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)p[2], 255.f), m2), s2);
  }
}

// ------------------------------------------------------------------------------------------ PIL bilinear resize (8 bpc)
// transforms.Resize((h, w)) on a PIL image (src/loaders.py:287-305, the `resize` loader mode -- neptune.yaml's default)
// = Image.resize(BILINEAR) = Pillow's ImagingResample: a horizontal pass into an 8-bit temporary, then a vertical
// pass, each output = clip8((2^21 + sum_k pixel_k * coef_k) >> 22) with per-output-index integer coefficient rows
// (triangle filter widened by the scale factor when shrinking, normalised, rounded to 22 fractional bits -- computed
// on the host in double precision exactly like Pillow's precompute_coeffs / normalize_coeffs_8bpc).  Integer
// arithmetic throughout -> bit-exact.  coef int32 [out][ksize], bounds int32 [out][2] = (first source index, taps).
constexpr int kPilPrecision = 32 - 8 - 2;
__device__ __forceinline__ uint8_t pil_clip8(int v) {
  v >>= kPilPrecision;
  return (uint8_t)min(max(v, 0), 255);
}
// in [n][H][W][C] -> tmp [n][H][Wo][C]
__global__ void pil_resize_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ tmp, const int* __restrict__ coef,
                                    const int* __restrict__ bounds, int ksize, int H, int W, int Wo, int C) {
  const int n = blockIdx.y;
  const long total = (long)H * Wo * C;
  const uint8_t* src = in + (long)n * H * W * C;
  uint8_t* dst = tmp + (long)n * total;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < total; q += (long)gridDim.x * blockDim.x) {
    const int c = q % C;
    const int xx = (q / C) % Wo;
    const int y = q / ((long)C * Wo);
    const int x0 = bounds[2 * xx], taps = bounds[2 * xx + 1];
    const int* k = coef + (long)xx * ksize;
    int acc = 1 << (kPilPrecision - 1);
    for (int t = 0; t < taps; ++t) acc += (int)src[((long)y * W + x0 + t) * C + c] * k[t];
    dst[q] = pil_clip8(acc);
  }
}
// tmp [n][H][Wo][C] -> out [n][Ho][Wo][C]
__global__ void pil_resize_v_kernel(const uint8_t* __restrict__ tmp, uint8_t* __restrict__ out, const int* __restrict__ coef,
                                    const int* __restrict__ bounds, int ksize, int H, int Ho, int Wo, int C) {
  const int n = blockIdx.y;
  const long row = (long)Wo * C, total = (long)Ho * row;
  const uint8_t* src = tmp + (long)n * H * row;
  uint8_t* dst = out + (long)n * total;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < total; q += (long)gridDim.x * blockDim.x) {
    const int yy = q / row;
    const long r = q % row;
    const int y0 = bounds[2 * yy], taps = bounds[2 * yy + 1];
    const int* k = coef + (long)yy * ksize;
    int acc = 1 << (kPilPrecision - 1);
    for (int t = 0; t < taps; ++t) acc += (int)src[(long)(y0 + t) * row + r] * k[t];
    dst[q] = pil_clip8(acc);
  }
}

// ------------------------------------------------------------------------------------------ exact EDT, two nearest
// scipy.ndimage.distance_transform_edt(1 - mask): Euclidean distance of every pixel to the nearest pixel of the
// instance, sqrt of the exact integer squared distance in float64.
// Batched over images: image n owns the instances [image_off[n], image_off[n + 1]) of a list whose entry k is plane
// plane_index[k] of `masks` (identity when plane_index is null; one image of K instances when image_off is null).
// cols (nullable) holds per plane the first and last column with a pixel at cols[4 p + 2], cols[4 p + 3]
// (mcb_plane_stats); both passes skip the columns outside, which hold no pixel and so never give the minimum.
// An empty plane gives what scipy returns for an input without background: sqrt((y + 1)^2 + x^2).
// Pass 1 (columns): g[k][y][x] = vertical distance to the nearest instance pixel of column x (kInfCol if none).
constexpr int kInfCol = 1 << 20;
__device__ __forceinline__ int edt_plane(const int* plane_index, int k) { return plane_index ? plane_index[k] : k; }
__global__ void edt_columns_kernel(const uint8_t* __restrict__ masks, const int* __restrict__ plane_index,
                                   const int* __restrict__ cols, int* __restrict__ g, int H, int W, int k0) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = k0 + blockIdx.y;
  const int p = edt_plane(plane_index, k);
  if (x >= W || (cols && (x < cols[4 * p + 2] || x > cols[4 * p + 3]))) return;
  const uint8_t* m = masks + (long)p * H * W;
  int* gk = g + (long)k * H * W;
  int d = kInfCol;
  for (int y = 0; y < H; ++y) {
    d = m[(long)y * W + x] ? 0 : min(d + 1, kInfCol);
    gk[(long)y * W + x] = d;
  }
  d = kInfCol;
  for (int y = H - 1; y >= 0; --y) {
    d = m[(long)y * W + x] ? 0 : min(d + 1, kInfCol);
    gk[(long)y * W + x] = min(gk[(long)y * W + x], d);
  }
}
// Pass 2 (rows) fused with the reduction over instances: one CTA per (image row, image); for each instance the row of
// g is staged in shared memory and every thread takes min over x' of (x - x')^2 + g^2 (exact int64), keeping the two
// smallest squared distances over instances.  clean_distances (src/preparation.py:159-168): sum of the two nearest
// distances as float16, the second nearest as float64; one instance -> it counts twice; none -> zeros.
__global__ void edt_rows_two_nearest_kernel(const int* __restrict__ g, const int* __restrict__ plane_index,
                                            const int* __restrict__ image_off, const int* __restrict__ cols,
                                            __half* __restrict__ dist_sum, double* __restrict__ second, int K, int H,
                                            int W) {
  extern __shared__ int s_g[];
  const int y = blockIdx.x;
  const int n = blockIdx.y;
  const int k0 = image_off ? image_off[n] : 0, k1 = image_off ? image_off[n + 1] : K;
  const long out_base = (long)n * H * W + (long)y * W;
  const int x = threadIdx.x;   // blockDim.x >= W handled by a strided loop below
  for (int xb = 0; xb < W; xb += blockDim.x) {
    const int xx = xb + x;
    long long b1 = -1, b2 = -1;   // two smallest squared distances (-1 = none yet)
    for (int k = k0; k < k1; ++k) {
      const int p = edt_plane(plane_index, k);
      const int c0 = cols ? cols[4 * p + 2] : 0, c1 = cols ? cols[4 * p + 3] : W - 1;
      __syncthreads();
      for (int i = c0 + threadIdx.x; i <= c1; i += blockDim.x) s_g[i] = g[((long)k * H + y) * W + i];
      __syncthreads();
      if (xx < W) {
        long long best = (long long)1 << 60;
        for (int xp = c0; xp <= c1; ++xp) {
          const long long gv = s_g[xp];
          if (gv >= kInfCol) continue;
          const long long dx = xx - xp;
          best = min(best, dx * dx + gv * gv);
        }
        if (best == ((long long)1 << 60)) best = (long long)(y + 1) * (y + 1) + (long long)xx * xx;
        if (b1 < 0 || best < b1) { b2 = b1; b1 = best; }
        else if (b2 < 0 || best < b2) { b2 = best; }
      }
    }
    if (xx < W) {
      double d1 = 0.0, d2 = 0.0;
      if (k1 - k0 == 1) { d1 = d2 = sqrt((double)b1); }
      else if (k1 - k0 >= 2) { d1 = sqrt((double)b1); d2 = sqrt((double)b2); }
      dist_sum[out_base + xx] = __double2half(d1 + d2);
      second[out_base + xx] = d2;
    }
  }
}

// ------------------------------------------------------------------------------------------ size map, target tensor
// get_size_matrix (src/preparation.py:189-195): pixel count of the pixel's connected component, 1 on background
__global__ void size_matrix_kernel(const int* __restrict__ labels, const int* __restrict__ area, long long* __restrict__ out,
                                   long hw) {
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw; q += (long)gridDim.x * blockDim.x) {
    const int l = labels[q];
    out[q] = l > 0 ? (long long)area[l - 1] : 1ll;
  }
}
// source pixel (within image n of H x W) of padded target pixel q of a Ho x Wo plane
__device__ __forceinline__ long target_src(long q, int n, int H, int W, int ph, int pw, int mode) {
  const int Wo = W + 2 * pw;
  const int y = q / Wo, x = q % Wo;
  return (long)n * H * W + (long)pad_src(y - ph, H, mode) * W + pad_src(x - pw, W, mode);
}
// one target value: a uint8 'L' plane through to_monochrome + to_tensor (src/loaders.py:520-529) is its byte as float32
__device__ __forceinline__ void store_target_u8(float* dst, long q, uint8_t v) { dst[q] = (float)v; }

// MetadataImageSegmentationDatasetDistances.__getitem__ (src/loaders.py:141-171) without the random augmentation:
//   M = mask image -> convert('L') -> float32;  D = distances.astype(uint16) -> uint8 (to_pil) -> float32;
//   S = sizes.astype(uint16) -> sqrt -> uint16 -> uint8 (to_pil) -> float32;  target = cat(M, D, S)
// optional symmetric padding (inference loaders pad the targets like the image).
__global__ void target_channels_kernel(const uint8_t* __restrict__ mask, const __half* __restrict__ dist,
                                       const long long* __restrict__ sizes, float* __restrict__ out, int H, int W, int ph,
                                       int pw, int mode) {
  const int n = blockIdx.y;
  const int Ho = H + 2 * ph, Wo = W + 2 * pw;
  const long plane = (long)Ho * Wo;
  float* dst = out + (long)n * 3 * plane;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < plane; q += (long)gridDim.x * blockDim.x) {
    const long p = target_src(q, n, H, W, ph, pw, mode);
    store_target_u8(dst, q, mask[p]);
    const float df = __half2float(dist[p]);                               // numpy float16 -> uint16: truncation
    const unsigned d16 = (unsigned)(unsigned short)(long long)df;
    store_target_u8(dst + plane, q, (uint8_t)(d16 & 0xFFu));
    const unsigned s16 = (unsigned)(unsigned short)sizes[p];
    const unsigned r16 = (unsigned)(unsigned short)__fsqrt_rn((float)s16);   // np.sqrt of a uint16 array is float32
    store_target_u8(dst + 2 * plane, q, (uint8_t)(r16 & 0xFFu));
  }
}
// the same target from planes that already went through the casts and to_pil (csrc/augment.cu):
// planes uint8 [n][H][W][C] -> out fp32 [n][C][Ho][Wo]
__global__ void target_channels_u8_kernel(const uint8_t* __restrict__ planes, float* __restrict__ out, int H, int W,
                                          int C, int ph, int pw, int mode) {
  const int n = blockIdx.y;
  const long plane = (long)(H + 2 * ph) * (W + 2 * pw);
  float* dst = out + (long)n * C * plane;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < plane; q += (long)gridDim.x * blockDim.x) {
    const long p = target_src(q, n, H, W, ph, pw, mode);
    for (int c = 0; c < C; ++c) store_target_u8(dst + c * plane, q, planes[p * C + c]);
  }
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

static dim3 grid_in(long items, int planes, int threads) {
  const int per_plane =
      (int)std::max(1L, std::min((items + threads - 1) / threads, (long)num_sms() * 8L / std::max(planes, 1) + 1));
  return dim3(per_plane, planes, 1);
}

extern "C" int mcb_image_pad_normalize(const uint8_t* img, float* out, int n, int h, int w, int pad_h, int pad_w,
                                       int pad_mode, const float* mean3, const float* std3, void* stream) {
  MCB_REQUIRE(img && out && mean3 && std3, "pad_normalize: null pointer");
  MCB_REQUIRE(n > 0 && h > 0 && w > 0 && pad_h >= 0 && pad_w >= 0 && pad_h < h && pad_w < w, "pad_normalize: bad shape");
  MCB_REQUIRE(pad_mode == 0 || pad_mode == 1, "pad_normalize: pad_mode %d (0 replicate, 1 reflect-101)", pad_mode);
  pad_normalize_kernel<<<grid_in((long)(h + 2 * pad_h) * (w + 2 * pad_w), n, 256), 256, 0, ST>>>(
      img, out, h, w, pad_h, pad_w, pad_mode, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_pil_resize_bilinear_u8(const uint8_t* in, uint8_t* tmp, uint8_t* out, const int* coef_h,
                                          const int* bounds_h, int ksize_h, const int* coef_v, const int* bounds_v,
                                          int ksize_v, int n, int h, int w, int c, int out_h, int out_w, void* stream) {
  MCB_REQUIRE(in && tmp && out && coef_h && bounds_h && coef_v && bounds_v, "pil_resize: null pointer");
  MCB_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && out_h > 0 && out_w > 0 && ksize_h > 0 && ksize_v > 0, "pil_resize: bad shape");
  pil_resize_h_kernel<<<grid_in((long)h * out_w * c, n, 256), 256, 0, ST>>>(in, tmp, coef_h, bounds_h, ksize_h, h, w, out_w, c);
  MCB_LAUNCH_CHECK();
  pil_resize_v_kernel<<<grid_in((long)out_h * out_w * c, n, 256), 256, 0, ST>>>(tmp, out, coef_v, bounds_v, ksize_v, h, out_h,
                                                                             out_w, c);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

static int edt_launch(const uint8_t* masks, const int* plane_index, const int* image_off, const int* cols, int k,
                      int n, int h, int w, int* workspace, void* dist_sum_f16, double* second_nearest, void* stream) {
  MCB_REQUIRE(h < kInfCol && w < kInfCol, "edt: image too large");
  constexpr int kMaxGridY = 65535;   // instances and images go on gridDim.y, in slices
  for (int k0 = 0; k0 < k; k0 += kMaxGridY) {
    edt_columns_kernel<<<dim3((w + 127) / 128, std::min(kMaxGridY, k - k0)), 128, 0, ST>>>(masks, plane_index, cols,
                                                                                         workspace, h, w, k0);
    MCB_LAUNCH_CHECK();
  }
  const int threads = std::min(1024, ((w + 31) / 32) * 32);
  const long hw = (long)h * w;
  for (int n0 = 0; n0 < n; n0 += kMaxGridY) {   // n > 1 only with image_off
    edt_rows_two_nearest_kernel<<<dim3(h, std::min(kMaxGridY, n - n0)), threads, (size_t)w * sizeof(int), ST>>>(
        workspace, plane_index, image_off ? image_off + n0 : nullptr, cols, (__half*)dist_sum_f16 + n0 * hw,
        second_nearest + n0 * hw, k, h, w);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_edt_two_nearest(const uint8_t* masks, int k, int h, int w, int* workspace, void* dist_sum_f16,
                                   double* second_nearest, void* stream) {
  MCB_REQUIRE(dist_sum_f16 && second_nearest && k >= 0 && h > 0 && w > 0, "edt: bad argument");
  MCB_REQUIRE(k == 0 || (masks && workspace), "edt: null pointer");
  return edt_launch(masks, nullptr, nullptr, nullptr, k, 1, h, w, workspace, dist_sum_f16, second_nearest, stream);
}

extern "C" int mcb_edt_two_nearest_batched(const uint8_t* masks, const int* plane_index, const int* image_off,
                                           const int* plane_stats, int k, int n, int h, int w, int* workspace,
                                           void* dist_sum_f16, double* second_nearest, void* stream) {
  MCB_REQUIRE(dist_sum_f16 && second_nearest && image_off && k >= 0 && n > 0 && h > 0 && w > 0, "edt: bad argument");
  MCB_REQUIRE(k == 0 || (masks && workspace), "edt: null pointer");
  return edt_launch(masks, plane_index, image_off, plane_stats, k, n, h, w, workspace, dist_sum_f16, second_nearest,
                    stream);
}

extern "C" int mcb_size_matrix(const int* labels, const int* area, long long* out, int h, int w, void* stream) {
  MCB_REQUIRE(labels && area && out, "size_matrix: null pointer");
  const long hw = (long)h * w;
  size_matrix_kernel<<<(unsigned)std::min((hw + 255) / 256, (long)num_sms() * 8), 256, 0, ST>>>(labels, area, out, hw);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_target_channels(const uint8_t* mask, const void* dist_f16, const long long* sizes, float* out, int n,
                                   int h, int w, int pad_h, int pad_w, int pad_mode, void* stream) {
  MCB_REQUIRE(mask && dist_f16 && sizes && out, "target_channels: null pointer");
  MCB_REQUIRE(pad_h >= 0 && pad_w >= 0 && pad_h < h && pad_w < w && (pad_mode == 0 || pad_mode == 1), "target_channels: bad padding");
  target_channels_kernel<<<grid_in((long)(h + 2 * pad_h) * (w + 2 * pad_w), n, 256), 256, 0, ST>>>(
      mask, (const __half*)dist_f16, sizes, out, h, w, pad_h, pad_w, pad_mode);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_target_channels_u8(const uint8_t* planes, float* out, int n, int h, int w, int c, int pad_h, int pad_w,
                                      int pad_mode, void* stream) {
  MCB_REQUIRE(planes && out, "target_channels_u8: null pointer");
  MCB_REQUIRE(n > 0 && h > 0 && w > 0 && (c == 1 || c == 3), "target_channels_u8: bad shape");
  MCB_REQUIRE(pad_h >= 0 && pad_w >= 0 && pad_h < h && pad_w < w && (pad_mode == 0 || pad_mode == 1),
              "target_channels_u8: bad padding");
  target_channels_u8_kernel<<<grid_in((long)(h + 2 * pad_h) * (w + 2 * pad_w), n, 256), 256, 0, ST>>>(
      planes, out, h, w, c, pad_h, pad_w, pad_mode);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
