// augment.cu — the random geometric augmentation of the training loaders (src/augmentation.py:5-10 fast_seq,
// :34-37 crop_seq + :91-135 RandomCropFixedSize, applied per sample through ImgAug, src/steps/pytorch/utils.py:108-129)
// for a whole batch.  Every plane of a sample (image bands, mask, distances, sizes) takes the same draw, so one thread
// computes the sample position of one output pixel once and gathers every plane from it.
//
// Per sample one parameter row (mcb_augment_row): flips before the warp, the 3x3 output -> input map of skimage's
// warp (np.linalg.inv of the imgaug Affine matrix, built on the host), flips after the warp, the crop offset.  Flips
// are index maps: a flip after the warp mirrors the output index, a flip before it mirrors the four integer neighbour
// indices after floor / ceil -- bit-identical to warping the flipped array.  The warp restates skimage's _warp_fast
// (order 1, mode 'constant', cval 0, preserve_range) in fp64 with explicitly rounded operations (no FMA contraction,
// like the C the Cython compiles to), then _clip_warp_output (clip to the input plane's [min, max]; pixels exactly
// at cval stay cval when cval lies outside that range) and imgaug's truncating astype back to the plane's dtype.
// uint16 planes (distances, sizes) are then cast to uint8 by to_pil (src/utils.py:284-289): wrap mod 256.
// Byte gathers from L2 (a sample's planes are ~0.7 MB); no tensor cores.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>
#include <cstring>

namespace mcb {

constexpr int kAugRowsPerLaunch = 64;   // rows travel as a kernel parameter (6 KB)
struct AugRows {
  mcb_augment_row r[kAugRowsPerLaunch];
};

// per-sample value range of every warped array, as uint32 pairs (0xFFFF - min, max) so that both reduce with
// atomicMax from a zeroed workspace: [sample][array: image, mask, distances, sizes][2]
__global__ void augment_range_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask,
                                     const uint16_t* __restrict__ dist, const uint16_t* __restrict__ size,
                                     const AugRows rows, int s0, unsigned* __restrict__ range, long hw) {
  const int j = blockIdx.y;
  if (!rows.r[j].warp) return;           // no warp, no clip
  const long s = s0 + j;
  unsigned lo[4] = {0xFFFFu, 0xFFFFu, 0xFFFFu, 0xFFFFu}, hi[4] = {0u, 0u, 0u, 0u};
  const uint8_t* im = img + s * hw * 3;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw * 3; q += (long)gridDim.x * blockDim.x) {
    const unsigned v = im[q];
    lo[0] = min(lo[0], v);
    hi[0] = max(hi[0], v);
  }
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw; q += (long)gridDim.x * blockDim.x) {
    const unsigned m = mask[s * hw + q];
    lo[1] = min(lo[1], m);
    hi[1] = max(hi[1], m);
    if (dist) {
      const unsigned d = dist[s * hw + q], z = size[s * hw + q];
      lo[2] = min(lo[2], d);
      hi[2] = max(hi[2], d);
      lo[3] = min(lo[3], z);
      hi[3] = max(hi[3], z);
    }
  }
  unsigned* rs = range + s * 8;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const unsigned l = __reduce_max_sync(0xFFFFFFFFu, 0xFFFFu - lo[a]);
    const unsigned h = __reduce_max_sync(0xFFFFFFFFu, hi[a]);
    if (lane == 0) {
      atomicMax(rs + 2 * a, l);
      atomicMax(rs + 2 * a + 1, h);
    }
  }
}

// skimage _clip_warp_output + imgaug's astype: clip to [lo, hi] (cval = 0 kept where lo > 0), truncate
__device__ __forceinline__ unsigned clip_trunc(double v, double lo, double hi) {
  if (lo > 0.0 && v == 0.0) return 0u;
  return (unsigned)(int)fmin(fmax(v, lo), hi);
}

// out[j][y][x] for every plane of sample s0 + j; img_out [n][oh][ow][3], tgt_out [n][oh][ow][T] (T = 3: mask,
// distances, sizes; T = 1: mask)
__global__ void augment_warp_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask,
                                    const uint16_t* __restrict__ dist, const uint16_t* __restrict__ size,
                                    const AugRows rows, int s0, const unsigned* __restrict__ range, int H, int W,
                                    int oh, int ow, uint8_t* __restrict__ img_out, uint8_t* __restrict__ tgt_out) {
  const int j = blockIdx.y;
  const long s = s0 + j;
  const mcb_augment_row& row = rows.r[j];
  const long hw = (long)H * W, ohw = (long)oh * ow;
  const int T = dist ? 3 : 1;
  const uint8_t* im = img + s * hw * 3;
  const uint8_t* mk = mask + s * hw;
  const uint16_t* ds = dist ? dist + s * hw : nullptr;
  const uint16_t* sz = dist ? size + s * hw : nullptr;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < ohw; q += (long)gridDim.x * blockDim.x) {
    int sy = (int)(q / ow) + row.top, sx = (int)(q % ow) + row.left;   // crop, then the post-warp flips
    if (row.post_flip & 1) sx = W - 1 - sx;
    if (row.post_flip & 2) sy = H - 1 - sy;
    uint8_t* io = img_out + (s * ohw + q) * 3;
    uint8_t* to = tgt_out + (s * ohw + q) * T;
    if (!row.warp) {
      if (row.pre_flip & 1) sx = W - 1 - sx;
      if (row.pre_flip & 2) sy = H - 1 - sy;
      const long p = (long)sy * W + sx;
      io[0] = im[p * 3];
      io[1] = im[p * 3 + 1];
      io[2] = im[p * 3 + 2];
      to[0] = mk[p];
      if (ds) {
        to[1] = (uint8_t)(ds[p] & 0xFFu);
        to[2] = (uint8_t)(sz[p] & 0xFFu);
      }
      continue;
    }
    // _transform_affine / _transform_projective (x = column, y = row of the output)
    const double* M = row.inv;
    const double x = (double)sx, y = (double)sy;
    double c = __dadd_rn(__dadd_rn(__dmul_rn(M[0], x), __dmul_rn(M[1], y)), M[2]);
    double r = __dadd_rn(__dadd_rn(__dmul_rn(M[3], x), __dmul_rn(M[4], y)), M[5]);
    if (!(M[6] == 0.0 && M[7] == 0.0 && M[8] == 1.0)) {
      const double z = __dadd_rn(__dadd_rn(__dmul_rn(M[6], x), __dmul_rn(M[7], y)), M[8]);
      c = __ddiv_rn(c, z);
      r = __ddiv_rn(r, z);
    }
    // bilinear_interpolation: floor / ceil neighbours, cval outside, weights from the unflipped position
    const double fr = floor(r), fc = floor(c);
    const long minr = (long)fr, minc = (long)fc, maxr = (long)ceil(r), maxc = (long)ceil(c);
    const double dr = __dsub_rn(r, (double)minr), dc = __dsub_rn(c, (double)minc);
    const double er = __dsub_rn(1.0, dr), ec = __dsub_rn(1.0, dc);
    const bool r0 = minr >= 0 && minr < H, r1 = maxr >= 0 && maxr < H;
    const bool c0 = minc >= 0 && minc < W, c1 = maxc >= 0 && maxc < W;
    const long yr0 = (row.pre_flip & 2) ? H - 1 - minr : minr, yr1 = (row.pre_flip & 2) ? H - 1 - maxr : maxr;
    const long xc0 = (row.pre_flip & 1) ? W - 1 - minc : minc, xc1 = (row.pre_flip & 1) ? W - 1 - maxc : maxc;
    const bool v00 = r0 && c0, v01 = r0 && c1, v10 = r1 && c0, v11 = r1 && c1;
    const long p00 = yr0 * W + xc0, p01 = yr0 * W + xc1, p10 = yr1 * W + xc0, p11 = yr1 * W + xc1;
    auto interp = [&](double tl, double tr, double bl, double br) {
      const double top = __dadd_rn(__dmul_rn(ec, tl), __dmul_rn(dc, tr));
      const double bottom = __dadd_rn(__dmul_rn(ec, bl), __dmul_rn(dc, br));
      return __dadd_rn(__dmul_rn(er, top), __dmul_rn(dr, bottom));
    };
    const unsigned* rs = range + s * 8;
    {
      const double lo = (double)(0xFFFFu - rs[0]), hi = (double)rs[1];
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const double v = interp(v00 ? (double)im[p00 * 3 + b] : 0.0, v01 ? (double)im[p01 * 3 + b] : 0.0,
                                v10 ? (double)im[p10 * 3 + b] : 0.0, v11 ? (double)im[p11 * 3 + b] : 0.0);
        io[b] = (uint8_t)clip_trunc(v, lo, hi);
      }
    }
    {
      const double v = interp(v00 ? (double)mk[p00] : 0.0, v01 ? (double)mk[p01] : 0.0, v10 ? (double)mk[p10] : 0.0,
                              v11 ? (double)mk[p11] : 0.0);
      to[0] = (uint8_t)clip_trunc(v, (double)(0xFFFFu - rs[2]), (double)rs[3]);
    }
    if (ds) {
      const double vd = interp(v00 ? (double)ds[p00] : 0.0, v01 ? (double)ds[p01] : 0.0, v10 ? (double)ds[p10] : 0.0,
                               v11 ? (double)ds[p11] : 0.0);
      to[1] = (uint8_t)(clip_trunc(vd, (double)(0xFFFFu - rs[4]), (double)rs[5]) & 0xFFu);   // uint16 -> uint8 wrap
      const double vs = interp(v00 ? (double)sz[p00] : 0.0, v01 ? (double)sz[p01] : 0.0, v10 ? (double)sz[p10] : 0.0,
                               v11 ? (double)sz[p11] : 0.0);
      to[2] = (uint8_t)(clip_trunc(vs, (double)(0xFFFFu - rs[6]), (double)rs[7]) & 0xFFu);
    }
  }
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int mcb_augment_warp(const uint8_t* img, const uint8_t* mask, const uint16_t* dist, const uint16_t* size,
                                const mcb_augment_row* rows, int n, int h, int w, int out_h, int out_w,
                                unsigned* range_ws, uint8_t* img_out, uint8_t* tgt_out, void* stream) {
  MCB_REQUIRE(img && mask && rows && range_ws && img_out && tgt_out, "augment_warp: null pointer");
  MCB_REQUIRE((dist == nullptr) == (size == nullptr), "augment_warp: distances and sizes come together");
  MCB_REQUIRE(n > 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0 && out_h <= h && out_w <= w,
              "augment_warp: bad shape (n %d, %dx%d -> %dx%d)", n, h, w, out_h, out_w);
  for (int i = 0; i < n; ++i) {
    const mcb_augment_row& r = rows[i];
    MCB_REQUIRE(r.warp == 0 || r.warp == 1, "augment_warp: row %d: warp %d", i, r.warp);
    MCB_REQUIRE((r.pre_flip & ~3) == 0 && (r.post_flip & ~3) == 0, "augment_warp: row %d: bad flip bits", i);
    MCB_REQUIRE(r.top >= 0 && r.left >= 0 && r.top + out_h <= h && r.left + out_w <= w,
                "augment_warp: row %d: crop (%d, %d) + %dx%d outside %dx%d", i, r.top, r.left, out_h, out_w, h, w);
  }
  const long hw = (long)h * w, ohw = (long)out_h * out_w;
  MCB_CHECK_CUDA(cudaMemsetAsync(range_ws, 0, sizeof(unsigned) * 8 * (size_t)n, ST));
  AugRows chunk;
  for (int s0 = 0; s0 < n; s0 += kAugRowsPerLaunch) {
    const int m = std::min(kAugRowsPerLaunch, n - s0);
    std::memcpy(chunk.r, rows + s0, sizeof(mcb_augment_row) * m);
    const int per_sample_r = (int)std::max(1L, std::min((hw * 3 + 255) / 256, (long)num_sms() * 4L / m + 1));
    augment_range_kernel<<<dim3(per_sample_r, m), 256, 0, ST>>>(img, mask, dist, size, chunk, s0, range_ws, hw);
    MCB_LAUNCH_CHECK();
    const int per_sample_w = (int)std::max(1L, std::min((ohw + 255) / 256, (long)num_sms() * 8L / m + 1));
    augment_warp_kernel<<<dim3(per_sample_w, m), 256, 0, ST>>>(img, mask, dist, size, chunk, s0, range_ws, h, w, out_h,
                                                              out_w, img_out, tgt_out);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}
