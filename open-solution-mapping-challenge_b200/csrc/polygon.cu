// polygon.cu — offline target preparation (src/preparation.py:18-198, overlay_masks) on the device:
//   * COCO polygon rasterisation, bit-exact to pycocotools' maskApi.c rleFrPoly + rleDecode (what the reference's
//     cocomask.frPyObjects(polys, h, w) followed by cocomask.decode computes);
//   * the per-instance bookkeeping of overlay_mask_one_image around it: plane statistics for the is_on_border test,
//     the erosion size gate and the distance-transform column ranges; the union of an image's kept instances per
//     category; the category overlay; the batched component-size map; the border class.
// The distance transform is input.cu's mcb_edt_two_nearest_batched, the morphology postproc.cu's
// mcb_binary_morph_rect, the labelling postproc.cu's mcb_ccl_label.  Integer / byte work; no tensor cores.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>
#include <climits>

namespace mcb {

// ------------------------------------------------------------------------------------------ rleFrPoly
// The host scales the vertices ((int)(5 x + .5), C truncation) and lays out one row per edge: edge_xy int32
// [E][4] = (xs, ys, xe, ye) of the closed polygon, edge_pt int64 [E + 1] = first upsampled point of every edge
// (max(|dx|, |dy|) + 1 points each, concatenated over all edges of all polygons), edge_plane int32 [E] = output plane.
// Point d of an edge is rleFrPoly's closed form; every product-plus-sum is rounded separately, as the C compiler of
// the reference evaluates it (no FMA contraction).
struct PolyPoint {
  long long u, v;
};
__device__ __forceinline__ PolyPoint edge_point(const int* __restrict__ edge_xy, int e, long long d) {
  long long xs = edge_xy[4 * e], ys = edge_xy[4 * e + 1], xe = edge_xy[4 * e + 2], ye = edge_xy[4 * e + 3];
  const long long dx = llabs(xe - xs), dy = llabs(ys - ye);
  const bool flip = (dx >= dy && xs > xe) || (dx < dy && ys > ye);
  if (flip) {
    long long t = xs; xs = xe; xe = t;
    t = ys; ys = ye; ye = t;
  }
  PolyPoint p;
  if (dx == 0 && dy == 0) {
    // s = 0.0 / 0 is NaN; x86's double -> int conversion (cvttsd2si) turns (int)NaN into INT_MIN
    p.u = xs;
    p.v = INT_MIN;
  } else if (dx >= dy) {
    const double s = __ddiv_rn((double)(ye - ys), (double)dx);
    const long long t = flip ? dx - d : d;
    p.u = t + xs;
    p.v = (int)__dadd_rn(__dadd_rn((double)ys, __dmul_rn(s, (double)t)), 0.5);
  } else {
    const double s = __ddiv_rn((double)(xe - xs), (double)dy);
    const long long t = flip ? dy - d : d;
    p.v = t + ys;
    p.u = (int)__dadd_rn(__dadd_rn((double)xs, __dmul_rn(s, (double)t)), 0.5);
  }
  return p;
}

// one thread per upsampled point j > 0 of a polygon: where u[j] != u[j-1] rleFrPoly records a column crossing
// (xd, yd) and the RLE toggles at the column-major position xd * h + yd; XOR-ing the toggles into a bit plane gives
// the RLE's run boundaries, duplicates cancelling as the zero-length runs merge in rleFrPoly.
__global__ void poly_crossings_kernel(const int* __restrict__ edge_xy, const long long* __restrict__ edge_pt,
                                      const int* __restrict__ edge_plane, int E, long long M,
                                      unsigned* __restrict__ bits, long long words, int h, int w) {
  const long long hw = (long long)h * w;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < M; g += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = E - 1;   // last edge with edge_pt[e] <= g
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (edge_pt[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const int e = lo;
    const long long d = g - edge_pt[e];
    const int plane = edge_plane[e];
    int ep = e;
    long long dp = d - 1;
    if (d == 0) {
      if (e == 0 || edge_plane[e - 1] != plane) continue;   // first point of its polygon
      ep = e - 1;
      dp = edge_pt[e] - edge_pt[e - 1] - 1;
    }
    const PolyPoint p1 = edge_point(edge_xy, e, d), p0 = edge_point(edge_xy, ep, dp);
    if (p1.u == p0.u) continue;
    double xd = (double)(p1.u < p0.u ? p1.u : p1.u - 1);
    xd = __dsub_rn(__ddiv_rn(__dadd_rn(xd, 0.5), 5.0), 0.5);
    if (floor(xd) != xd || xd < 0 || xd > w - 1) continue;
    double yd = (double)(p1.v < p0.v ? p1.v : p0.v);
    yd = __dsub_rn(__ddiv_rn(__dadd_rn(yd, 0.5), 5.0), 0.5);
    if (yd < 0) yd = 0;
    else if (yd > h) yd = h;
    yd = ceil(yd);
    const long long pos = (long long)xd * h + (long long)yd;
    if (pos >= hw) continue;   // y == h of the last column: past the plane
    atomicXor(bits + (long long)plane * words + (pos >> 5), 1u << (pos & 31));
  }
}

// inclusive XOR prefix over the bits of a word (bit 0 first)
__device__ __forceinline__ unsigned xor_prefix_bits(unsigned x) {
  x ^= x << 1;
  x ^= x << 2;
  x ^= x << 4;
  x ^= x << 8;
  x ^= x << 16;
  return x;
}

// rleDecode: one CTA per plane turns the toggle bits into mask bits in place by an XOR prefix over the whole
// column-major plane (not per column: a toggle at y == h lands on row 0 of the next column, as in maskApi).
constexpr int kScanThreads = 256;
__global__ void __launch_bounds__(kScanThreads) poly_scan_kernel(unsigned* __restrict__ bits, long long words) {
  __shared__ unsigned s_warp[kScanThreads / 32];
  unsigned* b = bits + (long long)blockIdx.x * words;
  const long long per = (words + kScanThreads - 1) / kScanThreads;
  const long long w0 = min(words, per * threadIdx.x), w1 = min(words, w0 + per);
  unsigned acc = 0;
  for (long long i = w0; i < w1; ++i) acc ^= b[i];
  const unsigned par = __popc(acc) & 1u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ball = __ballot_sync(0xffffffffu, par);
  unsigned carry = __popc(ball & ((1u << lane) - 1u)) & 1u;   // exclusive, within the warp
  if (lane == 0) s_warp[warp] = __popc(ball) & 1u;
  __syncthreads();
  for (int k = 0; k < warp; ++k) carry ^= s_warp[k];
  for (long long i = w0; i < w1; ++i) {
    unsigned x = xor_prefix_bits(b[i]);
    if (carry) x = ~x;
    b[i] = x;
    carry = x >> 31;
  }
}

// mask bits (column-major) -> uint8 plane [h][w] (row-major)
__global__ void poly_expand_kernel(const unsigned* __restrict__ bits, long long words, uint8_t* __restrict__ out,
                                   int h, int w) {
  const long long hw = (long long)h * w;
  const unsigned* b = bits + (long long)blockIdx.y * words;
  uint8_t* o = out + (long long)blockIdx.y * hw;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < hw; q += (long long)gridDim.x * blockDim.x) {
    const long long y = q / w, x = q % w;
    const long long pos = x * h + y;
    o[q] = (uint8_t)((b[pos >> 5] >> (pos & 31)) & 1u);
  }
}

// ------------------------------------------------------------------------------------------ per-plane statistics
// stats int32 [plane][4] = (pixel count, any pixel in [border : h - border, border : w - border] (not is_on_border),
// first column, last column with a pixel (w, -1 when empty)).  One CTA per plane.
constexpr int kStatThreads = 256;
__global__ void __launch_bounds__(kStatThreads) plane_stats_kernel(const uint8_t* __restrict__ planes,
                                                                   int* __restrict__ stats, int h, int w, int border) {
  __shared__ int s[4][kStatThreads / 32];
  const long long hw = (long long)h * w;
  const uint8_t* p = planes + (long long)blockIdx.x * hw;
  int area = 0, inner = 0, xmin = w, xmax = -1;
  for (long long q = threadIdx.x; q < hw; q += kStatThreads) {
    if (!p[q]) continue;
    const int y = (int)(q / w), x = (int)(q % w);
    ++area;
    inner |= (y >= border && y < h - border && x >= border && x < w - border);
    xmin = min(xmin, x);
    xmax = max(xmax, x);
  }
  for (int o = 16; o > 0; o >>= 1) {
    area += __shfl_xor_sync(0xffffffffu, area, o);
    inner |= __shfl_xor_sync(0xffffffffu, inner, o);
    xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
    xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s[0][warp] = area; s[1][warp] = inner; s[2][warp] = xmin; s[3][warp] = xmax; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < kStatThreads / 32; ++k) {
      area += s[0][k]; inner |= s[1][k]; xmin = min(xmin, s[2][k]); xmax = max(xmax, s[3][k]);
    }
    int* st = stats + 4 * (long long)blockIdx.x;
    st[0] = area; st[1] = inner; st[2] = xmin; st[3] = xmax;
  }
}

// ------------------------------------------------------------------------------------------ union, overlay
// out[g] = OR of planes index[off[g] .. off[g + 1]) (np.where(sum of the instances > 0, 1, 0).astype('uint8'))
__global__ void plane_union_kernel(const uint8_t* __restrict__ planes, const int* __restrict__ index,
                                   const int* __restrict__ off, uint8_t* __restrict__ out, long long hw) {
  const int g = blockIdx.y;
  const int k0 = off[g], k1 = off[g + 1];
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < hw; q += (long long)gridDim.x * blockDim.x) {
    uint8_t v = 0;
    for (int k = k0; k < k1 && !v; ++k) v = planes[(long long)index[k] * hw + q] != 0;
    out[(long long)g * hw + q] = v;
  }
}
// mask_overlayed = np.where(mask_c, category_nr[c], mask_overlayed) over the categories c in order;
// cat_masks uint8 [n][C][h][w] -> out uint8 [n][h][w]
__global__ void category_overlay_kernel(const uint8_t* __restrict__ cat_masks, const int* __restrict__ nr, int C,
                                        uint8_t* __restrict__ out, long long hw) {
  const int n = blockIdx.y;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < hw; q += (long long)gridDim.x * blockDim.x) {
    uint8_t v = 0;
    for (int c = 0; c < C; ++c)
      if (cat_masks[((long long)n * C + c) * hw + q]) v = (uint8_t)nr[c];
    out[(long long)n * hw + q] = v;
  }
}

// ------------------------------------------------------------------------------------------ sizes, border class
// get_size_matrix per plane from mcb_ccl_label's labels (1 .. count per plane): area is int32 workspace [n][h*w],
// zeroed by the caller
__global__ void label_area_kernel(const int* __restrict__ labels, int* __restrict__ area, long long hw) {
  const long long base = (long long)blockIdx.y * hw;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < hw; q += (long long)gridDim.x * blockDim.x) {
    const int l = labels[base + q];
    if (l > 0) atomicAdd(area + base + l - 1, 1);
  }
}
__global__ void size_from_area_kernel(const int* __restrict__ labels, const int* __restrict__ area,
                                      long long* __restrict__ out, long long hw) {
  const long long base = (long long)blockIdx.y * hw;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < hw; q += (long long)gridDim.x * blockDim.x) {
    const int l = labels[base + q];
    out[base + q] = l > 0 ? (long long)area[base + l - 1] : 1ll;
  }
}
// border class (src/preparation.py:83-86): (second_nearest < border_width) & (~mask_overlayed) is numpy's bitwise
// AND of a bool with the uint8 complement, so it holds where the class is even (background 0 included); the class id
// is the image's mask.max() + 1.  One CTA per image.
__global__ void __launch_bounds__(1024) border_class_kernel(uint8_t* __restrict__ mask, const double* __restrict__ second,
                                                            long long hw, double border_width) {
  __shared__ int s_max;
  uint8_t* m = mask + (long long)blockIdx.x * hw;
  const double* sn = second + (long long)blockIdx.x * hw;
  if (threadIdx.x == 0) s_max = 0;
  __syncthreads();
  int mx = 0;
  for (long long q = threadIdx.x; q < hw; q += blockDim.x) mx = max(mx, (int)m[q]);
  atomicMax(&s_max, mx);
  __syncthreads();
  const uint8_t cls = (uint8_t)(s_max + 1);
  for (long long q = threadIdx.x; q < hw; q += blockDim.x)
    if (sn[q] < border_width && !(m[q] & 1u)) m[q] = cls;
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

// grids put planes / images / groups on y; launches over more than kMaxGridY of them go in slices (gridDim.y <= 65535)
constexpr int kMaxGridY = 65535;
static dim3 plane_grid_poly(long long items, int planes, int threads) {
  const long long per = std::max(1LL, std::min((items + threads - 1) / threads,
                                               (long long)num_sms() * 8LL / std::max(planes, 1) + 1));
  return dim3((unsigned)per, (unsigned)planes, 1);
}

extern "C" int mcb_rasterize_polygons(const int* edge_xy, const long long* edge_pt, const int* edge_plane, int edges,
                                      long long points, unsigned* bits, uint8_t* out, int planes, int h, int w,
                                      void* stream) {
  MCB_REQUIRE(bits && out && planes > 0 && h > 0 && w > 0, "rasterize_polygons: bad argument");
  MCB_REQUIRE(edges >= 0 && points >= 0 && (edges == 0 || (edge_xy && edge_pt && edge_plane)),
              "rasterize_polygons: bad edge table");
  MCB_REQUIRE((long long)h * w < (1LL << 31), "rasterize_polygons: plane too large");
  const long long words = ((long long)h * w + 31) / 32;
  MCB_CHECK_CUDA(cudaMemsetAsync(bits, 0, (size_t)planes * words * sizeof(unsigned), ST));
  if (points > 0 && edges > 0) {
    const long long blocks = std::min((points + 255) / 256, (long long)num_sms() * 32);
    poly_crossings_kernel<<<(unsigned)blocks, 256, 0, ST>>>(edge_xy, edge_pt, edge_plane, edges, points, bits, words,
                                                            h, w);
    MCB_LAUNCH_CHECK();
  }
  poly_scan_kernel<<<planes, kScanThreads, 0, ST>>>(bits, words);
  MCB_LAUNCH_CHECK();
  for (int p0 = 0; p0 < planes; p0 += kMaxGridY) {
    const int cnt = std::min(kMaxGridY, planes - p0);
    poly_expand_kernel<<<plane_grid_poly((long long)h * w, cnt, 256), 256, 0, ST>>>(bits + (long long)p0 * words, words,
                                                                                   out + (long long)p0 * h * w, h, w);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_plane_stats(const uint8_t* planes, int count, int h, int w, int border, int* stats, void* stream) {
  MCB_REQUIRE(planes && stats && count > 0 && h > 0 && w > 0 && border >= 0, "plane_stats: bad argument");
  plane_stats_kernel<<<count, kStatThreads, 0, ST>>>(planes, stats, h, w, border);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_plane_union(const uint8_t* planes, const int* index, const int* group_off, int groups, int h, int w,
                               uint8_t* out, void* stream) {
  MCB_REQUIRE(planes && index && group_off && out && groups > 0 && h > 0 && w > 0, "plane_union: bad argument");
  const long long hw = (long long)h * w;
  for (int g0 = 0; g0 < groups; g0 += kMaxGridY) {
    const int cnt = std::min(kMaxGridY, groups - g0);
    plane_union_kernel<<<plane_grid_poly(hw, cnt, 256), 256, 0, ST>>>(planes, index, group_off + g0, out + g0 * hw, hw);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_category_overlay(const uint8_t* cat_masks, const int* category_nr, int categories, int n, int h,
                                    int w, uint8_t* out, void* stream) {
  MCB_REQUIRE(cat_masks && category_nr && out && categories > 0 && n > 0 && h > 0 && w > 0,
              "category_overlay: bad argument");
  const long long hw = (long long)h * w;
  for (int n0 = 0; n0 < n; n0 += kMaxGridY) {
    const int cnt = std::min(kMaxGridY, n - n0);
    category_overlay_kernel<<<plane_grid_poly(hw, cnt, 256), 256, 0, ST>>>(cat_masks + n0 * categories * hw, category_nr,
                                                                          categories, out + n0 * hw, hw);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_size_matrix_batched(const int* labels, int* area_ws, long long* out, int n, int h, int w,
                                       void* stream) {
  MCB_REQUIRE(labels && area_ws && out && n > 0 && h > 0 && w > 0, "size_matrix_batched: bad argument");
  const long long hw = (long long)h * w;
  MCB_CHECK_CUDA(cudaMemsetAsync(area_ws, 0, (size_t)n * hw * sizeof(int), ST));
  for (int n0 = 0; n0 < n; n0 += kMaxGridY) {
    const int cnt = std::min(kMaxGridY, n - n0);
    const dim3 grid = plane_grid_poly(hw, cnt, 256);
    label_area_kernel<<<grid, 256, 0, ST>>>(labels + n0 * hw, area_ws + n0 * hw, hw);
    MCB_LAUNCH_CHECK();
    size_from_area_kernel<<<grid, 256, 0, ST>>>(labels + n0 * hw, area_ws + n0 * hw, out + n0 * hw, hw);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_border_class(uint8_t* mask, const double* second_nearest, int n, int h, int w, double border_width,
                                void* stream) {
  MCB_REQUIRE(mask && second_nearest && n > 0 && h > 0 && w > 0, "border_class: bad argument");
  border_class_kernel<<<n, 1024, 0, ST>>>(mask, second_nearest, (long long)h * w, border_width);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
