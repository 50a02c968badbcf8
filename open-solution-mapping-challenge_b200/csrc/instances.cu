// instances.cu — the steps on either side of the per-pixel chain (SURVEY.md 8f-2, 8f-3) plus categorize_image:
//   * categorize_image (src/postprocessing.py:64-74): np.argmax over the channel axis;
//   * test-time augmentation (src/loaders.py:401-517): the 16 flip / rot90 variants as index maps, and the aggregator
//     fused with the class softmax and the inverse index map (no inverse-transformed copies are materialised);
//   * instance emission (src/utils.py:61-127): per-label area, bounding box and COCO run-length encoding
//     (pycocotools rleEncode / rleToBbox semantics, restated in oracle/instances_oracle.py), the pairwise IoU matrix of
//     the non-maximum suppression step (src/postprocessing.py:355-386) and the per-mask features of the scoring model
//     (src/postprocessing.py:284-306).
// All of it is HBM/L2-bound integer work: coalesced row-major reads, one plane (image, layer) per blockIdx.y or one
// warp per instance walking its bounding box.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>

namespace mcb {

// ------------------------------------------------------------------------------------------ categorize_image
// numpy argmax: index of the FIRST maximum; a NaN compares as the maximum (first NaN wins).
template <typename T>
__global__ void argmax_channels_kernel(const T* __restrict__ prob, long long* __restrict__ out, int C, long hw,
                                       int img0) {
  const int img = img0 + blockIdx.y;
  const T* p = prob + (long)img * C * hw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < hw; i += (long)gridDim.x * blockDim.x) {
    T best = p[i];
    int arg = 0;
    bool is_nan = best != best;
    for (int c = 1; c < C && !is_nan; ++c) {
      const T v = p[(long)c * hw + i];
      if (v != v) { arg = c; is_nan = true; }
      else if (v > best) { best = v; arg = c; }
    }
    out[(long)img * hw + i] = arg;
  }
}

// ------------------------------------------------------------------------------------------ test-time augmentation
// variant code: bits 0-1 = k (rotation by 90*k degrees counter-clockwise, np.rot90 convention), bits 2-3 = flip
// (0 none, 1 up-down, 2 left-right; the reference's `if ud ... elif lr` means a spec with both set applies ud only,
// src/loaders.py:471-474 — the host encodes that).  Forward: y = rot90(flip(x), k).
// Source coordinate of output pixel (i, j) of rot90(m, k), m of shape (H, W):
//   k=0: m[i, j]   k=1: m[j, W-1-i]   k=2: m[H-1-i, W-1-j]   k=3: m[H-1-j, i]
__device__ __forceinline__ void rot90_src(int k, int i, int j, int H, int W, int& si, int& sj) {
  switch (k & 3) {
    case 0: si = i; sj = j; break;
    case 1: si = j; sj = W - 1 - i; break;
    case 2: si = H - 1 - i; sj = W - 1 - j; break;
    default: si = H - 1 - j; sj = i; break;
  }
}

// source pixel (si, sj) of output pixel (i, j) of the variant with geometry code `cd` (bits 0-3) of an (H, W) image
__device__ __forceinline__ void tta_src(int cd, int i, int j, int H, int W, int& si, int& sj) {
  const int k = cd & 3, flip = (cd >> 2) & 3;
  rot90_src(k, i, j, H, W, si, sj);          // into the flipped image (H, W)
  if (flip == 1) si = H - 1 - si;
  else if (flip == 2) sj = W - 1 - sj;
}

// x [n][c][h][w] -> out [nv][c][ho][wo], (ho, wo) = (h, w) or (w, h) for odd k (square images keep their shape)
__global__ void tta_transform_kernel(const float* __restrict__ x, float* __restrict__ out, const int* __restrict__ img_of,
                                     const int* __restrict__ code, int C, int H, int W, int v0) {
  const int v = v0 + blockIdx.y;
  const int cd = code[v];
  const int k = cd & 3;
  const int Ho = (k & 1) ? W : H, Wo = (k & 1) ? H : W;
  const float* src = x + (long)img_of[v] * C * H * W;
  float* dst = out + (long)v * C * H * W;
  const long total = (long)C * H * W;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < total; q += (long)gridDim.x * blockDim.x) {
    const int c = q / ((long)Ho * Wo);
    const int r = q % ((long)Ho * Wo);
    const int i = r / Wo, j = r % Wo;
    int si, sj;
    tta_src(cd, i, j, H, W, si, sj);
    dst[q] = src[((long)c * H + si) * W + sj];
  }
}

// color_seq (src/augmentation.py:12-31, imgaug 0.2.5) on one uint8 RGB pixel.  branch 1-3: cv2 RGB2HSV (H in 0..179),
// Add `value` to channel branch-1 clipped at 255 (H too: imgaug clips at the dtype's maximum, not at 180), cv2 HSV2RGB;
// branch 4-6: Add `value` to R, G or B clipped at 255.
// RGB2HSV is cv2's integer path (12-bit fixed-point reciprocal tables; the rint of the division is taken here in integer
// arithmetic, which has no ties for these operands).  HSV2RGB is the map of cv2's AVX2 vector body (OpenCV 4.x
// HSV2RGB_b), derived by an exhaustive probe over all 2^24 inputs: fp32, the two `1 - s·t` terms fused (one rounding),
// every other product and difference rounded on its own, the result ×255 truncated.  The explicit __f*_rn intrinsics
// keep nvcc from contracting any other pair into an FMA.  cv2's scalar tail (the last columns of a row that do not fill
// a vector) rounds instead of truncating; DESIGN.md §4.5.
__device__ __forceinline__ void color_shift_px(int branch, int value, int& r, int& g, int& b) {
  if (branch >= 4) {
    if (branch == 4) r = min(255, r + value);
    else if (branch == 5) g = min(255, g + value);
    else b = min(255, b + value);
    return;
  }
  const int v = max(r, max(g, b));
  const int diff = v - min(r, min(g, b));
  const int sdiv = v ? ((255 << 13) + v) / (2 * v) : 0;                 // rint((255 << 12) / v)
  const int hdiv = diff ? ((180 << 13) + 6 * diff) / (12 * diff) : 0;   // rint((180 << 12) / (6 diff))
  const int num = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  int hh = (num * hdiv + 2048) >> 12, ss = (diff * sdiv + 2048) >> 12, vi = v;
  if (hh < 0) hh += 180;
  if (branch == 1) hh = min(255, hh + value);
  else if (branch == 2) ss = min(255, ss + value);
  else vi = min(255, vi + value);
  const float h = __fmul_rn((float)hh, 6.f / 180.f);
  const float s = __fmul_rn((float)ss, 1.f / 255.f);
  const float vv = __fmul_rn((float)vi, 1.f / 255.f);
  const float pre = truncf(h);
  const float f = __fsub_rn(h, pre);
  const float t1 = __fmul_rn(vv, __fsub_rn(1.f, s));
  const float t2 = __fmul_rn(vv, __fmaf_rn(-s, f, 1.f));
  const float t3 = __fmul_rn(vv, __fmaf_rn(-s, __fsub_rn(1.f, f), 1.f));
  const int sector = (int)pre - 6 * (int)truncf(__fmul_rn(pre, 1.f / 6.f));   // H up to 255 wraps: 200 = 20 (mod 180)
  // cv2's sector table {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0}: (b, g, r) picks from (vv, t1, t2, t3)
  const float fb = sector < 2 ? t1 : (sector == 2 ? t3 : (sector <= 4 ? vv : t2));
  const float fg = sector == 0 ? t3 : (sector <= 2 ? vv : (sector == 3 ? t2 : t1));
  const float fr = (sector == 0 || sector == 5) ? vv : (sector == 1 ? t2 : (sector == 4 ? t3 : t1));
  b = min(255, (int)__fmul_rn(fb, 255.f));
  g = min(255, (int)__fmul_rn(fg, 255.f));
  r = min(255, (int)__fmul_rn(fr, 255.f));
}

// The variant rows of the TTA loaders (MetadataImageSegmentationTTA.__getitem__ + test_time_augmentation_transform,
// src/loaders.py:94-111,477-487) on the decoded tiles: img uint8 [n][h][w][3] -> out uint8 [nv][h][w][3], row v from
// tile src[v].  code[v] = geometry (bits 0-3, as tta_transform_kernel) | colour branch << 4 | value << 8.  Colour is
// per pixel, so applying it at the source pixel equals the reference's colour-then-rotate order.  One thread per output
// pixel: 3 B in, 3 B out.
__global__ void tta_variants_u8_kernel(const uint8_t* __restrict__ img, uint8_t* __restrict__ out,
                                       const int* __restrict__ src, const int* __restrict__ code, int H, int W, int v0) {
  const int v = v0 + blockIdx.y;
  const int cd = code[v];
  const int branch = (cd >> 4) & 7, value = (cd >> 8) & 255;
  const int Wo = (cd & 1) ? H : W;
  const long hw = (long)H * W;
  const uint8_t* s = img + (long)src[v] * hw * 3;
  uint8_t* d = out + (long)v * hw * 3;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw; q += (long)gridDim.x * blockDim.x) {
    const int i = q / Wo, j = q % Wo;
    int si, sj;
    tta_src(cd, i, j, H, W, si, sj);
    const uint8_t* p = s + ((long)si * W + sj) * 3;
    int r = p[0], g = p[1], b = p[2];
    if (branch) color_shift_px(branch, value, r, g, b);
    d[q * 3] = (uint8_t)r;
    d[q * 3 + 1] = (uint8_t)g;
    d[q * 3 + 2] = (uint8_t)b;
  }
}

// Aggregation of the predictions of all variants of one image (TestTimeAugmentationAggregator.transform +
// test_time_augmentation_inverse_transform, src/loaders.py:437-497): inverse = flip(rot90(p, -k)), then
// gmean / mean / max / min over the variants.  pred [nv][c][h][w] are class probabilities, or logits when
// `from_logits` (the softmax over c is then taken here, in registers).  var_start [n+1] / var_index [nv] list the
// variants of each image.  Square maps for odd k.  method: 0 gmean, 1 mean, 2 max, 3 min.
constexpr int kTtaMaxC = 8;
__global__ void tta_aggregate_kernel(const float* __restrict__ pred, int from_logits, const int* __restrict__ var_start,
                                     const int* __restrict__ var_index, const int* __restrict__ code,
                                     float* __restrict__ out, int C, int H, int W, int method, int img0) {
  const int img = img0 + blockIdx.y;
  const int vb = var_start[img], ve = var_start[img + 1];
  const long hw = (long)H * W;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw; q += (long)gridDim.x * blockDim.x) {
    const int y = q / W, x = q % W;
    double acc[kTtaMaxC];
    for (int c = 0; c < C; ++c) acc[c] = (method == 2) ? -INFINITY : (method == 3 ? INFINITY : 0.0);
    for (int vi = vb; vi < ve; ++vi) {
      const int v = var_index[vi];
      const int cd = code[v];
      const int k = cd & 3, flip = (cd >> 2) & 3;
      // result R = F(Q), Q = rot90(P, -k): R[y, x] = Q[fy, fx]; Q[i, j] = P[source of rot90 by (4 - k)]
      int fy = y, fx = x;
      if (flip == 1) fy = H - 1 - y;
      else if (flip == 2) fx = W - 1 - x;
      int si, sj;
      const int Hp = (k & 1) ? W : H, Wp = (k & 1) ? H : W;   // shape of P (the variant's frame)
      rot90_src((4 - k) & 3, fy, fx, Hp, Wp, si, sj);
      const float* p = pred + (long)v * C * hw + (long)si * Wp + sj;
      float pv[kTtaMaxC];
      for (int c = 0; c < C; ++c) pv[c] = p[(long)c * hw];
      if (from_logits) {
        float m = pv[0];
        for (int c = 1; c < C; ++c) m = fmaxf(m, pv[c]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) { pv[c] = expf(pv[c] - m); s += pv[c]; }
        for (int c = 0; c < C; ++c) pv[c] = pv[c] / s;          // float32 probabilities, like utils.softmax
      }
      for (int c = 0; c < C; ++c) {
        const double t = (double)pv[c];
        if (method == 0) acc[c] += log(t);
        else if (method == 1) acc[c] += t;
        else if (method == 2) acc[c] = fmax(acc[c], t);
        else acc[c] = fmin(acc[c], t);
      }
    }
    const double inv = 1.0 / (double)max(ve - vb, 1);
    for (int c = 0; c < C; ++c) {
      double r = acc[c];
      if (method == 0) r = exp(r * inv);
      else if (method == 1) r = r * inv;
      out[((long)img * C + c) * hw + q] = (float)r;
    }
  }
}

// ------------------------------------------------------------------------------------------ instance geometry
// One pass over the label planes: per instance (slot = offsets[plane] + label - 1) the pixel count, the tight
// bounding box and the probability sum / maximum (FeatureExtractor: area, mean_prob, max_prob, get_bbox).  Threads walk
// contiguous row segments and flush once per label change.  geo: int32 [total][5] = {area, rmin, rmax, cmin, cmax}
// (initialised by the caller to {0, INT_MAX, -1, INT_MAX, -1}); psum fp64 [total]; pmax int64 [total], the
// order-preserving integer image of the fp64 maximum.  The maximum is kept in fp64 for both input types: the reference
// takes it over skimage's float64 resize, and an fp32 input widens exactly, so one path serves both.
__device__ __forceinline__ long long double_to_ordered(double d) {
  const long long i = __double_as_longlong(d);
  return i >= 0 ? i : i ^ 0x7FFFFFFFFFFFFFFFLL;
}

template <typename T>
__global__ void __launch_bounds__(256) instance_geometry_kernel(const int* __restrict__ labels, const T* __restrict__ prob,
                                                                const int* __restrict__ offsets,
                                                                const int* __restrict__ counts, int* __restrict__ geo,
                                                                double* __restrict__ psum, long long* __restrict__ pmax,
                                                                int H, int W, int seg, int plane0) {
  const int plane = plane0 + blockIdx.y;
  const int off = offsets[plane], K = counts[plane];
  const long hw = (long)H * W;
  const int* L = labels + (long)plane * hw;
  const T* P = prob ? prob + (long)plane * hw : nullptr;
  const int segs_per_row = (W + seg - 1) / seg;
  const long nseg = (long)H * segs_per_row;
  for (long sidx = blockIdx.x * (long)blockDim.x + threadIdx.x; sidx < nseg; sidx += (long)gridDim.x * blockDim.x) {
    const int r = sidx / segs_per_row;
    const int c0 = (int)(sidx % segs_per_row) * seg, c1 = min(W, c0 + seg);
    int cur = 0, cnt = 0, cs = 0;
    double sum = 0.0;
    double mx = -INFINITY;
    auto flush = [&](int cend) {
      if (cur > 0 && cur <= K) {
        int* g = geo + (long)(off + cur - 1) * 5;
        atomicAdd(g, cnt);
        atomicMin(g + 1, r);
        atomicMax(g + 2, r);
        atomicMin(g + 3, cs);
        atomicMax(g + 4, cend);
        if (P) { atomicAdd(psum + off + cur - 1, sum); atomicMax(pmax + off + cur - 1, double_to_ordered(mx)); }
      }
    };
    for (int c = c0; c < c1; ++c) {
      const int l = __ldg(L + (long)r * W + c);
      if (l != cur) {
        flush(c - 1);
        cur = l; cnt = 0; cs = c; sum = 0.0; mx = -INFINITY;
      }
      if (l > 0) {
        ++cnt;
        if (P) { const double pv = (double)__ldg(P + (long)r * W + c); sum += pv; mx = fmax(mx, pv); }
      }
    }
    flush(c1 - 1);
  }
}

// ------------------------------------------------------------------------------------------ COCO run-length encoding
// pycocotools rleEncode walks the mask in COLUMN-major order (Fortran order, src/utils.py:118-120) and emits the
// lengths of alternating runs, starting with a (possibly empty) run of zeros.  Equivalently: the sorted list of
// positions p (column-major, p = x*H + y) where the mask value differs from the value at p-1 (value 0 before the
// start); counts = differences of consecutive change positions, closed by H*W - last.
// The columns of an instance's bounding box [cmin, cmax] x [rmin, rmax] are INDEPENDENT tasks (one warp each, 32 rows
// per step): the scan's state on entering column x is 0 unless the box spans the full image height, in which case it
// is the instance's value at (H-1, x-1) -- one extra load, no serial dependency between columns (the background layer
// of every image is one instance as large as the image; walking its 300 columns serially took 1 ms).  A run that is
// still on at the last box row of a column ends at x*H + rmax + 1 unless the box spans the full height (then the next
// column's first pixel decides).  task_slot / task_x list the (instance, column) tasks in (instance, column) order, so
// change positions come out sorted.  Pass 1 (write == 0) counts the changes of each task, pass 2 writes them at
// task_start[t].  spans[slot] is set when a run of ones covers more than one column (rleToBbox then reports the full
// height).
__global__ void __launch_bounds__(128) rle_walk_kernel(const int* __restrict__ labels, const int* __restrict__ offsets,
                                                       const int* __restrict__ geo, const int* __restrict__ inst_plane,
                                                       const int* __restrict__ task_slot, const int* __restrict__ task_x,
                                                       const int* __restrict__ task_start, int* __restrict__ task_n,
                                                       int* __restrict__ changes, int* __restrict__ spans, int ntasks, int H,
                                                       int W, int write) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= ntasks) return;
  const int slot = task_slot[t], x = task_x[t];
  const int plane = inst_plane[slot];
  const int lab = slot - offsets[plane] + 1;
  const int* g = geo + (long)slot * 5;
  const int rmin = g[1], rmax = g[2], cmax = g[4];
  const bool full = (rmin == 0 && rmax == H - 1);
  const int* L = labels + (long)plane * H * W;
  int* dst = write ? changes + task_start[t] : nullptr;
  uint32_t carry = (full && x > 0) ? (uint32_t)(__ldg(L + (long)(H - 1) * W + (x - 1)) == lab) : 0u;
  int n = 0;
  for (int y0 = rmin; y0 <= rmax; y0 += 32) {
    const int y = y0 + lane;
    const bool on = (y <= rmax) && (__ldg(L + (long)y * W + x) == lab);
    const uint32_t bits = __ballot_sync(0xffffffffu, on);
    const int valid = min(32, rmax - y0 + 1);
    const uint32_t vmask = valid == 32 ? 0xffffffffu : ((1u << valid) - 1u);
    const uint32_t flips = (bits ^ ((bits << 1) | carry)) & vmask;
    if (write && ((flips >> lane) & 1u)) dst[n + __popc(flips & ((1u << lane) - 1u))] = x * H + y;
    // still on at the top of a column whose entry state is on: this run of ones started in an earlier column
    if (write && y0 == rmin && carry && (bits & 1u) && lane == 0) spans[slot] = 1;
    n += __popc(flips);
    carry = (bits >> (valid - 1)) & 1u;
  }
  // a run still on at the bottom of the box: it ends right below unless the scan continues into the next column
  // (full-height box, not the last column of the box) or the image ends here
  if (carry) {
    const bool continues = full && x < cmax;                 // the next column task sees it as its entry state
    const bool image_end = (x == W - 1 && rmax == H - 1);
    if (!continues && !image_end) {
      if (write && lane == 0) dst[n] = x * H + rmax + 1;
      ++n;
    }
  }
  if (!write && lane == 0) task_n[t] = n;
}

// counts from change positions: cnt[0] = p0, cnt[i] = p_i - p_{i-1}, cnt[n] = H*W - p_{n-1}  (n + 1 counts per instance;
// an empty instance gives the single count H*W).  One thread per output count.
__global__ void rle_counts_kernel(const int* __restrict__ changes, const int* __restrict__ nchanges,
                                  const int* __restrict__ out_start, const int* __restrict__ slot_of_count,
                                  uint32_t* __restrict__ cnts, long total_counts, int HW) {
  const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (i >= total_counts) return;
  const int slot = slot_of_count[i];
  // counts of slot s start at out_start[s] + s (one more count than changes per instance)
  const int first = out_start[slot] + slot;
  const int j = (int)(i - first);
  const int n = nchanges[slot];
  const int* p = changes + out_start[slot];
  const int hi = (j < n) ? p[j] : HW;
  const int lo = (j > 0) ? p[j - 1] : 0;
  cnts[i] = (uint32_t)(hi - lo);
}

// ------------------------------------------------------------------------------------------ non-maximum suppression
// Intersection counts between the instances of two label planes of the same image (remove_overlapping_masks compares
// every pair of instances of ALL layers of an image, src/postprocessing.py:355-386; instances of one layer never
// overlap).  inter [Ka][Kb] int32, zeroed by the caller; run-compressed like the geometry pass.
__global__ void __launch_bounds__(256) pair_intersection_kernel(const int* __restrict__ la, const int* __restrict__ lb,
                                                                int* __restrict__ inter, int Ka, int Kb, long hw,
                                                                int chunk) {
  const long b = ((long)blockIdx.x * blockDim.x + threadIdx.x) * chunk;
  const long e = min(hw, b + chunk);
  int ca = 0, cb = 0, cnt = 0;
  for (long i = b; i < e; ++i) {
    const int a = __ldg(la + i), bb = __ldg(lb + i);
    if (a != ca || bb != cb) {
      if (ca > 0 && cb > 0 && ca <= Ka && cb <= Kb && cnt) atomicAdd(inter + (long)(ca - 1) * Kb + (cb - 1), cnt);
      ca = a; cb = bb; cnt = 0;
    }
    ++cnt;
  }
  if (ca > 0 && cb > 0 && ca <= Ka && cb <= Kb && cnt) atomicAdd(inter + (long)(ca - 1) * Kb + (cb - 1), cnt);
}

// ------------------------------------------------------------------------------------------ contour length
// get_contour_length (src/postprocessing.py:340-352): cv2.findContours(RETR_TREE, CHAIN_APPROX_NONE) + drawContours
// with thickness 1 marks exactly the mask pixels that have a 4-neighbour outside the mask (image border counts as
// outside) -- outer and hole borders alike; the count of marked pixels per instance.  Pinned against cv2 itself in
// tests/test_oracle_pins.py.
__global__ void __launch_bounds__(256) contour_length_kernel(const int* __restrict__ labels,
                                                             const int* __restrict__ offsets,
                                                             const int* __restrict__ counts, int* __restrict__ clen,
                                                             int H, int W, int plane0) {
  const int plane = plane0 + blockIdx.y;
  const int off = offsets[plane], K = counts[plane];
  const long hw = (long)H * W;
  const int* L = labels + (long)plane * hw;
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < hw; q += (long)gridDim.x * blockDim.x) {
    const int l = L[q];
    if (l <= 0 || l > K) continue;
    const int y = q / W, x = q % W;
    const bool edge = y == 0 || x == 0 || y == H - 1 || x == W - 1 || L[q - W] != l || L[q + W] != l || L[q - 1] != l ||
                      L[q + 1] != l;
    if (edge) atomicAdd(clen + off + l - 1, 1);
  }
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

// grids put planes / images / variants on y; launches over more than kMaxGridY of them go in slices
// (gridDim.y <= 65535), each kernel adding its slice's first index to blockIdx.y
constexpr int kMaxGridY = 65535;
static dim3 grid2(long items, int planes, int threads) {
  const int per_plane =
      (int)std::max(1L, std::min((items + threads - 1) / threads, (long)num_sms() * 8L / std::max(planes, 1) + 1));
  return dim3(per_plane, planes, 1);
}

extern "C" int mcb_argmax_channels(const void* prob, int prob_is_f64, long long* out, int n, int c, int h, int w,
                                   void* stream) {
  MCB_REQUIRE(prob && out && n > 0 && c > 0 && h > 0 && w > 0, "argmax: bad argument");
  const long hw = (long)h * w;
  for (int i0 = 0; i0 < n; i0 += kMaxGridY) {
    const dim3 grid = grid2(hw, std::min(kMaxGridY, n - i0), 256);
    if (prob_is_f64) argmax_channels_kernel<double><<<grid, 256, 0, ST>>>((const double*)prob, out, c, hw, i0);
    else argmax_channels_kernel<float><<<grid, 256, 0, ST>>>((const float*)prob, out, c, hw, i0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_tta_transform(const float* x, float* out, const int* img_of, const int* code, int nv, int c, int h,
                                 int w, void* stream) {
  MCB_REQUIRE(x && out && img_of && code && nv > 0 && c > 0, "tta_transform: bad argument");
  for (int v0 = 0; v0 < nv; v0 += kMaxGridY) {
    tta_transform_kernel<<<grid2((long)c * h * w, std::min(kMaxGridY, nv - v0), 256), 256, 0, ST>>>(x, out, img_of, code,
                                                                                                  c, h, w, v0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_tta_variants_u8(const uint8_t* images, uint8_t* out, const int* src, const int* code, int nv, int h,
                                   int w, void* stream) {
  MCB_REQUIRE(images && out && src && code && nv > 0 && h > 0 && w > 0, "tta_variants_u8: bad argument");
  for (int v0 = 0; v0 < nv; v0 += kMaxGridY) {
    tta_variants_u8_kernel<<<grid2((long)h * w, std::min(kMaxGridY, nv - v0), 256), 256, 0, ST>>>(images, out, src, code,
                                                                                                h, w, v0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_tta_aggregate(const float* pred, int from_logits, const int* var_start, const int* var_index,
                                 const int* code, float* out, int n, int c, int h, int w, int method, void* stream) {
  MCB_REQUIRE(pred && var_start && var_index && code && out && n > 0, "tta_aggregate: null pointer");
  MCB_REQUIRE(c >= 1 && c <= kTtaMaxC, "tta_aggregate: %d classes (max %d)", c, kTtaMaxC);
  MCB_REQUIRE(method >= 0 && method <= 3, "tta_aggregate: method %d", method);
  for (int i0 = 0; i0 < n; i0 += kMaxGridY) {
    tta_aggregate_kernel<<<grid2((long)h * w, std::min(kMaxGridY, n - i0), 256), 256, 0, ST>>>(
        pred, from_logits, var_start, var_index, code, out, c, h, w, method, i0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_instance_geometry(const int* labels, const void* prob, int prob_is_f64, const int* offsets,
                                     const int* counts, int* geo, double* psum, long long* pmax, int planes, int h,
                                     int w, void* stream) {
  MCB_REQUIRE(labels && offsets && counts && geo, "instance_geometry: null pointer");
  MCB_REQUIRE(!prob || (psum && pmax), "instance_geometry: prob needs psum and pmax");
  const int seg = 32;
  const long nseg = (long)h * ((w + seg - 1) / seg);
  for (int p0 = 0; p0 < planes; p0 += kMaxGridY) {
    const dim3 grid = grid2(nseg, std::min(kMaxGridY, planes - p0), 256);
    if (prob && prob_is_f64)
      instance_geometry_kernel<double><<<grid, 256, 0, ST>>>(labels, (const double*)prob, offsets, counts, geo, psum,
                                                             pmax, h, w, seg, p0);
    else
      instance_geometry_kernel<float><<<grid, 256, 0, ST>>>(labels, (const float*)prob, offsets, counts, geo, psum, pmax,
                                                            h, w, seg, p0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_rle_walk(const int* labels, const int* offsets, const int* geo, const int* inst_plane,
                            const int* task_slot, const int* task_x, const int* task_start, int* task_n, int* changes,
                            int* spans, int ntasks, int h, int w, int write, void* stream) {
  if (ntasks <= 0) return MCB_OK;   // every instance empty: nothing to walk
  MCB_REQUIRE(labels && offsets && geo && inst_plane && task_slot && task_x && task_n, "rle_walk: null pointer");
  MCB_REQUIRE(!write || (task_start && changes && spans), "rle_walk: write pass needs task_start, changes, spans");
  MCB_REQUIRE((long)h * w < (1L << 31), "rle_walk: plane too large");
  if (ntasks <= 0) return MCB_OK;
  const int warps_per_block = 4;
  rle_walk_kernel<<<(ntasks + warps_per_block - 1) / warps_per_block, 32 * warps_per_block, 0, ST>>>(
      labels, offsets, geo, inst_plane, task_slot, task_x, task_start, task_n, changes, spans, ntasks, h, w, write);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_rle_counts(const int* changes, const int* nchanges, const int* out_start, const int* slot_of_count,
                              uint32_t* cnts, long total_counts, int hw, void* stream) {
  MCB_REQUIRE(nchanges && out_start && slot_of_count && cnts, "rle_counts: null pointer");
  if (total_counts <= 0) return MCB_OK;
  rle_counts_kernel<<<(unsigned)((total_counts + 255) / 256), 256, 0, ST>>>(changes, nchanges, out_start, slot_of_count,
                                                                         cnts, total_counts, hw);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_pair_intersections(const int* labels_a, const int* labels_b, int* inter, int ka, int kb, int h, int w,
                                      void* stream) {
  MCB_REQUIRE(labels_a && labels_b && inter, "pair_intersections: null pointer");
  if (ka <= 0 || kb <= 0) return MCB_OK;
  const long hw = (long)h * w;
  const int chunk = 64;
  const long threads = (hw + chunk - 1) / chunk;
  pair_intersection_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, ST>>>(labels_a, labels_b, inter, ka, kb, hw, chunk);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_contour_length(const int* labels, const int* offsets, const int* counts, int* clen, int planes, int h,
                                  int w, void* stream) {
  MCB_REQUIRE(labels && offsets && counts && clen, "contour_length: null pointer");
  for (int p0 = 0; p0 < planes; p0 += kMaxGridY) {
    contour_length_kernel<<<grid2((long)h * w, std::min(kMaxGridY, planes - p0), 256), 256, 0, ST>>>(labels, offsets,
                                                                                                   counts, clen, h, w, p0);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}
