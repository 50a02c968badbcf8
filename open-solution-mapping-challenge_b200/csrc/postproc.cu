// postproc.cu — the per-pixel mask post-processing of src/postprocessing.py:48-258 as batched CUDA kernels.
// Everything here is HBM/L2-bound integer or stencil work (no tensor cores): coalesced row-major accesses, one image
// per blockIdx.y, grids sized from the SM count.  Semantics follow the oracle (oracle/post_oracle.py) bit-for-bit for
// every integer/bool output and for the float64 resize.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>

namespace mcb {

static inline int blocks_for(long items, int threads) { return (int)std::max(1L, (items + threads - 1) / threads); }

// ------------------------------------------------------------------------------------------ resize (P1)
// skimage.transform.resize n-D branch == scipy map_coordinates(order=1, mode='constant', cval=0) on float64:
// coordinate c = (in/out)*(i+0.5)-0.5 per axis; output is cval when c is outside [0, in-1]; otherwise
// t = ((v00*1)*wy0)*wx0 + ((v01*1)*wy0)*wx1 + ((v10*1)*wy1)*wx0 + ((v11*1)*wy1)*wx1 accumulated in that order,
// w1 = c - floor(c), w0 = 1 - w1 (verified bit-exact against scipy 1.18); finally clipped to [min(img,0), max(img,0)].
__global__ void image_minmax_kernel(const float* __restrict__ x, float* __restrict__ mm, long per_image) {
  // one block per image
  const float* p = x + (long)blockIdx.x * per_image;
  float lo = INFINITY, hi = -INFINITY;
  for (long i = threadIdx.x; i < per_image; i += blockDim.x) {
    const float v = p[i];
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  __shared__ float slo[32], shi[32];
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) { slo[threadIdx.x >> 5] = lo; shi[threadIdx.x >> 5] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { lo = fminf(lo, slo[w]); hi = fmaxf(hi, shi[w]); }
    mm[2 * blockIdx.x] = fminf(lo, 0.f);
    mm[2 * blockIdx.x + 1] = fmaxf(hi, 0.f);
  }
}

__global__ void resize_bilinear_f64_kernel(const float* __restrict__ x, const float* __restrict__ mm,
                                           double* __restrict__ y, int C, int Hi, int Wi, int Ho, int Wo) {
  const int img = blockIdx.y;  // image index (batch)
  const double fy = (double)Hi / (double)Ho, fx = (double)Wi / (double)Wo;
  const double lo = (double)mm[2 * img], hi = (double)mm[2 * img + 1];
  const long per_out = (long)C * Ho * Wo;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < per_out; i += (long)gridDim.x * blockDim.x) {
    const int ox = i % Wo, oy = (i / Wo) % Ho, c = i / ((long)Wo * Ho);
    const double cy = __dadd_rn(__dmul_rn(fy, (double)oy + 0.5), -0.5);
    const double cx = __dadd_rn(__dmul_rn(fx, (double)ox + 0.5), -0.5);
    double t = 0.0;
    if (cy >= 0.0 && cy <= (double)(Hi - 1) && cx >= 0.0 && cx <= (double)(Wi - 1)) {
      const double fly = floor(cy), flx = floor(cx);
      const double wy1 = __dsub_rn(cy, fly), wx1 = __dsub_rn(cx, flx);
      const double wy0 = __dsub_rn(1.0, wy1), wx0 = __dsub_rn(1.0, wx1);
      const int y0 = (int)fly, x0 = (int)flx;
      const int y1 = min(y0 + 1, Hi - 1), x1 = min(x0 + 1, Wi - 1);  // weight is exactly 0 when clamped
      const float* p = x + ((long)img * C + c) * Hi * Wi;
      const double v00 = (double)p[(long)y0 * Wi + x0], v01 = (double)p[(long)y0 * Wi + x1];
      const double v10 = (double)p[(long)y1 * Wi + x0], v11 = (double)p[(long)y1 * Wi + x1];
      t = __dmul_rn(__dmul_rn(v00, wy0), wx0);
      t = __dadd_rn(t, __dmul_rn(__dmul_rn(v01, wy0), wx1));
      t = __dadd_rn(t, __dmul_rn(__dmul_rn(v10, wy1), wx0));
      t = __dadd_rn(t, __dmul_rn(__dmul_rn(v11, wy1), wx1));
    }
    t = fmin(fmax(t, lo), hi);
    y[(long)img * per_out + i] = t;
  }
}

// ------------------------------------------------------------------------------------------ threshold (P2)
// categorize_multilayer_image: layer l of channel c = prob[c] > thr[l]; layers are listed channel-major.
template <typename T>
__global__ void threshold_layers_kernel(const T* __restrict__ prob, const double* __restrict__ thr,
                                        const int* __restrict__ layer_channel, uint8_t* __restrict__ out, int C, int L,
                                        long hw) {
  const int img = blockIdx.y;
  const long total = (long)L * hw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int l = i / hw;
    const long q = i % hw;
    const double v = (double)prob[((long)img * C + layer_channel[l]) * hw + q];
    out[(long)img * total + i] = v > thr[l] ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------ CCL (P4)
// 4-connectivity union-find over the pixel grid (each root = smallest linear index of its component = its first pixel
// in raster order), then roots are ranked by an in-image prefix sum: labels 1..K in raster order of first pixel,
// exactly scipy.ndimage.label's numbering.  One "plane" = one (image, layer) 2-D mask.
__device__ __forceinline__ int uf_find(const int* L, int a) {
  int p = L[a];
  while (p != a) { a = p; p = L[a]; }
  return a;
}
__device__ __forceinline__ void uf_union(int* L, int a, int b) {
  while (true) {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a == b) return;
    if (a < b) { int t = a; a = b; b = t; }
    const int old = atomicMin(&L[a], b);  // a > b: hang the larger root under the smaller
    if (old == a) return;
    a = old;
  }
}
// Two launches.
//  (1) ccl_strip_kernel: a CTA labels one strip of 32 rows entirely in SHARED memory — horizontal runs get the index of
//      their first pixel (no atomics), one union per vertical contact between runs (shared-memory atomicMin hooks),
//      flatten — and writes strip-local roots as global pixel indices.
//  (2) ccl_plane_kernel: one CTA per plane stitches the strips (unions along the 32-row borders), flattens, ranks the
//      roots in raster order with a block-wide prefix sum (-> scipy.ndimage.label numbering) and relabels.
// RANK == false stops after the flatten (roots only; used by add_dropped_objects).
constexpr int CCL_STRIP = 32;

__device__ __forceinline__ int uf_find_s(const int* L, int a) {
  int p = L[a];
  while (p != a) { a = p; p = L[a]; }
  return a;
}
__device__ __forceinline__ void uf_union_s(int* L, int a, int b) {
  while (true) {
    a = uf_find_s(L, a);
    b = uf_find_s(L, b);
    if (a == b) return;
    if (a < b) { int t = a; a = b; b = t; }
    const int old = atomicMin(&L[a], b);
    if (old == a) return;
    a = old;
  }
}

template <typename T>
__global__ void __launch_bounds__(512) ccl_strip_kernel(const T* __restrict__ mask, int* __restrict__ L, int H, int W) {
  extern __shared__ int s_ccl[];
  const int y0 = blockIdx.x * CCL_STRIP;
  const int rows = min(CCL_STRIP, H - y0);
  const int n = rows * W;
  int* sl = s_ccl;                                              // [n] local parent (local linear index) or -1
  uint8_t* sm = reinterpret_cast<uint8_t*>(s_ccl + CCL_STRIP * W);  // [n] mask
  const long base = (long)blockIdx.y * H * W + (long)y0 * W;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sm[i] = mask[base + i] != 0 ? 1 : 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int x = i % W;
    if (!sm[i]) { sl[i] = -1; continue; }
    if (x > 0 && sm[i - 1]) continue;
    const int row_end = i - x + W;
    for (int j = i; j < row_end && sm[j]; ++j) sl[j] = i;
  }
  __syncthreads();
  for (int i = threadIdx.x + W; i < n; i += blockDim.x) {
    if (!sm[i] || !sm[i - W]) continue;
    const int x = i % W;
    if (x == 0 || !sm[i - 1] || !sm[i - W - 1]) uf_union_s(sl, sl[i], sl[i - W]);
  }
  __syncthreads();
  const int goff = y0 * W;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    L[base + i] = sm[i] ? goff + uf_find_s(sl, sl[i]) : -1;
}

template <typename T, bool RANK>
__global__ void __launch_bounds__(1024) ccl_plane_kernel(const T* __restrict__ mask, int* __restrict__ L,
                                                        int* __restrict__ out, int* __restrict__ count, int H, int W) {
  const long hw = (long)H * W;
  const T* mp = mask + (long)blockIdx.x * hw;
  int* Lp = L + (long)blockIdx.x * hw;
  int* op = RANK ? out + (long)blockIdx.x * hw : nullptr;
  // stitch the strips: one union per vertical contact across each 32-row border
  const int borders = (H - 1) / CCL_STRIP;
  for (int k = threadIdx.x; k < borders * W; k += blockDim.x) {
    const int x = k % W;
    const long i = (long)(k / W + 1) * CCL_STRIP * W + x;
    if (mp[i] == 0 || mp[i - W] == 0) continue;
    if (x == 0 || mp[i - 1] == 0 || mp[i - W - 1] == 0) uf_union(Lp, Lp[i], Lp[i - W]);
  }
  __syncthreads();
  for (long i = threadIdx.x; i < hw; i += blockDim.x)
    if (Lp[i] >= 0) Lp[i] = uf_find(Lp, Lp[i]);
  if (!RANK) return;
  __syncthreads();
  // rank the roots in raster order
  const long chunk = (hw + blockDim.x - 1) / blockDim.x;
  const long b = threadIdx.x * chunk, e = min(hw, b + chunk);
  int local = 0;
  for (long i = b; i < e; ++i) local += (Lp[i] == (int)i);
  __shared__ int warp_sums[32];
  __shared__ int total;
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += n;
  }
  if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int v = warp_sums[threadIdx.x];
    int sc = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, sc, o);
      if (threadIdx.x >= o) sc += n;
    }
    warp_sums[threadIdx.x] = sc - v;  // exclusive
    if (threadIdx.x == 31) total = sc;
  }
  __syncthreads();
  int run = warp_sums[threadIdx.x >> 5] + incl - local;
  for (long i = b; i < e; ++i)
    if (Lp[i] == (int)i) op[i] = ++run;
  if (threadIdx.x == 0 && count != nullptr) count[blockIdx.x] = total;
  __syncthreads();
  for (long i = threadIdx.x; i < hw; i += blockDim.x) {
    const int r = Lp[i];
    if (r < 0) op[i] = 0;
    else if (r != (int)i) op[i] = op[r];
  }
}

template <typename T, bool RANK>
static int launch_ccl(const T* mask, int* workspace, int* labels, int* counts, int planes, int h, int w,
                      cudaStream_t st) {
  const size_t smem = (size_t)CCL_STRIP * w * 5;
  if (smem > 200 * 1024) return fail(MCB_ERR_UNSUPPORTED, "ccl: width %d too large for the strip kernel", w);
  static bool attr_set = false;
  if (!attr_set && smem > 48 * 1024) {
    MCB_CHECK_CUDA(cudaFuncSetAttribute(ccl_strip_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  dim3 grid((h + CCL_STRIP - 1) / CCL_STRIP, planes);
  ccl_strip_kernel<T><<<grid, 512, smem, st>>>(mask, workspace, h, w);
  MCB_LAUNCH_CHECK();
  ccl_plane_kernel<T, RANK><<<planes, 1024, 0, st>>>(mask, workspace, labels, counts, h, w);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// ------------------------------------------------------------------------------------------ morphology (P3, P5)
// skimage erosion / dilation with rectangle(k, k): window offsets [lo, hi] per axis (even k is zero-padded on the
// top/left, so lo = -k/2 + 1), border mode 'reflect' == ignoring out-of-range taps for these windows.
template <typename T, bool IS_MAX>
__global__ void morph_rect_kernel(const T* __restrict__ in, T* __restrict__ out, int H, int W, int lo, int hi) {
  const long hw = (long)H * W;
  const T* ip = in + (long)blockIdx.y * hw;
  T* op = out + (long)blockIdx.y * hw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < hw; i += (long)gridDim.x * blockDim.x) {
    const int x = i % W, y = i / W;
    T acc = ip[i];
    for (int dy = lo; dy <= hi; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = lo; dx <= hi; ++dx) {
        const int xx = x + dx;
        if (xx < 0 || xx >= W) continue;
        const T v = ip[(long)yy * W + xx];
        acc = IS_MAX ? (v > acc ? v : acc) : (v < acc ? v : acc);
      }
    }
    op[i] = acc;
  }
}

// add_dropped_objects (src/utils.py:333-339): components of `original` without any pixel left in `processed`
// are added back.  roots = flattened union-find labels of `original`.
__global__ void dropped_mark_kernel(const int* __restrict__ roots, const uint8_t* __restrict__ processed,
                                    int* __restrict__ keep, long hw) {
  const long base = (long)blockIdx.y * hw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < hw; i += (long)gridDim.x * blockDim.x) {
    const int r = roots[base + i];
    if (r >= 0 && processed[base + i] != 0) keep[base + r] = 1;
  }
}
__global__ void dropped_restore_kernel(const int* __restrict__ roots, const uint8_t* __restrict__ processed,
                                       const int* __restrict__ keep, uint8_t* __restrict__ out, long hw) {
  const long base = (long)blockIdx.y * hw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < hw; i += (long)gridDim.x * blockDim.x) {
    const int r = roots[base + i];
    uint8_t v = processed[base + i];
    if (r >= 0 && keep[base + r] == 0) v = (uint8_t)(v + 1);
    out[base + i] = v;
  }
}

// ------------------------------------------------------------------------------------------ scores (P6)
// build_score: per plane, per label: sum of probabilities and pixel count (score = mean * sqrt(count) on the host side
// of the ABI is avoided: finalize kernel writes the score).  Scores are laid out per plane at `offsets[plane]`.
template <typename T>
__global__ void score_accumulate_kernel(const int* __restrict__ labels, const T* __restrict__ prob,
                                        const int* __restrict__ offsets, double* __restrict__ sums,
                                        int* __restrict__ counts, long hw) {
  const int plane = blockIdx.y;
  const long base = (long)plane * hw;
  const int off = offsets[plane];
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < hw; i += (long)gridDim.x * blockDim.x) {
    const int l = labels[base + i];
    if (l > 0) {
      atomicAdd(&sums[off + l - 1], (double)prob[base + i]);
      atomicAdd(&counts[off + l - 1], 1);
    }
  }
}
__global__ void score_finalize_kernel(const double* __restrict__ sums, const int* __restrict__ counts,
                                      double* __restrict__ scores, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = counts[i];
  scores[i] = c > 0 ? (sums[i] / (double)c) * sqrt((double)c) : nan("");
}

// build_score without a host round trip, scores at a fixed stride `kcap` per plane; counts[plane] = number of labels of
// the plane (from the labelling step).  Grid (S, planes): CTA (s, plane) owns a contiguous pixel span, every thread
// walks a CONTIGUOUS sub-range keeping a running (label, sum, count) and flushes with one native fp64 global atomic
// only when the label changes (a few times per thread, since instances are blobs) -- no same-address atomic storm and
// ~8 CTAs per SM in flight instead of one CTA per plane.  The accumulators are zeroed by the caller (memset) and
// turned into scores by score_finalize_strided_kernel.
template <typename T>
__global__ void __launch_bounds__(256) score_runs_kernel(const int* __restrict__ labels, const T* __restrict__ prob,
                                                         double* __restrict__ gsum, int* __restrict__ gcnt, long hw,
                                                         int kcap, int chunk) {
  const int plane = blockIdx.y;
  double* ps = gsum + (long)plane * kcap;
  int* pc = gcnt + (long)plane * kcap;
  const long base = (long)plane * hw;
  const long b = ((long)blockIdx.x * blockDim.x + threadIdx.x) * chunk;
  const long e = min(hw, b + chunk);
  int cur = 0, cnt = 0;
  double sum = 0.0;
  for (long i = b; i < e; ++i) {
    const int l = __ldg(labels + base + i);
    if (l != cur) {
      if (cur > 0 && cur <= kcap) { atomicAdd(&ps[cur - 1], sum); atomicAdd(&pc[cur - 1], cnt); }
      cur = l; cnt = 0; sum = 0.0;
    }
    if (l > 0) { sum += (double)__ldg(prob + base + i); ++cnt; }
  }
  if (cur > 0 && cur <= kcap) { atomicAdd(&ps[cur - 1], sum); atomicAdd(&pc[cur - 1], cnt); }
}
__global__ void score_finalize_strided_kernel(const double* __restrict__ gsum, const int* __restrict__ gcnt,
                                              const int* __restrict__ counts, double* __restrict__ scores, int kcap) {
  const int plane = blockIdx.x;
  const int K = min(counts[plane], kcap);
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const int c = gcnt[(long)plane * kcap + i];
    const double sm = gsum[(long)plane * kcap + i];
    scores[(long)plane * kcap + i] = c > 0 ? (sm / (double)c) * sqrt((double)c) : nan("");
  }
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

static dim3 plane_grid(long hw, int planes, int threads) {
  const int per_plane = (int)std::max(1L, std::min((hw + threads - 1) / threads, (long)num_sms() * 8L / std::max(planes, 1) + 1));
  return dim3(per_plane, planes, 1);
}

extern "C" int mcb_resize_bilinear_f64(const float* x, double* y, float* minmax_ws, int n, int c, int hi, int wi,
                                       int ho, int wo, void* stream) {
  MCB_REQUIRE(x && y && minmax_ws, "resize: null pointer");
  MCB_REQUIRE(n > 0 && c > 0 && hi > 1 && wi > 1 && ho > 0 && wo > 0, "resize: bad shape");
  image_minmax_kernel<<<n, 512, 0, ST>>>(x, minmax_ws, (long)c * hi * wi);
  MCB_LAUNCH_CHECK();
  resize_bilinear_f64_kernel<<<plane_grid((long)c * ho * wo, n, 256), 256, 0, ST>>>(x, minmax_ws, y, c, hi, wi, ho, wo);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_threshold_layers(const void* prob, int prob_is_f64, const double* thresholds,
                                    const int* layer_channel, uint8_t* out, int n, int c, int layers, int h, int w,
                                    void* stream) {
  MCB_REQUIRE(prob && thresholds && layer_channel && out, "threshold: null pointer");
  const long hw = (long)h * w;
  dim3 grid = plane_grid(hw * layers, n, 256);
  if (prob_is_f64)
    threshold_layers_kernel<double><<<grid, 256, 0, ST>>>((const double*)prob, thresholds, layer_channel, out, c, layers, hw);
  else
    threshold_layers_kernel<float><<<grid, 256, 0, ST>>>((const float*)prob, thresholds, layer_channel, out, c, layers, hw);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_ccl_label(const void* mask, int mask_is_i32, int* labels, int* workspace, int* counts, int planes,
                             int h, int w, void* stream) {
  MCB_REQUIRE(mask && labels && workspace, "ccl: null pointer");
  MCB_REQUIRE((long)h * w < (1L << 31), "ccl: plane too large");
  if (mask_is_i32) return launch_ccl<int, true>((const int*)mask, workspace, labels, counts, planes, h, w, ST);
  return launch_ccl<uint8_t, true>((const uint8_t*)mask, workspace, labels, counts, planes, h, w, ST);
}

extern "C" int mcb_morph_rect(const void* in, void* out, int is_i32, int is_dilation, int size, int planes, int h,
                              int w, void* stream) {
  MCB_REQUIRE(in && out && in != out, "morph: null or aliased pointer");
  MCB_REQUIRE(size >= 1 && size <= 31, "morph: size %d", size);
  const int kp = (size % 2 == 0) ? size + 1 : size;
  const int hi = (kp - 1) / 2;
  const int lo = (size % 2 == 0) ? -hi + 1 : -hi;
  dim3 grid = plane_grid((long)h * w, planes, 256);
  if (is_i32) {
    if (is_dilation) morph_rect_kernel<int, true><<<grid, 256, 0, ST>>>((const int*)in, (int*)out, h, w, lo, hi);
    else morph_rect_kernel<int, false><<<grid, 256, 0, ST>>>((const int*)in, (int*)out, h, w, lo, hi);
  } else {
    if (is_dilation) morph_rect_kernel<uint8_t, true><<<grid, 256, 0, ST>>>((const uint8_t*)in, (uint8_t*)out, h, w, lo, hi);
    else morph_rect_kernel<uint8_t, false><<<grid, 256, 0, ST>>>((const uint8_t*)in, (uint8_t*)out, h, w, lo, hi);
  }
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// skimage <= 0.17 binary_erosion / binary_dilation with rectangle(k, k) (src/preparation.py:170-186), i.e.
// ndi.binary_erosion(structure, border_value=True) / ndi.binary_dilation(structure), on {0,1} uint8 planes.  Dilation
// takes the same window as the grey dilation above; scipy centres an even binary erosion at index k/2, so its window
// is [-k/2, k/2 - 1] where the grey erosion's is [-k/2 + 1, k/2].  Out-of-range taps are ignored in both (border_value
// True for the erosion, 0 for the dilation).
extern "C" int mcb_binary_morph_rect(const uint8_t* in, uint8_t* out, int is_dilation, int size, int planes, int h, int w,
                                     void* stream) {
  MCB_REQUIRE(in && out && in != out, "binary_morph: null or aliased pointer");
  MCB_REQUIRE(size >= 1 && size <= 31, "binary_morph: size %d", size);
  constexpr int kMaxGridY = 65535;   // planes go on gridDim.y, in slices
  const long hw = (long)h * w;
  for (int p0 = 0; p0 < planes; p0 += kMaxGridY) {
    const int cnt = std::min(kMaxGridY, planes - p0);
    if (is_dilation || size % 2 == 1) {
      if (int r = mcb_morph_rect(in + p0 * hw, out + p0 * hw, 0, is_dilation, size, cnt, h, w, stream)) return r;
      continue;
    }
    morph_rect_kernel<uint8_t, false><<<plane_grid(hw, cnt, 256), 256, 0, ST>>>(in + p0 * hw, out + p0 * hw, h, w,
                                                                               -size / 2, size / 2 - 1);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}

extern "C" int mcb_add_dropped_objects(const uint8_t* original, const uint8_t* processed, uint8_t* out, int* workspace,
                                       int planes, int h, int w, void* stream) {
  MCB_REQUIRE(original && processed && out && workspace, "add_dropped: null pointer");
  const long hw = (long)h * w;
  int* roots = workspace;
  int* keep = workspace + (long)planes * hw;
  dim3 grid = plane_grid(hw, planes, 256);
  if (int r = launch_ccl<uint8_t, false>(original, roots, nullptr, nullptr, planes, h, w, ST)) return r;
  MCB_CHECK_CUDA(cudaMemsetAsync(keep, 0, (size_t)planes * hw * sizeof(int), ST));
  dropped_mark_kernel<<<grid, 256, 0, ST>>>(roots, processed, keep, hw);
  MCB_LAUNCH_CHECK();
  dropped_restore_kernel<<<grid, 256, 0, ST>>>(roots, processed, keep, out, hw);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_instance_scores(const int* labels, const void* prob, int prob_is_f64, const int* offsets,
                                   double* sums, int* counts, double* scores, int total_instances, int planes, int h,
                                   int w, void* stream) {
  MCB_REQUIRE(labels && prob && offsets && sums && counts && scores, "scores: null pointer");
  if (total_instances <= 0) return MCB_OK;
  const long hw = (long)h * w;
  MCB_CHECK_CUDA(cudaMemsetAsync(sums, 0, (size_t)total_instances * sizeof(double), ST));
  MCB_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)total_instances * sizeof(int), ST));
  dim3 grid = plane_grid(hw, planes, 256);
  if (prob_is_f64)
    score_accumulate_kernel<double><<<grid, 256, 0, ST>>>(labels, (const double*)prob, offsets, sums, counts, hw);
  else
    score_accumulate_kernel<float><<<grid, 256, 0, ST>>>(labels, (const float*)prob, offsets, sums, counts, hw);
  MCB_LAUNCH_CHECK();
  score_finalize_kernel<<<blocks_for(total_instances, 256), 256, 0, ST>>>(sums, counts, scores, total_instances);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_instance_scores_strided(const int* labels, const void* prob, int prob_is_f64, const int* counts,
                                           double* scores, double* gsum_ws, int* gcnt_ws, int kcap, int planes, int h,
                                           int w, void* stream) {
  MCB_REQUIRE(labels && prob && counts && scores && gsum_ws && gcnt_ws, "scores_strided: null pointer");
  MCB_REQUIRE(kcap >= 1, "scores_strided: kcap %d", kcap);
  const long hw = (long)h * w;
  MCB_CHECK_CUDA(cudaMemsetAsync(gsum_ws, 0, (size_t)planes * kcap * sizeof(double), ST));
  MCB_CHECK_CUDA(cudaMemsetAsync(gcnt_ws, 0, (size_t)planes * kcap * sizeof(int), ST));
  const int S = (int)std::max(1L, std::min(64L, (long)num_sms() * 8L / std::max(planes, 1)));
  const int chunk = (int)(((hw + (long)S * 256 - 1) / ((long)S * 256) + 3) / 4 * 4);  // pixels per thread
  const int ctas = (int)((hw + (long)chunk * 256 - 1) / ((long)chunk * 256));
  dim3 grid(ctas, planes);
  if (prob_is_f64)
    score_runs_kernel<double><<<grid, 256, 0, ST>>>(labels, (const double*)prob, gsum_ws, gcnt_ws, hw, kcap, chunk);
  else
    score_runs_kernel<float><<<grid, 256, 0, ST>>>(labels, (const float*)prob, gsum_ws, gcnt_ws, hw, kcap, chunk);
  MCB_LAUNCH_CHECK();
  score_finalize_strided_kernel<<<planes, 256, 0, ST>>>(gsum_ws, gcnt_ws, counts, scores, kcap);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
