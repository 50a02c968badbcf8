// crf.cu — dense-CRF mean-field (src/postprocessing.py:183-225 -> pydensecrf DenseCRF2D) as shared-memory-tiled
// kernels.  PARITY UNPINNED: pydensecrf is absent; semantics follow oracle/post_oracle.py::dense_crf, which restates the
// published algorithm (Kraehenbuehl & Koltun 2011) with EXACT Gaussian filtering inside a (2R+1)^2 window instead of
// the library's permutohedral-lattice approximation (with sxy = 1 the tail beyond R = 6 is < 1.5e-8).
//
//   U = -log(max(p, 1e-5)); Q0 = softmax(-U)
//   K_g(i,j) = exp(-|pi-pj|^2 / (2 sxy_g^2)),  K_b(i,j) = exp(-|pi-pj|^2/(2 sxy_b^2) - |Ii-Ij|^2/(2 srgb^2))
//   n_k = 1/sqrt(K_k 1 + 1e-20)  (symmetric normalisation);  msg_k = n_k (.) K_k (n_k (.) Q)
//   Q <- softmax(-U + compat_g msg_g + compat_b msg_b), `iterations` times.
//
// One launch per iteration (every pixel needs its 13x13 neighbourhood of the previous iterate); Q ping-pongs through
// L2 (2 x 300 x 300 x 4 B per image).  A CTA of 8 warps owns 32x32 outputs and stages (pre-scaled RGB, Q*n_b, Q*n_g)
// with a 6-pixel halo in shared memory.  The kernel is bound by fp32 issue (169 bilateral taps per pixel and
// iteration), so the tap body is cut to the bone:
//   * every thread owns FOUR vertically adjacent outputs and walks the 16 source rows they share, so each staged
//     pixel is loaded once for up to four taps; lanes run along x (conflict-free 16-byte shared-memory loads);
//   * the four outputs are processed as two PAIRS (f2 helpers below): colour difference, squared distance and both
//     class accumulations cost 16 FADD / FFMA + 2 MUFU.EX2 per pair of taps;
//   * colours are pre-scaled by sqrt(log2(e) / (2 srgb^2)) and the horizontal spatial weight enters as an addend of the
//     exponent, so one ex2 yields the complete horizontal x colour weight; the vertical weight multiplies the row sum;
//   * out-of-image pixels are staged with a far-away colour (weight underflows to exactly 0) -- no per-tap branch;
//   * the purely spatial Gaussian message is separable: 13 + 13 taps through a shared-memory row buffer.
// HBM/L2 traffic is one read of (Q, norms, RGB) and one write of Q per iteration; no tensor cores.
#include "host_common.h"
#include "../../include/mcb200.h"
#include <algorithm>
#include <math.h>

namespace mcb {

constexpr int CRF_R = 6;
constexpr int CRF_D = 2 * CRF_R + 1;
constexpr int CRF_T = 32;                 // outputs per CTA edge
constexpr int CRF_S = CRF_T + 2 * CRF_R;  // staged tile edge (44)
constexpr int CRF_ROWS = 4;               // outputs per thread (vertical)
constexpr int CRF_THREADS = CRF_T * (CRF_T / CRF_ROWS);   // 256
// 73 KB per CTA -> three CTAs per SM within the 227 KB of shared memory an SM offers
constexpr size_t CRF_SMEM = (size_t)CRF_S * CRF_S * (sizeof(float4) + sizeof(float2) + sizeof(float2)) +
                            (size_t)CRF_S * CRF_T * sizeof(float2);

__constant__ float c_g1g[CRF_D];    // 1-D spatial weights exp(-d^2 / (2 sxy^2)), Gaussian kernel
__constant__ float c_g1b[CRF_D];    // ... bilateral kernel
__constant__ float c_e1b[CRF_D];    // d^2 * log2(e) / (2 sxy_b^2)  (>= 0): exponent addend of the horizontal weight

// de-normalise (x*std+mean)*255 and cast like numpy's float64 -> uint8 C cast (truncate, wrap modulo 256)
__global__ void crf_rgb_kernel(const float* __restrict__ img, uint8_t* __restrict__ rgb, long hw, long total) {
  const double mean[3] = {0.485, 0.456, 0.406}, stdv[3] = {0.229, 0.224, 0.225};
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = i % 3;
    const long p = (i / 3) % hw, n = i / (3 * hw);
    const double v = ((double)img[(n * 3 + c) * hw + p] * stdv[c] + mean[c]) * 255.0;
    rgb[i] = (uint8_t)(long long)v;
  }
}

// fp32 pairs: sm_90 has no packed fp32x2 arithmetic, so each helper is two scalar FADD / FFMA with the same
// round-to-nearest results the packed form gives
typedef float2 f2;
__device__ __forceinline__ f2 pk(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk(f2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float ex2_approx(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// MODE 0: norms (writes n_g, n_b).  MODE 1: one mean-field iteration.
template <int MODE>
__global__ void __launch_bounds__(CRF_THREADS) crf_kernel(const float* __restrict__ probs, const float* __restrict__ q_in,
                                                          const uint8_t* __restrict__ rgb, float* __restrict__ norms,
                                                          float* __restrict__ q_out, int H, int W, float color_scale,
                                                          float compat_g, float compat_b, int first_iter) {
  extern __shared__ __align__(16) uint8_t crf_smem[];
  float4(*s_rgb)[CRF_S] = reinterpret_cast<float4(*)[CRF_S]>(crf_smem);                      // scaled r, g, b, -
  float2(*s_qb)[CRF_S] = reinterpret_cast<float2(*)[CRF_S]>(crf_smem + sizeof(float4) * CRF_S * CRF_S);  // q0 q1 (x n_b)
  float2(*s_qg)[CRF_S] = reinterpret_cast<float2(*)[CRF_S]>(crf_smem + (sizeof(float4) + sizeof(float2)) * CRF_S * CRF_S);  // q0 q1 (x n_g)
  float2(*s_hg)[CRF_T] = reinterpret_cast<float2(*)[CRF_T]>(crf_smem + (sizeof(float4) + 2 * sizeof(float2)) * CRF_S * CRF_S);
  const int img = blockIdx.z;
  const long hw = (long)H * W;
  const int x0 = blockIdx.x * CRF_T, y0 = blockIdx.y * CRF_T;
  const float* ng = norms + (long)img * 2 * hw;
  const float* nb = ng + hw;
  // ---- stage the halo tile
  for (int i = threadIdx.x; i < CRF_S * CRF_S; i += CRF_THREADS) {
    const int sy = i / CRF_S, sx = i % CRF_S;
    const int y = y0 + sy - CRF_R, x = x0 + sx - CRF_R;
    float4 c = make_float4(1e9f, 1e9f, 1e9f, 0.f);   // outside the image: the colour weight underflows to exactly 0
    float2 qb = make_float2(0.f, 0.f);
    float2 qg = make_float2(0.f, 0.f);
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const long p = (long)y * W + x;
      const uint8_t* cp = rgb + ((long)img * hw + p) * 3;
      c = make_float4((float)cp[0] * color_scale, (float)cp[1] * color_scale, (float)cp[2] * color_scale, 0.f);
      if (MODE == 1) {
        float q0, q1;
        if (first_iter) {
          // Q0 = softmax(-U) = clipped probabilities renormalised
          const float p0 = fmaxf(probs[((long)img * 2) * hw + p], 1e-5f), p1 = fmaxf(probs[((long)img * 2 + 1) * hw + p], 1e-5f);
          const float u0 = -logf(p0), u1 = -logf(p1);
          const float m = fmaxf(-u0, -u1);
          const float e0 = expf(-u0 - m), e1 = expf(-u1 - m);
          q0 = e0 / (e0 + e1);
          q1 = e1 / (e0 + e1);
        } else {
          q0 = q_in[((long)img * 2) * hw + p];
          q1 = q_in[((long)img * 2 + 1) * hw + p];
        }
        const float a = ng[p], b = nb[p];
        qg = make_float2(q0 * a, q1 * a);
        qb = make_float2(q0 * b, q1 * b);
      } else {
        qg = make_float2(1.f, 1.f);   // MODE 0: the separable pass then sums the in-image Gaussian weights
      }
    }
    s_rgb[sy][sx] = c;
    s_qb[sy][sx] = qb;
    s_qg[sy][sx] = qg;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  // ---- separable Gaussian kernel, horizontal pass: s_hg[row][x] = sum_dx g(dx) * s_qg[row][x + dx]
  {
    float g1[CRF_D];
#pragma unroll
    for (int d = 0; d < CRF_D; ++d) g1[d] = c_g1g[d];
    for (int r = wrp; r < CRF_S; r += CRF_THREADS / 32) {
      float h0 = 0.f, h1 = 0.f;
#pragma unroll
      for (int d = 0; d < CRF_D; ++d) {
        const float2 v = s_qg[r][lane + d];
        h0 = fmaf(g1[d], v.x, h0);
        h1 = fmaf(g1[d], v.y, h1);
      }
      s_hg[r][lane] = make_float2(h0, h1);
    }
  }
  // ---- bilateral kernel: outputs (ry + j, x), j = 0..3, as two packed pairs (0,1) and (2,3)
  const int ry = wrp * CRF_ROWS;                 // first output row of this thread inside the tile
  f2 mr[2], mg[2], mb[2];
#pragma unroll
  for (int pr = 0; pr < 2; ++pr) {
    const float4 a = s_rgb[ry + 2 * pr + CRF_R][lane + CRF_R], b = s_rgb[ry + 2 * pr + 1 + CRF_R][lane + CRF_R];
    mr[pr] = pk(a.x, b.x); mg[pr] = pk(a.y, b.y); mb[pr] = pk(a.z, b.z);
  }
  f2 ex[CRF_D];
#pragma unroll
  for (int d = 0; d < CRF_D; ++d) ex[d] = pk(c_e1b[d], c_e1b[d]);
  f2 acc0[2] = {pk(0.f, 0.f), pk(0.f, 0.f)}, acc1[2] = {pk(0.f, 0.f), pk(0.f, 0.f)};   // MODE 1: class-0 / class-1 messages; MODE 0: acc0 = weight sums
#pragma unroll 1
  for (int s = 0; s < CRF_D + CRF_ROWS - 1; ++s) {
    f2 r0[2] = {pk(0.f, 0.f), pk(0.f, 0.f)}, r1[2] = {pk(0.f, 0.f), pk(0.f, 0.f)};
#pragma unroll
    for (int d = 0; d < CRF_D; ++d) {
      const float4 o = s_rgb[ry + s][lane + d];
      const f2 orr = pk(o.x, o.x), og = pk(o.y, o.y), ob = pk(o.z, o.z);
      f2 q0p = pk(0.f, 0.f), q1p = pk(0.f, 0.f);   // (q0, q0), (q1, q1)
      if (MODE == 1) {
        const float2 q = s_qb[ry + s][lane + d];
        q0p = pk(q.x, q.x);
        q1p = pk(q.y, q.y);
      }
#pragma unroll
      for (int pr = 0; pr < 2; ++pr) {
        const f2 dr = sub2(mr[pr], orr), dg = sub2(mg[pr], og), db = sub2(mb[pr], ob);
        f2 t = fma2(dr, dr, ex[d]);
        t = fma2(dg, dg, t);
        t = fma2(db, db, t);
        float t0, t1;
        upk(t, t0, t1);
        const f2 k = pk(ex2_approx(-t0), ex2_approx(-t1));
        if (MODE == 1) {
          r0[pr] = fma2(k, q0p, r0[pr]);
          r1[pr] = fma2(k, q1p, r1[pr]);
        } else {
          r0[pr] = add2(r0[pr], k);
        }
      }
    }
    // vertical weight of source row s for output j: g(s - j - R) when 0 <= s - j <= 2R, else 0
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      const int u0 = s - 2 * pr, u1 = s - 2 * pr - 1;
      const f2 wy = pk((u0 >= 0 && u0 < CRF_D) ? c_g1b[u0] : 0.f, (u1 >= 0 && u1 < CRF_D) ? c_g1b[u1] : 0.f);
      acc0[pr] = fma2(wy, r0[pr], acc0[pr]);
      if (MODE == 1) acc1[pr] = fma2(wy, r1[pr], acc1[pr]);
    }
  }
  __syncthreads();   // s_hg complete
  float mb0[CRF_ROWS], mb1[CRF_ROWS];
  upk(acc0[0], mb0[0], mb0[1]); upk(acc0[1], mb0[2], mb0[3]);
  upk(acc1[0], mb1[0], mb1[1]); upk(acc1[1], mb1[2], mb1[3]);
#pragma unroll
  for (int j = 0; j < CRF_ROWS; ++j) {
    const int x = x0 + lane, y = y0 + ry + j;
    if (x >= W || y >= H) continue;
    // separable Gaussian kernel, vertical pass
    float mg0 = 0.f, mg1 = 0.f;
#pragma unroll
    for (int d = 0; d < CRF_D; ++d) {
      const float2 v = s_hg[ry + j + d][lane];
      mg0 = fmaf(c_g1g[d], v.x, mg0);
      mg1 = fmaf(c_g1g[d], v.y, mg1);
    }
    const long p = (long)y * W + x;
    if (MODE == 0) {
      norms[(long)img * 2 * hw + p] = 1.f / sqrtf(mg0 + 1e-20f);
      norms[(long)img * 2 * hw + hw + p] = 1.f / sqrtf(mb0[j] + 1e-20f);
    } else {
      const float a = ng[p], b = nb[p];
      const float p0 = fmaxf(probs[((long)img * 2) * hw + p], 1e-5f), p1 = fmaxf(probs[((long)img * 2 + 1) * hw + p], 1e-5f);
      const float e0 = logf(p0) + compat_g * (mg0 * a) + compat_b * (mb0[j] * b);   // -U = log p
      const float e1 = logf(p1) + compat_g * (mg1 * a) + compat_b * (mb1[j] * b);
      const float m = fmaxf(e0, e1);
      const float x0e = expf(e0 - m), x1e = expf(e1 - m);
      q_out[((long)img * 2) * hw + p] = x0e / (x0e + x1e);
      q_out[((long)img * 2 + 1) * hw + p] = x1e / (x0e + x1e);
    }
  }
}

}  // namespace mcb

using namespace mcb;

extern "C" int mcb_crf_rgb_from_normalized(const float* img, uint8_t* rgb, int n, int h, int w, void* stream) {
  MCB_REQUIRE(img && rgb, "crf_rgb: null pointer");
  const long hw = (long)h * w, total = hw * 3 * n;
  const int grid = (int)std::max(1L, std::min((total + 255) / 256, (long)num_sms() * 8));
  crf_rgb_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, rgb, hw, total);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_dense_crf(const float* probs, const uint8_t* rgb, float* out, float* workspace, int n, int h, int w,
                             float compat_gaussian, float sxy_gaussian, float compat_bilateral, float sxy_bilateral,
                             float srgb, int iterations, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(probs && rgb && out && workspace, "dense_crf: null pointer");
  MCB_REQUIRE(iterations >= 1, "dense_crf: iterations %d", iterations);
  MCB_REQUIRE(sxy_gaussian > 0.f && sxy_bilateral > 0.f && srgb > 0.f, "dense_crf: kernel widths must be positive");
  float g1g[CRF_D], g1b[CRF_D], e1b[CRF_D];
  const double log2e = 1.4426950408889634;
  for (int d = -CRF_R; d <= CRF_R; ++d) {
    const double d2 = (double)(d * d);
    g1g[d + CRF_R] = (float)exp(-0.5 * d2 / ((double)sxy_gaussian * sxy_gaussian));
    g1b[d + CRF_R] = (float)exp(-0.5 * d2 / ((double)sxy_bilateral * sxy_bilateral));
    e1b[d + CRF_R] = (float)(0.5 * d2 / ((double)sxy_bilateral * sxy_bilateral) * log2e);
  }
  MCB_CHECK_CUDA(cudaMemcpyToSymbolAsync(c_g1g, g1g, sizeof(g1g), 0, cudaMemcpyHostToDevice, st));
  MCB_CHECK_CUDA(cudaMemcpyToSymbolAsync(c_g1b, g1b, sizeof(g1b), 0, cudaMemcpyHostToDevice, st));
  MCB_CHECK_CUDA(cudaMemcpyToSymbolAsync(c_e1b, e1b, sizeof(e1b), 0, cudaMemcpyHostToDevice, st));
  static bool attr_set = false;
  if (!attr_set) {
    MCB_CHECK_CUDA(cudaFuncSetAttribute(crf_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CRF_SMEM));
    MCB_CHECK_CUDA(cudaFuncSetAttribute(crf_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CRF_SMEM));
    attr_set = true;
  }
  const long plane = (long)n * 2 * h * w;
  float* norms = workspace;            // [n][2][h][w]
  float* qa = workspace + plane;       // ping
  float* qb = workspace + 2 * plane;   // pong
  dim3 grid((w + CRF_T - 1) / CRF_T, (h + CRF_T - 1) / CRF_T, n);
  // colours enter pre-scaled so that |dI|^2 is the base-2 exponent: exp(-|dI|^2 / (2 srgb^2)) = 2^-(s^2 |dI|^2)
  const float color_scale = (float)sqrt(0.5 * log2e / ((double)srgb * srgb));
  crf_kernel<0><<<grid, CRF_THREADS, CRF_SMEM, st>>>(probs, nullptr, rgb, norms, nullptr, h, w, color_scale,
                                                    compat_gaussian, compat_bilateral, 0);
  MCB_LAUNCH_CHECK();
  const float* qin = nullptr;
  for (int it = 0; it < iterations; ++it) {
    float* qout = (it == iterations - 1) ? out : ((it & 1) ? qb : qa);
    crf_kernel<1><<<grid, CRF_THREADS, CRF_SMEM, st>>>(probs, qin, rgb, norms, qout, h, w, color_scale, compat_gaussian,
                                                      compat_bilateral, it == 0 ? 1 : 0);
    MCB_LAUNCH_CHECK();
    qin = qout;
  }
  return MCB_OK;
}
