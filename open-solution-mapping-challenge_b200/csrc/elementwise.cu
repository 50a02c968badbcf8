// elementwise.cu — the HBM-bound glue of the U-Net step: layout conversion, stem im2col, BatchNorm (train/eval,
// forward/backward), 2x2 max-pool, per-channel sums, the final 1x1 classifier, fused Adam.
// All NHWC bf16 kernels move 16 bytes (8 channels) per thread per access; grids are sized in multiples of the SM count.
#include "host_common.h"
#include "../../include/mcb200.h"
#include "detsum.cuh"
#include <algorithm>
#include <math.h>

namespace mcb {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

static inline int grid_for(long work_items, int threads, int per_sm = 8) {
  long blocks = (work_items + threads - 1) / threads;
  long cap = (long)num_sms() * per_sm;
  return (int)std::max(1L, std::min(blocks, cap));
}

// ------------------------------------------------------------------------------------------ layout conversion
__global__ void nchw_f32_to_nhwc_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, int N, int C, int H,
                                             int W) {
  mcb::pdl_prologue();
  const long total = (long)N * H * W * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = i % C;
    const long p = i / C;
    const int w = p % W;
    const int h = (p / W) % H;
    const int n = p / ((long)W * H);
    y[i] = __float2bfloat16(x[(((long)n * C + c) * H + h) * W + w]);
  }
}
__global__ void nhwc_bf16_to_nchw_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, int N, int C, int H,
                                             int W) {
  mcb::pdl_prologue();
  const long total = (long)N * H * W * C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int w = i % W;
    const int h = (i / W) % H;
    const int c = (i / ((long)W * H)) % C;
    const int n = i / ((long)W * H * C);
    y[i] = __bfloat162float(x[(((long)n * H + h) * W + w) * C + c]);
  }
}

// ------------------------------------------------------------------------------------------ stem im2col
// 7x7 stride-2 pad-3 conv over a 3-channel fp32 NCHW image becomes a [N*Ho*Wo] x 192 bf16 matrix
// (k = (ky*7 + kx)*3 + c for k < 147, zero beyond) consumed by the 1x1 GEMM path.
constexpr int STEM_SW = 32;                      // output pixels per strip (one output row)
constexpr int STEM_COLS = 2 * STEM_SW + 5;       // input columns a strip touches
// One CTA = one strip of 32 output pixels of one output row: the 7 x 69 x 3 input patch is staged in shared memory
// with coalesced loads (each input element is read from global once per strip instead of once per tap), then every
// thread assembles 16-byte groups of 8 k-values; consecutive threads write consecutive 16-byte groups.
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, bf16* __restrict__ col, int N,
                                                          int H, int W) {
  mcb::pdl_prologue();
  __shared__ float s[3][7][STEM_COLS + 1];
  const int Ho = H / 2, Wo = W / 2;
  const int strips = (Wo + STEM_SW - 1) / STEM_SW;
  const int strip = blockIdx.x % strips;
  const int oy = (blockIdx.x / strips) % Ho;
  const int n = blockIdx.x / (strips * Ho);
  const int ox0 = strip * STEM_SW;
  const int ix0 = 2 * ox0 - 3, iy0 = 2 * oy - 3;
  for (int e = threadIdx.x; e < 3 * 7 * STEM_COLS; e += blockDim.x) {
    const int cc = e % STEM_COLS;
    const int r = (e / STEM_COLS) % 7;
    const int c = e / (STEM_COLS * 7);
    const int iy = iy0 + r, ix = ix0 + cc;
    float v = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(x + (((long)n * 3 + c) * H + iy) * W + ix);
    s[c][r][cc] = v;
  }
  __syncthreads();
  const int npx = min(STEM_SW, Wo - ox0);
  const long base = (((long)n * Ho + oy) * Wo + ox0) * 24;
  for (int e = threadIdx.x; e < npx * 24; e += blockDim.x) {
    const int g = e % 24;
    const int pl = e / 24;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      float v = 0.f;
      if (k < 147) {
        const int c = k % 3, kx = (k / 3) % 7, ky = k / 21;
        v = s[c][ky][2 * pl + kx];
      }
      f[j] = v;
    }
    reinterpret_cast<uint4*>(col)[base + e] = pack8(f);
  }
}
// master stem weight fp32 [7][7][64][3] (tap-major like every conv) <-> GEMM operand bf16 [64][192]
__global__ void stem_pack_weight_kernel(const float* __restrict__ w, bf16* __restrict__ wp) {
  mcb::pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 192) return;
  const int k = i % 192, co = i / 192;
  float v = 0.f;
  if (k < 147) {
    const int c = k % 3, tap = k / 3;
    v = w[((long)tap * 64 + co) * 3 + c];
  }
  wp[i] = __float2bfloat16(v);
}
__global__ void stem_unpack_wgrad_kernel(const float* __restrict__ dwp, float* __restrict__ dw) {
  mcb::pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 49 * 64 * 3) return;
  const int c = i % 3, co = (i / 3) % 64, tap = i / 192;
  dw[i] += dwp[(long)co * 192 + tap * 3 + c];
}

// ------------------------------------------------------------------------------------------ BatchNorm
// stats = [sum(C), sumsq(C)] of the bf16 conv output -> per-channel affine (scale, shift) + saved mean / invstd,
// running statistics updated like nn.BatchNorm2d (momentum, unbiased variance)
__global__ void bn_finalize_kernel(const float* __restrict__ stats, float count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, float momentum, float eps,
                                   float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean_out,
                                   float* __restrict__ invstd_out, int C) {
  mcb::pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mean = stats[c] / count;
  float var = stats[C + c] / count - mean * mean;
  var = fmaxf(var, 0.f);
  const float invstd = rsqrtf(var + eps);
  const float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - mean * sc;
  mean_out[c] = mean;
  invstd_out[c] = invstd;
  if (running_mean != nullptr) {
    const float unbiased = var * (count / fmaxf(count - 1.f, 1.f));
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
}
__global__ void bn_eval_params_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ rm, const float* __restrict__ rv, float eps,
                                      float* __restrict__ scale, float* __restrict__ shift, int C) {
  mcb::pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float sc = gamma[c] * rsqrtf(rv[c] + eps);
  scale[c] = sc;
  shift[c] = beta[c] - rm[c] * sc;
}

// every BatchNorm of the net in one launch (inference): table rows = {gamma, beta, running_mean, running_var, scale,
// shift, C} as 64-bit values; blockIdx.y = BN index
__global__ void bn_eval_params_batched_kernel(const long long* __restrict__ table, float eps) {
  mcb::pdl_prologue();
  const long long* row = table + (long long)blockIdx.y * 7;
  const float* gamma = reinterpret_cast<const float*>(row[0]);
  const float* beta = reinterpret_cast<const float*>(row[1]);
  const float* rm = reinterpret_cast<const float*>(row[2]);
  const float* rv = reinterpret_cast<const float*>(row[3]);
  float* scale = reinterpret_cast<float*>(row[4]);
  float* shift = reinterpret_cast<float*>(row[5]);
  const int C = (int)row[6];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    const float sc = gamma[c] * rsqrtf(rv[c] + eps);
    scale[c] = sc;
    shift[c] = beta[c] - rm[c] * sc;
  }
}

// y = [relu]( z*scale + shift  [+ r*rscale + rshift | + r] )
// The grid stride is a multiple of C/8, so every thread keeps ONE channel group for its whole loop and the per-channel
// coefficients live in registers; two independent 16-byte loads per stream are in flight per iteration.
template <int RES>  // 0: none, 1: activation residual, 2: residual with its own BN affine
__global__ void __launch_bounds__(256) bn_apply_kernel(const uint4* __restrict__ z, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, const uint4* __restrict__ r,
                                                       const float* __restrict__ rscale, const float* __restrict__ rshift,
                                                       int relu, uint4* __restrict__ y, long total8, int C8) {
  mcb::pdl_prologue();
  const long stride = (long)gridDim.x * blockDim.x;
  long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const int c0 = (int)(i % C8) * 8;
  float sc[8], sh[8], rs[8], rh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = __ldg(scale + c0 + j);
    sh[j] = __ldg(shift + c0 + j);
    if (RES == 2) { rs[j] = __ldg(rscale + c0 + j); rh[j] = __ldg(rshift + c0 + j); }
  }
  for (; i < total8; i += 2 * stride) {
    const long i2 = i + stride;
    const bool has2 = i2 < total8;
    const uint4 za = __ldg(z + i);
    uint4 zb = za, ra = za, rb = za;
    if (has2) zb = __ldg(z + i2);
    if (RES) { ra = __ldg(r + i); if (has2) rb = __ldg(r + i2); }
    float f[8], g[8];
    unpack8(za, f);
    if (RES) unpack8(ra, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      f[j] = fmaf(f[j], sc[j], sh[j]);
      if (RES == 1) f[j] += g[j];
      if (RES == 2) f[j] += fmaf(g[j], rs[j], rh[j]);
      if (relu) f[j] = fmaxf(f[j], 0.f);
    }
    y[i] = pack8(f);
    if (has2) {
      unpack8(zb, f);
      if (RES) unpack8(rb, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        f[j] = fmaf(f[j], sc[j], sh[j]);
        if (RES == 1) f[j] += g[j];
        if (RES == 2) f[j] += fmaf(g[j], rs[j], rh[j]);
        if (relu) f[j] = fmaxf(f[j], 0.f);
      }
      y[i2] = pack8(f);
    }
  }
}

// Training-mode BatchNorm with the statistics finalisation folded in: every thread derives the affine of ITS 8
// channels from the conv epilogue's (sum, sumsq); the first C/8 threads of block 0 also publish mean / invstd for the
// backward pass and update the running statistics (momentum, unbiased variance) — no separate finalize launch.
struct BNTrain {
  const float* stats;   // [2C] sum, sumsq
  const float* gamma;
  const float* beta;
  float* running_mean;  // may be null
  float* running_var;
  float* mean;          // saved for backward
  float* invstd;
};
__device__ __forceinline__ void bn_train_coef(const BNTrain& b, int C, int c0, float count, float eps, float momentum,
                                              bool writer, float (&sc)[8], float (&sh)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    const float mean = __ldg(b.stats + c) / count;
    const float var = fmaxf(__ldg(b.stats + C + c) / count - mean * mean, 0.f);
    const float invstd = rsqrtf(var + eps);
    sc[j] = __ldg(b.gamma + c) * invstd;
    sh[j] = __ldg(b.beta + c) - mean * sc[j];
    if (writer) {
      b.mean[c] = mean;
      b.invstd[c] = invstd;
      if (b.running_mean != nullptr) {
        const float unbiased = var * (count / fmaxf(count - 1.f, 1.f));
        b.running_mean[c] = (1.f - momentum) * b.running_mean[c] + momentum * mean;
        b.running_var[c] = (1.f - momentum) * b.running_var[c] + momentum * unbiased;
      }
    }
  }
}
template <int RES>
__global__ void __launch_bounds__(256) bn_train_apply_kernel(const uint4* __restrict__ z, BNTrain bn,
                                                             const uint4* __restrict__ r, BNTrain rbn, int relu,
                                                             uint4* __restrict__ y, long total8, int C8, float count,
                                                             float eps, float momentum) {
  mcb::pdl_prologue();
  const long stride = (long)gridDim.x * blockDim.x;
  long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const int c0 = (int)(i % C8) * 8;
  const bool writer = (i < C8);
  float sc[8], sh[8], rs[8], rh[8];
  bn_train_coef(bn, C8 * 8, c0, count, eps, momentum, writer, sc, sh);
  if (RES == 2) bn_train_coef(rbn, C8 * 8, c0, count, eps, momentum, writer, rs, rh);
  for (; i < total8; i += 2 * stride) {
    const long i2 = i + stride;
    const bool has2 = i2 < total8;
    const uint4 za = __ldg(z + i);
    uint4 zb = za, ra = za, rb = za;
    if (has2) zb = __ldg(z + i2);
    if (RES) { ra = __ldg(r + i); if (has2) rb = __ldg(r + i2); }
    float f[8], g[8];
    unpack8(za, f);
    if (RES) unpack8(ra, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      f[j] = fmaf(f[j], sc[j], sh[j]);
      if (RES == 1) f[j] += g[j];
      if (RES == 2) f[j] += fmaf(g[j], rs[j], rh[j]);
      if (relu) f[j] = fmaxf(f[j], 0.f);
    }
    y[i] = pack8(f);
    if (has2) {
      unpack8(zb, f);
      if (RES) unpack8(rb, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        f[j] = fmaf(f[j], sc[j], sh[j]);
        if (RES == 1) f[j] += g[j];
        if (RES == 2) f[j] += fmaf(g[j], rs[j], rh[j]);
        if (relu) f[j] = fmaxf(f[j], 0.f);
      }
      y[i2] = pack8(f);
    }
  }
}

// per-block partial rows of channel_reduce_kernel ([out0 | out1] over C channels) and final_conv_bwd_kernel ([dW | db]),
// summed in block order by the finishing kernels (detsum.cuh)
constexpr long kChannelRedCap = 1024L * 2 * 2048;
constexpr long kFinalRedCap = 1024L * 66;
MCB_DET_WORKSPACE(float, g_channel_red, kChannelRedCap, channel_red_finish_kernel)
MCB_DET_WORKSPACE(float, g_final_red, kFinalRedCap, final_red_finish_kernel)

// Per-channel reductions over NHWC: block = 256 threads = (256 / C8) pixel lanes x C8 channel groups (C8 = C/8 <= 256).
// MODE 0: sum(x)                                  -> out0                 (bias gradient)
// MODE 1: g = dy * (y > 0); sum(g), sum(g * xhat) -> out0 (dbeta), out1 (dgamma)   xhat = (z - mean) * invstd
template <int MODE>
__global__ void channel_reduce_kernel(const uint4* __restrict__ a, const uint4* __restrict__ ymask,
                                      const uint4* __restrict__ z, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, float* __restrict__ out0,
                                      float* __restrict__ out1, long pixels, int C8) {
  mcb::pdl_prologue();
  extern __shared__ float red[];  // [2][256][8]
  const int cg = threadIdx.x % C8;
  const int lane_p = threadIdx.x / C8;
  const int lanes = blockDim.x / C8;
  float s0[8], s1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
  float mu[8], is[8];
  if (MODE == 1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mu[j] = __ldg(mean + cg * 8 + j);
      is[j] = __ldg(invstd + cg * 8 + j);
    }
  }
  if (lane_p < lanes) {
    const long pstride = (long)gridDim.x * lanes;
    for (long p = (long)blockIdx.x * lanes + lane_p; p < pixels; p += 2 * pstride) {
      const long ia = p * C8 + cg;
      const long ib = (p + pstride) * C8 + cg;
      const bool hb = (p + pstride) < pixels;
      const uint4 va = __ldg(a + ia);
      uint4 vb = va, za = va, zb = va, ma = va, mb = va;
      if (hb) vb = __ldg(a + ib);
      if (MODE == 1) {
        za = __ldg(z + ia);
        if (hb) zb = __ldg(z + ib);
        if (ymask != nullptr) {
          ma = __ldg(ymask + ia);
          if (hb) mb = __ldg(ymask + ib);
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (u == 1 && !hb) break;
        float f[8];
        unpack8(u ? vb : va, f);
        if (MODE == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) s0[j] += f[j];
        } else {
          float m[8], zz[8];
          unpack8(u ? zb : za, zz);
          if (ymask != nullptr) {
            unpack8(u ? mb : ma, m);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = (m[j] > 0.f) ? f[j] : 0.f;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            s0[j] += f[j];
            s1[j] += f[j] * ((zz[j] - mu[j]) * is[j]);
          }
        }
      }
    }
  }
  float* r0 = red;
  float* r1 = red + blockDim.x * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    r0[threadIdx.x * 8 + j] = s0[j];
    if (MODE == 1) r1[threadIdx.x * 8 + j] = s1[j];
  }
  __syncthreads();
  // threads 0 .. C8*8-1 each own one channel and sum over the pixel lanes into this block's row
  float* row = g_channel_red + (size_t)blockIdx.x * 2 * (C8 * 8);
  for (int ch = threadIdx.x; ch < C8 * 8; ch += blockDim.x) {
    const int g = ch / 8, j = ch % 8;
    float t0 = 0.f, t1 = 0.f;
    for (int l = 0; l < lanes; ++l) {
      t0 += r0[(l * C8 + g) * 8 + j];
      if (MODE == 1) t1 += r1[(l * C8 + g) * 8 + j];
    }
    row[ch] = t0;
    if (MODE == 1) row[C8 * 8 + ch] = t1;
  }
}

// dz = gamma*invstd * (g - dbeta/M - xhat * dgamma/M),  g = dy * (y > 0); optionally also emits g (the gradient that
// flows to the residual branch): g_out = g (store) or g_out += g (accumulate).  Per-channel coefficients in registers
// (fixed channel group per thread), two independent loads per stream in flight.
template <bool MASK, int GOUT>  // GOUT 0: none, 1: store, 2: accumulate
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ ymask,
                                                           const uint4* __restrict__ z, const float* __restrict__ mean,
                                                           const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                           const float* __restrict__ dbeta, const float* __restrict__ dgamma,
                                                           float inv_count, uint4* __restrict__ dz, uint4* __restrict__ g_out,
                                                           long total8, int C8) {
  mcb::pdl_prologue();
  const long stride = (long)gridDim.x * blockDim.x;
  long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
  const int c0 = (int)(i % C8) * 8;
  float mu[8], is[8], a[8], k1[8], k2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mu[j] = __ldg(mean + c0 + j);
    is[j] = __ldg(invstd + c0 + j);
    a[j] = __ldg(gamma + c0 + j) * is[j];
    k1[j] = __ldg(dbeta + c0 + j) * inv_count;
    k2[j] = __ldg(dgamma + c0 + j) * inv_count;
  }
  for (; i < total8; i += 2 * stride) {
    const long idx[2] = {i, i + stride};
    const bool has[2] = {true, idx[1] < total8};
    uint4 vdy[2], vz[2], vm[2], vg[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (has[u]) {
        vdy[u] = __ldg(dy + idx[u]);
        vz[u] = __ldg(z + idx[u]);
        if (MASK) vm[u] = __ldg(ymask + idx[u]);
        if (GOUT == 2) vg[u] = g_out[idx[u]];
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (!has[u]) continue;
      float g[8], zz[8], o[8];
      unpack8(vdy[u], g);
      unpack8(vz[u], zz);
      if (MASK) {
        float m[8];
        unpack8(vm[u], m);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = (m[j] > 0.f) ? g[j] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (zz[j] - mu[j]) * is[j];
        o[j] = a[j] * (g[j] - k1[j] - xh * k2[j]);
      }
      dz[idx[u]] = pack8(o);
      if (GOUT) {
        if (GOUT == 2) {
          float e[8];
          unpack8(vg[u], e);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] += e[j];
        }
        g_out[idx[u]] = pack8(g);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ 2x2 max-pool
__global__ void maxpool2_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int N, int H, int W, int C8) {
  mcb::pdl_prologue();
  const int Ho = H / 2, Wo = W / 2;
  const long total = (long)N * Ho * Wo * C8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int cg = i % C8;
    const long p = i / C8;
    const int ox = p % Wo, oy = (p / Wo) % Ho;
    const long n = p / ((long)Wo * Ho);
    const long base = ((n * H + 2 * oy) * W + 2 * ox) * C8 + cg;
    float a[8], b[8], c[8], d[8];
    unpack8(__ldg(x + base), a);
    unpack8(__ldg(x + base + C8), b);
    unpack8(__ldg(x + base + (long)W * C8), c);
    unpack8(__ldg(x + base + (long)W * C8 + C8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = fmaxf(fmaxf(a[j], b[j]), fmaxf(c[j], d[j]));
    y[i] = pack8(a);
  }
}
// gradient goes to the FIRST maximum in window scan order (torch's max_pool2d backward);
// dx = (store | accumulate) routed gradient
__global__ void maxpool2_bwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ dy, uint4* __restrict__ dx,
                                    int accumulate, int N, int H, int W, int C8) {
  mcb::pdl_prologue();
  const int Ho = H / 2, Wo = W / 2;
  const long total = (long)N * Ho * Wo * C8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int cg = i % C8;
    const long p = i / C8;
    const int ox = p % Wo, oy = (p / Wo) % Ho;
    const long n = p / ((long)Wo * Ho);
    const long base = ((n * H + 2 * oy) * W + 2 * ox) * C8 + cg;
    const long idx[4] = {base, base + C8, base + (long)W * C8, base + (long)W * C8 + C8};
    float v[4][8], g[8], o[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) unpack8(__ldg(x + idx[k]), v[k]);
    unpack8(__ldg(dy + i), g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int best = 0;
      float m = v[0][j];
#pragma unroll
      for (int k = 1; k < 4; ++k)
        if (v[k][j] > m) { m = v[k][j]; best = k; }
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k][j] = (k == best) ? g[j] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (accumulate) {
        float e[8];
        unpack8(dx[idx[k]], e);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[k][j] += e[j];
      }
      dx[idx[k]] = pack8(o[k]);
    }
  }
}

// ------------------------------------------------------------------------------------------ final 1x1 classifier
// logits[n][k][h][w] (fp32 NCHW, the reference's output layout) = W[k][:] . x[n][h][w][:] + b[k];  C = 32, K = 2
__global__ void final_conv_fwd_kernel(const uint4* __restrict__ x, const float* __restrict__ w,
                                      const float* __restrict__ b, float* __restrict__ logits, long pixels_per_img,
                                      long pixels, int C, int K) {
  mcb::pdl_prologue();
  extern __shared__ float sw[];  // K*C + K
  for (int i = threadIdx.x; i < K * C + K; i += blockDim.x) sw[i] = (i < K * C) ? w[i] : b[i - K * C];
  __syncthreads();
  const int C8 = C / 8;
  for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pixels; p += (long)gridDim.x * blockDim.x) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int g = 0; g < C8; ++g) {
      float f[8];
      unpack8(__ldg(x + p * C8 + g), f);
      for (int k = 0; k < K; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[k] = fmaf(f[j], sw[k * C + g * 8 + j], acc[k]);
    }
    const long n = p / pixels_per_img, q = p % pixels_per_img;
    for (int k = 0; k < K; ++k) logits[(n * K + k) * pixels_per_img + q] = acc[k] + sw[K * C + k];
  }
}
// backward: dx[p][c] = (x[p][c] > 0) * sum_k dlogits[k][p] W[k][c];  dW[k][c] += sum_p dlogits[k][p] x[p][c];
// db[k] += sum_p dlogits[k][p].   x is the ReLU output of dec0, so the mask folds dec0's ReLU backward in.
__global__ void final_conv_bwd_kernel(const uint4* __restrict__ x, const float* __restrict__ w,
                                      const float* __restrict__ dlogits, uint4* __restrict__ dx,
                                      float* __restrict__ dw, float* __restrict__ db, long pixels_per_img,
                                      long pixels, int C, int K) {
  mcb::pdl_prologue();
  extern __shared__ float sm[];  // K*C weights, then per warp K*C + K accumulators
  float* sw = sm;
  float* sacc = sm + K * C;
  for (int i = threadIdx.x; i < K * C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int C8 = C / 8;
  float lw[2][32];  // per-thread partial dW (K <= 2, C <= 32)
  float lb[2] = {0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int c = 0; c < 32; ++c) lw[k][c] = 0.f;
  for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pixels; p += (long)gridDim.x * blockDim.x) {
    const long n = p / pixels_per_img, q = p % pixels_per_img;
    float d[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      d[k] = __ldg(dlogits + (n * K + k) * pixels_per_img + q);
      lb[k] += d[k];
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      float f[8], o[8];
      unpack8(__ldg(x + p * C8 + g), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = g * 8 + j;
        lw[0][c] = fmaf(d[0], f[j], lw[0][c]);
        lw[1][c] = fmaf(d[1], f[j], lw[1][c]);
        o[j] = (f[j] > 0.f) ? (d[0] * sw[c] + d[1] * sw[C + c]) : 0.f;
      }
      dx[p * C8 + g] = pack8(o);
    }
  }
  // warp reduce into per-warp slots, then the warps in order into this block's row [dW | db]
  const int n_acc = K * C + K, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      float v = lw[k][c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0) sacc[wid * n_acc + k * C + c] = v;
    }
    float v = lb[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sacc[wid * n_acc + K * C + k] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_acc; i += blockDim.x) {
    float t = 0.f;
    for (int w8 = 0; w8 < (int)(blockDim.x >> 5); ++w8) t += sacc[w8 * n_acc + i];
    g_final_red[(size_t)blockIdx.x * n_acc + i] = t;
  }
}

// ------------------------------------------------------------------------------------------ fused Adam
// torch.optim.Adam with L2 weight decay folded into the gradient (src/models.py:57,287-292), over one flat fp32
// parameter arena; also refreshes the bf16 operand copy of the weights (same layout) for the next forward.
// hyper (optional, device): {lr, bc1, sqrt(bc2)} of this step -- lets the launch sit inside a replayed CUDA graph
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, bf16* __restrict__ p_bf16, long n, float lr, float beta1,
                            float beta2, float eps, float wd, float bc1, float bc2_sqrt, float grad_scale,
                            const float* __restrict__ hyper) {
  mcb::pdl_prologue();
  if (hyper != nullptr) {
    lr = __ldg(hyper);
    bc1 = __ldg(hyper + 1);
    bc2_sqrt = __ldg(hyper + 2);
  }
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float pi = p[i];
    const float gi = g[i] * grad_scale + wd * pi;
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pi -= (lr / bc1) * (mi / denom);
    p[i] = pi;
    if (p_bf16 != nullptr) p_bf16[i] = __float2bfloat16(pi);
  }
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, bf16* __restrict__ y, long n) {
  mcb::pdl_prologue();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(x[i]);
}

}  // namespace mcb

using namespace mcb;
#define ST static_cast<cudaStream_t>(stream)

extern "C" int mcb_nchw_f32_to_nhwc_bf16(const float* x, void* y, int n, int c, int h, int w, void* stream) {
  MCB_REQUIRE(x && y, "null pointer");
  const long total = (long)n * c * h * w;
  launch_pdl(nchw_f32_to_nhwc_bf16_kernel, grid_for(total, 256), 256, 0, ST, x, (bf16*)y, n, c, h, w);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_nhwc_bf16_to_nchw_f32(const void* x, float* y, int n, int c, int h, int w, void* stream) {
  MCB_REQUIRE(x && y, "null pointer");
  const long total = (long)n * c * h * w;
  launch_pdl(nhwc_bf16_to_nchw_f32_kernel, grid_for(total, 256), 256, 0, ST, (const bf16*)x, y, n, c, h, w);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_stem_im2col(const float* x, void* col, int n, int h, int w, void* stream) {
  MCB_REQUIRE(x && col, "null pointer");
  MCB_REQUIRE(h % 2 == 0 && w % 2 == 0, "stem_im2col: odd size");
  const long ctas = (long)n * (h / 2) * (((w / 2) + STEM_SW - 1) / STEM_SW);  // one per strip of an output row
  MCB_REQUIRE(ctas < (1L << 31), "stem_im2col: too many strips");
  launch_pdl(stem_im2col_kernel, dim3((unsigned)ctas), 256, 0, ST, x, (bf16*)col, n, h, w);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_stem_pack_weight(const float* w, void* wp, void* stream) {
  MCB_REQUIRE(w && wp, "null pointer");
  launch_pdl(stem_pack_weight_kernel, (64 * 192 + 255) / 256, 256, 0, ST, w, (bf16*)wp);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_stem_unpack_wgrad(const float* dwp, float* dw, void* stream) {
  MCB_REQUIRE(dwp && dw, "null pointer");
  launch_pdl(stem_unpack_wgrad_kernel, (49 * 64 * 3 + 255) / 256, 256, 0, ST, dwp, dw);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_bn_finalize(const float* stats, long count, const float* gamma, const float* beta,
                               float* running_mean, float* running_var, float momentum, float eps, float* scale,
                               float* shift, float* mean, float* invstd, int c, void* stream) {
  MCB_REQUIRE(stats && gamma && beta && scale && shift && mean && invstd, "bn_finalize: null pointer");
  launch_pdl(bn_finalize_kernel, (c + 127) / 128, 128, 0, ST, stats, (float)count, gamma, beta, running_mean, running_var,
                                                      momentum, eps, scale, shift, mean, invstd, c);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_bn_eval_params(const float* gamma, const float* beta, const float* running_mean,
                                  const float* running_var, float eps, float* scale, float* shift, int c,
                                  void* stream) {
  MCB_REQUIRE(gamma && beta && running_mean && running_var && scale && shift, "bn_eval_params: null pointer");
  launch_pdl(bn_eval_params_kernel, (c + 127) / 128, 128, 0, ST, gamma, beta, running_mean, running_var, eps, scale, shift, c);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_bn_eval_params_batched(const long long* table, int n_bn, int max_c, float eps, void* stream) {
  MCB_REQUIRE(table && n_bn > 0 && max_c > 0, "bn_eval_params_batched: bad arguments");
  dim3 grid((max_c + 255) / 256, n_bn);
  launch_pdl(bn_eval_params_batched_kernel, grid, 256, 0, ST, table, eps);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_bn_apply(const void* z, const float* scale, const float* shift, const void* residual,
                            const float* res_scale, const float* res_shift, int relu, void* y, long pixels, int c,
                            void* stream) {
  MCB_REQUIRE(z && scale && shift && y, "bn_apply: null pointer");
  MCB_REQUIRE(c % 8 == 0, "bn_apply: channels %d not a multiple of 8", c);
  MCB_REQUIRE(256 % (c / 8) == 0, "bn_apply: channels %d (c/8 must divide 256)", c);
  const long total8 = pixels * (c / 8);
  const int grid = grid_for((total8 + 1) / 2, 256);
  if (residual == nullptr)
    launch_pdl(bn_apply_kernel<0>, grid, 256, 0, ST, (const uint4*)z, scale, shift, nullptr, nullptr, nullptr, relu, (uint4*)y,
                                             total8, c / 8);
  else if (res_scale == nullptr)
    launch_pdl(bn_apply_kernel<1>, grid, 256, 0, ST, (const uint4*)z, scale, shift, (const uint4*)residual, nullptr, nullptr,
                                             relu, (uint4*)y, total8, c / 8);
  else
    launch_pdl(bn_apply_kernel<2>, grid, 256, 0, ST, (const uint4*)z, scale, shift, (const uint4*)residual, res_scale,
                                             res_shift, relu, (uint4*)y, total8, c / 8);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_bn_train_apply(const void* z, const mcb_bn_train* bn, const void* residual,
                                  const mcb_bn_train* res_bn, int relu, void* y, long pixels, int c, float momentum,
                                  float eps, void* stream) {
  return mcb_bn_train_apply_global(z, bn, residual, res_bn, relu, y, pixels, pixels, c, momentum, eps, stream);
}
extern "C" int mcb_bn_train_apply_global(const void* z, const mcb_bn_train* bn, const void* residual,
                                         const mcb_bn_train* res_bn, int relu, void* y, long pixels, long stat_count,
                                         int c, float momentum, float eps, void* stream) {
  MCB_REQUIRE(stat_count >= pixels, "bn_train_apply: stat_count %ld < pixels %ld", stat_count, pixels);
  MCB_REQUIRE(z && bn && y && bn->stats && bn->gamma && bn->beta && bn->mean && bn->invstd, "bn_train_apply: null pointer");
  MCB_REQUIRE(c % 8 == 0 && 256 % (c / 8) == 0, "bn_train_apply: channels %d (c/8 must divide 256)", c);
  MCB_REQUIRE(!(res_bn && !residual), "bn_train_apply: res_bn without residual");
  const long total8 = pixels * (c / 8);
  const int grid = grid_for((total8 + 1) / 2, 256);
  BNTrain b{bn->stats, bn->gamma, bn->beta, bn->running_mean, bn->running_var, bn->mean, bn->invstd};
  BNTrain rb{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  if (res_bn) rb = BNTrain{res_bn->stats, res_bn->gamma, res_bn->beta, res_bn->running_mean, res_bn->running_var,
                           res_bn->mean, res_bn->invstd};
  const float count = (float)stat_count;
  if (residual == nullptr)
    launch_pdl(bn_train_apply_kernel<0>, grid, 256, 0, ST, (const uint4*)z, b, nullptr, rb, relu, (uint4*)y, total8, c / 8, count, eps, momentum);
  else if (res_bn == nullptr)
    launch_pdl(bn_train_apply_kernel<1>, grid, 256, 0, ST, (const uint4*)z, b, (const uint4*)residual, rb, relu, (uint4*)y, total8, c / 8, count, eps, momentum);
  else
    launch_pdl(bn_train_apply_kernel<2>, grid, 256, 0, ST, (const uint4*)z, b, (const uint4*)residual, rb, relu, (uint4*)y, total8, c / 8, count, eps, momentum);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

static int reduce_cfg(int c, int* threads, int* c8) {
  *c8 = c / 8;
  if (c % 8 != 0 || *c8 > 256) return fail(MCB_ERR_UNSUPPORTED, "channel reduce: channels %d", c);
  *threads = 256 - (256 % *c8);
  if (*threads < *c8) *threads = *c8;
  return MCB_OK;
}
extern "C" int mcb_channel_sum(const void* x, float* out, long pixels, int c, void* stream) {
  MCB_REQUIRE(x && out, "channel_sum: null pointer");
  int threads, c8;
  if (int r = reduce_cfg(c, &threads, &c8)) return r;
  const int lanes = threads / c8;
  const int grid = (int)std::max(1L, std::min((pixels + lanes * 4 - 1) / (lanes * 4), (long)num_sms() * 4));
  MCB_REQUIRE((long)grid * 2 * c <= kChannelRedCap, "channel_sum: %d blocks x %d channels exceed the workspace", grid, c);
  launch_pdl(channel_reduce_kernel<0>, grid, threads, (size_t)threads * 8 * 2 * sizeof(float), ST, 
      (const uint4*)x, nullptr, nullptr, nullptr, nullptr, out, nullptr, pixels, c8);
  launch_pdl(channel_red_finish_kernel, det_finish_grid(c), kDetFinishThreads, 0, ST, 0L, grid, 2L * c, (long)c,
             (long)c, out, 0L);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_bn_bwd_reduce(const void* dy, const void* y_mask, const void* z, const float* mean,
                                 const float* invstd, float* dbeta, float* dgamma, long pixels, int c, void* stream) {
  MCB_REQUIRE(dy && z && mean && invstd && dbeta && dgamma, "bn_bwd_reduce: null pointer");
  int threads, c8;
  if (int r = reduce_cfg(c, &threads, &c8)) return r;
  const int lanes = threads / c8;
  const int grid = (int)std::max(1L, std::min((pixels + lanes * 4 - 1) / (lanes * 4), (long)num_sms() * 4));
  MCB_REQUIRE((long)grid * 2 * c <= kChannelRedCap, "bn_bwd_reduce: %d blocks x %d channels exceed the workspace", grid, c);
  launch_pdl(channel_reduce_kernel<1>, grid, threads, (size_t)threads * 8 * 2 * sizeof(float), ST, 
      (const uint4*)dy, (const uint4*)y_mask, (const uint4*)z, mean, invstd, dbeta, dgamma, pixels, c8);
  launch_pdl(channel_red_finish_kernel, det_finish_grid(c), kDetFinishThreads, 0, ST, 0L, grid, 2L * c, (long)c,
             (long)c, dbeta, 0L);
  launch_pdl(channel_red_finish_kernel, det_finish_grid(c), kDetFinishThreads, 0, ST, (long)c, grid, 2L * c, (long)c,
             (long)c, dgamma, 0L);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_bn_bwd_apply(const void* dy, const void* y_mask, const void* z, const float* mean,
                                const float* invstd, const float* gamma, const float* dbeta, const float* dgamma,
                                void* dz, void* g_out, int g_accumulate, long pixels, int c, void* stream) {
  return mcb_bn_bwd_apply_global(dy, y_mask, z, mean, invstd, gamma, dbeta, dgamma, dz, g_out, g_accumulate, pixels,
                                 pixels, c, stream);
}
extern "C" int mcb_bn_bwd_apply_global(const void* dy, const void* y_mask, const void* z, const float* mean,
                                       const float* invstd, const float* gamma, const float* dbeta, const float* dgamma,
                                       void* dz, void* g_out, int g_accumulate, long pixels, long stat_count, int c,
                                       void* stream) {
  MCB_REQUIRE(stat_count >= pixels, "bn_bwd_apply: stat_count %ld < pixels %ld", stat_count, pixels);
  MCB_REQUIRE(dy && z && mean && invstd && gamma && dbeta && dgamma && dz, "bn_bwd_apply: null pointer");
  MCB_REQUIRE(c % 8 == 0, "bn_bwd_apply: channels %d", c);
  MCB_REQUIRE(256 % (c / 8) == 0, "bn_bwd_apply: channels %d (c/8 must divide 256)", c);
  const long total8 = pixels * (c / 8);
  const int grid = grid_for((total8 + 1) / 2, 256);
  const float ic = 1.0f / (float)stat_count;
#define MCB_BWD(MASK, GOUT)                                                                                         \
  launch_pdl(bn_bwd_apply_kernel<MASK, GOUT>, grid, 256, 0, ST, (const uint4*)dy, (const uint4*)y_mask, (const uint4*)z, mean, \
                                                        invstd, gamma, dbeta, dgamma, ic, (uint4*)dz, (uint4*)g_out,  \
                                                        total8, c / 8)
  const int gout = g_out == nullptr ? 0 : (g_accumulate ? 2 : 1);
  if (y_mask != nullptr) {
    if (gout == 0) MCB_BWD(true, 0); else if (gout == 1) MCB_BWD(true, 1); else MCB_BWD(true, 2);
  } else {
    if (gout == 0) MCB_BWD(false, 0); else if (gout == 1) MCB_BWD(false, 1); else MCB_BWD(false, 2);
  }
#undef MCB_BWD
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_maxpool2_fwd(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  MCB_REQUIRE(x && y, "maxpool2_fwd: null pointer");
  MCB_REQUIRE(c % 8 == 0 && h % 2 == 0 && w % 2 == 0, "maxpool2_fwd: shape");
  const long total = (long)n * (h / 2) * (w / 2) * (c / 8);
  launch_pdl(maxpool2_fwd_kernel, grid_for(total, 256), 256, 0, ST, (const uint4*)x, (uint4*)y, n, h, w, c / 8);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_maxpool2_bwd(const void* x, const void* dy, void* dx, int accumulate, int n, int h, int w, int c,
                                void* stream) {
  MCB_REQUIRE(x && dy && dx, "maxpool2_bwd: null pointer");
  MCB_REQUIRE(c % 8 == 0 && h % 2 == 0 && w % 2 == 0, "maxpool2_bwd: shape");
  const long total = (long)n * (h / 2) * (w / 2) * (c / 8);
  launch_pdl(maxpool2_bwd_kernel, grid_for(total, 256), 256, 0, ST, (const uint4*)x, (const uint4*)dy, (uint4*)dx, accumulate,
                                                            n, h, w, c / 8);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_final_conv_fwd(const void* x, const float* w, const float* b, float* logits, int n, int h, int wd,
                                  int c, int k, void* stream) {
  MCB_REQUIRE(x && w && b && logits, "final_conv_fwd: null pointer");
  MCB_REQUIRE(c % 8 == 0 && k >= 1 && k <= 4, "final_conv_fwd: c %d k %d", c, k);
  const long ppi = (long)h * wd, pixels = ppi * n;
  launch_pdl(final_conv_fwd_kernel, grid_for(pixels, 256), 256, (size_t)(k * c + k) * sizeof(float), ST, 
      (const uint4*)x, w, b, logits, ppi, pixels, c, k);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_final_conv_bwd(const void* x, const float* w, const float* dlogits, void* dx, float* dw, float* db,
                                  int n, int h, int wd, int c, int k, void* stream) {
  MCB_REQUIRE(x && w && dlogits && dx && dw && db, "final_conv_bwd: null pointer");
  MCB_REQUIRE(c == 32 && k == 2, "final_conv_bwd: only the reference's 32 -> 2 classifier is built");
  const long ppi = (long)h * wd, pixels = ppi * n;
  const int grid = grid_for(pixels, 128, 4), n_acc = k * c + k;
  MCB_REQUIRE((long)grid * n_acc <= kFinalRedCap, "final_conv_bwd: %d blocks exceed the workspace", grid);
  launch_pdl(final_conv_bwd_kernel, grid, 128, (size_t)(k * c + 4 * n_acc) * sizeof(float), ST, 
      (const uint4*)x, w, dlogits, (uint4*)dx, dw, db, ppi, pixels, c, k);
  launch_pdl(final_red_finish_kernel, det_finish_grid(k * c), kDetFinishThreads, 0, ST, 0L, grid, (long)n_acc,
             (long)(k * c), (long)(k * c), dw, 0L);
  launch_pdl(final_red_finish_kernel, det_finish_grid(k), kDetFinishThreads, 0, ST, (long)(k * c), grid, (long)n_acc,
             (long)k, (long)k, db, 0L);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_adam_step(float* p, const float* g, float* m, float* v, void* p_bf16, long n, float lr, float beta1,
                             float beta2, float eps, float weight_decay, int step, float grad_scale, void* stream) {
  MCB_REQUIRE(p && g && m && v, "adam_step: null pointer");
  MCB_REQUIRE(step >= 1, "adam_step: step %d", step);
  // bias corrections in double, like torch.optim.Adam's Python-side arithmetic
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  launch_pdl(adam_kernel, grid_for(n, 256), 256, 0, ST, p, g, m, v, (bf16*)p_bf16, n, lr, beta1, beta2, eps, weight_decay,
                                                (float)bc1, (float)sqrt(bc2), grad_scale, (const float*)nullptr);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_adam_step_dyn(float* p, const float* g, float* m, float* v, void* p_bf16, long n,
                                 const float* hyper, float beta1, float beta2, float eps, float weight_decay,
                                 float grad_scale, void* stream) {
  MCB_REQUIRE(p && g && m && v && hyper, "adam_dyn: null pointer");
  if (n == 0) return MCB_OK;
  launch_pdl(adam_kernel, grid_for(n, 256), 256, 0, ST, p, g, m, v, (bf16*)p_bf16, n, 0.f, beta1, beta2, eps,
             weight_decay, 1.f, 1.f, grad_scale, hyper);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
extern "C" int mcb_cast_f32_bf16(const float* x, void* y, long n, void* stream) {
  MCB_REQUIRE(x && y, "cast: null pointer");
  launch_pdl(cast_f32_bf16_kernel, grid_for(n, 256), 256, 0, ST, x, (bf16*)y, n);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
