// loss.cu — the reference's training losses as two-phase fused kernels (SURVEY.md Appendix C):
//   mode 0: PyTorchUNetWeighted  L = dice_w * Dice_1 + ce_w * mean(w * CE)      (src/models.py:149-161,310-454,
//           src/steps/pytorch/validation.py:8-16), w = distance weight * size weight (src/models.py:339-381)
//   mode 1: PyTorchUNet          L = mean(CE)                                     (src/steps/pytorch/validation.py:25-28)
// Phase 1 reduces the four global sums (I = sum p1*t, P = sum p1, T = sum t, S = sum w*ce) — the only cross-pixel
// (and cross-GPU: all-reduce them between the phases) coupling; phase 2 writes the loss and d(loss)/d(logits).
#include "host_common.h"
#include "../../include/mcb200.h"
#include "detsum.cuh"
#include <algorithm>

namespace mcb {

struct LossCfg {
  int mode;
  float w0, sigma2, C;      // distance / size weights
  float dice_w, ce_w, smooth, eps;
};

__device__ __forceinline__ float pixel_weight(const LossCfg& cfg, float d, float s) {
  float wd = 1.f + cfg.w0 * expf(-(d * d) / cfg.sigma2);
  if (d == 0.f) wd = 1.f;
  float s_ = (s == 0.f) ? 1.f : s;
  float ws = cfg.C / s_;
  if (s_ == 1.f) ws = 1.f;
  return wd * ws;
}

// per-block rows of the four loss sums, added in block order by loss_red_finish_kernel (detsum.cuh)
constexpr long kLossRedCap = 2048L * 4;
MCB_DET_WORKSPACE(double, g_loss_red, kLossRedCap, loss_red_finish_kernel)

__global__ void loss_partials_kernel(const float* __restrict__ logits, const float* __restrict__ target, LossCfg cfg,
                                     double* __restrict__ sums, long ppi, long pixels, int tch) {
  mcb::pdl_prologue();
  float aI = 0.f, aP = 0.f, aT = 0.f, aS = 0.f;
  for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pixels; p += (long)gridDim.x * blockDim.x) {
    const long n = p / ppi, q = p % ppi;
    const float z0 = __ldg(logits + (n * 2) * ppi + q), z1 = __ldg(logits + (n * 2 + 1) * ppi + q);
    const float t = (float)(long)__ldg(target + (n * tch) * ppi + q);  // .long() truncation like the reference
    const float m = fmaxf(z0, z1);
    const float e0 = expf(z0 - m), e1 = expf(z1 - m);
    const float se = e0 + e1;
    const float p1 = e1 / se;
    const float ce = m + logf(se) - (t != 0.f ? z1 : z0);
    float w = 1.f;
    if (cfg.mode == 0) w = pixel_weight(cfg, __ldg(target + (n * tch + 1) * ppi + q), __ldg(target + (n * tch + 2) * ppi + q));
    const float t1 = (t == 1.f) ? 1.f : 0.f;
    aI += p1 * t1;
    aP += p1;
    aT += t1;
    aS += w * ce;
  }
  __shared__ float red[4][32];
  float v[4] = {aI, aP, aT, aS};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += (double)red[threadIdx.x][w];
    g_loss_red[(size_t)blockIdx.x * 4 + threadIdx.x] = t;
  }
}

__global__ void loss_grad_kernel(const float* __restrict__ logits, const float* __restrict__ target, LossCfg cfg,
                                 const double* __restrict__ sums, double global_pixels, float grad_scale,
                                 float* __restrict__ dlogits, float* __restrict__ loss_out, long ppi, long pixels,
                                 int tch) {
  mcb::pdl_prologue();
  const double I = sums[0], P = sums[1], T = sums[2], S = sums[3];
  const double Dn = P + T + (double)cfg.smooth + (double)cfg.eps;
  const double num = 2.0 * I + (double)cfg.smooth;
  if (blockIdx.x == 0 && threadIdx.x == 0 && loss_out != nullptr) {
    double L = (double)cfg.ce_w * S / global_pixels;
    if (cfg.mode == 0) L += (double)cfg.dice_w * (1.0 - num / Dn);
    *loss_out = (float)L;
  }
  const float inv_M = (float)(1.0 / global_pixels);
  const float gA = (float)(-2.0 / Dn);            // d(1 - num/Dn)/dp1 = -(2 t Dn - num)/Dn^2 = t*gA + gB
  const float gB = (float)(num / (Dn * Dn));
  for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pixels; p += (long)gridDim.x * blockDim.x) {
    const long n = p / ppi, q = p % ppi;
    const float z0 = __ldg(logits + (n * 2) * ppi + q), z1 = __ldg(logits + (n * 2 + 1) * ppi + q);
    const float t = (float)(long)__ldg(target + (n * tch) * ppi + q);
    const float m = fmaxf(z0, z1);
    const float e0 = expf(z0 - m), e1 = expf(z1 - m);
    const float se = e0 + e1;
    const float p1 = e1 / se, p0 = e0 / se;
    float w = 1.f;
    if (cfg.mode == 0) w = pixel_weight(cfg, __ldg(target + (n * tch + 1) * ppi + q), __ldg(target + (n * tch + 2) * ppi + q));
    const float oh1 = (t != 0.f) ? 1.f : 0.f;  // CE target class (class index t)
    float d1 = cfg.ce_w * w * inv_M * (p1 - oh1);
    float d0 = cfg.ce_w * w * inv_M * (p0 - (1.f - oh1));
    if (cfg.mode == 0) {
      const float t1 = (t == 1.f) ? 1.f : 0.f;
      const float g = cfg.dice_w * (t1 * gA + gB) * p1 * p0;
      d1 += g;
      d0 -= g;
    }
    dlogits[(n * 2) * ppi + q] = d0 * grad_scale;
    dlogits[(n * 2 + 1) * ppi + q] = d1 * grad_scale;
  }
}

// numpy softmax over the class axis of NCHW logits (src/utils.py:231-273 as used at src/models.py:88-92)
__global__ void softmax2_kernel(const float* __restrict__ logits, float* __restrict__ probs, long ppi, long pixels) {
  mcb::pdl_prologue();
  for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pixels; p += (long)gridDim.x * blockDim.x) {
    const long n = p / ppi, q = p % ppi;
    const float z0 = logits[(n * 2) * ppi + q], z1 = logits[(n * 2 + 1) * ppi + q];
    const float m = fmaxf(z0, z1);
    const float e0 = expf(z0 - m), e1 = expf(z1 - m);
    const float se = e0 + e1;
    probs[(n * 2) * ppi + q] = e0 / se;
    probs[(n * 2 + 1) * ppi + q] = e1 / se;
  }
}

static LossCfg make_cfg(const mcb_loss_args* a) {
  LossCfg c;
  c.mode = a->mode;
  c.w0 = a->w0;
  c.sigma2 = a->sigma * a->sigma;
  c.C = a->size_c;
  c.dice_w = a->dice_weight;
  c.ce_w = a->ce_weight;
  c.smooth = a->dice_smooth;
  c.eps = 1e-7f;
  return c;
}
static int loss_grid(long pixels) {
  return (int)std::max(1L, std::min((pixels + 255) / 256, (long)num_sms() * 8));
}

}  // namespace mcb

using namespace mcb;

extern "C" int mcb_loss_partials(const mcb_loss_args* a, double* sums, void* stream) {
  MCB_REQUIRE(a && a->logits && a->target && sums, "loss_partials: null pointer");
  MCB_REQUIRE(a->mode == 0 || a->mode == 1, "loss: mode %d", a->mode);
  const long ppi = (long)a->h * a->w, pixels = ppi * a->n;
  const int grid = loss_grid(pixels);
  MCB_REQUIRE((long)grid * 4 <= kLossRedCap, "loss_partials: %d blocks exceed the workspace", grid);
  launch_pdl(loss_partials_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), 
      a->logits, a->target, make_cfg(a), sums, ppi, pixels, a->mode == 0 ? 3 : 1);
  launch_pdl(loss_red_finish_kernel, det_finish_grid(4), kDetFinishThreads, 0, static_cast<cudaStream_t>(stream), 0L,
             grid, 4L, 4L, 4L, sums, 0L);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_loss_grad(const mcb_loss_args* a, const double* sums, long global_pixels, float grad_scale,
                             float* dlogits, float* loss_out, void* stream) {
  MCB_REQUIRE(a && a->logits && a->target && sums && dlogits, "loss_grad: null pointer");
  MCB_REQUIRE(a->mode == 0 || a->mode == 1, "loss: mode %d", a->mode);
  const long ppi = (long)a->h * a->w, pixels = ppi * a->n;
  launch_pdl(loss_grad_kernel, loss_grid(pixels), 256, 0, static_cast<cudaStream_t>(stream), 
      a->logits, a->target, make_cfg(a), sums, (double)global_pixels, grad_scale, dlogits, loss_out, ppi, pixels,
      a->mode == 0 ? 3 : 1);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_softmax2(const float* logits, float* probs, int n, int h, int w, void* stream) {
  MCB_REQUIRE(logits && probs, "softmax2: null pointer");
  const long ppi = (long)h * w, pixels = ppi * n;
  launch_pdl(softmax2_kernel, loss_grid(pixels), 256, 0, static_cast<cudaStream_t>(stream), logits, probs, ppi, pixels);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
