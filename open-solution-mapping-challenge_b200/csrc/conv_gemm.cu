// conv_gemm.cu — host side of the convolution family: decomposes each conv / transposed conv / gradient into
// taps + phases, picks pixel tiles, encodes the TMA tensor maps and launches the wgmma kernels of conv_gemm.cuh.
// Exposed through the C ABI declared in include/mcb200.h.
#include "host_common.h"
#include "conv_gemm.cuh"
#include "../../include/mcb200.h"
#include <algorithm>
#include <mutex>
#include <stdlib.h>

namespace mcb {

// choose a pixel box (bw, bh, bn) with rows = bw*bh*bn <= max_rows, rows % row_mult == 0, maximising the fraction
// of useful rows over all tiles; ties prefer wide boxes (contiguous memory).
static void pick_tile(int Wv, int Hv, int N, int max_rows, int row_mult, int* pbw, int* pbh, int* pbn) {
  double best = -1.0;
  int bbw = 1, bbh = 1, bbn = 1;
  for (int bw = 1; bw <= std::min(max_rows, std::min(Wv, 256)); ++bw) {
    for (int bh = 1; bw * bh <= max_rows && bh <= std::min(Hv, 256); ++bh) {
      const int bn_max = std::min(256, max_rows / (bw * bh));
      for (int bn = 1; bn <= bn_max; ++bn) {
        // the batch extent may overhang (zero-filled by TMA) only to reach the row multiple the MMA K step needs
        if (bn > N && row_mult == 1) break;
        const int rows = bw * bh * bn;
        if (rows % row_mult != 0) continue;
        const long tiles = (long)((Wv + bw - 1) / bw) * ((Hv + bh - 1) / bh) * ((N + bn - 1) / bn);
        const double eff = (double)Wv * Hv * N / ((double)tiles * max_rows);
        const double score = eff + 1e-6 * bw + 1e-9 * bh;  // ties: prefer wide rows (contiguous memory)
        if (score > best) {
          best = score;
          bbw = bw; bbh = bh; bbn = bn;
        }
      }
    }
  }
  *pbw = bbw; *pbh = bbh; *pbn = bbn;
}

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

template <int BN, int BK, bool B_MN, bool HALO>
static int launch_conv_inst(const ConvGemmParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    MCB_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, BK, B_MN, HALO>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  launch_pdl(conv_gemm_kernel<BN, BK, B_MN, HALO>, grid, kConvThreads, smem, st, p);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

template <int BK, bool B_MN, bool HALO>
static int launch_conv_bn(int BN, const ConvGemmParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  switch (BN) {
    case 256: return launch_conv_inst<256, BK, B_MN, HALO>(p, grid, smem, st);
    case 128: return launch_conv_inst<128, BK, B_MN, HALO>(p, grid, smem, st);
    case 64: return launch_conv_inst<64, BK, B_MN, HALO>(p, grid, smem, st);
    case 32: return launch_conv_inst<32, BK, B_MN, HALO>(p, grid, smem, st);
  }
  return fail(MCB_ERR_UNSUPPORTED, "unsupported BN %d", BN);
}

static int launch_conv(int BN, int BK, bool b_mn, ConvGemmParams& p, int m_tiles, int n_tiles, int phases,
                       cudaStream_t st, bool halo = false) {
  const int a_bytes = halo ? ((kHaloW * kHaloH * BK * 2 + 1023) / 1024) * 1024 : 128 * BK * 2;
  const int b_bytes = BN * BK * 2;
  const int stage = halo ? b_bytes : a_bytes + b_bytes;
  const int out_bufs = BN <= 64 ? 4 : (BN == 128 ? 2 : 1);
  const int out_bytes = out_bufs * 128 * BN * 2;
  const int aux_bytes = p.aux_mode != 0 ? 2 * 128 * (BN >= 64 ? 64 : 32) * 2 : 0;  // one aux chunk per MMA warpgroup
  const int fixed = out_bytes + aux_bytes + kStatBytes + 1024 /*align*/ + 1536 /*barriers, row table*/ +
                    (halo ? 2 * a_bytes : 0);
  const int budget = std::min(env_int("MCB_SMEM_BUDGET_KB", 227) * 1024, 232448);
  int stages = std::max(2, std::min(env_int("MCB_MAX_STAGES", halo ? 9 : 6), (budget - fixed) / stage));
  if (p.b_resident) {
    // resident weights need one ring slot per tap, a single N tile and a single phase
    if (halo && n_tiles == 1 && phases == 1 && (budget - fixed) / stage >= 9) stages = 9;
    else p.b_resident = 0;
  }
  p.stages = stages;
  p.m_tiles = m_tiles; p.n_tiles = n_tiles; p.phases = phases;
  const size_t smem = (size_t)stages * stage + fixed;
  const long total = (long)m_tiles * n_tiles * phases;
  dim3 grid((unsigned)std::min<long>(total, num_sms()), 1, 1);
  const int nch = n_tiles * BN;  // N extent of this launch, channels p.n_off ..
  const bool red = p.stats != nullptr || p.aux_mode == 2 || (p.aux_mode == 1 && p.bn_dbeta != nullptr);
  p.red_stride = 2 * nch;
  if (red && (long)grid.x * p.red_stride > kConvRedCap)
    return fail(MCB_ERR_UNSUPPORTED, "conv: reduction rows %u x %d exceed the workspace", grid.x, p.red_stride);
  int r;
  if (halo) {
    if (BK == 64) r = b_mn ? launch_conv_bn<64, true, true>(BN, p, grid, smem, st) : launch_conv_bn<64, false, true>(BN, p, grid, smem, st);
    else r = b_mn ? launch_conv_bn<32, true, true>(BN, p, grid, smem, st) : launch_conv_bn<32, false, true>(BN, p, grid, smem, st);
  } else {
    if (BK == 64) r = b_mn ? launch_conv_bn<64, true, false>(BN, p, grid, smem, st) : launch_conv_bn<64, false, false>(BN, p, grid, smem, st);
    else r = b_mn ? launch_conv_bn<32, true, false>(BN, p, grid, smem, st) : launch_conv_bn<32, false, false>(BN, p, grid, smem, st);
  }
  if (r || !red) return r;
  // per-channel sums of the CTAs' rows, in CTA order (detsum.cuh)
  const int rows = (int)grid.x;
  if (p.aux_mode == 0) {
    launch_pdl(conv_red_finish_kernel, det_finish_grid(2L * nch), kDetFinishThreads, 0, st, 0L, rows,
               (long)p.red_stride, 2L * nch, (long)nch, p.stats + p.n_off, (long)p.stats_c);
  } else {
    launch_pdl(conv_red_finish_kernel, det_finish_grid(nch), kDetFinishThreads, 0, st, 0L, rows, (long)p.red_stride,
               (long)nch, (long)nch, p.bn_dbeta + p.n_off, 0L);
    if (p.aux_mode == 2)
      launch_pdl(conv_red_finish_kernel, det_finish_grid(nch), kDetFinishThreads, 0, st, (long)nch, rows,
                 (long)p.red_stride, (long)nch, (long)nch, p.bn_dgamma + p.n_off, 0L);
  }
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// haloed 3x3 path: worth it when 8x16 single-image tiles cover the image without much waste
// k_channels = channels per tap of the GEMM-K dimension.  The haloed tile saves the nine per-tap fetches where they make
// the kernel L2-bound (>= 128 channels on large images whose extent the 8x16 tile divides); on thin layers the
// per-tile issue cost dominates and ragged small images waste rows.
// MCB_HALO: 0 never, 1 whenever the tile covers >= 80%, 2 (default) the rule above.
static bool use_halo(int ksize, int stride, int W, int H, int k_channels) {
  const int mode = env_int("MCB_HALO", 2);
  if (ksize != 3 || stride != 1 || mode == 0) return false;
  // experimental (MCB_BRES=1, off by default): one-chunk layers (32 / 64 channels) take the haloed tile with
  // RESIDENT weights -- one TMA load and 18 / 36 back-to-back MMAs per tile instead of 18 loads and 9 barrier waits
  if (env_int("MCB_BRES", 0) == 1 && k_channels <= 64 && W % 8 == 0 && H % 16 == 0) return true;
  if (mode == 2) return k_channels >= env_int("MCB_HALO_MINC", 128) && W % 8 == 0 && H % 16 == 0 && W >= 80;
  const double eff = (double)W * H / ((double)((W + 7) / 8) * 8 * ((H + 15) / 16) * 16);
  return eff >= 0.8;
}

static int pick_bn(int n_total, long m_tiles, int phases) {
  int bn = 32;
  for (int cand : {256, 128, 64, 32}) {
    if (n_total % cand == 0) { bn = cand; break; }
  }
  // keep the machine filled when the pixel dimension is small
  const long sms = num_sms();
  // (fat tiles beat many thin ones: go below 128 only when even 128-wide tiles leave most SMs idle; one round of
  // 256-wide tiles beats two rounds of 128-wide ones until the tile count falls below ~0.6 of a wave)
  if (bn > 128 && m_tiles * phases * (n_total / bn) * 10 < sms * env_int("MCB_BN256_MIN_WAVE_X10", 6)) bn = 128;
  if (bn > 64 && n_total % 64 == 0 && m_tiles * phases * (n_total / bn) < sms / 3) bn = 64;
  int forced = env_int("MCB_FORCE_BN", 0);
  if (forced && n_total % forced == 0) bn = forced;
  return bn;
}

// weight tensor map: bf16 [taps][rows = cout][cols = cin_total], viewed as (cin_total, cout, taps)
static int encode_weight(CUtensorMap* m, const void* w, int taps, int cout, int cin_total, int box_inner, int box_rows,
                         int swizzle) {
  uint64_t dims[3] = {(uint64_t)cin_total, (uint64_t)cout, (uint64_t)taps};
  uint64_t str[2] = {(uint64_t)cin_total * 2, (uint64_t)cin_total * cout * 2};
  uint32_t box[3] = {(uint32_t)box_inner, (uint32_t)box_rows, 1};
  return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, w, dims, str, box, swizzle);
}

// 1-D decomposition helpers ------------------------------------------------------------------------
struct Tap1D { int k; int d; int parity; };  // kernel index, offset in the (possibly parity) view, source parity

// forward conv, stride 2, k=3, pad=1: input coordinate 2*o - 1 + k
static int fwd_s2_taps(int ksize, Tap1D* out) {
  if (ksize == 1) { out[0] = {0, 0, 0}; return 1; }
  out[0] = {0, -1, 1}; out[1] = {1, 0, 0}; out[2] = {2, 0, 1};
  return 3;
}
// data gradient of a stride-2 conv for output parity py: da[2y+py] = sum_k dz[(2y+py+pad-k)/2] W[k], parity must match
static int dgrad_s2_taps(int ksize, int py, Tap1D* out) {
  if (ksize == 1) { if (py == 0) { out[0] = {0, 0, 0}; return 1; } return 0; }
  if (py == 0) { out[0] = {1, 0, 0}; return 1; }
  out[0] = {0, 1, 0}; out[1] = {2, 0, 0};
  return 2;
}
// transposed conv k=4 s=2 p=1 forward for output parity py: out[2y+py] += in[y+d] W[k]
static int convt_fwd_taps(int py, Tap1D* out) {
  if (py == 0) { out[0] = {1, 0, 0}; out[1] = {3, -1, 0}; }
  else { out[0] = {0, 1, 0}; out[1] = {2, 0, 0}; }
  return 2;
}
// transposed conv data gradient: din[y] = sum_k dout[2y - 1 + k] W[k]  (parity view of dout, offset d)
static int convt_dgrad_taps(Tap1D* out) {
  out[0] = {0, -1, 1}; out[1] = {1, 0, 0}; out[2] = {2, 0, 1}; out[3] = {3, 1, 0};
  return 4;
}

static int check_c(int c, const char* what) {
  if (c % 32 != 0) return fail(MCB_ERR_UNSUPPORTED, "%s channels %d not a multiple of 32", what, c);
  if (c % 64 != 0 && c != 32) return fail(MCB_ERR_UNSUPPORTED, "%s channels %d: only 32 or multiples of 64", what, c);
  return MCB_OK;
}

}  // namespace mcb

using namespace mcb;

// =====================================================================================================
extern "C" int mcb_conv_fwd(const mcb_conv_fwd_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->x[0] && a->weight && a->y, "conv_fwd: null pointer");
  MCB_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv_fwd: ksize %d", a->ksize);
  MCB_REQUIRE(a->stride == 1 || a->stride == 2, "conv_fwd: stride %d", a->stride);
  const int nsrc = a->x[1] ? 2 : 1;
  MCB_REQUIRE(!(nsrc == 2 && a->stride == 2), "conv_fwd: concat + stride 2 unsupported");
  const int cin_total = a->cin[0] + (nsrc == 2 ? a->cin[1] : 0);
  for (int s = 0; s < nsrc; ++s)
    if (int r = check_c(a->cin[s], "conv_fwd input")) return r;
  if (int r = check_c(a->cout, "conv_fwd output")) return r;
  const int BK = (a->cin[0] % 64 == 0 && (nsrc == 1 || a->cin[1] % 64 == 0)) ? 64 : 32;
  MCB_REQUIRE(!(BK == 32 && nsrc == 2), "conv_fwd: 32-channel concat unsupported");
  const int H = a->h, W = a->w, N = a->n;
  MCB_REQUIRE(a->stride == 1 || (H % 2 == 0 && W % 2 == 0), "conv_fwd: stride 2 needs even H, W");
  const int Ho = H / a->stride, Wo = W / a->stride;
  const int pad = a->ksize / 2;

  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  const bool halo = use_halo(a->ksize, a->stride, Wo, Ho, nsrc == 2 ? std::min(a->cin[0], a->cin[1]) : a->cin[0]);
  if (halo) { p.bw = 8; p.bh = 16; p.bn = 1; }
  else pick_tile(Wo, Ho, N, 128, 1, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  p.Wv = Wo; p.Hv = Ho; p.Nimg = N;
  p.tiles_x = (Wo + p.bw - 1) / p.bw;
  p.tiles_y = (Ho + p.bh - 1) / p.bh;
  const long m_tiles = (long)p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  const int BN = pick_bn(a->cout, m_tiles, 1);
  const int swz = BK * 2;

  int nt = 0;
  if (a->stride == 1) {
    for (int s = 0; s < nsrc; ++s)
      if (int r = encode_nhwc_view(&p.tmA[s], a->x[s], N, H, W, a->cin[s], 0, a->cin[s], -1, -1, BK,
                                   halo ? kHaloW : p.bw, halo ? kHaloH : p.bh, p.bn, swz)) return r;
    for (int ky = 0; ky < a->ksize; ++ky)
      for (int kx = 0; kx < a->ksize; ++kx)
        for (int s = 0; s < nsrc; ++s) {
          TapDesc& t = p.taps[nt++];
          t.src = s; t.dx = kx - pad; t.dy = ky - pad; t.nchunks = a->cin[s] / BK;
          t.wk0 = (s == 0) ? 0 : a->cin[0]; t.wtap = ky * a->ksize + kx;
        }
  } else {
    Tap1D ty[3], tx[3];
    const int ny = fwd_s2_taps(a->ksize, ty), nx = fwd_s2_taps(a->ksize, tx);
    bool used[4] = {false, false, false, false};
    for (int i = 0; i < ny; ++i)
      for (int j = 0; j < nx; ++j) {
        TapDesc& t = p.taps[nt++];
        t.src = ty[i].parity * 2 + tx[j].parity; used[t.src] = true;
        t.dx = tx[j].d; t.dy = ty[i].d; t.nchunks = a->cin[0] / BK; t.wk0 = 0;
        t.wtap = ty[i].k * a->ksize + tx[j].k;
      }
    for (int v = 0; v < 4; ++v)
      if (used[v])
        if (int r = encode_nhwc_view(&p.tmA[v], a->x[0], N, H, W, a->cin[0], 0, a->cin[0], v >> 1, v & 1, BK, p.bw,
                                     p.bh, p.bn, swz)) return r;
  }
  p.tap_start[0] = 0; p.tap_count[0] = nt;
  if (int r = encode_weight(&p.tmB, a->weight, a->ksize * a->ksize, a->cout, cin_total, BK, BN, swz)) return r;
  const int out_cw = BN >= 64 ? 64 : 32;
  if (int r = encode_nhwc_view(&p.tmD[0], a->y, N, Ho, Wo, a->cout, 0, a->cout, -1, -1, out_cw, p.bw, p.bh, p.bn,
                               out_cw * 2)) return r;
  p.bias = a->bias; p.relu = a->relu; p.stats = a->stats; p.stats_c = a->cout;
  p.scale = a->scale;
  p.b_resident = (halo && nsrc == 1 && a->cin[0] == BK && env_int("MCB_BRES", 0) == 1) ? 1 : 0;
  if (a->residual) {
    p.residual = static_cast<const __nv_bfloat16*>(a->residual);
    p.mask_H = Ho; p.mask_W = Wo; p.mask_C = a->cout; p.mask_s = 1;
  }
  return launch_conv(BN, BK, false, p, (int)m_tiles, a->cout / BN, 1, st, halo);
}

// =====================================================================================================
extern "C" int mcb_conv_dgrad(const mcb_conv_dgrad_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->dy && a->weight && a->dx, "conv_dgrad: null pointer");
  MCB_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv_dgrad: ksize %d", a->ksize);
  MCB_REQUIRE(a->stride == 1 || a->stride == 2, "conv_dgrad: stride %d", a->stride);
  MCB_REQUIRE(!(a->relu_mask && a->accumulate), "conv_dgrad: relu_mask with accumulate is ill-defined");
  MCB_REQUIRE(!(a->relu_mask && a->bn_z), "conv_dgrad: with bn_z the mask is derived from bn_z (relu_mask must be NULL)");
  if (int r = check_c(a->cout, "conv_dgrad dy")) return r;
  if (int r = check_c(a->cin, "conv_dgrad dx")) return r;
  const int H = a->h, W = a->w, N = a->n;
  const int Ho = H / a->stride, Wo = W / a->stride;
  const int pad = a->ksize / 2;
  const int BK = (a->cout % 64 == 0) ? 64 : 32;  // GEMM-K is cout here

  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  const int Wv = (a->stride == 1) ? W : W / 2, Hv = (a->stride == 1) ? H : H / 2;
  const bool halo = use_halo(a->ksize, a->stride, Wv, Hv, a->cout);
  if (halo) { p.bw = 8; p.bh = 16; p.bn = 1; }
  else pick_tile(Wv, Hv, N, 128, 1, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  p.Wv = Wv; p.Hv = Hv; p.Nimg = N;
  p.tiles_x = (Wv + p.bw - 1) / p.bw;
  p.tiles_y = (Hv + p.bh - 1) / p.bh;
  const long m_tiles = (long)p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  int phases = 1;
  int nt = 0;
  if (int r = encode_nhwc_view(&p.tmA[0], a->dy, N, Ho, Wo, a->cout, 0, a->cout, -1, -1, BK, halo ? kHaloW : p.bw,
                               halo ? kHaloH : p.bh, p.bn, BK * 2)) return r;
  int phase_map[4] = {0, 0, 0, 0};  // launch phase -> (py*2+px)
  if (a->stride == 1) {
    for (int ky = 0; ky < a->ksize; ++ky)
      for (int kx = 0; kx < a->ksize; ++kx) {
        TapDesc& t = p.taps[nt++];
        t.src = 0; t.dx = pad - kx; t.dy = pad - ky; t.nchunks = a->cout / BK; t.wk0 = 0; t.wtap = ky * a->ksize + kx;
      }
    p.tap_start[0] = 0; p.tap_count[0] = nt;
  } else {
    MCB_REQUIRE(H % 2 == 0 && W % 2 == 0, "conv_dgrad: stride 2 needs even H, W");
    phases = 0;
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        Tap1D ty[2], tx[2];
        const int ny = dgrad_s2_taps(a->ksize, py, ty), nx = dgrad_s2_taps(a->ksize, px, tx);
        if (ny * nx == 0) continue;
        p.tap_start[phases] = nt;
        for (int i = 0; i < ny; ++i)
          for (int j = 0; j < nx; ++j) {
            TapDesc& t = p.taps[nt++];
            t.src = 0; t.dx = tx[j].d; t.dy = ty[i].d; t.nchunks = a->cout / BK; t.wk0 = 0;
            t.wtap = ty[i].k * a->ksize + tx[j].k;
          }
        p.tap_count[phases] = nt - p.tap_start[phases];
        phase_map[phases] = py * 2 + px;
        ++phases;
      }
    if (a->ksize == 1 && !a->accumulate) {
      // only the (even, even) input pixels receive gradient; the rest is zero
      MCB_CHECK_CUDA(cudaMemsetAsync(a->dx, 0, (size_t)N * H * W * a->cin * 2, st));
    }
  }
  // the kernel derives the mask parity from blockIdx.z as (py, px) = (z >> 1, z & 1); with all four phases present
  // (3x3) launch order == parity order; the 1x1 case has the single phase (0,0).
  const int BN = pick_bn(a->cin, m_tiles, phases);
  const int bmn_cw = BN >= 64 ? 64 : 32;
  // MN-major B: weight slice [taps][cout][ci_off : ci_off + cin] viewed as (cin inner = N, cout = K rows, taps),
  // row pitch cin_total; box (bmn_cw, BK, 1)
  {
    const char* wb = static_cast<const char*>(a->weight) + (size_t)a->ci_off * 2;
    uint64_t dims[3] = {(uint64_t)a->cin, (uint64_t)a->cout, (uint64_t)(a->ksize * a->ksize)};
    uint64_t str[2] = {(uint64_t)a->cin_total * 2, (uint64_t)a->cin_total * a->cout * 2};
    uint32_t box[3] = {(uint32_t)bmn_cw, (uint32_t)BK, 1};
    if (int r = encode_tmap(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, wb, dims, str, box, bmn_cw * 2)) return r;
  }
  const int out_cw = BN >= 64 ? 64 : 32;
  const void* aux = a->bn_z ? a->bn_z : a->relu_mask;  // tensor with the geometry of dx, tiled like the output
  for (int ph = 0; ph < phases; ++ph) {
    const int py = (a->stride == 1) ? -1 : (phase_map[ph] >> 1), px = (a->stride == 1) ? -1 : (phase_map[ph] & 1);
    if (int r = encode_nhwc_view(&p.tmD[ph], a->dx, N, H, W, a->cin, 0, a->cin, py, px, out_cw, p.bw, p.bh, p.bn,
                                 out_cw * 2)) return r;
    if (aux)
      if (int r = encode_nhwc_view(&p.tmX[ph], aux, N, H, W, a->cin, 0, a->cin, py, px, out_cw, p.bw, p.bh, p.bn,
                                   out_cw * 2)) return r;
  }
  p.accumulate = a->accumulate;
  p.b_resident = (halo && a->cout == BK && env_int("MCB_BRES", 0) == 1) ? 1 : 0;
  p.aux_mode = a->bn_z ? 2 : (a->relu_mask ? 1 : 0);
  MCB_REQUIRE(!(a->dx_channel_sum && (!a->relu_mask || a->accumulate)),
              "conv_dgrad: dx_channel_sum needs relu_mask and a complete (non-accumulated) gradient");
  if (a->dx_channel_sum) p.bn_dbeta = a->dx_channel_sum;
  if (a->bn_z) {
    MCB_REQUIRE(a->bn_mean && a->bn_invstd && a->bn_gamma && a->bn_beta && a->bn_dbeta && a->bn_dgamma,
                "conv_dgrad: incomplete bn reduction args");
    MCB_REQUIRE(!a->accumulate, "conv_dgrad: bn reduction needs the complete gradient (no accumulate)");
    MCB_REQUIRE(!(a->stride == 2 && a->ksize == 1), "conv_dgrad: bn reduction with a 1x1 stride-2 conv is unsupported");
    p.bn_mean = a->bn_mean; p.bn_invstd = a->bn_invstd; p.bn_gamma = a->bn_gamma; p.bn_beta = a->bn_beta;
    p.bn_dbeta = a->bn_dbeta; p.bn_dgamma = a->bn_dgamma;
  }
  return launch_conv(BN, BK, true, p, (int)m_tiles, a->cin / BN, phases, st, halo);
}

// =====================================================================================================
extern "C" int mcb_convt_fwd(const mcb_convt_fwd_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->x && a->weight && a->y, "convt_fwd: null pointer");
  if (int r = check_c(a->cin, "convt_fwd input")) return r;
  if (int r = check_c(a->cout, "convt_fwd output")) return r;
  const int H = a->h, W = a->w, N = a->n;
  const int BK = (a->cin % 64 == 0) ? 64 : 32;
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  pick_tile(W, H, N, 128, 1, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  p.Wv = W; p.Hv = H; p.Nimg = N;
  p.tiles_x = (W + p.bw - 1) / p.bw;
  p.tiles_y = (H + p.bh - 1) / p.bh;
  const long m_tiles = (long)p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  const int BN = pick_bn(a->cout, m_tiles, 4);
  if (int r = encode_nhwc_view(&p.tmA[0], a->x, N, H, W, a->cin, 0, a->cin, -1, -1, BK, p.bw, p.bh, p.bn, BK * 2))
    return r;
  int nt = 0;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      const int ph = py * 2 + px;
      Tap1D ty[2], tx[2];
      convt_fwd_taps(py, ty); convt_fwd_taps(px, tx);
      p.tap_start[ph] = nt;
      for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) {
          TapDesc& t = p.taps[nt++];
          t.src = 0; t.dx = tx[j].d; t.dy = ty[i].d; t.nchunks = a->cin / BK; t.wk0 = 0; t.wtap = ty[i].k * 4 + tx[j].k;
        }
      p.tap_count[ph] = 4;
      const int out_cw = BN >= 64 ? 64 : 32;
      if (int r = encode_nhwc_view(&p.tmD[ph], a->y, N, 2 * H, 2 * W, a->cout, 0, a->cout, py, px, out_cw, p.bw, p.bh,
                                   p.bn, out_cw * 2)) return r;
    }
  if (int r = encode_weight(&p.tmB, a->weight, 16, a->cout, a->cin, BK, BN, BK * 2)) return r;
  p.bias = a->bias; p.relu = a->relu;
  return launch_conv(BN, BK, false, p, (int)m_tiles, a->cout / BN, 4, st);
}

extern "C" int mcb_convt_dgrad(const mcb_convt_dgrad_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->dy && a->weight && a->dx, "convt_dgrad: null pointer");
  MCB_REQUIRE(!(a->relu_mask && a->accumulate), "convt_dgrad: relu_mask with accumulate is ill-defined");
  if (int r = check_c(a->cin, "convt_dgrad dx")) return r;
  if (int r = check_c(a->cout, "convt_dgrad dy")) return r;
  const int H = a->h, W = a->w, N = a->n;  // input (dx) dims; dy is 2H x 2W
  const int BK = (a->cout % 64 == 0) ? 64 : 32;
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  pick_tile(W, H, N, 128, 1, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  p.Wv = W; p.Hv = H; p.Nimg = N;
  p.tiles_x = (W + p.bw - 1) / p.bw;
  p.tiles_y = (H + p.bh - 1) / p.bh;
  const long m_tiles = (long)p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  const int BN = pick_bn(a->cin, m_tiles, 1);
  for (int v = 0; v < 4; ++v)
    if (int r = encode_nhwc_view(&p.tmA[v], a->dy, N, 2 * H, 2 * W, a->cout, 0, a->cout, v >> 1, v & 1, BK, p.bw,
                                 p.bh, p.bn, BK * 2)) return r;
  Tap1D t1[4];
  convt_dgrad_taps(t1);
  int nt = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      TapDesc& t = p.taps[nt++];
      t.src = t1[i].parity * 2 + t1[j].parity; t.dx = t1[j].d; t.dy = t1[i].d; t.nchunks = a->cout / BK; t.wk0 = 0;
      t.wtap = t1[i].k * 4 + t1[j].k;
    }
  p.tap_start[0] = 0; p.tap_count[0] = nt;
  const int bmn_cw = BN >= 64 ? 64 : 32;
  if (int r = encode_weight(&p.tmB, a->weight, 16, a->cout, a->cin, bmn_cw, BK, bmn_cw * 2)) return r;
  const int out_cw = BN >= 64 ? 64 : 32;
  if (int r = encode_nhwc_view(&p.tmD[0], a->dx, N, H, W, a->cin, 0, a->cin, -1, -1, out_cw, p.bw, p.bh, p.bn,
                               out_cw * 2)) return r;
  p.accumulate = a->accumulate;
  if (a->relu_mask) {
    if (int r = encode_nhwc_view(&p.tmX[0], a->relu_mask, N, H, W, a->cin, 0, a->cin, -1, -1, out_cw, p.bw, p.bh, p.bn,
                                 out_cw * 2)) return r;
    p.aux_mode = 1;
  }
  MCB_REQUIRE(!(a->dx_channel_sum && (!a->relu_mask || a->accumulate)),
              "convt_dgrad: dx_channel_sum needs relu_mask and a complete (non-accumulated) gradient");
  p.bn_dbeta = a->dx_channel_sum;
  return launch_conv(BN, BK, true, p, (int)m_tiles, a->cin / BN, 1, st);
}

// =====================================================================================================
namespace mcb {

template <int BN>
static int launch_wgrad_inst(const WgradParams& p, dim3 grid, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    MCB_CHECK_CUDA(cudaFuncSetAttribute(wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  launch_pdl(wgrad_kernel<BN>, grid, kGemmThreads, smem, st, p);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// Region of g_wgrad_red for launches on stream st.  Launches of one stream are serialised; launches of different
// streams may overlap, so each stream keeps its own region (the kWgradRegions most recently used streams do; a step
// uses two streams at a time).
static long wgrad_region_offset(cudaStream_t st) {
  static std::mutex mu;
  static cudaStream_t owner[kWgradRegions];
  static unsigned long last_use[kWgradRegions];
  static unsigned long clock = 0;
  std::lock_guard<std::mutex> lock(mu);
  ++clock;
  int r = 0;
  for (int i = 0; i < kWgradRegions; ++i) {
    if (last_use[i] != 0 && owner[i] == st) { r = i; break; }
    if (last_use[i] < last_use[r]) r = i;   // otherwise: the least recently used region
  }
  owner[r] = st;
  last_use[r] = clock;
  return (long)r * kWgradRegionCap;
}

static int launch_wgrad(WgradParams& p, int cin_src, cudaStream_t st) {
  int BN = 32;
  for (int cand : {256, 128, 64, 32})
    if (cin_src % cand == 0) { BN = cand; break; }
  const int m_tiles = (p.cout + 127) / 128;
  const int n_tiles = cin_src / BN;
  // split-K over the pixel tiles so the grid covers the machine a few times
  // Every split adds a full fp32 output tile with red.add (atomic traffic = splits x |dW|), while the operand
  // streams are L2/HBM-bound and want every SM busy.  So: exactly ONE resident wave of CTAs (never a ragged second
  // wave; the 384-thread CTA takes the whole register file, one CTA per SM) and at least `min_kb` K blocks per CTA.
  const long base = (long)m_tiles * n_tiles * p.ntaps;
  const long cap = (long)num_sms() * env_int("MCB_WGRAD_WAVES_X10", 10) / 10;
  int splits = (int)std::max(1L, std::min((long)p.tiles_total, cap / std::max(1L, base)));
  const int min_kb = env_int("MCB_WGRAD_MIN_KB", 6);
  splits = std::max(1, std::min(splits, std::max(1, p.tiles_total / min_kb)));
  // short reductions (deep layers: few pixel tiles, many weights) are bound by the fp32 red.add epilogues, not by the
  // operand streams: aim for `kb_target` K blocks per CTA, but keep at least 0.4 of a wave busy (on the full step
  // these GEMMs share the SMs with the BatchNorm-backward kernels)
  const int kb_target = env_int("MCB_WGRAD_KB_TARGET", 64);
  if (kb_target > 0) {
    const long lo_cap = cap * env_int("MCB_WGRAD_MIN_WAVE_X10", 4) / 10;
    const int lo = (int)std::max(1L, lo_cap / std::max(1L, base));
    const int want = std::max(1, p.tiles_total / kb_target);
    splits = std::max(1, std::min(splits, std::max(lo, want)));
  }
  int forced = env_int("MCB_WGRAD_SPLITS", 0);
  if (forced > 0) splits = std::min(forced, p.tiles_total);
  // several splits store their partial products in split-ordered rows of the workspace (summed deterministically below)
  p.cin_src = cin_src;
  p.slice = (long)p.ntaps * p.cout * cin_src;
  if (splits > 1) splits = (int)std::max(1L, std::min((long)splits, kWgradRegionCap / p.slice));
  p.ws_off = splits > 1 ? wgrad_region_offset(st) : 0;
  p.splits = splits;
  const int b_cw = BN >= 64 ? 64 : 32;
  const int stage = 2 * 64 * 128 + (BN / b_cw) * 64 * b_cw * 2;
  const int budget = env_int("MCB_SMEM_BUDGET_KB", 227) * 1024;
  const int per = (p.tiles_total + splits - 1) / splits;
  p.stages = std::max(2, std::min(std::min(per, 8), budget / stage));
  const size_t smem = (size_t)p.stages * stage + 1024 + 512;
  dim3 grid(n_tiles, m_tiles, p.ntaps * splits);
  int r;
  switch (BN) {
    case 256: r = launch_wgrad_inst<256>(p, grid, smem, st); break;
    case 128: r = launch_wgrad_inst<128>(p, grid, smem, st); break;
    case 64: r = launch_wgrad_inst<64>(p, grid, smem, st); break;
    default: r = launch_wgrad_inst<32>(p, grid, smem, st); break;
  }
  if (r || splits == 1) return r;
  // the splits that own pixel tiles, summed in split order into dW[tap][cout][ci_off + ci] (detsum.cuh)
  const int rows = (p.tiles_total + per - 1) / per;
  launch_pdl(wgrad_red_finish_kernel, det_finish_grid(p.slice), kDetFinishThreads, 0, st, p.ws_off, rows, p.slice, p.slice,
             (long)cin_src, p.dw + p.ci_off, (long)p.cin_total);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

static int wgrad_common_setup(WgradParams& p, int Wv, int Hv, int N, int cout, int cin_src) {
  pick_tile(Wv, Hv, N, 64, 16, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  if (p.rows % 16 != 0 || p.rows > 64) return fail(MCB_ERR_UNSUPPORTED, "wgrad: no pixel box for %dx%dx%d", Wv, Hv, N);
  p.Wv = Wv; p.Hv = Hv; p.Nimg = N;
  p.tiles_x = (Wv + p.bw - 1) / p.bw;
  p.tiles_y = (Hv + p.bh - 1) / p.bh;
  p.tiles_total = p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  p.a_cw = (cout % 64 == 0) ? 64 : 32;
  p.a_chunks = (cout >= 128) ? 2 : 1;
  (void)cin_src;
  return MCB_OK;
}

}  // namespace mcb

extern "C" int mcb_conv_wgrad(const mcb_conv_wgrad_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->dy && a->x && a->dw, "conv_wgrad: null pointer");
  MCB_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv_wgrad: ksize %d", a->ksize);
  MCB_REQUIRE(a->stride == 1 || a->stride == 2, "conv_wgrad: stride %d", a->stride);
  if (int r = check_c(a->cout, "conv_wgrad dy")) return r;
  if (int r = check_c(a->cin, "conv_wgrad x")) return r;
  MCB_REQUIRE(a->cout % 128 == 0 || a->cout == 64 || a->cout == 32, "conv_wgrad: cout %d", a->cout);
  const int H = a->h, W = a->w, N = a->n;
  const int Ho = H / a->stride, Wo = W / a->stride;
  const int pad = a->ksize / 2;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  if (int r = wgrad_common_setup(p, Wo, Ho, N, a->cout, a->cin)) return r;
  const int b_cw = (a->cin % 64 == 0) ? 64 : 32;
  if (int r = encode_nhwc_view(&p.tmA[0], a->dy, N, Ho, Wo, a->cout, 0, a->cout, -1, -1, p.a_cw, p.bw, p.bh, p.bn,
                               p.a_cw * 2)) return r;
  int nt = 0;
  if (a->stride == 1) {
    if (int r = encode_nhwc_view(&p.tmB[0], a->x, N, H, W, a->cin, 0, a->cin, -1, -1, b_cw, p.bw, p.bh, p.bn,
                                 b_cw * 2)) return r;
    for (int ky = 0; ky < a->ksize; ++ky)
      for (int kx = 0; kx < a->ksize; ++kx) {
        WgradTap& t = p.taps[nt++];
        t.srcA = 0; t.ax = 0; t.ay = 0; t.srcB = 0; t.bx = kx - pad; t.by = ky - pad; t.wtap = ky * a->ksize + kx;
      }
  } else {
    MCB_REQUIRE(H % 2 == 0 && W % 2 == 0, "conv_wgrad: stride 2 needs even H, W");
    Tap1D ty[3], tx[3];
    const int ny = fwd_s2_taps(a->ksize, ty), nx = fwd_s2_taps(a->ksize, tx);
    bool used[4] = {false, false, false, false};
    for (int i = 0; i < ny; ++i)
      for (int j = 0; j < nx; ++j) {
        WgradTap& t = p.taps[nt++];
        t.srcA = 0; t.ax = 0; t.ay = 0;
        t.srcB = ty[i].parity * 2 + tx[j].parity; used[t.srcB] = true;
        t.bx = tx[j].d; t.by = ty[i].d; t.wtap = ty[i].k * a->ksize + tx[j].k;
      }
    for (int v = 0; v < 4; ++v)
      if (used[v])
        if (int r = encode_nhwc_view(&p.tmB[v], a->x, N, H, W, a->cin, 0, a->cin, v >> 1, v & 1, b_cw, p.bw, p.bh,
                                     p.bn, b_cw * 2)) return r;
  }
  p.ntaps = nt;
  p.dw = a->dw; p.cout = a->cout; p.cin_total = a->cin_total; p.ci_off = a->ci_off;
  return launch_wgrad(p, a->cin, st);
}

extern "C" int mcb_convt_wgrad(const mcb_convt_wgrad_args* a, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MCB_REQUIRE(a && a->dy && a->x && a->dw, "convt_wgrad: null pointer");
  if (int r = check_c(a->cout, "convt_wgrad dy")) return r;
  if (int r = check_c(a->cin, "convt_wgrad x")) return r;
  MCB_REQUIRE(a->cout % 128 == 0 || a->cout == 64 || a->cout == 32, "convt_wgrad: cout %d", a->cout);
  const int H = a->h, W = a->w, N = a->n;  // input dims; dy is 2H x 2W
  WgradParams p;
  memset(&p, 0, sizeof(p));
  if (int r = wgrad_common_setup(p, W, H, N, a->cout, a->cin)) return r;
  const int b_cw = (a->cin % 64 == 0) ? 64 : 32;
  for (int v = 0; v < 4; ++v)
    if (int r = encode_nhwc_view(&p.tmA[v], a->dy, N, 2 * H, 2 * W, a->cout, 0, a->cout, v >> 1, v & 1, p.a_cw, p.bw,
                                 p.bh, p.bn, p.a_cw * 2)) return r;
  if (int r = encode_nhwc_view(&p.tmB[0], a->x, N, H, W, a->cin, 0, a->cin, -1, -1, b_cw, p.bw, p.bh, p.bn, b_cw * 2))
    return r;
  Tap1D t1[4];
  convt_dgrad_taps(t1);
  int nt = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      WgradTap& t = p.taps[nt++];
      t.srcA = t1[i].parity * 2 + t1[j].parity; t.ax = t1[j].d; t.ay = t1[i].d;
      t.srcB = 0; t.bx = 0; t.by = 0; t.wtap = t1[i].k * 4 + t1[j].k;
    }
  p.ntaps = nt;
  p.dw = a->dw; p.cout = a->cout; p.cin_total = a->cin; p.ci_off = 0;
  return launch_wgrad(p, a->cin, st);
}
