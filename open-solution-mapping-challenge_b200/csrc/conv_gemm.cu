// conv_gemm.cu — host side of the convolution family.  Each entry point validates its arguments, sets the epilogue
// fields and describes its op: the tensors it reads and writes (View) and the per-axis tap rule (TapRule).  plan_conv /
// plan_wgrad turn that description into taps + phases, pixel tiles and TMA tensor maps and launch the wgmma kernels of
// conv_gemm.cuh.  Exposed through the C ABI declared in include/mcb200.h.
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

// Launch rules.  The integer expressions that use these constants fix every launch's BN, stages and splits, and with
// them the fp32 summation order: rewriting one can change a rounding, a split count and so the results' last bits.
constexpr int kSmemBudget = 227 * 1024;               // dynamic shared memory of one CTA (the sm_90 maximum)
constexpr int kMaxStagesHalo = 9, kMaxStages = 6;     // operand ring depth, haloed / per-tap path
constexpr int kWgradMaxStages = 8;                    // ... of the weight-gradient GEMMs
constexpr int kTwoStagingMinStages = 3;               // two epilogue staging buffers while the ring keeps this many stages
constexpr int kHaloMinChannels = 128;                 // haloed tile from this many channels per tap
constexpr int kBn256MinWaveX10 = 6;                   // 256-wide N tiles down to 0.6 of a wave
constexpr int kWgradWavesX10 = 10;                    // weight-gradient grid: one wave
constexpr int kWgradMinKb = 6;                        // K blocks (pixel tiles) per weight-gradient CTA, at least
constexpr int kWgradKbTarget = 64;                    // ... and aimed at for short reductions
constexpr int kWgradMinWaveX10 = 4;                   // ... keeping at least 0.4 of a wave busy

static_assert(conv_smem(32, 32, true, kMaxStagesHalo, 1, 0).fits && conv_smem(32, 32, false, kMaxStages, 1, 0).fits &&
                  wgrad_smem(32, kWgradMaxStages).fits, "the mbarriers outgrow their reserve at the deepest rings");

// Test hooks: they force a regime that a test's shapes would not reach under the launch rules.  Unset (the default),
// the rules decide, and that is the only path the library takes in use.  Read on every launch, so that a test can
// change them between calls.
//   MCB_FORCE_BN      N tile width (ignored unless it divides the N extent)
//   MCB_HALO          0 never the haloed 3x3 tile, 1 whenever it covers >= 80% of the view, 2 (default) use_halo's rule
//   MCB_WGRAD_SPLITS  split-K count of the weight-gradient GEMMs
struct TestHooks { int force_bn, halo, wgrad_splits; };
static TestHooks test_hooks() {
  auto get = [](const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
  };
  return {get("MCB_FORCE_BN", 0), get("MCB_HALO", 2), get("MCB_WGRAD_SPLITS", 0)};
}

// Launches one kernel instantiation; its first launch raises its dynamic shared-memory limit to kSmemBudget
template <auto Kernel, class Params>
static int launch_kernel(const Params& p, dim3 grid, int threads, size_t smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    MCB_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget));
    attr_set = true;
  }
  Kernel<<<grid, threads, smem, st>>>(p);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// the conv_gemm_kernel instantiation for (BN, BK, b_mn, halo); with_flag passes a run-time flag as a template argument
static int launch_conv_kernel(int BN, int BK, bool b_mn, bool halo, const ConvGemmParams& p, dim3 grid, size_t smem,
                              cudaStream_t st) {
  auto with_flag = [](bool v, auto f) { return v ? f(std::true_type()) : f(std::false_type()); };
  return with_flag(BK == 64, [&](auto bk64) { return with_flag(b_mn, [&](auto mn) { return with_flag(halo, [&](auto h) {
    constexpr int K = decltype(bk64)::value ? 64 : 32;
    constexpr bool M = decltype(mn)::value, H = decltype(h)::value;
    switch (BN) {
      case 256: return launch_kernel<conv_gemm_kernel<256, K, M, H>>(p, grid, kConvThreads, smem, st);
      case 128: return launch_kernel<conv_gemm_kernel<128, K, M, H>>(p, grid, kConvThreads, smem, st);
      case 64: return launch_kernel<conv_gemm_kernel<64, K, M, H>>(p, grid, kConvThreads, smem, st);
      case 32: return launch_kernel<conv_gemm_kernel<32, K, M, H>>(p, grid, kConvThreads, smem, st);
    }
    return fail(MCB_ERR_UNSUPPORTED, "unsupported BN %d", BN);
  }); }); });
}

static int launch_conv(int BN, int BK, bool b_mn, ConvGemmParams& p, int m_tiles, int n_tiles, int phases,
                       cudaStream_t st, bool halo = false) {
  auto layout = [&](int stages, int out_bufs) { return conv_smem(BN, BK, halo, stages, out_bufs, p.aux_mode != 0); };
  // (layout(0, b).bytes: everything but the operand ring)
  const int stage = layout(0, 0).stage, max_stages = halo ? kMaxStagesHalo : kMaxStages;
  p.out_bufs = (kSmemBudget - layout(0, 2).bytes) / stage >= kTwoStagingMinStages ? 2 : 1;
  p.stages = std::max(2, std::min(max_stages, (kSmemBudget - layout(0, p.out_bufs).bytes) / stage));
  p.m_tiles = m_tiles; p.n_tiles = n_tiles; p.phases = phases;
  const size_t smem = layout(p.stages, p.out_bufs).bytes;
  const long total = (long)m_tiles * n_tiles * phases;
  dim3 grid((unsigned)std::min<long>(total, num_sms()), 1, 1);
  const int nch = n_tiles * BN;  // N extent of this launch, channels p.n_off ..
  const bool red = conv_reduces(p);
  p.red_stride = 2 * nch;
  if (red && (long)grid.x * p.red_stride > kConvRedCap)
    return fail(MCB_ERR_UNSUPPORTED, "conv: reduction rows %u x %d exceed the workspace", grid.x, p.red_stride);
  const int r = launch_conv_kernel(BN, BK, b_mn, halo, p, grid, smem, st);
  if (r || !red) return r;
  // per-channel sums of the CTAs' rows, in CTA order (detsum.cuh)
  const int rows = (int)grid.x;
  if (p.aux_mode == 0) {
    conv_red_finish_kernel<<<det_finish_grid(2L * nch, rows), kDetFinishThreads, 0, st>>>(
        0L, rows, (long)p.red_stride, 2L * nch, (long)nch, p.stats + p.n_off, (long)p.stats_c);
  } else {
    conv_red_finish_kernel<<<det_finish_grid(nch, rows), kDetFinishThreads, 0, st>>>(
        0L, rows, (long)p.red_stride, (long)nch, (long)nch, p.bn_dbeta + p.n_off, 0L);
    if (p.aux_mode == 2)
      conv_red_finish_kernel<<<det_finish_grid(nch, rows), kDetFinishThreads, 0, st>>>(
          (long)nch, rows, (long)p.red_stride, (long)nch, (long)nch, p.bn_dgamma + p.n_off, 0L);
  }
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

// haloed 3x3 path: worth it when 8x16 single-image tiles cover the image without much waste
// k_channels = channels per tap of the GEMM-K dimension.  The haloed tile saves the nine per-tap fetches where they make
// the kernel L2-bound (>= 128 channels on large images whose extent the 8x16 tile divides); on thin layers the
// per-tile issue cost dominates and ragged small images waste rows.
// (MCB_HALO overrides the rule in tests: see test_hooks)
static bool use_halo(int ksize, int stride, int W, int H, int k_channels) {
  const int mode = test_hooks().halo;
  if (ksize != 3 || stride != 1 || mode == 0) return false;
  if (mode == 2) return k_channels >= kHaloMinChannels && W % 8 == 0 && H % 16 == 0 && W >= 80;
  const double eff = (double)W * H / ((double)((W + 7) / 8) * 8 * ((H + 15) / 16) * 16);
  return eff >= 0.8;
}

// the widest N tile that divides n channels
static int widest_bn(int n) {
  for (int bn : {256, 128, 64})
    if (n % bn == 0) return bn;
  return 32;
}

static int pick_bn(int n_total, long m_tiles, int phases) {
  int bn = widest_bn(n_total);
  // keep the machine filled when the pixel dimension is small
  const long sms = num_sms();
  // (fat tiles beat many thin ones: go below 128 only when even 128-wide tiles leave most SMs idle; one round of
  // 256-wide tiles beats two rounds of 128-wide ones until the tile count falls below ~0.6 of a wave)
  if (bn > 128 && m_tiles * phases * (n_total / bn) * 10 < sms * kBn256MinWaveX10) bn = 128;
  if (bn > 64 && n_total % 64 == 0 && m_tiles * phases * (n_total / bn) < sms / 3) bn = 64;
  const int forced = test_hooks().force_bn;
  if (forced && n_total % forced == 0) bn = forced;
  return bn;
}

// weight tensor map: bf16 [taps][rows][pitch], columns [c_off, c_off + cols) viewed as (cols, rows, taps)
static int encode_weight(CUtensorMap* m, const void* w, int taps, int rows, int pitch, int c_off, int cols,
                         int box_inner, int box_rows) {
  uint64_t dims[3] = {(uint64_t)cols, (uint64_t)rows, (uint64_t)taps};
  uint64_t str[2] = {(uint64_t)pitch * 2, (uint64_t)pitch * rows * 2};
  uint32_t box[3] = {(uint32_t)box_inner, (uint32_t)box_rows, 1};
  return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, static_cast<const char*>(w) + (size_t)c_off * 2, dims, str,
                     box, box_inner * 2);
}

// NHWC bf16 tensor
struct View { const void* p; int n, h, w, c; };

// tensor map of t (slot < 0) or of its 2x2 parity view (py, px) = (slot >> 1, slot & 1); box (box_c, bw, bh, bn)
static int encode_view(CUtensorMap* m, const View& t, int slot, int box_c, int bw, int bh, int bn) {
  return encode_nhwc_view(m, t.p, t.n, t.h, t.w, t.c, 0, t.c, slot < 0 ? -1 : slot >> 1, slot < 0 ? -1 : slot & 1,
                          box_c, bw, bh, bn, box_c * 2);
}

// 1-D decomposition ------------------------------------------------------------------------------------------------
// One axis of a convolution with kernel size ksize, padding pad and stride 1 or 2: output o reads input
// stride * o - pad + k.  gather: the taps of that convolution; scatter: the taps of its data gradient (the transposed
// conv of stride 2, padding 1 is the data gradient of such a conv).  Taps are listed by increasing kernel index k, or
// decreasing with k_desc: the order within a phase is the fp32 accumulation order of the kernel.
struct TapRule { int ksize, pad, stride; bool scatter = false, k_desc = false; };
struct Tap1D { int k; int d; int parity; };  // kernel index, offset in the (possibly parity) view, source parity

// gather: offset floor((k - pad) / stride) in the input parity view (k - pad) mod stride, for every k.
// scatter, for parity `parity` of the convolution's input (the data gradient's output): input stride * y + parity
// receives output y + (parity + pad - k) / stride, for the k where that divides (stride 1: parity 0 and every k)
static int taps_1d(const TapRule& r, int parity, Tap1D* out) {
  int n = 0;
  for (int i = 0; i < r.ksize; ++i) {
    const int k = r.k_desc ? r.ksize - 1 - i : i;
    if (!r.scatter) {
      const int s = k - r.pad, par = (s % r.stride + r.stride) % r.stride;
      out[n++] = {k, (s - par) / r.stride, par};
    } else if ((parity + r.pad - k) % r.stride == 0) {
      out[n++] = {k, (parity + r.pad - k) / r.stride, 0};
    }
  }
  return n;
}

// Calls f(slot, dx, dy, wtap) for the 2-D taps of phase (py, px), y-major: slot = py * 2 + px of the source parity view
// the tap reads (0 for stride-1 ops), (dx, dy) its offset in that view, wtap its weight tap
template <class F>
static void for_each_tap(const TapRule& r, int py, int px, F f) {
  Tap1D ty[4], tx[4];
  const int ny = taps_1d(r, py, ty), nx = taps_1d(r, px, tx);
  for (int i = 0; i < ny; ++i)
    for (int j = 0; j < nx; ++j) f(ty[i].parity * 2 + tx[j].parity, tx[j].d, ty[i].d, ty[i].k * r.ksize + tx[j].k);
}

static int convt_ksize(int ksize) { return ksize == 0 ? 4 : ksize; }

static int check_c(int c, const char* what) {
  if (c % 32 != 0) return fail(MCB_ERR_UNSUPPORTED, "%s channels %d not a multiple of 32", what, c);
  if (c % 64 != 0 && c != 32) return fail(MCB_ERR_UNSUPPORTED, "%s channels %d: only 32 or multiples of 64", what, c);
  return MCB_OK;
}

// One conv_gemm_kernel launch for an op whose taps follow `rule` along both axes.  GEMM M runs over the pixels of the
// output view, N over out.c, K over taps x the channels of the A sources.
//  - gather (forward conv, transposed-conv data gradient): one phase.  A is the concatenated sources a[0 .. nsrc) at
//    stride 1 (slot = source), or the 2x2 parity views of a[0] at stride 2 (slot = py * 2 + px).
//  - scatter (conv data gradient, transposed-conv forward): A is a[0].  At stride 2 there is one phase per parity view of
//    out that receives taps, packed in (py, px) order.
// Weights are bf16 [ksize^2][rows][w_pitch]: K-major for forward ops (rows = out.c, the A sources' channels side by
// side), MN-major for data gradients (b_mn: rows = a[0].c, columns [w_off, w_off + out.c)).  aux: a tensor with the
// geometry of out that the epilogue reads (p.aux_mode), or null.  The caller has set the epilogue fields of p.
static int plan_conv(ConvGemmParams& p, const TapRule& rule, const View* a, int nsrc, const View& out, const void* aux,
                     const void* w, int w_pitch, int w_off, bool b_mn, cudaStream_t st) {
  const bool phased = rule.scatter && rule.stride == 2, parity_a = !rule.scatter && rule.stride == 2;
  const int Wv = phased ? out.w / 2 : out.w, Hv = phased ? out.h / 2 : out.h, N = out.n;
  int BK = 64;
  for (int s = 0; s < nsrc; ++s)
    if (a[s].c % 64 != 0) BK = 32;
  const bool halo = use_halo(rule.ksize, rule.stride, Wv, Hv, nsrc == 2 ? std::min(a[0].c, a[1].c) : a[0].c);
  if (halo) { p.bw = 8; p.bh = 16; p.bn = 1; }
  else pick_tile(Wv, Hv, N, 128, 1, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  p.Wv = Wv; p.Hv = Hv; p.Nimg = N;
  p.tiles_x = (Wv + p.bw - 1) / p.bw;
  p.tiles_y = (Hv + p.bh - 1) / p.bh;
  const long m_tiles = (long)p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);

  bool used[4] = {false, false, false, false};  // A slots the taps read
  int phases = 0, nt = 0, phase_slot[4];
  for (int v = 0; v < (phased ? 4 : 1); ++v) {
    const int start = nt;
    // y, then x, then the concat source (the HALO producer indexes tap_begin + t * nsrc + s); concat sources come only
    // with stride-1 gathers, whose taps all read slot 0
    for_each_tap(rule, v >> 1, v & 1, [&](int slot, int dx, int dy, int wtap) {
      for (int s = 0; s < nsrc; ++s) {
        TapDesc& t = p.taps[nt++];
        t.src = slot + s; t.dx = dx; t.dy = dy; t.nchunks = a[s].c / BK; t.wk0 = s == 0 ? 0 : a[0].c; t.wtap = wtap;
        used[slot + s] = true;
      }
    });
    if (nt == start) continue;
    p.tap_start[phases] = start; p.tap_count[phases] = nt - start;
    phase_slot[phases++] = phased ? v : -1;
  }
  for (int v = 0; v < 4; ++v)
    if (used[v])
      if (int r = encode_view(&p.tmA[v], a[parity_a ? 0 : v], parity_a ? v : -1, BK, halo ? kHaloW : p.bw,
                              halo ? kHaloH : p.bh, p.bn)) return r;

  const int BN = pick_bn(out.c, m_tiles, phases);
  const int wtaps = rule.ksize * rule.ksize;
  if (int r = b_mn ? encode_weight(&p.tmB, w, wtaps, a[0].c, w_pitch, w_off, out.c, chunk_width(BN), BK)
                   : encode_weight(&p.tmB, w, wtaps, out.c, w_pitch, 0, w_pitch, BK, BN)) return r;
  const View aux_view = {aux, out.n, out.h, out.w, out.c};
  for (int ph = 0; ph < phases; ++ph) {
    if (int r = encode_view(&p.tmD[ph], out, phase_slot[ph], chunk_width(BN), p.bw, p.bh, p.bn)) return r;
    if (aux)
      if (int r = encode_view(&p.tmX[ph], aux_view, phase_slot[ph], chunk_width(BN), p.bw, p.bh, p.bn)) return r;
  }
  return launch_conv(BN, BK, b_mn, p, (int)m_tiles, out.c / BN, phases, st, halo);
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

static int launch_wgrad(WgradParams& p, int BN, int cin_src, cudaStream_t st) {
  const int m_tiles = (p.cout + 127) / 128;
  const int n_tiles = cin_src / BN;
  // split-K over the pixel tiles so the grid covers the machine a few times
  // Every split adds a full fp32 output tile with red.add (atomic traffic = splits x |dW|), while the operand
  // streams are L2/HBM-bound and want every SM busy.  So: exactly ONE resident wave of CTAs (never a ragged second
  // wave; the 384-thread CTA takes the whole register file, one CTA per SM) and at least `min_kb` K blocks per CTA.
  const long base = (long)m_tiles * n_tiles * p.ntaps;
  const long cap = (long)num_sms() * kWgradWavesX10 / 10;
  int splits = (int)std::max(1L, std::min((long)p.tiles_total, cap / std::max(1L, base)));
  splits = std::max(1, std::min(splits, std::max(1, p.tiles_total / kWgradMinKb)));
  // short reductions (deep layers: few pixel tiles, many weights) are bound by the fp32 red.add epilogues, not by the
  // operand streams: aim for kWgradKbTarget K blocks per CTA, but keep at least 0.4 of a wave busy (on the full step
  // these GEMMs share the SMs with the BatchNorm-backward kernels)
  const long lo_cap = cap * kWgradMinWaveX10 / 10;
  const int lo = (int)std::max(1L, lo_cap / std::max(1L, base));
  const int want = std::max(1, p.tiles_total / kWgradKbTarget);
  splits = std::max(1, std::min(splits, std::max(lo, want)));
  const int forced = test_hooks().wgrad_splits;
  if (forced > 0) splits = std::min(forced, p.tiles_total);
  // several splits store their partial products in split-ordered rows of the workspace (summed deterministically below)
  p.cin_src = cin_src;
  p.slice = (long)p.ntaps * p.cout * cin_src;
  if (splits > 1) splits = (int)std::max(1L, std::min((long)splits, kWgradRegionCap / p.slice));
  p.ws_off = splits > 1 ? wgrad_region_offset(st) : 0;
  p.splits = splits;
  const int per = (p.tiles_total + splits - 1) / splits;
  p.stages = std::max(2, std::min(std::min(per, kWgradMaxStages), kSmemBudget / wgrad_smem(BN, 0).stage));
  const size_t smem = wgrad_smem(BN, p.stages).bytes;
  dim3 grid(n_tiles, m_tiles, p.ntaps * splits);
  int r;
  switch (BN) {
    case 256: r = launch_kernel<wgrad_kernel<256>>(p, grid, kGemmThreads, smem, st); break;
    case 128: r = launch_kernel<wgrad_kernel<128>>(p, grid, kGemmThreads, smem, st); break;
    case 64: r = launch_kernel<wgrad_kernel<64>>(p, grid, kGemmThreads, smem, st); break;
    default: r = launch_kernel<wgrad_kernel<32>>(p, grid, kGemmThreads, smem, st); break;
  }
  if (r || splits == 1) return r;
  // the splits that own pixel tiles, summed in split order into dW[tap][cout][ci_off + ci] (detsum.cuh)
  const int rows = (p.tiles_total + per - 1) / per;
  wgrad_red_finish_kernel<<<det_finish_grid(p.slice, rows), kDetFinishThreads, 0, st>>>(
      p.ws_off, rows, p.slice, p.slice, (long)cin_src, p.dw + p.ci_off, (long)p.cin_total);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

static int wgrad_common_setup(WgradParams& p, int Wv, int Hv, int N, int cout) {
  pick_tile(Wv, Hv, N, 64, 16, &p.bw, &p.bh, &p.bn);
  p.rows = p.bw * p.bh * p.bn;
  if (p.rows % 16 != 0 || p.rows > 64) return fail(MCB_ERR_UNSUPPORTED, "wgrad: no pixel box for %dx%dx%d", Wv, Hv, N);
  p.Wv = Wv; p.Hv = Hv; p.Nimg = N;
  p.tiles_x = (Wv + p.bw - 1) / p.bw;
  p.tiles_y = (Hv + p.bh - 1) / p.bh;
  p.tiles_total = p.tiles_x * p.tiles_y * ((N + p.bn - 1) / p.bn);
  p.a_cw = (cout % 64 == 0) ? 64 : 32;
  p.a_chunks = (cout >= 128) ? 2 : 1;
  return MCB_OK;
}

// One wgrad_kernel launch: dW[tap][cout][ci_off + ci] += sum over pixels of dy[.., cout] x[.., ci] at the offsets of the
// taps of `rule` (a gather).  The taps read x for a conv weight gradient and dy for a transposed-conv one (through the
// stride-2 conv over dy that is its data gradient); the other operand is read plainly and the pixel tiles cover it.
// The caller has set dw, cout, cin_total and ci_off.
static int plan_wgrad(WgradParams& p, const TapRule& rule, const View& dy, const View& x, bool taps_on_dy,
                      cudaStream_t st) {
  const View& plain = taps_on_dy ? x : dy;
  if (int r = wgrad_common_setup(p, plain.w, plain.h, plain.n, dy.c)) return r;
  bool used_a[4] = {!taps_on_dy, false, false, false}, used_b[4] = {taps_on_dy, false, false, false};
  bool* used = taps_on_dy ? used_a : used_b;
  int nt = 0;
  for_each_tap(rule, 0, 0, [&](int slot, int ox, int oy, int wtap) {
    WgradTap& t = p.taps[nt++];
    if (taps_on_dy) { t.srcA = slot; t.ax = ox; t.ay = oy; }
    else { t.srcB = slot; t.bx = ox; t.by = oy; }
    t.wtap = wtap;
    used[slot] = true;
  });
  p.ntaps = nt;
  const bool parity = rule.stride == 2;
  const int BN = widest_bn(x.c);
  for (int v = 0; v < 4; ++v) {
    if (used_a[v])
      if (int r = encode_view(&p.tmA[v], dy, taps_on_dy && parity ? v : -1, p.a_cw, p.bw, p.bh, p.bn)) return r;
    if (used_b[v])
      if (int r = encode_view(&p.tmB[v], x, !taps_on_dy && parity ? v : -1, chunk_width(BN), p.bw, p.bh, p.bn))
        return r;
  }
  return launch_wgrad(p, BN, x.c, st);
}

}  // namespace mcb

using namespace mcb;

// =====================================================================================================
extern "C" int mcb_conv_fwd(const mcb_conv_fwd_args* a, void* stream) {
  MCB_REQUIRE(a && a->x[0] && a->weight && a->y, "conv_fwd: null pointer");
  MCB_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv_fwd: ksize %d", a->ksize);
  MCB_REQUIRE(a->stride == 1 || a->stride == 2, "conv_fwd: stride %d", a->stride);
  const int nsrc = a->x[1] ? 2 : 1;
  MCB_REQUIRE(!(nsrc == 2 && a->stride == 2), "conv_fwd: concat + stride 2 unsupported");
  for (int s = 0; s < nsrc; ++s)
    if (int r = check_c(a->cin[s], "conv_fwd input")) return r;
  if (int r = check_c(a->cout, "conv_fwd output")) return r;
  // a 32-channel source makes the whole launch BK = 32 (plan_conv): each source is read in 32-channel chunks
  MCB_REQUIRE(a->stride == 1 || (a->h % 2 == 0 && a->w % 2 == 0), "conv_fwd: stride 2 needs even H, W");
  const int Ho = a->h / a->stride, Wo = a->w / a->stride;
  const View x[2] = {{a->x[0], a->n, a->h, a->w, a->cin[0]}, {a->x[1], a->n, a->h, a->w, a->cin[1]}};

  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.bias = a->bias; p.relu = a->relu; p.stats = a->stats; p.stats_c = a->cout;
  p.scale = a->scale;
  if (a->residual) {
    p.residual = static_cast<const __nv_bfloat16*>(a->residual);
    p.mask_H = Ho; p.mask_W = Wo; p.mask_C = a->cout; p.mask_s = 1;
  }
  return plan_conv(p, {a->ksize, a->ksize / 2, a->stride}, x, nsrc, {a->y, a->n, Ho, Wo, a->cout}, nullptr, a->weight,
                   a->cin[0] + (nsrc == 2 ? a->cin[1] : 0), 0, false, static_cast<cudaStream_t>(stream));
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
  MCB_REQUIRE(a->stride == 1 || (a->h % 2 == 0 && a->w % 2 == 0), "conv_dgrad: stride 2 needs even H, W");
  MCB_REQUIRE(!(a->dx_channel_sum && (!a->relu_mask || a->accumulate)),
              "conv_dgrad: dx_channel_sum needs relu_mask and a complete (non-accumulated) gradient");
  if (a->bn_z) {
    MCB_REQUIRE(a->bn_mean && a->bn_invstd && a->bn_gamma && a->bn_beta && a->bn_dbeta && a->bn_dgamma,
                "conv_dgrad: incomplete bn reduction args");
    MCB_REQUIRE(!a->accumulate, "conv_dgrad: bn reduction needs the complete gradient (no accumulate)");
    MCB_REQUIRE(!(a->stride == 2 && a->ksize == 1), "conv_dgrad: bn reduction with a 1x1 stride-2 conv is unsupported");
  }

  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.accumulate = a->accumulate;
  p.aux_mode = a->bn_z ? 2 : (a->relu_mask ? 1 : 0);
  p.bn_dbeta = a->dx_channel_sum;
  if (a->bn_z) {
    p.bn_mean = a->bn_mean; p.bn_invstd = a->bn_invstd; p.bn_gamma = a->bn_gamma; p.bn_beta = a->bn_beta;
    p.bn_dbeta = a->bn_dbeta; p.bn_dgamma = a->bn_dgamma;
  }
  if (a->stride == 2 && a->ksize == 1 && !a->accumulate) {
    // only the (even, even) input pixels receive gradient; the rest is zero
    MCB_CHECK_CUDA(cudaMemsetAsync(a->dx, 0, (size_t)a->n * a->h * a->w * a->cin * 2, st));
  }
  const View dy = {a->dy, a->n, a->h / a->stride, a->w / a->stride, a->cout};
  // aux: the tensor the ReLU mask is derived from
  return plan_conv(p, {a->ksize, a->ksize / 2, a->stride, true}, &dy, 1, {a->dx, a->n, a->h, a->w, a->cin},
                   a->bn_z ? a->bn_z : a->relu_mask, a->weight, a->cin_total, a->ci_off, true, st);
}

// =====================================================================================================
// ConvTranspose2d(ksize, stride 2, padding 1): four sub-pixel phases, the data gradient of a stride-2 conv.  ksize 3
// (output_padding 1, same 2x output) reads the zero row past the bottom / right edge (TMA out-of-bounds fill).
extern "C" int mcb_convt_fwd(const mcb_convt_fwd_args* a, void* stream) {
  MCB_REQUIRE(a && a->x && a->weight && a->y, "convt_fwd: null pointer");
  if (int r = check_c(a->cin, "convt_fwd input")) return r;
  if (int r = check_c(a->cout, "convt_fwd output")) return r;
  const int K = convt_ksize(a->ksize);
  MCB_REQUIRE(K == 3 || K == 4, "convt_fwd: ksize %d", a->ksize);
  const View x = {a->x, a->n, a->h, a->w, a->cin};
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.bias = a->bias; p.relu = a->relu;
  // the 3x3 kernel sums the two taps of an odd parity as k = 2, then k = 0
  return plan_conv(p, {K, 1, 2, true, K == 3}, &x, 1, {a->y, a->n, 2 * a->h, 2 * a->w, a->cout}, nullptr, a->weight,
                   a->cin, 0, false, static_cast<cudaStream_t>(stream));
}

extern "C" int mcb_convt_dgrad(const mcb_convt_dgrad_args* a, void* stream) {
  MCB_REQUIRE(a && a->dy && a->weight && a->dx, "convt_dgrad: null pointer");
  MCB_REQUIRE(!(a->relu_mask && a->accumulate), "convt_dgrad: relu_mask with accumulate is ill-defined");
  if (int r = check_c(a->cin, "convt_dgrad dx")) return r;
  if (int r = check_c(a->cout, "convt_dgrad dy")) return r;
  const int K = convt_ksize(a->ksize);
  MCB_REQUIRE(K == 3 || K == 4, "convt_dgrad: ksize %d", a->ksize);
  MCB_REQUIRE(!(a->dx_channel_sum && (!a->relu_mask || a->accumulate)),
              "convt_dgrad: dx_channel_sum needs relu_mask and a complete (non-accumulated) gradient");
  const View dy = {a->dy, a->n, 2 * a->h, 2 * a->w, a->cout};  // dx is h x w
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.accumulate = a->accumulate;
  p.aux_mode = a->relu_mask ? 1 : 0;
  p.bn_dbeta = a->dx_channel_sum;
  return plan_conv(p, {K, 1, 2}, &dy, 1, {a->dx, a->n, a->h, a->w, a->cin}, a->relu_mask, a->weight, a->cin, 0, true,
                   static_cast<cudaStream_t>(stream));
}

// =====================================================================================================
extern "C" int mcb_conv_wgrad(const mcb_conv_wgrad_args* a, void* stream) {
  MCB_REQUIRE(a && a->dy && a->x && a->dw, "conv_wgrad: null pointer");
  MCB_REQUIRE(a->ksize == 1 || a->ksize == 3, "conv_wgrad: ksize %d", a->ksize);
  MCB_REQUIRE(a->stride == 1 || a->stride == 2, "conv_wgrad: stride %d", a->stride);
  if (int r = check_c(a->cout, "conv_wgrad dy")) return r;
  if (int r = check_c(a->cin, "conv_wgrad x")) return r;
  MCB_REQUIRE(a->cout % 128 == 0 || a->cout == 64 || a->cout == 32, "conv_wgrad: cout %d", a->cout);
  MCB_REQUIRE(a->stride == 1 || (a->h % 2 == 0 && a->w % 2 == 0), "conv_wgrad: stride 2 needs even H, W");
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.dw = a->dw; p.cout = a->cout; p.cin_total = a->cin_total; p.ci_off = a->ci_off;
  const View dy = {a->dy, a->n, a->h / a->stride, a->w / a->stride, a->cout}, x = {a->x, a->n, a->h, a->w, a->cin};
  return plan_wgrad(p, {a->ksize, a->ksize / 2, a->stride}, dy, x, false, static_cast<cudaStream_t>(stream));
}

extern "C" int mcb_convt_wgrad(const mcb_convt_wgrad_args* a, void* stream) {
  MCB_REQUIRE(a && a->dy && a->x && a->dw, "convt_wgrad: null pointer");
  if (int r = check_c(a->cout, "convt_wgrad dy")) return r;
  if (int r = check_c(a->cin, "convt_wgrad x")) return r;
  MCB_REQUIRE(a->cout % 128 == 0 || a->cout == 64 || a->cout == 32, "convt_wgrad: cout %d", a->cout);
  const int K = convt_ksize(a->ksize);
  MCB_REQUIRE(K == 3 || K == 4, "convt_wgrad: ksize %d", a->ksize);
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.dw = a->dw; p.cout = a->cout; p.cin_total = a->cin; p.ci_off = 0;
  const View dy = {a->dy, a->n, 2 * a->h, 2 * a->w, a->cout}, x = {a->x, a->n, a->h, a->w, a->cin};
  return plan_wgrad(p, {K, 1, 2}, dy, x, true, static_cast<cudaStream_t>(stream));
}
