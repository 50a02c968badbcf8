// conv_gemm.cuh — device kernels for every convolution-shaped op of the U-Net, as wgmma implicit GEMMs.
//
//   conv_gemm_kernel<BN, BK, B_MN>   forward convs / transposed convs / data gradients
//       D[pixel, n] = sum over taps t, channels k:  A_t[pixel + off_t, k] * B_t[n, k]
//       A tiles: NHWC bf16 activations fetched by 4-D tiled TMA boxes (channels, bw, bh, bn) placed at the tap
//       offset — out-of-bounds rows/columns are zero-filled by the TMA unit, which IS the conv zero padding.
//       B tiles: bf16 weights [tap][cout][cin]; K-major for forward, MN-major (same storage) for dgrad.
//       Accumulator: 128 x BN fp32 in registers, 64 rows per MMA warpgroup.  Epilogue: bias / ReLU / ReLU-mask /
//       BN-statistics, bf16, TMA store (or TMA reduce-add for gradient accumulation).
//
//   wgrad_kernel<BN>                 weight gradients
//       dW_t[co, ci] += sum over pixels: dY[pixel + offA_t, co] * X[pixel + offB_t, ci]
//       both operands MN-major (the pixel axis is GEMM-K), split-K over pixel tiles, deterministic split sum.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one warp issues, the register file goes to the others),
// warpgroups 1 and 2 = MMA + epilogue, rows 0..63 and 64..127 of the 128-row tile.
#pragma once
#include "tc.cuh"
#include "detsum.cuh"

namespace mcb {

constexpr int kMaxTaps = 24;

// per-CTA partial rows of the epilogue's per-channel reductions (conv_gemm_kernel) and of split-K weight gradients
// (wgrad_kernel); summed in a fixed order by the finishing kernels (detsum.cuh)
constexpr long kConvRedCap = 256L * 4096;         // rows (CTAs) x [sum | second sum] over <= 2048 channels
// weight-gradient GEMMs of one step run on two streams at once (main chain and side stream): one region per stream
constexpr int kWgradRegions = 4;
constexpr long kWgradRegionCap = 4L * 1024 * 1024;   // splits x weight-gradient elements of one launch
MCB_DET_WORKSPACE(float, g_conv_red, kConvRedCap, conv_red_finish_kernel)
MCB_DET_WORKSPACE(float, g_wgrad_red, kWgradRegions * kWgradRegionCap, wgrad_red_finish_kernel)
constexpr int kGemmThreads = 384;
constexpr int kProducerRegs = 40, kMmaRegs = 232;  // 128 x 40 + 256 x 232 <= 64 K registers

struct TapDesc {
  int16_t src;      // index into tmA
  int16_t dx, dy;   // offset in the source view (W, H coordinates)
  int16_t nchunks;  // number of BK-channel chunks of this source
  int32_t wk0;      // first K coordinate in the weight tensor for this source (concat offset)
  int32_t wtap;     // tap coordinate in the weight tensor
};

struct ConvGemmParams {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  CUtensorMap tmD[4];  // one per phase (blockIdx.z)
  TapDesc taps[kMaxTaps];
  int tap_start[4];
  int tap_count[4];
  int Wv, Hv, Nimg;  // extents of the output view
  int bw, bh, bn, rows;
  int tiles_x, tiles_y;
  int m_tiles, n_tiles, phases;  // persistent tile space: phases x m_tiles x n_tiles
  int stages;
  int b_resident;  // HALO only, experimental: the 9 per-tap weight tiles are loaded ONCE per CTA into ring slots 0..8
                   // (single N tile, one channel chunk) instead of once per pixel tile
  int n_off;  // first N (weight row / column) coordinate of this launch (concat source slice for dgrad)
  // epilogue:  v = acc * scale[c] + bias[c] + residual[pix][c];  v = relu(v);  v = mask ? v : 0
  const float* scale;              // per-channel multiplier (inference-mode BatchNorm folded into the epilogue), or null
  const __nv_bfloat16* residual;   // NHWC bf16 with the geometry of the output tensor (mask_H/W/C), or null
  const float* bias;
  float* stats;
  int stats_c;  // number of channels in stats (cout)
  int mask_H, mask_W, mask_C, mask_s;  // geometry of `residual`: full dims; mask_s = 1 (plain) or 2 (parity view)
  int relu;
  int accumulate;
  // Auxiliary tile (dgrad only): a tensor with the geometry of the OUTPUT, fetched chunk by chunk with TMA (tmX, same
  // boxes as tmD) into shared memory while the main loop of the tile still runs.
  //   aux_mode 1: the ReLU output y of the producing layer:  g = acc * (y > 0)
  //   aux_mode 2: the BatchNorm input z of the producing conv-BN-ReLU unit: the mask is that unit's own output sign,
  //               (fma(z, gamma*invstd, beta - mean*gamma*invstd) > 0), and the BatchNorm-backward reductions of the
  //               stored gradient ride along:  dbeta += sum g,  dgamma += sum g * (z - mean) * invstd
  CUtensorMap tmX[4];
  int aux_mode;
  const float* bn_mean;
  const float* bn_invstd;
  const float* bn_gamma;
  const float* bn_beta;
  float* bn_dbeta;
  float* bn_dgamma;
  int red_stride;  // 2 x the N extent of the launch: one g_conv_red row per CTA, [sum | second sum] per channel
};

struct WgradTap {
  int16_t srcA, ax, ay;
  int16_t srcB, bx, by;
  int32_t wtap;
};

struct WgradParams {
  CUtensorMap tmA[4];  // dY views, box (64 | 32 channels, bw, bh, bn)
  CUtensorMap tmB[4];  // X views
  WgradTap taps[16];
  int ntaps;
  int Wv, Hv, Nimg;
  int bw, bh, bn, rows;  // rows % 16 == 0, rows <= 64
  int tiles_x, tiles_y, tiles_total;
  int splits;
  int stages;
  float* dw;  // [tap][cout][cin_total]
  int cout, cin_total, ci_off;
  int a_cw;  // channel width of one A chunk: 64 (SW128) or 32 (SW64)
  int a_chunks;  // chunks actually loaded (1 or 2); missing ones alias chunk 0 (LBO = 0)
  int cin_src;   // input channels of this launch (the N extent)
  long slice;    // splits > 1: elements of one split's g_wgrad_red row, ntaps x cout x cin_src
  long ws_off;   // first element of this launch's stream's region of g_wgrad_red
};

// (pointer + offset, not an integer round trip: the result provably stays in the shared window, so every access below
// compiles to LDS/STS with 32-bit addressing instead of generic LD/ST with 64-bit address arithmetic)
__device__ __forceinline__ uint8_t* align_up_1024(uint8_t* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  return p + ((1024u - (a & 1023u)) & 1023u);
}


// -------------------------------------------------------------------------------------------------
// Persistent, warp-specialised: one CTA per SM walks tiles t = blockIdx.x, += gridDim.x (n fastest, so CTAs that run
// together share the A pixel tile in L2).  The TMA ring (full/empty mbarriers) runs continuously across tiles, so the
// producer loads the operands of tile i+1 while the MMA warpgroups run the epilogue of tile i.
constexpr int kConvThreads = 384;  // warpgroup 0 TMA producer, warpgroups 1, 2 MMA + epilogue

// HALO (3x3, stride 1): the pixel tile is 8 wide x 16 tall in one image and ONE haloed TMA box (BK channels, 10, 18, 1)
// per channel chunk serves all nine taps: tap (dy, dx) is the same shared-memory tile read through a descriptor whose
// start is shifted by ((1+dy)*10 + (1+dx)) rows and whose 8-row groups are 10 rows apart (the swizzle is a function of
// the absolute shared-memory address, which both TMA and wgmma apply, so unaligned starts and a non-atom SBO address
// the same bytes TMA wrote).  A and B then travel in separate mbarrier rings: 1 A load + 9 B loads per channel chunk.
constexpr int kHaloW = 10, kHaloH = 18;  // (8 + 2) x (16 + 2)

// per-channel reduction scratch: per MMA warpgroup 4 warps x (up to) 8 channel groups x 16 floats
constexpr int kStatBytes = 2 * 4 * 8 * 16 * 4;

__device__ __forceinline__ void mma_wg_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int BN, int BK, bool B_MN, bool HALO>
__global__ void __launch_bounds__(kConvThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
  static_assert(BK == 64 || BK == 32, "BK");
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN");
  constexpr int A_ROW_BYTES = BK * 2;              // 128 (SW128) or 64 (SW64)
  constexpr int A_BYTES = HALO ? ((kHaloW * kHaloH * A_ROW_BYTES + 1023) / 1024) * 1024 : 128 * A_ROW_BYTES;
  constexpr int B_BYTES = BN * BK * 2;
  constexpr int STAGE_BYTES = HALO ? B_BYTES : A_BYTES + B_BYTES;  // HALO: the ring holds B tiles; A has its own 2 slots
  constexpr int A_RING_BYTES = HALO ? 2 * A_BYTES : 0;
  constexpr uint32_t A_LAYOUT = (BK == 64) ? tc::LAYOUT_SW128 : tc::LAYOUT_SW64;
  // MN-major B: rows are K (BK of them), each row holds min(BN,64) n-values
  constexpr int BMN_CW = (BN >= 64) ? 64 : 32;          // n-values per sub-tile row
  constexpr int BMN_ROW_BYTES = BMN_CW * 2;             // 128 or 64
  constexpr int BMN_SUB_BYTES = BK * BMN_ROW_BYTES;     // one sub-tile
  constexpr uint32_t BMN_LAYOUT = (BMN_CW == 64) ? tc::LAYOUT_SW128 : tc::LAYOUT_SW64;
  // output staging: chunks of OUT_CW channels (one TMA store each)
  constexpr int OUT_CW = (BN >= 64) ? 64 : 32;
  constexpr int OUT_ROW_BYTES = OUT_CW * 2;
  constexpr int OUT_CHUNK_BYTES = 128 * OUT_ROW_BYTES;
  constexpr int OUT_CHUNKS = BN / OUT_CW;
  // small tiles finish faster than a TMA store drains: rotate several staging buffers so the epilogue of tile i+1 never
  // waits for the store of tile i
  constexpr int OUT_BUFS = (BN <= 64) ? 4 : (BN == 128 ? 2 : 1);
  constexpr int OUT_BYTES = OUT_BUFS * OUT_CHUNKS * OUT_CHUNK_BYTES;
  constexpr int ACC = BN / 2;  // fp32 accumulators per thread (64 x BN per warpgroup)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_up_1024(smem_raw);
  const int stages = p.stages;
  const int aux_mode = p.aux_mode;
  uint8_t* a_ring = smem + (size_t)stages * STAGE_BYTES;               // HALO only: 2 haloed A tiles
  uint8_t* out_stage = a_ring + A_RING_BYTES;                          // 1024-aligned (all pieces are)
  uint8_t* aux_stage = out_stage + OUT_BYTES;                          // aux modes: one chunk per MMA warpgroup
  float* stat_scratch = reinterpret_cast<float*>(aux_stage + (aux_mode != 0 ? 2 * OUT_CHUNK_BYTES : 0));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stat_scratch) + kStatBytes);
  uint64_t* empty_bar = full_bar + stages;
  uint64_t* a_full_bar = empty_bar + stages;      // [2] (HALO)
  uint64_t* a_empty_bar = a_full_bar + 2;         // [2] (HALO)
  uint64_t* aux_full_bar = a_empty_bar + 2;       // [2] one per MMA warpgroup
  int* row_pix = reinterpret_cast<int*>(aux_full_bar + 2);  // [128] pixel index in the full-resolution tensor, -1 = invalid

  // the shuffle makes the warp index provably warp-uniform, so the role loops below compile onto the uniform datapath
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int tiles_per_phase = p.m_tiles * p.n_tiles;
  const int total_tiles = tiles_per_phase * p.phases;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < stages; ++s) {
      tc::mbar_init(&full_bar[s], 1);
      tc::mbar_init(&empty_bar[s], 2);  // one arrival per MMA warpgroup
    }
    tc::mbar_init(&a_full_bar[0], 1);
    tc::mbar_init(&a_full_bar[1], 1);
    tc::mbar_init(&a_empty_bar[0], 2);
    tc::mbar_init(&a_empty_bar[1], 2);
    tc::mbar_init(&aux_full_bar[0], 1);
    tc::mbar_init(&aux_full_bar[1], 1);
    tc::fence_barrier_init();
    tc::prefetch_tmap(&p.tmB);
    tc::prefetch_tmap(&p.tmA[0]);
  }
  __syncthreads();
  pdl_prologue();  // everything above touched only shared memory / kernel parameters

  if (warp < 4) {
    tc::regs_dealloc<kProducerRegs>();
    if (warp != 0) return;
    // ===================================================== TMA producer (whole warp walks the loop, one elected lane issues)
    const uint32_t a_bytes = (uint32_t)p.rows * A_ROW_BYTES;
    uint32_t ag = 0;  // HALO: haloed A tiles issued so far
    int ring_s = 0;            // pipeline slot / phase parity, advanced without integer division: the single-thread
    uint32_t ring_ph = 0;      // producer loop is a latency chain, every instruction in it is exposed
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      // tile order: phase fastest (the phases of one pixel tile share the A tile in L2), then pixel tile, N tile
      // slowest (CTAs running together share the weight tile; a CTA keeps its N tile for many tiles in a row)
      const int phase_id = t % p.phases;
      const int mt = (t / p.phases) % p.m_tiles;
      const int nt = t / (p.phases * p.m_tiles);
      const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tn = mt / (p.tiles_x * p.tiles_y);
      const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = tn * p.bn;
      const int ncol0 = nt * BN;
      const int tap_begin = p.tap_start[phase_id], tap_end = tap_begin + p.tap_count[phase_id];
      auto load_b = [&](uint8_t* sb, uint64_t* bar, const TapDesc& tap, int ch) {
        if (!B_MN) {
          tc::tma_load_3d(sb, &p.tmB, bar, tap.wk0 + ch * BK, p.n_off + ncol0, tap.wtap);
        } else {
#pragma unroll
          for (int j = 0; j < BN / BMN_CW; ++j)
            tc::tma_load_3d(sb + j * BMN_SUB_BYTES, &p.tmB, bar, p.n_off + ncol0 + j * BMN_CW, tap.wk0 + ch * BK,
                            tap.wtap);
        }
      };
      if (HALO) {
        // taps are listed tap-major, source-minor: entry (t, s) at tap_begin + t * nsrc + s
        const int nsrc = (tap_end - tap_begin) / 9;
        for (int sidx = 0; sidx < nsrc; ++sidx) {
          const TapDesc t0 = p.taps[tap_begin + sidx];
          for (int ch = 0; ch < t0.nchunks; ++ch, ++ag) {
            const int as = ag & 1;
            tc::mbar_wait(&a_empty_bar[as], ((ag >> 1) & 1) ^ 1);
            if (tc::elect_one()) {
              tc::mbar_expect_tx(&a_full_bar[as], (uint32_t)(kHaloW * kHaloH * A_ROW_BYTES));
              tc::tma_load_4d(a_ring + (size_t)as * A_BYTES, &p.tmA[t0.src], &a_full_bar[as], ch * BK, x0 - 1, y0 - 1, n0);
            }
            for (int t = 0; t < 9; ++t) {
              const TapDesc tap = p.taps[tap_begin + t * nsrc + sidx];
              int s = ring_s;
              const uint32_t ph = ring_ph;
              if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
              if (p.b_resident) {
                if (ag != 0) continue;   // weights of tap t already sit in slot t
                s = t;
              } else {
                tc::mbar_wait(&empty_bar[s], ph ^ 1);
              }
              uint8_t* sb = smem + (size_t)s * STAGE_BYTES;
              if (tc::elect_one()) {
                tc::mbar_expect_tx(&full_bar[s], B_BYTES);
                load_b(sb, &full_bar[s], tap, ch);
              }
            }
          }
        }
        continue;
      }
      for (int tp = tap_begin; tp < tap_end; ++tp) {
        const TapDesc tap = p.taps[tp];
        const CUtensorMap* mA = &p.tmA[tap.src];
        for (int ch = 0; ch < tap.nchunks; ++ch) {
          const int s = ring_s;
          const uint32_t ph = ring_ph;
          if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
          tc::mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + (size_t)s * STAGE_BYTES;
          if (tc::elect_one()) {
            tc::mbar_expect_tx(&full_bar[s], a_bytes + B_BYTES);
            tc::tma_load_4d(sa, mA, &full_bar[s], ch * BK, x0 + tap.dx, y0 + tap.dy, n0);
            load_b(sa + A_BYTES, &full_bar[s], tap, ch);
          }
        }
      }
    }
    return;
  }

  // ===================================================== MMA + epilogue (warpgroups 1, 2)
  tc::regs_alloc<kMmaRegs>();
  const int wg = (warp >> 2) - 1;              // rows 64 * wg .. 64 * wg + 63 of the tile
  const int wtid = threadIdx.x & 127;          // thread index inside the warpgroup
  const int ww = wtid >> 5;                    // warp inside the warpgroup
  const int bar_id = 2 + wg;
  const int r_lo = wg * 64 + ww * 16 + (lane >> 2);  // accumulator rows r_lo and r_lo + 8 (tc::wgmma_bf16 layout)
  constexpr int CH = (OUT_CHUNKS + 1) / 2;   // chunks per warpgroup in the second pass (warpgroup 1 may own fewer)
  constexpr int CGc = OUT_CW / 8;            // 8-channel groups per chunk
  constexpr int RGc = 128 / CGc;             // row groups
  constexpr int ROWSc = 128 / RGc;           // rows per thread in the reduction
  float* my_scratch = stat_scratch + wg * (4 * CGc * 16);
  const int my_chunks = (OUT_CHUNKS - wg + 1) / 2;   // warpgroup wg owns chunks wg, wg + 2, ...
  // per-channel reductions are kept in registers (threads wtid < OUT_CW, one channel per chunk) across all tiles of
  // this CTA that share an N tile, and flushed with one atomic per channel when the N tile changes / at the end
  float racc1[CH], racc2[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) racc1[j] = racc2[j] = 0.f;
  int racc_nt = -1;
  // aux 1 with bn_dbeta set: per-channel sum of the masked gradient (bias gradient of the producing layer)
  const bool do_red = (p.stats != nullptr || aux_mode == 2 || (aux_mode == 1 && p.bn_dbeta != nullptr));
  uint8_t* abuf = aux_stage + (size_t)wg * OUT_CHUNK_BYTES;
  uint32_t aux_n = 0;
  auto issue_aux = [&](int t2, int chunk2) {   // one thread: fetch the aux chunk of tile t2 into abuf
    const int ph2 = t2 % p.phases;
    const int mt2 = (t2 / p.phases) % p.m_tiles;
    const int nt2 = t2 / (p.phases * p.m_tiles);
    const int tx2 = mt2 % p.tiles_x, ty2 = (mt2 / p.tiles_x) % p.tiles_y, tn2 = mt2 / (p.tiles_x * p.tiles_y);
    tc::mbar_expect_tx(&aux_full_bar[wg], (uint32_t)p.rows * OUT_ROW_BYTES);
    tc::tma_load_4d(abuf, &p.tmX[ph2], &aux_full_bar[wg], p.n_off + nt2 * BN + chunk2 * OUT_CW, tx2 * p.bw,
                    ty2 * p.bh, tn2 * p.bn);
  };
  if (aux_mode != 0 && wtid == 0 && my_chunks > 0 && (int)blockIdx.x < total_tiles) issue_aux(blockIdx.x, wg);
  // this CTA's row of per-channel partial sums; zeroed here, before the first flush (several barriers later)
  float* red_row = g_conv_red + (size_t)blockIdx.x * p.red_stride;
  const int red_half = p.red_stride >> 1;
  if (do_red)
    for (int i = threadIdx.x - 128; i < p.red_stride; i += 256) red_row[i] = 0.f;
  auto flush_reductions = [&]() {
    if (racc_nt >= 0 && wtid < OUT_CW) {
#pragma unroll
      for (int j = 0; j < CH; ++j) {
        if (j < my_chunks) {
          const int ch = racc_nt * BN + (wg + 2 * j) * OUT_CW + wtid;   // relative to p.n_off
          red_row[ch] += racc1[j];
          red_row[red_half + ch] += racc2[j];
          racc1[j] = racc2[j] = 0.f;
        }
      }
    }
  };

  float acc[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) acc[i] = 0.f;
  uint32_t ag = 0;
  int ring_s = 0;
  uint32_t ring_ph = 0;
  int it = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++it) {
    const int phase_id = t % p.phases;
    const int tap_begin = p.tap_start[phase_id], tap_end = tap_begin + p.tap_count[phase_id];
    // ---------------------------------------------------- main loop: one wgmma group per ring slot; the slot (and, in
    // HALO mode, the A tile after its ninth tap) is released once the NEXT group is issued and this one has completed
    {
      int prev_s = -1, prev_as = -1;
      auto release_prev = [&]() {
        if (wtid == 0) {
          if (prev_s >= 0) tc::mbar_arrive(&empty_bar[prev_s]);
          if (prev_as >= 0) tc::mbar_arrive(&a_empty_bar[prev_as]);
        }
      };
      auto mma_block = [&](uint64_t da0, uint64_t db0, bool first) {
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t da = da0 + (uint64_t)((k * 32) >> 4);
          const uint64_t db = B_MN ? db0 + (uint64_t)((k * 16 * BMN_ROW_BYTES) >> 4) : db0 + (uint64_t)((k * 32) >> 4);
          tc::wgmma_bf16<BN, 0, B_MN ? 1 : 0>(acc, da, db, (!first || k > 0) ? 1u : 0u);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        release_prev();
      };
      auto b_desc = [&](uint32_t sb) {
        return B_MN ? tc::make_smem_desc(sb, BMN_SUB_BYTES, 8 * BMN_ROW_BYTES, BMN_LAYOUT)
                    : tc::make_smem_desc(sb, 16, 8 * A_ROW_BYTES, A_LAYOUT);
      };
      if (HALO) {
        const int nsrc = (tap_end - tap_begin) / 9;
        int i = 0;
        for (int sidx = 0; sidx < nsrc; ++sidx) {
          const int nch = p.taps[tap_begin + sidx].nchunks;
          for (int ch = 0; ch < nch; ++ch, ++ag) {
            const int as = ag & 1;
            tc::mbar_wait(&a_full_bar[as], (ag >> 1) & 1);
            // this warpgroup's 64 output rows are image rows 8 wg .. 8 wg + 7 of the tile
            const uint32_t a_base = tc::smem_u32(a_ring + (size_t)as * A_BYTES) + (uint32_t)(wg * 8 * kHaloW * A_ROW_BYTES);
            for (int tt = 0; tt < 9; ++tt, ++i) {
              const TapDesc tap = p.taps[tap_begin + tt * nsrc + sidx];
              int s = ring_s;
              const uint32_t ph = ring_ph;
              if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
              if (p.b_resident) {
                s = tt;
                if (ag == 0) tc::mbar_wait(&full_bar[s], 0);   // first tile of this CTA only
              } else {
                tc::mbar_wait(&full_bar[s], ph);
              }
              const uint32_t sa = a_base + (uint32_t)(((1 + tap.dy) * kHaloW + (1 + tap.dx)) * A_ROW_BYTES);
              mma_block(tc::make_smem_desc(sa, 16, kHaloW * A_ROW_BYTES, A_LAYOUT),
                        b_desc(tc::smem_u32(smem + (size_t)s * STAGE_BYTES)), i == 0);
              prev_s = p.b_resident ? -1 : s;
              prev_as = (tt == 8) ? as : -1;
            }
          }
        }
      } else {
        int num_kb = 0;
        for (int tp = tap_begin; tp < tap_end; ++tp) num_kb += p.taps[tp].nchunks;
        for (int i = 0; i < num_kb; ++i) {
          const int s = ring_s;
          const uint32_t ph = ring_ph;
          if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
          tc::mbar_wait(&full_bar[s], ph);
          const uint32_t sa = tc::smem_u32(smem + (size_t)s * STAGE_BYTES);
          mma_block(tc::make_smem_desc(sa + (uint32_t)(wg * 64 * A_ROW_BYTES), 16, 8 * A_ROW_BYTES, A_LAYOUT),
                    b_desc(sa + A_BYTES), i == 0);
          prev_s = s;
        }
      }
      tc::wgmma_wait<0>();
      tc::fence_acc(acc);
      release_prev();
    }

    // ---------------------------------------------------- epilogue
    const int mt = (t / p.phases) % p.m_tiles;
    const int nt = t / (p.phases * p.m_tiles);
    const int tx = mt % p.tiles_x, ty = (mt / p.tiles_x) % p.tiles_y, tn = mt / (p.tiles_x * p.tiles_y);
    const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = tn * p.bn;
    const int ncol0 = nt * BN;
    // every row of the tile is a real output pixel (the common case): the second pass skips the per-row checks
    const bool tile_full = p.rows == 128 && x0 + p.bw <= p.Wv && y0 + p.bh <= p.Hv && n0 + p.bn <= p.Nimg;
    if (do_red && nt != racc_nt) {
      flush_reductions();
      racc_nt = nt;
    }
    // staging buffer of this tile: the TMA stores that last read it (OUT_BUFS tiles ago) must have finished reading
    if (wtid == 0) tc::tma_store_wait_read<OUT_BUFS - 1>();
    mma_wg_sync();
    uint8_t* obuf = out_stage + (size_t)(it % OUT_BUFS) * OUT_CHUNKS * OUT_CHUNK_BYTES;
    // registers -> scale / bias / residual / ReLU -> bf16 -> swizzled staging (the layout the TMA store reads)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_lo + 8 * h;
      const int wi = row % p.bw, hi = (row / p.bw) % p.bh, ni = row / (p.bw * p.bh);
      const int ox = x0 + wi, oy = y0 + hi, on = n0 + ni;
      const bool valid = row < p.rows && ox < p.Wv && oy < p.Hv && on < p.Nimg;
      int pix = -1;
      if (valid) {
        pix = 0;
        if (p.mask_H > 0) {
          const int fy = oy * p.mask_s + (p.mask_s == 2 ? (phase_id >> 1) : 0);
          const int fx = ox * p.mask_s + (p.mask_s == 2 ? (phase_id & 1) : 0);
          pix = (on * p.mask_H + fy) * p.mask_W + fx;
        }
      }
      if ((lane & 3) == 0) row_pix[row] = pix;
      const __nv_bfloat16* rrow = nullptr;
      if (p.residual != nullptr && valid) rrow = p.residual + (size_t)pix * p.mask_C + p.n_off + ncol0;
      uint8_t* rowp = obuf + (size_t)row * OUT_ROW_BYTES;
      const int swz = (OUT_CW == 64) ? (row & 7) : ((row >> 1) & 3);   // SWIZZLE_128B / SWIZZLE_64B
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (p.scale != nullptr) {
          const float2 sv = __ldg(reinterpret_cast<const float2*>(p.scale + p.n_off + ncol0 + col));
          v0 *= sv.x; v1 *= sv.y;
        }
        if (p.bias != nullptr) {
          const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + p.n_off + ncol0 + col));
          v0 += bv.x; v1 += bv.y;
        }
        if (rrow != nullptr) {
          const float2 rv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(rrow + col));
          v0 += rv.x; v1 += rv.y;
        }
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        constexpr int UNITS = OUT_CW / 8;   // 16-byte units per staged row
        const int chunk = j / UNITS, unit = (j % UNITS) ^ swz;
        *reinterpret_cast<uint32_t*>(rowp + (size_t)chunk * OUT_CHUNK_BYTES + unit * 16 + 4 * (lane & 3)) =
            tc::pack_bf16x2(v0, v1);
      }
    }
    tc::fence_proxy_async_smem();
    mma_wg_sync();

    for (int cj = 0; cj < my_chunks; ++cj) {
      const int chunk = wg + 2 * cj;
      uint8_t* cbuf = obuf + (size_t)chunk * OUT_CHUNK_BYTES;
      if (do_red || aux_mode != 0) {
        // Second pass over the STORED (bf16) chunk in a (row group, 8-channel group) layout: 16-byte smem accesses,
        // per-channel coefficients in registers.
        //   forward:  (sum v, sum v^2) of the valid rows -> BatchNorm batch statistics of the following layer
        //   aux 1:    g = v * (y > 0), written back in place
        //   aux 2:    g = v * (bn(z) > 0) written back, (sum g, sum g * xhat) -> dbeta / dgamma of that BatchNorm
        if (cj > 0) asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // scratch of the previous chunk read
        if (aux_mode != 0) {
          tc::mbar_wait(&aux_full_bar[wg], aux_n & 1);
          ++aux_n;
        }
        const bool bnred = aux_mode == 2;
        const int cg = wtid % CGc, rg = wtid / CGc;
        const int ch0 = p.n_off + ncol0 + chunk * OUT_CW + cg * 8;
        float s1[8], s2[8], mu[8], is[8], sc[8], sh[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s1[j] = s2[j] = mu[j] = is[j] = sc[j] = sh[j] = 0.f;
        if (bnred) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            mu[j] = __ldg(p.bn_mean + ch0 + j);
            is[j] = __ldg(p.bn_invstd + ch0 + j);
            sc[j] = __ldg(p.bn_gamma + ch0 + j) * is[j];       // same expressions as the forward's
            sh[j] = __ldg(p.bn_beta + ch0 + j) - mu[j] * sc[j];  // bn_train_coef (elementwise.cu)
          }
        }
        // rows rg*ROWSc .. +ROWSc-1; the swizzle term of row r depends only on rr (OUT_CW 64: r & 7 == rr; 32:
        // (r >> 1) & 3 == ((rg & 1) * 2 + (rr >> 1))), so every offset is base + compile-time pieces
        const uint32_t row0_off = (uint32_t)(rg * ROWSc) * OUT_ROW_BYTES;
        const int swz_rg = (OUT_CW == 64) ? 0 : (rg & 1) * 2;
#pragma unroll
        for (int rr = 0; rr < ROWSc; ++rr) {
          if (!tile_full && row_pix[rg * ROWSc + rr] < 0) continue;   // ragged tiles only
          const int unit = (OUT_CW == 64) ? (cg ^ rr) : (cg ^ (swz_rg + (rr >> 1)));
          const uint32_t off = row0_off + (uint32_t)rr * OUT_ROW_BYTES + (uint32_t)unit * 16;
          const uint4 pk = *reinterpret_cast<const uint4*>(cbuf + off);
          const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&pk);
          if (aux_mode == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 xy = __bfloat1622float2(h2[j]);
              s1[2 * j] += xy.x; s2[2 * j] += xy.x * xy.x;
              s1[2 * j + 1] += xy.y; s2[2 * j + 1] += xy.y * xy.y;
            }
          } else if (aux_mode == 1) {
            const uint4 ak = *reinterpret_cast<const uint4*>(abuf + off);
            const uint32_t w[4] = {ak.x, ak.y, ak.z, ak.w};
            uint32_t o[4] = {pk.x, pk.y, pk.z, pk.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              // bf16 > 0  <=>  sign bit clear and magnitude nonzero
              const uint32_t lo = w[e] & 0xFFFFu, hi2 = w[e] >> 16;
              if (!(lo != 0 && lo < 0x8000u)) o[e] &= 0xFFFF0000u;
              if (!(hi2 != 0 && hi2 < 0x8000u)) o[e] &= 0x0000FFFFu;
            }
            *reinterpret_cast<uint4*>(cbuf + off) = make_uint4(o[0], o[1], o[2], o[3]);
            if (do_red) {
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                s1[2 * e] += __uint_as_float(o[e] << 16);
                s1[2 * e + 1] += __uint_as_float(o[e] & 0xFFFF0000u);
              }
            }
          } else {
            const uint4 zk = *reinterpret_cast<const uint4*>(abuf + off);
            const __nv_bfloat162* z2 = reinterpret_cast<const __nv_bfloat162*>(&zk);
            uint32_t o[4] = {pk.x, pk.y, pk.z, pk.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float2 g = __bfloat1622float2(h2[j]);
              const float2 zz = __bfloat1622float2(z2[j]);
              if (!(fmaf(zz.x, sc[2 * j], sh[2 * j]) > 0.f)) { g.x = 0.f; o[j] &= 0xFFFF0000u; }
              if (!(fmaf(zz.y, sc[2 * j + 1], sh[2 * j + 1]) > 0.f)) { g.y = 0.f; o[j] &= 0x0000FFFFu; }
              s1[2 * j] += g.x; s2[2 * j] += g.x * ((zz.x - mu[2 * j]) * is[2 * j]);
              s1[2 * j + 1] += g.y; s2[2 * j + 1] += g.y * ((zz.y - mu[2 * j + 1]) * is[2 * j + 1]);
            }
            *reinterpret_cast<uint4*>(cbuf + off) = make_uint4(o[0], o[1], o[2], o[3]);
          }
        }
        if (aux_mode != 0) tc::fence_proxy_async_smem();  // the masked chunk is read by the TMA store below
        if (do_red) {
          // combine the row groups of this warp with shuffles (lanes l, l+CGc, ... share a channel group), then the
          // four warps through a small shared-memory table
#pragma unroll
          for (int off = CGc; off < 32; off <<= 1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              s1[j] += __shfl_xor_sync(0xffffffffu, s1[j], off);
              s2[j] += __shfl_xor_sync(0xffffffffu, s2[j], off);
            }
          }
          if (lane < CGc) {
            float4* scq = reinterpret_cast<float4*>(my_scratch + ((size_t)ww * CGc + lane) * 16);
            scq[0] = make_float4(s1[0], s2[0], s1[1], s2[1]);
            scq[1] = make_float4(s1[2], s2[2], s1[3], s2[3]);
            scq[2] = make_float4(s1[4], s2[4], s1[5], s2[5]);
            scq[3] = make_float4(s1[6], s2[6], s1[7], s2[7]);
          }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
        if (do_red && wtid < OUT_CW) {
          float a1 = 0.f, a2 = 0.f;
#pragma unroll
          for (int w4 = 0; w4 < 4; ++w4) {
            const float2 v2 = *reinterpret_cast<const float2*>(my_scratch + ((size_t)w4 * CGc + (wtid >> 3)) * 16 + (wtid & 7) * 2);
            a1 += v2.x;
            a2 += v2.y;
          }
#pragma unroll
          for (int j = 0; j < CH; ++j)
            if (j == cj) { racc1[j] += a1; racc2[j] += a2; }
        }
      }

      if (wtid == 0) {
        const CUtensorMap* mD = &p.tmD[phase_id];
        if (p.accumulate) tc::tma_reduce_add_4d(mD, cbuf, p.n_off + ncol0 + chunk * OUT_CW, x0, y0, n0);
        else tc::tma_store_4d(mD, cbuf, p.n_off + ncol0 + chunk * OUT_CW, x0, y0, n0);
        if (aux_mode != 0) {
          // abuf is free (every thread of the warpgroup passed the barrier after its last read): fetch the next chunk
          if (cj + 1 < my_chunks) issue_aux(t, chunk + 2);
          else if (t + (int)gridDim.x < total_tiles) issue_aux(t + (int)gridDim.x, wg);
        }
      }
    }
    if (wtid == 0 && my_chunks > 0) tc::tma_store_commit();   // one bulk group per tile (see the wait above)
  }
  if (do_red) flush_reductions();
  if (wtid == 0) tc::tma_store_wait_read0();
}

// -------------------------------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1) wgrad_kernel(const __grid_constant__ WgradParams p) {
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN");
  constexpr int KROWS = 64;                       // max pixel rows per K block
  constexpr int B_CW = (BN >= 64) ? 64 : 32;      // channels per B sub-tile row
  constexpr int B_ROW_BYTES = B_CW * 2;
  constexpr int B_SUB_BYTES = KROWS * B_ROW_BYTES;
  constexpr int B_SUBS = BN / B_CW;
  constexpr int B_BYTES = B_SUBS * B_SUB_BYTES;
  constexpr uint32_t B_LAYOUT = (B_CW == 64) ? tc::LAYOUT_SW128 : tc::LAYOUT_SW64;
  constexpr int A_SUB_BYTES = KROWS * 128;        // sized for the 64-channel case
  constexpr int A_BYTES = 2 * A_SUB_BYTES;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_up_1024(smem_raw);
  const int stages = p.stages;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)stages * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + stages;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);  // provably warp-uniform
  const int lane = threadIdx.x & 31;
  const int ncol0 = blockIdx.x * BN;       // cin tile
  const int m0 = blockIdx.y * 128;         // cout tile
  const int tap_id = blockIdx.z / p.splits;
  const int split = blockIdx.z % p.splits;
  const WgradTap tap = p.taps[tap_id];
  // K blocks (pixel tiles) of this split
  const int per = (p.tiles_total + p.splits - 1) / p.splits;
  const int kb_begin = split * per;
  const int kb_end = min(p.tiles_total, kb_begin + per);
  const int num_kb = max(0, kb_end - kb_begin);
  const int a_row_bytes = p.a_cw * 2;
  const uint32_t a_layout = (p.a_cw == 64) ? tc::LAYOUT_SW128 : tc::LAYOUT_SW64;
  // M = 128 output channels = one 64-row slice per MMA warpgroup; with <= 64 channels loaded the second one idles
  const int mma_wgs = (p.a_chunks * p.a_cw > 64) ? 2 : 1;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < stages; ++s) {
      tc::mbar_init(&full_bar[s], 1);
      tc::mbar_init(&empty_bar[s], mma_wgs);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();
  pdl_prologue();  // everything above touched only shared memory / kernel parameters
  if (num_kb == 0) return;

  if (warp < 4) {
    tc::regs_dealloc<kProducerRegs>();
    if (warp != 0) return;
    const CUtensorMap* mA = &p.tmA[tap.srcA];
    const CUtensorMap* mB = &p.tmB[tap.srcB];
    const uint32_t tx_bytes = (uint32_t)p.rows * (uint32_t)(a_row_bytes * p.a_chunks + B_ROW_BYTES * B_SUBS);
    int ring_s = 0;
    uint32_t ring_ph = 0;
    // pixel-tile coordinates advance incrementally (no integer division inside the single-thread issue loop)
    int tx = kb_begin % p.tiles_x;
    int ty = (kb_begin / p.tiles_x) % p.tiles_y;
    int tn = kb_begin / (p.tiles_x * p.tiles_y);
    for (int i = 0; i < num_kb; ++i) {
      const int s = ring_s;
      const uint32_t ph = ring_ph;
      if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
      const int x0 = tx * p.bw, y0 = ty * p.bh, n0 = tn * p.bn;
      if (++tx == p.tiles_x) { tx = 0; if (++ty == p.tiles_y) { ty = 0; ++tn; } }
      tc::mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* sa = smem + (size_t)s * STAGE_BYTES;
      uint8_t* sb = sa + A_BYTES;
      if (tc::elect_one()) {
        tc::mbar_expect_tx(&full_bar[s], tx_bytes);
        for (int j = 0; j < p.a_chunks; ++j)
          tc::tma_load_4d(sa + j * A_SUB_BYTES, mA, &full_bar[s], m0 + j * p.a_cw, x0 + tap.ax, y0 + tap.ay, n0);
#pragma unroll
        for (int j = 0; j < B_SUBS; ++j)
          tc::tma_load_4d(sb + j * B_SUB_BYTES, mB, &full_bar[s], ncol0 + j * B_CW, x0 + tap.bx, y0 + tap.by, n0);
      }
    }
    return;
  }

  tc::regs_alloc<kMmaRegs>();
  const int wg = (warp >> 2) - 1;
  if (wg >= mma_wgs) return;
  const int wtid = threadIdx.x & 127;
  const int ksteps = p.rows / 16;
  // A (MN-major): this warpgroup's 64 output channels are A sub-tile wg.  With 32-channel chunks (a single chunk) the
  // second 32-wide swizzle atom of the 64-row slice points at the unused sub-tile 1; those rows are never stored.
  const uint32_t a_off = (uint32_t)(wg * A_SUB_BYTES);
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int ring_s = 0;
  uint32_t ring_ph = 0;
  int prev_s = -1;
  for (int i = 0; i < num_kb; ++i) {
    const int s = ring_s;
    const uint32_t ph = ring_ph;
    if (++ring_s == stages) { ring_s = 0; ring_ph ^= 1; }
    tc::mbar_wait(&full_bar[s], ph);
    const uint32_t sa = tc::smem_u32(smem + (size_t)s * STAGE_BYTES);
    const uint32_t sb = sa + A_BYTES;
    const uint64_t da0 = tc::make_smem_desc(sa + a_off, A_SUB_BYTES, 8 * a_row_bytes, a_layout);
    const uint64_t db0 = tc::make_smem_desc(sb, B_SUB_BYTES, 8 * B_ROW_BYTES, B_LAYOUT);
    tc::wgmma_fence();
    for (int k = 0; k < ksteps; ++k) {
      const uint64_t da = da0 + (uint64_t)((k * 16 * a_row_bytes) >> 4);
      const uint64_t db = db0 + (uint64_t)((k * 16 * B_ROW_BYTES) >> 4);
      tc::wgmma_bf16<BN, 1, 1>(acc, da, db, (i > 0 || k > 0) ? 1u : 0u);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<1>();
    if (prev_s >= 0 && wtid == 0) tc::mbar_arrive(&empty_bar[prev_s]);
    prev_s = s;
  }
  tc::wgmma_wait<0>();
  tc::fence_acc(acc);
  if (wtid == 0) tc::mbar_arrive(&empty_bar[prev_s]);

  // the 64 x BN partial product (rows = output channels, columns = input channels): with one split, the only
  // contribution to these weight-gradient elements, added in place; with several, stored into this split's row of
  // g_wgrad_red and summed in split order by wgrad_red_finish_kernel
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + (wtid >> 5) * 16 + (lane >> 2) + 8 * h;
    const int co = m0 + m;
    if (m >= p.a_chunks * p.a_cw || co >= p.cout) continue;
    if (p.splits > 1) {
      float* prow = g_wgrad_red + p.ws_off + (size_t)split * p.slice + ((size_t)tap.wtap * p.cout + co) * p.cin_src + ncol0 +
                    2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        *reinterpret_cast<float2*>(prow + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      continue;
    }
    float* drow = p.dw + ((size_t)tap.wtap * p.cout + co) * p.cin_total + p.ci_off + ncol0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(drow + 8 * j), "f"(acc[4 * j + 2 * h]),
                   "f"(acc[4 * j + 2 * h + 1])
                   : "memory");
  }
}

}  // namespace mcb
