// watershed.cu — marker-based watershed on the relief -prob (4-connectivity).  NOT a reference function (SURVEY 0.4:
// `grep -ri watershed` finds nothing in the reference); named by BASELINE.json's north_star.  PARITY UNPINNED: the
// semantics are DEFINED by oracle/post_oracle.py::minimax_watershed, chosen so that every relaxation schedule reaches
// the same fixed point (three monotone stages), which is what makes a parallel implementation bit-exact against it:
//   level(p) = clip(floor((1 - prob(p)) * (levels - 1)))
//   1. cost(p)  = min over marker->p paths inside the mask of the max level on the path (markers: 0)
//   2. dist(p)  = fewest steps along tight moves q->p  (cost(p) == max(cost(q), level(p)))
//   3. label(p) = smallest marker label reachable through tight moves that decrease dist by exactly one
// One CTA per plane (planes are independent -> no grid-wide sync): the CTA sweeps its 32x32 tiles, relaxing each tile to
// a local fixed point in shared memory (1-pixel halo), alternating sweep direction, until a whole sweep changes nothing.
#include "host_common.h"
#include "../../include/mcb200.h"

namespace mcb {

constexpr int WS_T = 32;
constexpr int WS_INF = 0x3fffffff;          // cost / dist: unreached
constexpr unsigned WS_NO_LABEL = 0xffffffffu; // label stage: unreached.  Labels are compared as unsigned, so every
                                              // positive int32 marker label (up to 2^31 - 1) sorts below it
constexpr int WS_MAX_TILES = 1024;   // tile-activity table in shared memory (larger planes sweep every tile)

template <int STAGE>
__device__ void ws_stage(const int* __restrict__ lev, int* __restrict__ cost, int* __restrict__ dist,
                         int* __restrict__ lab, const int* __restrict__ markers, const uint8_t* __restrict__ mask, int H,
                         int W, const unsigned char* __restrict__ tile_on) {
  __shared__ int s_var[WS_T + 2][WS_T + 2];   // the variable being relaxed in this stage
  __shared__ int s_cost[WS_T + 2][WS_T + 2];  // stage >= 2
  __shared__ int s_dist[WS_T + 2][WS_T + 2];  // stage 3
  __shared__ int s_flag;
  int* var = STAGE == 1 ? cost : (STAGE == 2 ? dist : lab);
  const int var_inf = STAGE == 3 ? (int)WS_NO_LABEL : WS_INF;
  // stages 1-2 relax signed costs / distances, stage 3 relaxes labels as unsigned values (see WS_NO_LABEL)
  auto less = [](int a, int b) { return STAGE == 3 ? (unsigned)a < (unsigned)b : a < b; };
  const int tx = threadIdx.x % WS_T, ty = threadIdx.x / WS_T;
  const int tiles_x = (W + WS_T - 1) / WS_T, tiles_y = (H + WS_T - 1) / WS_T;
  const int ntiles = tiles_x * tiles_y;
  for (int sweep = 0;; ++sweep) {
    int sweep_changed = 0;
    for (int ti = 0; ti < ntiles; ++ti) {
      const int t = (sweep & 1) ? (ntiles - 1 - ti) : ti;
      if (tile_on != nullptr && !tile_on[t]) continue;   // no mask / marker pixel in this tile: nothing can change
      const int x0 = (t % tiles_x) * WS_T, y0 = (t / tiles_x) * WS_T;
      // stage the tile + halo
      for (int i = threadIdx.x; i < (WS_T + 2) * (WS_T + 2); i += blockDim.x) {
        const int sy = i / (WS_T + 2), sx = i % (WS_T + 2);
        const int y = y0 + sy - 1, x = x0 + sx - 1;
        const bool in = (y >= 0 && y < H && x >= 0 && x < W);
        const long p = (long)y * W + x;
        s_var[sy][sx] = in ? var[p] : var_inf;
        if (STAGE >= 2) s_cost[sy][sx] = in ? cost[p] : WS_INF;
        if (STAGE == 3) s_dist[sy][sx] = in ? dist[p] : WS_INF;
      }
      __syncthreads();
      const int x = x0 + tx, y = y0 + ty;
      const bool inside = (x < W && y < H);
      const long p = (long)y * W + x;
      bool active = false;
      int lv = 0, my_cost = WS_INF, my_dist = WS_INF;
      if (inside) {
        const bool is_m = markers[p] > 0;
        active = (mask[p] != 0 || is_m) && !is_m;
        lv = lev[p];
        if (STAGE >= 2) { my_cost = s_cost[ty + 1][tx + 1]; active = active && my_cost < WS_INF; }
        if (STAGE == 3) { my_dist = s_dist[ty + 1][tx + 1]; active = active && my_dist < WS_INF; }
      }
      bool tile_changed = false;
      for (int it = 0; it < 4 * WS_T; ++it) {
        int nv = s_var[ty + 1][tx + 1];
        if (active) {
          const int ny[4] = {ty, ty + 2, ty + 1, ty + 1}, nx[4] = {tx + 1, tx + 1, tx, tx + 2};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (STAGE == 1) {
              const int c = s_var[ny[k]][nx[k]];
              nv = min(nv, max(c, lv));
            } else {
              const int cq = s_cost[ny[k]][nx[k]];
              const bool tight = cq < WS_INF && max(cq, lv) == my_cost;
              if (STAGE == 2) {
                if (tight) nv = min(nv, s_var[ny[k]][nx[k]] + (s_var[ny[k]][nx[k]] < WS_INF ? 1 : 0));
              } else {
                if (tight && s_dist[ny[k]][nx[k]] + 1 == my_dist && less(s_var[ny[k]][nx[k]], nv)) nv = s_var[ny[k]][nx[k]];
              }
            }
          }
        }
        const bool ch = active && less(nv, s_var[ty + 1][tx + 1]);
        const int any = __syncthreads_or(ch ? 1 : 0);
        if (ch) s_var[ty + 1][tx + 1] = nv;
        if (!any) break;
        tile_changed = true;
        __syncthreads();
      }
      if (tile_changed) {
        if (inside) var[p] = s_var[ty + 1][tx + 1];
        sweep_changed = 1;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) s_flag = sweep_changed;
    __syncthreads();
    const int f = s_flag;
    __syncthreads();
    if (!f) break;
  }
}

template <typename T>
__global__ void __launch_bounds__(WS_T* WS_T) watershed_kernel(const T* __restrict__ prob, const int* __restrict__ markers,
                                                             const uint8_t* __restrict__ mask, int* __restrict__ out,
                                                             int* __restrict__ work, int H, int W, int levels) {
  const long hw = (long)H * W;
  const long base = (long)blockIdx.x * hw;
  int* lev = work + (long)blockIdx.x * 3 * hw;
  int* cost = lev + hw;
  int* dist = cost + hw;
  int* lab = out + base;
  const int* mk = markers + base;
  const uint8_t* ms = mask + base;
  for (long i = threadIdx.x; i < hw; i += blockDim.x) {
    const double v = floor((1.0 - (double)prob[base + i]) * (double)(levels - 1));
    const int l = v < 0.0 ? 0 : (v > (double)(levels - 1) ? levels - 1 : (int)v);
    const int m = mk[i];
    lev[i] = l;
    cost[i] = m > 0 ? 0 : WS_INF;
    dist[i] = m > 0 ? 0 : WS_INF;
    lab[i] = m > 0 ? m : (int)WS_NO_LABEL;
  }
  __syncthreads();
  // tiles without a single mask / marker pixel never hold an active pixel in any stage: mark them once, skip them in
  // every sweep (building maps cover ~20 % of a tile map)
  __shared__ unsigned char s_tile_on[WS_MAX_TILES];
  const int tiles_x = (W + WS_T - 1) / WS_T, tiles_y = (H + WS_T - 1) / WS_T;
  const unsigned char* tile_on = nullptr;
  if (tiles_x * tiles_y <= WS_MAX_TILES) {
    const int tx = threadIdx.x % WS_T, ty = threadIdx.x / WS_T;
    for (int t = 0; t < tiles_x * tiles_y; ++t) {
      const int x = (t % tiles_x) * WS_T + tx, y = (t / tiles_x) * WS_T + ty;
      const bool on = (x < W && y < H) && (ms[(long)y * W + x] != 0 || mk[(long)y * W + x] > 0);
      const int any = __syncthreads_or(on ? 1 : 0);
      if (threadIdx.x == 0) s_tile_on[t] = (unsigned char)(any != 0);
    }
    __syncthreads();
    tile_on = s_tile_on;
  }
  ws_stage<1>(lev, cost, dist, lab, mk, ms, H, W, tile_on);
  __syncthreads();
  ws_stage<2>(lev, cost, dist, lab, mk, ms, H, W, tile_on);
  __syncthreads();
  ws_stage<3>(lev, cost, dist, lab, mk, ms, H, W, tile_on);
  __syncthreads();
  for (long i = threadIdx.x; i < hw; i += blockDim.x)
    if (lab[i] == (int)WS_NO_LABEL) lab[i] = 0;
}

}  // namespace mcb

using namespace mcb;

extern "C" int mcb_watershed(const void* prob, int prob_is_f64, const int* markers, const uint8_t* mask, int* labels,
                             int* workspace, int planes, int h, int w, int levels, void* stream) {
  MCB_REQUIRE(prob && markers && mask && labels && workspace, "watershed: null pointer");
  MCB_REQUIRE(levels >= 2 && levels <= 65536, "watershed: levels %d", levels);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (prob_is_f64)
    watershed_kernel<double><<<planes, WS_T * WS_T, 0, st>>>((const double*)prob, markers, mask, labels, workspace, h, w, levels);
  else
    watershed_kernel<float><<<planes, WS_T * WS_T, 0, st>>>((const float*)prob, markers, mask, labels, workspace, h, w, levels);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
