// evaluation.cu — the per-pair and per-image work of the COCO segmentation evaluation (src/cocoeval.py, driven by
// src/utils.py:308-321 and the validation callback src/callbacks.py:133-151):
//   * mask IoU of (detection, ground truth) pairs from their column-major COCO run lists (pycocotools rleIou, called
//     as maskUtils.iou(d, g, iscrowd) at src/cocoeval.py:196);
//   * COCOeval.evaluateImg (src/cocoeval.py:242-320): the greedy matching of score-ordered detections to ground truths,
//     one warp per (image, area range), one lane per IoU threshold.
// Every output element is written by exactly one thread; nothing is accumulated in completion order.
#include "host_common.h"
#include "../../include/mcb200.h"

namespace mcb {

// ------------------------------------------------------------------------------------------ rleIou
// One thread per listed pair.  The run lists of label-map instances are short (about two runs per bounding-box column),
// and the merge of two lists is a serial walk, so a thread per pair keeps every lane busy where a warp per pair would
// leave most lanes idle.  The walk is pycocotools' rleIou loop verbatim (unsigned 32-bit counters).
__global__ void rle_pair_iou_kernel(const uint32_t* __restrict__ dt_cnts, const long long* __restrict__ dt_starts,
                                    const uint32_t* __restrict__ gt_cnts, const long long* __restrict__ gt_starts,
                                    const uint8_t* __restrict__ gt_crowd, const int* __restrict__ pair_dt,
                                    const int* __restrict__ pair_gt, const long long* __restrict__ pair_out,
                                    double* __restrict__ iou, int npairs) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  const int d = pair_dt[p], g = pair_gt[p];
  const uint32_t* A = dt_cnts + dt_starts[d];
  const uint32_t* B = gt_cnts + gt_starts[g];
  const long ka = (long)(dt_starts[d + 1] - dt_starts[d]), kb = (long)(gt_starts[g + 1] - gt_starts[g]);
  uint32_t ca = A[0], cb = B[0], i = 0, u = 0, ct = 1;
  long a = 1, b = 1;
  bool va = false, vb = false;
  while (ct > 0) {
    const uint32_t c = min(ca, cb);
    if (va || vb) {
      u += c;
      if (va && vb) i += c;
    }
    ct = 0;
    ca -= c;
    if (!ca && a < ka) { ca = A[a++]; va = !va; }
    ct += ca;
    cb -= c;
    if (!cb && b < kb) { cb = B[b++]; vb = !vb; }
    ct += cb;
  }
  if (i == 0) {
    u = 1;
  } else if (gt_crowd[g]) {  // crowd ground truth: the union is the detection's area (rleArea)
    u = 0;
    for (long j = 1; j < ka; j += 2) u += A[j];
  }
  iou[pair_out[p]] = (double)i / (double)u;
}

// ------------------------------------------------------------------------------------------ evaluateImg
// Task = (unit, area range), unit = one (image, category) of the evaluation.  Ground truths are visited in the order of
// the stable sort by `_ignore`: the non-ignored ones in their own order, then the ignored ones.  The sweep of lane t
// reads the IoU row of each detection (the same address in every lane: one broadcast) and its own matched-flag row.
__global__ void coco_match_kernel(const double* __restrict__ iou, const long long* __restrict__ iou_off,
                                  const int* __restrict__ nd, const int* __restrict__ ng,
                                  const long long* __restrict__ dt_off, const long long* __restrict__ dt_id,
                                  const double* __restrict__ dt_area, const long long* __restrict__ gt_off,
                                  const long long* __restrict__ gt_id, const uint8_t* __restrict__ gt_crowd,
                                  const double* __restrict__ gt_area, const double* __restrict__ area_rng,
                                  const double* __restrict__ thr, int units, int A, int T, long long d_total,
                                  long long g_total, long long* __restrict__ dt_match, uint8_t* __restrict__ dt_ignore,
                                  uint8_t* __restrict__ gt_ignore, uint8_t* __restrict__ gt_taken) {
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= (long)units * A) return;
  const int unit = (int)(warp / A), a = (int)(warp % A);
  const int D = nd[unit], G = ng[unit];
  const long long d0 = dt_off[unit], g0 = gt_off[unit];
  const double lo = area_rng[2 * a], hi = area_rng[2 * a + 1];
  auto ignored = [&](int g) -> bool {
    const double ar = gt_area[g0 + g];
    return gt_crowd[g0 + g] || ar < lo || ar > hi;
  };
  int n_kept = 0;
  for (int g = 0; g < G; ++g) n_kept += !ignored(g);
  for (int j = lane; j < G; j += 32) gt_ignore[(long long)a * g_total + g0 + j] = j >= n_kept;
  if (lane >= T) return;
  const double t = fmin(thr[lane], 1 - 1e-10);
  uint8_t* taken = gt_taken + ((long long)a * T + lane) * g_total + g0;
  const double* tab = iou + iou_off[unit];
  long long* out_m = dt_match + ((long long)a * T + lane) * d_total + d0;
  uint8_t* out_ig = dt_ignore + ((long long)a * T + lane) * d_total + d0;
  for (int d = 0; d < D; ++d) {
    double best = t;
    int m = -1;
    bool m_ig = false;
    for (int pass = 0; pass < 2; ++pass) {
      if (pass == 1 && m > -1 && !m_ig) break;  // matched a regular ground truth: the ignored ones are not tried
      for (int g = 0; g < G; ++g) {
        const bool ig = ignored(g);
        if (ig != (pass == 1)) continue;
        if (taken[g] && !gt_crowd[g0 + g]) continue;
        const double v = tab[(long)d * G + g];
        if (v < best) continue;
        best = v;
        m = g;
        m_ig = ig;
      }
    }
    long long match = 0;
    bool dig = false;
    if (m > -1) {
      match = gt_id[g0 + m];
      dig = m_ig;
      if (dt_id[d0 + d] > 0) taken[m] = 1;  // gtm holds the detection id; the sweep tests gtm > 0
    }
    // unmatched detections outside the area range are ignored; "unmatched" tests the stored id, so a match to a ground
    // truth with id 0 counts as unmatched here and in accumulate
    const double ar = dt_area[d0 + d];
    out_m[d] = match;
    out_ig[d] = dig || (match == 0 && (ar < lo || ar > hi));
  }
}

// ------------------------------------------------------------------------------------------ get_iou
// Row r of a ragged IoU table (one instance against the ground truths of its image and category) reduces to its
// maximum, NaN for a row without ground truths (the reference's `None`).  One thread per row: rows are a few dozen
// entries, and the maximum of non-NaN values does not depend on the visiting order.
__global__ void iou_row_max_kernel(const double* __restrict__ iou, const long long* __restrict__ row_off, int rows,
                                   double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const long long b = row_off[r], e = row_off[r + 1];
  double m = b < e ? iou[b] : __longlong_as_double(0x7FF8000000000000LL);
  for (long long j = b + 1; j < e; ++j) m = fmax(m, iou[j]);
  out[r] = m;
}

}  // namespace mcb

using namespace mcb;
#define ST ((cudaStream_t)stream)

extern "C" int mcb_rle_pair_iou(const uint32_t* dt_cnts, const long long* dt_starts, const uint32_t* gt_cnts,
                                const long long* gt_starts, const uint8_t* gt_crowd, const int* pair_dt,
                                const int* pair_gt, const long long* pair_out, double* iou, int npairs, void* stream) {
  if (npairs <= 0) return MCB_OK;
  MCB_REQUIRE(dt_cnts && dt_starts && gt_cnts && gt_starts && gt_crowd && pair_dt && pair_gt && pair_out && iou,
              "rle_pair_iou: null pointer");
  rle_pair_iou_kernel<<<(npairs + 127) / 128, 128, 0, ST>>>(dt_cnts, dt_starts, gt_cnts, gt_starts, gt_crowd, pair_dt,
                                                            pair_gt, pair_out, iou, npairs);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_iou_row_max(const double* iou, const long long* row_off, int rows, double* out, void* stream) {
  MCB_REQUIRE(rows >= 0, "iou_row_max: negative row count %d", rows);
  if (rows == 0) return MCB_OK;
  MCB_REQUIRE(iou && row_off && out, "iou_row_max: null pointer");
  iou_row_max_kernel<<<(rows + 127) / 128, 128, 0, ST>>>(iou, row_off, rows, out);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_coco_match(const double* iou, const long long* iou_off, const int* nd, const int* ng,
                              const long long* dt_off, const long long* dt_id, const double* dt_area,
                              const long long* gt_off, const long long* gt_id, const uint8_t* gt_crowd,
                              const double* gt_area, const double* area_rng, const double* thr, int units, int A, int T,
                              long long d_total, long long g_total, long long* dt_match, uint8_t* dt_ignore,
                              uint8_t* gt_ignore, uint8_t* gt_taken, void* stream) {
  if (units <= 0 || A <= 0) return MCB_OK;
  MCB_REQUIRE(T >= 1 && T <= 32, "coco_match: 1..32 IoU thresholds (one lane each), got %d", T);
  MCB_REQUIRE(iou_off && nd && ng && dt_off && gt_off && area_rng && thr, "coco_match: null pointer");
  MCB_REQUIRE(d_total == 0 || (dt_id && dt_area && dt_match && dt_ignore), "coco_match: null detection table");
  MCB_REQUIRE(g_total == 0 || (gt_id && gt_crowd && gt_area && gt_ignore && gt_taken), "coco_match: null ground truth");
  const long warps = (long)units * A;
  const int warps_per_block = 4;
  coco_match_kernel<<<(unsigned)((warps + warps_per_block - 1) / warps_per_block), 32 * warps_per_block, 0, ST>>>(
      iou, iou_off, nd, ng, dt_off, dt_id, dt_area, gt_off, gt_id, gt_crowd, gt_area, area_rng, thr, units, A, T,
      d_total, g_total, dt_match, dt_ignore, gt_ignore, gt_taken);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
