// forest.cu — prediction of the second-level scoring model's tree ensembles (src/models.py:212-282): a RandomForest
// (sklearn's ForestRegressor.predict) or a LightGBM booster (GBDT::Predict over Tree::NumericalDecision), both
// flattened into one node format by mcb200.forest.
//
// Two kernels per chunk of trees:
//   * traverse: one thread per (tree, row) pair of the chunk writes that tree's leaf value to buf[tree][row];
//   * accumulate: one thread per row adds the chunk's leaf values in tree order to the row's running float64 sum, and
//     after the last chunk divides by the tree count when the forest averages.
// The sum of every row is 0.0 + leaf(tree 0) + leaf(tree 1) + ... in tree order, exactly the loop of both libraries, so
// the result is bit-exact.  No atomics; nothing depends on completion order.
#include "host_common.h"
#include "../../include/mcb200.h"

namespace mcb {

// LightGBM's kZeroThreshold (include/LightGBM/meta.h): a double initialised from the float literal 1e-35f
__device__ __forceinline__ double lgbm_zero_threshold() { return (double)1e-35f; }

template <int SEMANTICS>
__device__ __forceinline__ bool goes_left(double x, double threshold, uint8_t flags) {
  if (SEMANTICS == MCB_FOREST_SKLEARN) {
    // sklearn casts the features to float32 (check_array(dtype=DTYPE)) and compares against the float64 threshold;
    // NaN follows missing_go_to_left (Tree._apply_dense)
    const float v = (float)x;
    if (isnan(v)) return flags & MCB_FOREST_DEFAULT_LEFT;
    return (double)v <= threshold;
  } else {
    // the C API's dense rows drop |x| <= kZeroThreshold, so such a value reaches the tree as 0.0; then
    // Tree::NumericalDecision
    const double kz = lgbm_zero_threshold();
    double v = fabs(x) <= kz ? 0.0 : x;
    const int missing = (flags >> 2) & 3;
    if (isnan(v) && missing != MCB_FOREST_MISSING_NAN) v = 0.0;
    if ((missing == MCB_FOREST_MISSING_ZERO && v >= -kz && v <= kz) || (missing == MCB_FOREST_MISSING_NAN && isnan(v)))
      return flags & MCB_FOREST_DEFAULT_LEFT;
    return v <= threshold;
  }
}

template <int SEMANTICS>
__global__ void __launch_bounds__(256) forest_traverse_kernel(const double* __restrict__ x, int rows, int n_features,
                                                              const int* __restrict__ tree_root, int tree0, int trees,
                                                              const int* __restrict__ feature,
                                                              const double* __restrict__ threshold,
                                                              const int* __restrict__ left,
                                                              const int* __restrict__ right,
                                                              const uint8_t* __restrict__ flags,
                                                              const double* __restrict__ leaf_value,
                                                              double* __restrict__ buf) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)trees * rows) return;
  const int t = (int)(i / rows), r = (int)(i - (long long)t * rows);
  const double* xr = x + (long long)r * n_features;
  int n = tree_root[tree0 + t];
  while (n >= 0) n = goes_left<SEMANTICS>(xr[feature[n]], threshold[n], flags[n]) ? left[n] : right[n];
  buf[i] = leaf_value[~n];
}

__global__ void __launch_bounds__(256) forest_accumulate_kernel(const double* __restrict__ buf, int rows, int trees,
                                                                int first, int last_divisor, double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  double s = first ? 0.0 : out[r];
  for (int t = 0; t < trees; ++t) s += buf[(long long)t * rows + r];
  out[r] = last_divisor > 0 ? s / (double)last_divisor : s;
}

}  // namespace mcb

using namespace mcb;
#define ST ((cudaStream_t)stream)

extern "C" int mcb_forest_predict(const double* x, int rows, int n_features, const int* tree_root, int n_trees,
                                  const int* feature, const double* threshold, const int* left, const int* right,
                                  const uint8_t* flags, const double* leaf_value, int semantics, int average,
                                  double* work, int chunk_trees, double* out, void* stream) {
  MCB_REQUIRE(rows >= 0 && n_features >= 1 && n_trees >= 1, "forest_predict: rows %d, features %d, trees %d", rows,
              n_features, n_trees);
  MCB_REQUIRE(semantics == MCB_FOREST_SKLEARN || semantics == MCB_FOREST_LIGHTGBM,
              "forest_predict: unknown semantics %d", semantics);
  MCB_REQUIRE(chunk_trees >= 1, "forest_predict: chunk_trees %d", chunk_trees);
  if (rows == 0) return MCB_OK;
  MCB_REQUIRE(x && tree_root && feature && threshold && left && right && flags && leaf_value && work && out,
              "forest_predict: null pointer");
  for (int t0 = 0; t0 < n_trees; t0 += chunk_trees) {
    const int cnt = n_trees - t0 < chunk_trees ? n_trees - t0 : chunk_trees;
    const long long pairs = (long long)cnt * rows;
    const unsigned blocks = (unsigned)((pairs + 255) / 256);
    if (semantics == MCB_FOREST_SKLEARN)
      forest_traverse_kernel<MCB_FOREST_SKLEARN><<<blocks, 256, 0, ST>>>(x, rows, n_features, tree_root, t0, cnt,
                                                                         feature, threshold, left, right, flags,
                                                                         leaf_value, work);
    else
      forest_traverse_kernel<MCB_FOREST_LIGHTGBM><<<blocks, 256, 0, ST>>>(x, rows, n_features, tree_root, t0, cnt,
                                                                          feature, threshold, left, right, flags,
                                                                          leaf_value, work);
    MCB_LAUNCH_CHECK();
    const bool last = t0 + cnt >= n_trees;
    forest_accumulate_kernel<<<(rows + 255) / 256, 256, 0, ST>>>(work, rows, cnt, t0 == 0,
                                                                  last && average ? n_trees : 0, out);
    MCB_LAUNCH_CHECK();
  }
  return MCB_OK;
}
