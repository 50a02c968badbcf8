"""TEST INFRASTRUCTURE — numpy restatement of the tree-ensemble prediction of the second-level scoring model
(src/models.py:212-282) over the flattened forest of mcb200.forest.  Only tests/ and scripts/ import this file.

Order: per row, 0.0 plus the trees' leaf values in tree order in float64 (`out += leaf` one tree at a time is that
per-row loop), then division by the tree count when the forest averages.  That is sklearn's ForestRegressor.predict at
n_jobs=1 (`y_hat += prediction` per estimator under its lock, then `y_hat /= len(self.estimators_)`) and LightGBM's
GBDT::PredictRaw loop (`output[k] += models_[i]->Predict(features)`, then `/= num_iteration_for_pred_` when
average_output).

Split rules:
  * sklearn (sklearn/tree/_tree.pyx, Tree._apply_dense): X is cast to float32 by check_array(dtype=DTYPE); at a node,
    a NaN goes left if missing_go_to_left, else right; otherwise left iff x <= threshold (float32 against float64).
  * LightGBM (include/LightGBM/tree.h, Tree::NumericalDecision, and the C API's dense-row path in c_api.cpp):
      - the C API keeps a dense value only when fabs(x) > kZeroThreshold or x is NaN, into a zeroed buffer, so
        |x| <= kZeroThreshold reaches the tree as 0.0 (kZeroThreshold = 1e-35f, a float widened to double);
      - missing_type = (decision_type >> 2) & 3 (0 None, 1 Zero, 2 NaN); a NaN under a type other than NaN becomes
        0.0;
      - a zero (IsZero: -kZeroThreshold <= x <= kZeroThreshold) under Zero, or a NaN under NaN, goes left if
        decision_type & 2 (kDefaultLeftMask), else right;
      - otherwise left iff x <= threshold;
      - a tree with num_leaves = 1 returns leaf_value[0] (its root is a leaf).
"""
import numpy as np

SKLEARN, LIGHTGBM = 0, 1
DEFAULT_LEFT = 2
K_ZERO_THRESHOLD = float(np.float32(1e-35))


def _goes_left(semantics, v, threshold, flags):
    default_left = (flags & DEFAULT_LEFT) != 0
    if semantics == SKLEARN:
        return np.where(np.isnan(v), default_left, v <= threshold)
    with np.errstate(invalid="ignore"):
        v = np.where(np.abs(v) <= K_ZERO_THRESHOLD, 0.0, v)
        missing = (flags >> 2) & 3
        v = np.where(np.isnan(v) & (missing != 2), 0.0, v)
        default = ((missing == 1) & (v >= -K_ZERO_THRESHOLD) & (v <= K_ZERO_THRESHOLD)) | ((missing == 2) & np.isnan(v))
        return np.where(default, default_left, v <= threshold)


def tree_leaves(forest, x, t):
    """leaf value of tree t for every row of x (already in the library's input precision)"""
    rows = x.shape[0]
    node = np.full(rows, int(forest.tree_root[t]), np.int64)
    active = np.nonzero(node >= 0)[0]
    while active.size:
        n = node[active]
        go = _goes_left(forest.semantics, x[active, forest.feature[n]], forest.threshold[n], forest.flags[n])
        node[active] = np.where(go, forest.left[n], forest.right[n])
        active = active[node[active] >= 0]
    return forest.leaf_value[~node]


def predict(forest, x):
    """float64 [rows] for x [rows][n_features]; `forest` is anything with mcb200.forest.Forest's arrays"""
    x = np.asarray(x, np.float64)
    if forest.semantics == SKLEARN:
        x = x.astype(np.float32).astype(np.float64)     # float32 widens exactly: the comparison is float vs double
    out = np.zeros(x.shape[0], np.float64)
    for t in range(forest.tree_root.size):
        out += tree_leaves(forest, x, t)
    if forest.average:
        out /= forest.tree_root.size
    return out


# ---------------------------------------------------------------------------------------------------------------------
# seeded LightGBM-format forests
# ---------------------------------------------------------------------------------------------------------------------
def random_tree_text(rs, index, n_features, leaves, max_depth):
    """one `Tree=` block with `leaves` leaves and depth <= max_depth, splits on random features with random
    decision_type (default-left and missing type None / Zero / NaN), thresholds drawn from {0, +-1e-36, +-1e-35f, N(0, 1)}"""
    # grow by splitting a random leaf that is still shallower than max_depth; LightGBM numbers internal nodes in
    # creation order and a split leaf keeps its index for the left child (Tree::Split)
    split_feature, threshold, decision, left, right = [], [], [], [], []
    leaf_parent, leaf_depth = [-1], [0]            # per leaf: parent node (-1 = root), depth
    leaf_side = [0]
    cand = [0] if max_depth > 0 else []          # leaves shallower than max_depth
    for node in range(leaves - 1):
        ci = rs.randint(len(cand))
        k = cand[ci]
        p = leaf_parent[k]
        if p >= 0:
            (left if leaf_side[k] == 0 else right)[p] = node
        split_feature.append(int(rs.randint(n_features)))
        c = rs.randint(6)
        threshold.append([0.0, 1e-36, -1e-36, K_ZERO_THRESHOLD, float(rs.randn()), float(rs.randn())][c])
        decision.append(int(rs.choice([0, 2])) | (int(rs.randint(3)) << 2))
        new = len(leaf_depth)
        left.append(~k)
        right.append(~new)
        d = leaf_depth[k] + 1
        leaf_parent[k], leaf_side[k], leaf_depth[k] = node, 0, d
        leaf_parent.append(node)
        leaf_side.append(1)
        leaf_depth.append(d)
        if d < max_depth:
            cand.append(new)
        else:
            cand[ci] = cand[-1]
            cand.pop()
    values = rs.randn(leaves) * 0.01
    fmt = " ".join
    return "\n".join([
        "Tree=%d" % index, "num_leaves=%d" % leaves, "num_cat=0",
        "split_feature=" + fmt(str(v) for v in split_feature),
        "split_gain=" + fmt("1" for _ in split_feature),
        "threshold=" + fmt(repr(v) for v in threshold),
        "decision_type=" + fmt(str(v) for v in decision),
        "left_child=" + fmt(str(v) for v in left),
        "right_child=" + fmt(str(v) for v in right),
        "leaf_value=" + fmt(repr(float(v)) for v in values),
        "is_linear=0", "shrinkage=0.01", "", ""])


def model_text(trees, n_features, average=False, objective="regression", num_class=1):
    """a LightGBM text model around `Tree=` blocks (as Booster.model_to_string writes it)"""
    head = ["tree", "version=v4", "num_class=%d" % num_class, "num_tree_per_iteration=1", "label_index=0",
            "max_feature_idx=%d" % (n_features - 1), "objective=%s" % objective]
    if average:
        head.append("average_output")
    head += ["feature_names=" + " ".join("f%d" % i for i in range(n_features)),
             "feature_infos=" + " ".join("[-1:1]" for _ in range(n_features)), "tree_sizes=0", ""]
    return "\n".join(head) + "\n" + "\n".join(trees) + "\nend of trees\n\nparameters:\nend of parameters\n"


def random_lightgbm_model(seed, n_trees, n_features=10, leaves=500, max_depth=20, average=False):
    rs = np.random.RandomState(seed)
    return model_text([random_tree_text(rs, t, n_features, leaves if t % 7 else int(rs.randint(1, 4)), max_depth)
                       for t in range(n_trees)], n_features, average=average)


def rows_with_specials(seed, rows, n_features):
    """N(0, 1) rows with exact zeros, -0.0, +-1e-36, +-1e-35f and NaN scattered in"""
    rs = np.random.RandomState(seed)
    x = rs.randn(rows, n_features)
    specials = np.array([0.0, -0.0, 1e-36, -1e-36, K_ZERO_THRESHOLD, -K_ZERO_THRESHOLD, np.nan])
    mask = rs.rand(rows, n_features) < 0.2
    x[mask] = specials[rs.randint(specials.size, size=int(mask.sum()))]
    return x
