"""Tree-ensemble prediction of the second-level scoring model (src/models.py:212-282) on the H100.

`Forest` is the flattened node format of include/mcb200.h (`mcb_forest_predict`) that both importers produce:
  * `from_sklearn(RandomForestRegressor)` reads every `estimators_[i].tree_`;
  * `from_lightgbm_string(text)` parses LightGBM's text model (`Booster.model_to_string(num_iteration=None)`, which
    writes the trees up to the best iteration, the ones `Booster.predict` uses).

Per row the device sums the trees' leaf values in tree order in float64, starting at 0.0, and divides by the tree count
when the forest averages: sklearn's ForestRegressor.predict at n_jobs=1 and LightGBM's GBDT::PredictRaw loop, so the
prediction is bit-exact.  The split rules of each library are in csrc/forest.cu and restated in oracle/forest_oracle.py.

Models are input from outside the program, so everything is validated before a node reaches the device: every tree is
a proper binary tree reached from its root, without cycles, and every child, leaf and feature index is in range.  What
the kernel does not implement is refused by name with NotImplementedError: categorical splits, linear trees, more than
one class, and any LightGBM objective other than plain L2 `regression`.
"""
import numpy as np

from . import _lib as L

SKLEARN, LIGHTGBM = 0, 1                       # MCB_FOREST_SKLEARN / MCB_FOREST_LIGHTGBM
CATEGORICAL, DEFAULT_LEFT = 1, 2               # LightGBM's kCategoricalMask / kDefaultLeftMask
MISSING_NONE, MISSING_ZERO, MISSING_NAN = 0, 1, 2
CHUNK_PAIRS = 1 << 22                          # (tree, row) pairs per chunk: 32 MiB of float64 leaf values


class Forest:
    """a validated, flattened tree ensemble.  Nodes of all trees share one set of arrays: feature int32, threshold
    float64, left / right int32 (a node index, or ~k for leaf_value[k]) and flags uint8 (decision_type layout:
    DEFAULT_LEFT, missing type in bits 2-3); tree_root int32 holds each tree's root (~k for a one-leaf tree)."""

    def __init__(self, semantics, n_features, tree_root, feature, threshold, left, right, flags, leaf_value,
                 average):
        self.semantics = int(semantics)
        self.n_features = int(n_features)
        self.tree_root = np.ascontiguousarray(tree_root, np.int32)
        self.feature = np.ascontiguousarray(feature, np.int32)
        self.threshold = np.ascontiguousarray(threshold, np.float64)
        self.left = np.ascontiguousarray(left, np.int32)
        self.right = np.ascontiguousarray(right, np.int32)
        self.flags = np.ascontiguousarray(flags, np.uint8)
        self.leaf_value = np.ascontiguousarray(leaf_value, np.float64)
        self.average = bool(average)
        self._validate()
        self._device = {}

    @property
    def n_trees(self):
        return int(self.tree_root.size)

    def _validate(self):
        if self.semantics not in (SKLEARN, LIGHTGBM):
            raise ValueError("forest: unknown semantics %r" % self.semantics)
        if self.n_features < 1 or self.n_trees < 1:
            raise ValueError("forest: %d features, %d trees" % (self.n_features, self.n_trees))
        n, k = self.feature.size, self.leaf_value.size
        if not (self.threshold.size == self.left.size == self.right.size == self.flags.size == n):
            raise ValueError("forest: node arrays of different lengths")
        if n >= 2 ** 31 - 1 or k >= 2 ** 31 - 1:
            raise ValueError("forest: more than 2^31 - 2 nodes or leaves")
        if n and (self.feature.min() < 0 or self.feature.max() >= self.n_features):
            raise ValueError("forest: feature index out of range [0, %d)" % self.n_features)
        if np.any(self.flags & CATEGORICAL):
            raise NotImplementedError("forest: categorical splits are not supported")
        if np.any(self.flags > 15) or np.any((self.flags >> 2) & 3 == 3):
            raise ValueError("forest: invalid split flags")
        refs = np.concatenate([self.tree_root, self.left, self.right]).astype(np.int64)
        nodes, leaves = refs[refs >= 0], ~refs[refs < 0]
        if (nodes.size and nodes.max() >= n) or (leaves.size and leaves.max() >= k):
            raise ValueError("forest: child index out of range")
        # every node and every leaf is referenced exactly once (by a root or by one parent) ...
        if np.any(np.bincount(nodes, minlength=n) != 1) or np.any(np.bincount(leaves, minlength=k) != 1):
            raise ValueError("forest: a node or leaf is shared, or unreachable")
        # ... and is reached from a root: a cycle would hold nodes that no root reaches
        seen, frontier = 0, self.tree_root[self.tree_root >= 0]
        while frontier.size:
            seen += frontier.size
            children = np.concatenate([self.left[frontier], self.right[frontier]])
            frontier = children[children >= 0]
        if seen != n:
            raise ValueError("forest: %d nodes are not reached from any root (a cycle)" % (n - seen))

    def _arrays(self, device):
        import torch
        key = str(device)
        if key not in self._device:
            self._device[key] = tuple(torch.from_numpy(a).to(device) for a in (
                self.tree_root, self.feature, self.threshold, self.left, self.right, self.flags, self.leaf_value))
        return self._device[key]

    def predict(self, x, device="cuda"):
        """x float64 [rows][n_features] (anything np.asarray takes) -> float64 [rows]: one upload, one
        mcb_forest_predict, one readback.  Zero rows launch nothing."""
        import torch
        x = np.ascontiguousarray(x, np.float64)
        if x.ndim != 2 or x.shape[1] != self.n_features:
            raise ValueError("forest: expected rows of %d features, got shape %s" % (self.n_features, x.shape))
        rows = x.shape[0]
        if rows == 0:
            return np.zeros(0, np.float64)
        if rows >= 2 ** 31:
            raise ValueError("forest: %d rows (at most 2^31 - 1)" % rows)
        if not torch.cuda.is_available():
            raise RuntimeError("forest: prediction needs a CUDA device; there is no CPU fallback")
        device = torch.device(device)
        root, feature, threshold, left, right, flags, leaf = self._arrays(device)
        with torch.cuda.device(device):
            xd = torch.from_numpy(x).to(device)
            chunk = max(1, min(self.n_trees, CHUNK_PAIRS // rows))
            work = torch.empty(chunk * rows, dtype=torch.float64, device=device)
            out = torch.empty(rows, dtype=torch.float64, device=device)
            L.fcall("mcb_forest_predict", L.dp(xd), rows, self.n_features, L.dp(root), self.n_trees, L.dp(feature),
                    L.dp(threshold), L.dp(left), L.dp(right), L.dp(flags), L.dp(leaf), self.semantics,
                    int(self.average), L.dp(work), chunk, L.dp(out))
            return out.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# sklearn
# ---------------------------------------------------------------------------------------------------------------------
def from_sklearn(estimator):
    """RandomForestRegressor (fitted) -> Forest.  Reads estimators_[i].tree_: children_left / children_right (-1 marks
    a leaf), feature, threshold, missing_go_to_left and value[:, 0, 0]; averages over the trees."""
    trees = getattr(estimator, "estimators_", None)
    if not trees:
        raise ValueError("from_sklearn: the estimator is not a fitted forest (no estimators_)")
    if getattr(estimator, "n_outputs_", 1) != 1:
        raise NotImplementedError("from_sklearn: multi-output forests are not supported (n_outputs_ = %d)"
                                  % estimator.n_outputs_)
    n_features = int(estimator.n_features_in_)
    roots, parts = [], []
    node_off = leaf_off = 0
    for ti, est in enumerate(trees):
        t = est.tree_
        cl, cr = np.asarray(t.children_left, np.int64), np.asarray(t.children_right, np.int64)
        count = cl.size
        value = np.asarray(t.value)
        if value.ndim != 3 or value.shape[0] != count or value.shape[1:] != (1, 1):
            raise NotImplementedError("from_sklearn: tree %d has values of shape %s, only single-output regression "
                                      "trees are supported" % (ti, value.shape))
        internal = cl != -1
        if count == 0 or np.any(cr[~internal] != -1) or np.any(cr[internal] == -1):
            raise ValueError("from_sklearn: tree %d has a node with a single child" % ti)
        kids = np.concatenate([cl[internal], cr[internal]])
        if kids.size and (kids.min() < 1 or kids.max() >= count):
            raise ValueError("from_sklearn: tree %d has a child index out of range" % ti)
        n_int = int(internal.sum())
        index = np.empty(count, np.int64)
        index[internal] = node_off + np.arange(n_int)
        index[~internal] = ~(leaf_off + np.arange(count - n_int))
        missing_left = np.asarray(t.missing_go_to_left, bool)[internal]
        parts.append((np.asarray(t.feature, np.int64)[internal], np.asarray(t.threshold, np.float64)[internal],
                      index[cl[internal]], index[cr[internal]],
                      np.where(missing_left, DEFAULT_LEFT, 0).astype(np.uint8), value[~internal, 0, 0]))
        roots.append(index[0])
        node_off += n_int
        leaf_off += count - n_int
    cols = [np.concatenate([p[i] for p in parts]) for i in range(6)]
    return Forest(SKLEARN, n_features, np.asarray(roots), *cols[:5], cols[5], average=True)


# ---------------------------------------------------------------------------------------------------------------------
# LightGBM text model
# ---------------------------------------------------------------------------------------------------------------------
def _values(block, key, n, kind, where):
    """the n space-separated values of `key` (an absent or empty line holds none)"""
    text = block.get(key) or ""
    try:
        vals = [kind(v) for v in text.split()]
    except ValueError:
        raise ValueError("LightGBM model: %s: malformed %s" % (where, key)) from None
    if len(vals) != n:
        raise ValueError("LightGBM model: %s: %s has %d values, expected %d" % (where, key, len(vals), n))
    return vals


def _int(block, key, where):
    try:
        return int(block[key])
    except (KeyError, TypeError, ValueError):
        raise ValueError("LightGBM model: %s: missing or malformed %s" % (where, key)) from None


def parse_lightgbm_model(text):
    """LightGBM's text model -> (header dict, [tree dict]).  `key=value` lines; a bare line (`average_output`) maps to
    None.  The header runs to the first `Tree=` line and the trees to `end of trees`."""
    lines = [ln.strip() for ln in text.splitlines()]
    body = [ln for ln in lines if ln]
    if not body or body[0] != "tree":
        raise ValueError("LightGBM model: the text does not start with `tree`")
    if "end of trees" not in body:
        raise ValueError("LightGBM model: no `end of trees` line (truncated text?)")
    header, trees, block = {}, [], None
    for ln in body[1:body.index("end of trees")]:
        if ln.startswith("Tree="):
            block = {}
            trees.append(block)
            continue
        key, sep, val = ln.partition("=")
        target = header if block is None else block
        if key in target:
            raise ValueError("LightGBM model: duplicate line %r" % key)
        target[key] = val if sep else None
    return header, trees


def from_lightgbm_string(text):
    """LightGBM text model (Booster.model_to_string(num_iteration=None)) -> Forest with LightGBM's split rules; the
    forest averages when the header has `average_output` (boosting_type 'rf')."""
    header, trees = parse_lightgbm_model(text)
    if _int(header, "num_class", "header") != 1:
        raise NotImplementedError("LightGBM model: multiclass models are not supported (num_class = %s)"
                                  % header["num_class"])
    if _int(header, "num_tree_per_iteration", "header") != 1:
        raise NotImplementedError("LightGBM model: more than one tree per iteration is not supported")
    objective = header.get("objective")
    if objective != "regression":
        raise NotImplementedError("LightGBM model: objective %r is not supported (only plain L2 'regression', whose "
                                  "output is the raw score)" % objective)
    n_features = _int(header, "max_feature_idx", "header") + 1
    if n_features < 1:
        raise ValueError("LightGBM model: max_feature_idx %d" % (n_features - 1))
    names = (header.get("feature_names") or "").split()
    if len(names) != n_features:
        raise ValueError("LightGBM model: %d feature_names for max_feature_idx %d" % (len(names), n_features - 1))
    if not trees:
        raise ValueError("LightGBM model: no trees")
    roots, parts = [], []
    node_off = leaf_off = 0
    for ti, b in enumerate(trees):
        where = "tree %d" % ti
        nl = _int(b, "num_leaves", where)
        if nl < 1:
            raise ValueError("LightGBM model: %s: num_leaves %d" % (where, nl))
        if "num_cat" in b and _int(b, "num_cat", where) != 0:
            raise NotImplementedError("LightGBM model: %s: categorical splits are not supported" % where)
        if "is_linear" in b and _int(b, "is_linear", where) != 0:
            raise NotImplementedError("LightGBM model: %s: linear trees (is_linear=1) are not supported" % where)
        ni = nl - 1
        feature = np.asarray(_values(b, "split_feature", ni, int, where), np.int64)
        threshold = np.asarray(_values(b, "threshold", ni, float, where), np.float64)
        decision = np.asarray(_values(b, "decision_type", ni, int, where), np.int64)
        left = np.asarray(_values(b, "left_child", ni, int, where), np.int64)
        right = np.asarray(_values(b, "right_child", ni, int, where), np.int64)
        leaf = np.asarray(_values(b, "leaf_value", nl, float, where), np.float64)
        if np.any(decision & CATEGORICAL):
            raise NotImplementedError("LightGBM model: %s: categorical splits (decision_type & 1) are not supported"
                                      % where)
        if np.any((decision < 0) | (decision > 15) | ((decision >> 2) & 3 == 3)):
            raise ValueError("LightGBM model: %s: invalid decision_type" % where)
        if ni and (feature.min() < 0 or feature.max() >= n_features):
            raise ValueError("LightGBM model: %s: split_feature out of range [0, %d)" % (where, n_features))
        kids = np.concatenate([left, right])
        if ni and (kids.min() < -nl or kids.max() > ni - 1):
            raise ValueError("LightGBM model: %s: child index out of range" % where)

        def glob(c):
            return np.where(c >= 0, c + node_off, ~(~c + leaf_off))
        parts.append((feature, threshold, glob(left), glob(right), decision.astype(np.uint8), leaf))
        roots.append(node_off if ni else ~leaf_off)
        node_off += ni
        leaf_off += nl
    cols = [np.concatenate([p[i] for p in parts]) for i in range(6)]
    try:
        return Forest(LIGHTGBM, n_features, np.asarray(roots), *cols[:5], cols[5], average="average_output" in header)
    except ValueError as e:
        raise ValueError("LightGBM model: %s" % e) from None
