"""The second-level scoring model's forests without a GPU: the importers of mcb200.forest, the numpy restatement in
oracle/forest_oracle.py and the host side of mcb200.models.ScoringRandomForest / ScoringLightGBM.

* sklearn: the restatement over the imported arrays equals RandomForestRegressor.predict (n_jobs=1) bit for bit on the
  scoring features of tests/golden/scoring_features.npz, with NaNs in training and at predict time; the imported
  nodes equal each `tree_`, node for node.
* LightGBM: lightgbm is not installed here, so the parser and the split rules are pinned to the published algorithm
  (Tree::NumericalDecision and the C API's dense-row path) by hand-derived known-answer vectors: every decision_type,
  +-0, +-1e-36, +-1e-35f, NaN under each missing type, one-leaf trees and average_output.
* Every refusal raises with its name; malformed text raises ValueError.
* The transformers keep the reference's constructor signatures and joblib (estimator, feature_names) files.
"""
import ast
import inspect
import os

import numpy as np
import pytest

from oracle import forest_oracle as O
from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEATURES = ('threshold', 'area', 'mean_prob', 'max_prob', 'bbox_ar', 'bbox_area', 'bbox_fill', 'min_dist_to_border',
            'max_dist_to_border', 'contour_length')
KZ = O.K_ZERO_THRESHOLD


def golden_rows(prefix):
    g = np.load(os.path.join(ROOT, "tests", "golden", "scoring_features.npz"))
    return np.stack([g[prefix + c] for c in FEATURES], 1).astype(np.float64), g[prefix + "iou"]


def trained_forest(n_estimators=40, seed=0, **kw):
    from sklearn.ensemble import RandomForestRegressor
    x, y = golden_rows("ann_")
    keep = ~np.isnan(y)
    x, y = x[keep], y[keep]
    rs = np.random.RandomState(seed)
    x[rs.rand(*x.shape) < 0.05] = np.nan
    params = dict(n_estimators=n_estimators, max_depth=20, min_samples_split=10, min_samples_leaf=5,
                  max_features=1.0, n_jobs=1, random_state=seed)
    params.update(kw)
    return RandomForestRegressor(**params).fit(x, y)


def predict_rows(seed=1):
    x, _ = golden_rows("none_")
    rs = np.random.RandomState(seed)
    x[rs.rand(*x.shape) < 0.05] = np.nan
    return x


# ---------------------------------------------------------------------------------------------------------------------
# sklearn
# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_equals_sklearn_predict_bit_for_bit(mcb):
    from mcb200 import forest as F
    model = trained_forest()
    forest = F.from_sklearn(model)
    x = predict_rows()
    assert x.shape[0] > 4000 and np.isnan(x).any()
    got = O.predict(forest, x)
    assert np.array_equal(got, model.predict(x))
    # the configured shape: min_samples_* 100, max_leaf_nodes 500
    model = trained_forest(n_estimators=20, min_samples_split=100, min_samples_leaf=100, max_leaf_nodes=500)
    assert np.array_equal(O.predict(F.from_sklearn(model), x), model.predict(x))


def test_sklearn_float32_cast_decides_ties(mcb):
    """a value that rounds to float32 onto the threshold goes left although the float64 value is above it"""
    from sklearn.ensemble import RandomForestRegressor
    from mcb200 import forest as F
    x = np.array([[0.0], [1.0]] * 10)
    model = RandomForestRegressor(n_estimators=1, bootstrap=False, random_state=0).fit(x, x[:, 0])
    forest = F.from_sklearn(model)
    thr = forest.threshold[0]
    probe = np.array([[np.nextafter(np.float64(np.float32(thr)), 2.0)], [thr], [np.nan]])
    assert np.float32(probe[0, 0]) == np.float32(thr)
    assert np.array_equal(O.predict(forest, probe), model.predict(probe))


def test_importer_arrays_equal_tree_(mcb):
    from mcb200 import forest as F
    model = trained_forest(n_estimators=6)
    forest = F.from_sklearn(model)
    assert forest.n_trees == 6 and forest.average and forest.n_features == len(FEATURES)
    for t, est in enumerate(model.estimators_):
        tr = est.tree_
        stack = [(0, int(forest.tree_root[t]))]
        visited = 0
        while stack:
            i, n = stack.pop()
            visited += 1
            if tr.children_left[i] == -1:
                assert n < 0 and forest.leaf_value[~n] == tr.value[i, 0, 0]
                continue
            assert n >= 0
            assert forest.feature[n] == tr.feature[i] and forest.threshold[n] == tr.threshold[i]
            assert bool(forest.flags[n] & 2) == bool(tr.missing_go_to_left[i])
            stack += [(tr.children_left[i], int(forest.left[n])), (tr.children_right[i], int(forest.right[n]))]
        assert visited == tr.node_count


# ---------------------------------------------------------------------------------------------------------------------
# LightGBM known answers
# ---------------------------------------------------------------------------------------------------------------------
def stump(index, threshold, decision_type, right_value, left_value=0.0, feature=0):
    return "\n".join(["Tree=%d" % index, "num_leaves=2", "num_cat=0", "split_feature=%d" % feature,
                      "split_gain=1", "threshold=%r" % threshold, "decision_type=%d" % decision_type,
                      "left_child=-1", "right_child=-2", "leaf_value=%r %r" % (left_value, right_value),
                      "leaf_weight=1 1", "leaf_count=1 1", "internal_value=0", "internal_weight=1",
                      "internal_count=2", "is_linear=0", "shrinkage=1", "", ""])


ABOVE_KZ = float(np.nextafter(KZ, 1.0))
# x -> (the value a None- or NaN-type node compares, hand-derived; whether a Zero-type node takes its default
# direction; whether a NaN-type node takes its default direction)
# The C API zeroes |x| <= kZeroThreshold (1e-35f); NaN becomes 0.0 under None and Zero; IsZero is |x| <= 1e-35f.
KNOWN = [
    (0.0, 0.0, True, False),
    (-0.0, 0.0, True, False),
    (1e-36, 0.0, True, False),
    (-1e-36, 0.0, True, False),
    (1e-35, 0.0, True, False),           # below 1e-35f (a float is 1.0000000180e-35)
    (KZ, 0.0, True, False),
    (-KZ, 0.0, True, False),
    (ABOVE_KZ, ABOVE_KZ, False, False),
    (-ABOVE_KZ, -ABOVE_KZ, False, False),
    (np.nan, 0.0, True, True),           # None / Zero see 0.0 (Zero then defaults); NaN type defaults
    (0.5, 0.5, False, False),
    (-0.5, -0.5, False, False),
]


def test_lightgbm_decision_rules_known_answers(mcb):
    """one stump per (decision_type, threshold); tree j sends its right leaf 2^j, so the sum spells every decision"""
    from mcb200 import forest as F
    thresholds = (0.0, -0.25, 0.25, 1e-36)
    combos = [(dt, thr) for dt in (0, 2, 4, 6, 8, 10) for thr in thresholds]
    text = O.model_text([stump(j, thr, dt, float(2 ** j)) for j, (dt, thr) in enumerate(combos)], 1)
    forest = F.from_lightgbm_string(text)
    assert forest.n_trees == 24 and not forest.average
    x = np.array([[k[0]] for k in KNOWN])
    want = []
    for _, value, zero_default, nan_default in KNOWN:
        s = 0.0
        for j, (dt, thr) in enumerate(combos):
            missing, default_left = dt >> 2, bool(dt & 2)
            default = (missing == 1 and zero_default) or (missing == 2 and nan_default)
            left = default_left if default else value <= thr
            s += 0.0 if left else float(2 ** j)
        want.append(s)
    assert np.array_equal(O.predict(forest, x), np.array(want))
    # spot checks written out: 1e-36 under a None node at threshold 0 compares as 0.0 <= 0 -> left (raw it would
    # go right); just above 1e-35f it goes right
    none0 = combos.index((0, 0.0))
    bits = O.predict(forest, np.array([[1e-36], [ABOVE_KZ]])).astype(np.int64)
    assert not (bits[0] >> none0) & 1 and (bits[1] >> none0) & 1


def test_lightgbm_tree_shapes_and_average_output(mcb):
    """a three-leaf tree, a one-leaf tree (empty split arrays) and average_output, with literal answers"""
    from mcb200 import forest as F
    three = "\n".join(["Tree=0", "num_leaves=3", "num_cat=0", "split_feature=1 0", "threshold=0.5 -1",
                       "decision_type=2 10", "left_child=1 -1", "right_child=-2 -3", "leaf_value=0.25 4 -2",
                       "is_linear=0", "shrinkage=1", ""])
    one = "\n".join(["Tree=1", "num_leaves=1", "num_cat=0", "split_feature=", "split_gain=", "threshold=",
                     "decision_type=", "left_child=", "right_child=", "leaf_value=1.5", "is_linear=0",
                     "shrinkage=1", ""])
    x = np.array([[0.0, 0.0],          # f1 0 <= .5 -> node 1: f0 0 <= -1 no -> leaf 2 (-2)
                  [-3.0, 0.0],         # -> node 1: -3 <= -1 -> leaf 0 (0.25)
                  [np.nan, 0.0],       # node 1 NaN-type, default left -> leaf 0
                  [0.0, 1.0],          # f1 1 > .5 -> leaf 1 (4)
                  [0.0, np.nan]])      # node 0 None-type: NaN -> 0.0 <= .5 -> node 1 -> leaf 2
    tree_only = [-2.0, 0.25, 0.25, 4.0, -2.0]
    f = F.from_lightgbm_string(O.model_text([three, one], 2))
    assert np.array_equal(O.predict(f, x), np.array(tree_only) + 1.5)
    f = F.from_lightgbm_string(O.model_text([three, one], 2, average=True))
    assert f.average and np.array_equal(O.predict(f, x), (np.array(tree_only) + 1.5) / 2)
    f = F.from_lightgbm_string(O.model_text([one.replace("Tree=1", "Tree=0")], 2))
    assert f.tree_root[0] < 0 and np.array_equal(O.predict(f, x), np.full(5, 1.5))


def test_seeded_lightgbm_model_parses_to_its_trees(mcb):
    from mcb200 import forest as F
    f = F.from_lightgbm_string(O.random_lightgbm_model(3, 30, leaves=40, max_depth=6))
    assert f.n_trees == 30 and f.leaf_value.size == f.feature.size + 30
    # depth <= 6: at most 6 decisions from every root
    depth = np.zeros(f.feature.size, np.int64)
    frontier, d = f.tree_root[f.tree_root >= 0], 1
    while frontier.size:
        depth[frontier] = d
        kids = np.concatenate([f.left[frontier], f.right[frontier]])
        frontier, d = kids[kids >= 0], d + 1
    assert depth.max() <= 6
    x = O.rows_with_specials(4, 500, 10)
    assert np.isfinite(O.predict(f, x)).all()


# ---------------------------------------------------------------------------------------------------------------------
# refusals and malformed input
# ---------------------------------------------------------------------------------------------------------------------
GOOD = "\n".join(["Tree=0", "num_leaves=3", "num_cat=0", "split_feature=1 0", "threshold=0.5 -1",
                  "decision_type=2 10", "left_child=1 -1", "right_child=-2 -3", "leaf_value=0.25 4 -2",
                  "is_linear=0", "shrinkage=1", ""])


@pytest.mark.parametrize("text, name", [
    (O.model_text([GOOD.replace("decision_type=2 10", "decision_type=3 10")], 2), "categorical"),
    (O.model_text([GOOD.replace("num_cat=0", "num_cat=1")], 2), "categorical"),
    (O.model_text([GOOD.replace("is_linear=0", "is_linear=1")], 2), "linear"),
    (O.model_text([GOOD], 2, num_class=3), "multiclass"),
    (O.model_text([GOOD], 2, objective="regression sqrt"), "regression sqrt"),
    (O.model_text([GOOD], 2, objective="binary sigmoid:1"), "binary"),
    (O.model_text([GOOD], 2, objective="huber"), "huber"),
])
def test_lightgbm_refusals_are_named(mcb, text, name):
    from mcb200 import forest as F
    with pytest.raises(NotImplementedError, match=name):
        F.from_lightgbm_string(text)


@pytest.mark.parametrize("edit", [
    lambda t: t.replace("left_child=1 -1", "left_child=0 -1"),          # cycle through the root
    lambda t: t.replace("left_child=1 -1", "left_child=1 1"),           # node 1 its own child
    lambda t: t.replace("left_child=1 -1", "left_child=2 -1"),          # child out of range
    lambda t: t.replace("right_child=-2 -3", "right_child=-2 -4"),      # leaf out of range
    lambda t: t.replace("right_child=-2 -3", "right_child=-1 -3"),      # leaf 0 twice, leaf 1 never
    lambda t: t.replace("split_feature=1 0", "split_feature=2 0"),      # feature out of range
    lambda t: t.replace("split_feature=1 0", "split_feature=1"),        # short array
    lambda t: t.replace("threshold=0.5 -1", "threshold=0.5 x"),         # not a number
    lambda t: t.replace("decision_type=2 10", "decision_type=2 12"),    # missing type 3
    lambda t: t.replace("num_leaves=3", "num_leaves=0"),
    lambda t: t.replace("num_leaves=3", "num_leaves=three"),
    lambda t: t.replace("end of trees", ""),                            # truncated
    lambda t: t.replace("tree\n", "", 1),                               # not a model
    lambda t: t.replace("max_feature_idx=1", "max_feature_idx=2"),      # feature_names count
    lambda t: t.replace("Tree=0", "Tree=0\nnum_leaves=3"),              # duplicate key
])
def test_lightgbm_malformed_text_raises_value_error(mcb, edit):
    from mcb200 import forest as F
    text = O.model_text([GOOD], 2)
    F.from_lightgbm_string(text)
    with pytest.raises(ValueError):
        F.from_lightgbm_string(edit(text))


def test_forest_validation_of_arrays(mcb):
    from mcb200 import forest as F
    ok = dict(semantics=F.SKLEARN, n_features=1, tree_root=[0], feature=[0, 0], threshold=[0.0, 1.0], left=[1, -1],
              right=[-3, -2], flags=[0, 0], leaf_value=[1.0, 2.0, 3.0], average=True)
    F.Forest(**ok)
    bad = [dict(left=[1, 0], right=[-3, -2]),                    # a cycle 0 -> 1 -> 0 (root also referenced)
           dict(tree_root=[~2], left=[1, 0], right=[-2, -1]),    # a cycle no root reaches
           dict(feature=[0, 1]), dict(flags=[0, 12]), dict(tree_root=[]),
           dict(leaf_value=[1.0, 2.0]), dict(threshold=[0.0])]
    for b in bad:
        with pytest.raises(ValueError):
            F.Forest(**dict(ok, **b))
    with pytest.raises(NotImplementedError, match="categorical"):
        F.Forest(**dict(ok, flags=[1, 0]))
    with pytest.raises(ValueError):
        F.Forest(**ok).predict(np.zeros((3, 2)))
    assert F.Forest(**ok).predict(np.zeros((0, 1))).shape == (0,)     # zero rows: no device needed, no launch


def test_sklearn_refusals(mcb):
    from sklearn.ensemble import RandomForestRegressor
    from mcb200 import forest as F
    with pytest.raises(ValueError, match="not a fitted forest"):
        F.from_sklearn(RandomForestRegressor())
    x = np.random.RandomState(0).rand(50, 2)
    multi = RandomForestRegressor(n_estimators=2, random_state=0).fit(x, np.stack([x[:, 0], x[:, 1]], 1))
    with pytest.raises(NotImplementedError, match="multi-output"):
        F.from_sklearn(multi)


# ---------------------------------------------------------------------------------------------------------------------
# transformers
# ---------------------------------------------------------------------------------------------------------------------
REFERENCE_SIGNATURES = {"ScoringLightGBM": ["model_params", "training_params", "train_size", "target"],
                        "ScoringRandomForest": ["train_size", "target", "model_params"]}


def test_constructor_signatures_equal_the_reference(mcb):
    from mcb200 import models
    for name, params in REFERENCE_SIGNATURES.items():
        assert list(inspect.signature(getattr(models, name).__init__).parameters)[1:] == params, name


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree (MCB_REFERENCE_ROOT) absent")
def test_pinned_signatures_are_the_reference_source():
    with open(os.path.join(ref_shim.REFERENCE_ROOT, "src", "models.py")) as fh:
        tree = ast.parse(fh.read())
    found = {}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name in REFERENCE_SIGNATURES:
            init = next(b for b in node.body if isinstance(b, ast.FunctionDef) and b.name == "__init__")
            found[node.name] = [a.arg for a in init.args.args][1:]
    assert found == REFERENCE_SIGNATURES


def frames(x, counts):
    import pandas as pd
    out, at = [], 0
    for image in counts:
        layers = []
        for k in image:
            df = pd.DataFrame(x[at:at + k], columns=list(FEATURES))
            df["area"] = df["area"].fillna(0).astype(np.int64)        # an int64 column, as the features have
            layers.append(df)
            at += k
        out.append(layers)
    return out


def test_random_forest_fit_and_joblib_round_trip(mcb, tmp_path):
    """fit from the reference's feature frames (background layer skipped, `iou` the target), save, load into a
    fresh transformer: same estimator, same feature names, same host predictions"""
    from mcb200 import models
    x, y = golden_rows("ann_")
    keep = ~np.isnan(y)
    x, y = x[keep][:600], y[keep][:600]
    fr = frames(x, [[0, 100, 100], [0, 200, 200]])
    at = 0
    for image in fr:
        for df in image:
            df["iou"] = y[at:at + len(df)]
            at += len(df)
    m = models.ScoringRandomForest(0.8, "iou", {"n_estimators": 5, "max_depth": 4, "random_state": 0}).fit(fr)
    assert m.feature_names == list(FEATURES)
    # train_test_split at train_size 0.8 of the 600 rows of the non-background layers
    assert all(e.tree_.weighted_n_node_samples[0] == 480 for e in m.estimator.estimators_)
    path = str(tmp_path / "rf.pkl")
    m.save(path)
    import joblib
    est, names = joblib.load(path)
    assert names == list(FEATURES) and type(est).__name__ == "RandomForestRegressor"
    m2 = models.ScoringRandomForest(0.8, "iou", {}).load(path)
    assert m2.feature_names == m.feature_names
    assert np.array_equal(m2.estimator.predict(x), m.estimator.predict(x))
    from mcb200 import forest as F
    assert np.array_equal(O.predict(F.from_sklearn(m2.estimator), x), m.estimator.predict(x))


def test_transform_without_rows_launches_nothing(mcb):
    """zero rows end before any device call: this runs on a machine without one"""
    import pandas as pd
    from mcb200 import models
    m = models.ScoringRandomForest(0.8, "iou", {"n_estimators": 2, "random_state": 0})
    x, y = golden_rows("ann_")
    keep = ~np.isnan(y)
    m.estimator.fit(x[keep][:200], y[keep][:200])
    m.feature_names = list(FEATURES)
    empty = pd.DataFrame(columns=list(FEATURES))
    assert m.transform([[empty, empty], [empty]]) == {"scores": [[[], []], [[]]]}
    assert m.transform([]) == {"scores": []}
