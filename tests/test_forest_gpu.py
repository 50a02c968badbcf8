"""The second-level scoring model's forests on the device (csrc/forest.cu through mcb200.forest and
mcb200.models.ScoringRandomForest / ScoringLightGBM) against oracle/forest_oracle.py, bit for bit:

* the scoring batch (20 tiles of 300 x 300, CATEGORY_LAYERS [1, 19]: the 4 136 instance rows of
  tests/golden/scoring_features.npz) through a RandomForest of the configured shape (500 trees, max_depth 20,
  min_samples_split / min_samples_leaf 100, max_leaf_nodes 500; squared_error and max_features=1.0, the current names
  of 'mse' and 'auto'), with NaNs in training and at predict time; also equal to RandomForestRegressor.predict;
* a seeded LightGBM-format forest of 3 000 trees of 500 leaves and depth <= 20 on rows holding zeros, -0.0, +-1e-36,
  +-1e-35f and NaNs, plain and with average_output;
* 1 row, 0 rows, row counts that are not a multiple of the 256-thread block, and a chunk so small that every row's sum
  is carried across many launches;
* the inference chain FeatureExtractor -> ScoringRandomForest (device) -> ScoreImageJoiner -> NonMaximumSupression ->
  create_annotations gives the same annotations as the chain with the host forest's predict per (image, layer).
"""
import numpy as np
import pytest

from oracle import forest_oracle as O
from oracle import instances_oracle as I
from oracle import scoring_oracle as S

pytestmark = pytest.mark.gpu

FEATURES = ('threshold', 'area', 'mean_prob', 'max_prob', 'bbox_ar', 'bbox_area', 'bbox_fill', 'min_dist_to_border',
            'max_dist_to_border', 'contour_length')


def golden_rows(prefix):
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "scoring_features.npz"))
    return np.stack([g[prefix + c] for c in FEATURES], 1).astype(np.float64), g[prefix + "iou"]


@pytest.fixture(scope="module")
def configured_forest():
    from sklearn.ensemble import RandomForestRegressor
    x, y = golden_rows("ann_")
    keep = ~np.isnan(y)
    x, y = x[keep], y[keep]
    rs = np.random.RandomState(0)
    x[rs.rand(*x.shape) < 0.05] = np.nan
    return RandomForestRegressor(n_estimators=500, criterion="squared_error", max_depth=20, min_samples_split=100,
                                 min_samples_leaf=100, max_features=1.0, max_leaf_nodes=500, n_jobs=1,
                                 random_state=0).fit(x, y)


@pytest.fixture(scope="module")
def batch_rows():
    x, _ = golden_rows("none_")
    rs = np.random.RandomState(1)
    x[rs.rand(*x.shape) < 0.05] = np.nan
    return x


@pytest.fixture(scope="module")
def lightgbm_text():
    return O.random_lightgbm_model(7, 3000, n_features=10, leaves=500, max_depth=20)


def test_random_forest_scoring_batch(mcb, cuda, configured_forest, batch_rows):
    from mcb200 import forest as F
    forest = F.from_sklearn(configured_forest)
    assert forest.n_trees == 500 and batch_rows.shape[0] > 4000
    got = forest.predict(batch_rows)
    assert np.array_equal(got, O.predict(forest, batch_rows))
    assert np.array_equal(got, configured_forest.predict(batch_rows))


@pytest.mark.parametrize("average", [False, True])
def test_lightgbm_forest_3000_trees(mcb, cuda, lightgbm_text, average):
    from mcb200 import forest as F
    text = lightgbm_text.replace("objective=regression\n", "objective=regression\naverage_output\n") if average \
        else lightgbm_text
    forest = F.from_lightgbm_string(text)
    assert forest.n_trees == 3000 and forest.average == average and forest.leaf_value.max() != 0
    x = O.rows_with_specials(8, 4100, 10)
    got = forest.predict(x)
    assert np.array_equal(got, O.predict(forest, x))


@pytest.mark.parametrize("rows", [1, 2, 255, 257, 1001, 4099])
def test_row_counts(mcb, cuda, configured_forest, batch_rows, rows):
    from mcb200 import forest as F
    forest = F.from_sklearn(configured_forest)
    x = batch_rows[:rows]
    assert np.array_equal(forest.predict(x), O.predict(forest, x))


def test_zero_rows_and_small_chunks(mcb, cuda, configured_forest, batch_rows, monkeypatch):
    from mcb200 import forest as F
    forest = F.from_sklearn(configured_forest)
    assert forest.predict(np.zeros((0, len(FEATURES)))).shape == (0,)
    want = O.predict(forest, batch_rows[:300])
    monkeypatch.setattr(F, "CHUNK_PAIRS", 300 * 7)        # 7 trees per launch pair: 72 chunks, the last of 3 trees
    assert np.array_equal(forest.predict(batch_rows[:300]), want)
    monkeypatch.setattr(F, "CHUNK_PAIRS", 1)              # one tree per chunk
    assert np.array_equal(forest.predict(batch_rows[:300]), want)


def test_lightgbm_transformer_on_a_text_model(mcb, cuda, lightgbm_text):
    """ScoringLightGBM.transform from a booster's text model (a stand-in booster: lightgbm is not needed to predict)"""
    import pandas as pd
    from mcb200 import models

    class Booster:
        def model_to_string(self, num_iteration=None):
            assert num_iteration is None
            return lightgbm_text.replace(" ".join("f%d" % i for i in range(10)), " ".join(FEATURES))

    m = models.ScoringLightGBM({}, {}, 0.7, "iou")
    m.estimator, m.feature_names = Booster(), list(FEATURES)
    x = O.rows_with_specials(9, 700, 10)
    frames = [[pd.DataFrame(x[:0], columns=FEATURES), pd.DataFrame(x[:300], columns=FEATURES)],
              [pd.DataFrame(x[300:301], columns=FEATURES), pd.DataFrame(x[301:], columns=FEATURES)]]
    frames[1][1]["iou"] = None                                 # extra columns are not features
    got = m.transform(frames)["scores"]
    want = O.predict(m._device_forest(), x)
    assert [len(l) for im in got for l in im] == [0, 300, 1, 399]
    assert np.array_equal(np.array([v for im in got for l in im for v in l]), want)


def stream(fn, *iterables):
    return (fn(*args) for args in zip(*iterables))


def test_inference_chain_device_forest_equals_host_forest(mcb, cuda, monkeypatch):
    """FeatureExtractor -> ScoringRandomForest -> ScoreImageJoiner -> NonMaximumSupression -> create_annotations, once
    with the device forest and once with the same fitted estimator's host predict per (image, layer), as
    src/models.py:267-278 calls it"""
    from mcb200 import models
    from mcb200 import postprocessing as G
    from mcb200 import utils as U
    monkeypatch.setattr(G, "CATEGORY_LAYERS", list(S.SCORING_LAYERS))
    probs, labels, annotations = S.scoring_case(n=5, size=64, seed=11)
    f_train = G.FeatureExtractor().transform(list(labels[1:]), list(probs[1:]), annotations[1:])["features"]
    model = models.ScoringRandomForest(0.8, "iou", {"n_estimators": 100, "max_depth": 20, "min_samples_leaf": 2,
                                                    "n_jobs": 1, "random_state": 0}).fit(f_train)
    features = G.FeatureExtractor().transform(list(labels), list(probs))["features"]
    s_dev = model.transform(features)["scores"]
    s_host = [[list(model.estimator.predict(l[model.feature_names])) if len(l) > 0 else [] for l in im]
              for im in features]
    assert s_dev == s_host and sum(len(l) for im in s_dev for l in im) > 20
    assert len({v for im in s_dev for l in im for v in l}) > 10
    results = []
    for scores in (s_dev, s_host):
        joined = G.ScoreImageJoiner().transform(list(labels), scores)["images_with_scores"]
        kept = G.NonMaximumSupression(0.5).transform(joined)["images_with_scores"]
        results.append(U.create_annotations(list(range(len(kept))), kept, None, [None, 100], [1, 19]))
    assert results[0] == results[1] and len(results[0]) > 10
    ora = [I.remove_overlapping_masks(*p, iou_threshold=0.5) for p in S.score_image_joiner(list(labels),
                                                                                         s_host)["images_with_scores"]]
    assert results[1] == I.create_annotations(list(range(len(ora))), ora, [None, 100], [1, 19])
