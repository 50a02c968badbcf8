"""The second-level scoring features on the device (mcb200.postprocessing.FeatureExtractor and the per-image
functions), at the inference batch size: 20 images of 300 x 300 with CATEGORY_LAYERS = [1, 19] (20 layers), against
tests/golden/scoring_features.npz (the unmodified reference's output) and against oracle/scoring_oracle.py on the
same seeded inputs.  The case holds an image without annotations, an image whose building layers above 0.5 have no
instances, an annotation covering the whole image, multi-polygon and overlapping annotations, and instances on the
border.

Bars: integer features, threshold, box ratios, border distances and contour_length exact; max_prob exact in the
probabilities' own precision (float64); mean_prob within area * 2^-53 relative of the exactly rounded mean (float64
summation of `area` non-negative terms in any order, as tests/test_instances_scale_gpu.py derives it); iou exact (a
ratio of integer pixel counts, compared as the float64 the reference computes); column order and dtypes equal.

Mutations these tests catch:
  * [1, 1] used despite a [1, 19] configuration: 2 layers per image instead of the golden's 20;
  * every polygon of a segmentation used instead of the first: the multi-polygon annotations change `iou`;
  * `iou = 0` where the reference gives None: the golden's `iou_none` layers and the object dtype of their column;
  * the IoU max taken over all categories instead of the layer's own: the background layer's `iou` turns numeric.

The pipeline test wires the transformers as src/pipelines.py does after the network: the train pipeline in stream
mode (generators from the mask chain into FeatureExtractor), a ScoringRandomForest fitted once, and the inference
chain FeatureExtractor -> forest -> ScoreImageJoiner -> NonMaximumSupression -> create_annotations, against the same
chain on the oracle restatements with their own features.
"""
import math

import numpy as np
import pytest
import torch

from oracle import instances_oracle as I
from oracle import scoring_oracle as S

pytestmark = pytest.mark.gpu

U53 = 2.0 ** -53
EXACT = ("counts", "iou_none", "dtypes", "iou", "threshold", "area", "bbox_ar", "bbox_area", "bbox_fill",
         "min_dist_to_border", "max_dist_to_border", "contour_length", "max_prob")


@pytest.fixture(autouse=True)
def scoring_config(monkeypatch):
    """the scoring workflow's src/pipeline_config.py (CATEGORY_LAYERS = [1, 19]); the reference tree is not importable
    here, so the module defaults stand in for it"""
    from mcb200 import postprocessing as G
    monkeypatch.setattr(G, "CATEGORY_LAYERS", list(S.SCORING_LAYERS))


@pytest.fixture(scope="module")
def case():
    return S.scoring_case()


@pytest.fixture(scope="module")
def golden():
    import os
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "scoring_features.npz"))


def check_flat(got, want, labels, probs):
    for k in EXACT:
        assert np.array_equal(got[k], want[k], equal_nan=got[k].dtype.kind == "f"), k
    # mean_prob against the exactly rounded mean of each instance's probabilities
    n, nl = labels.shape[:2]
    inds = np.cumsum(S.SCORING_LAYERS)
    offs = np.concatenate([[0], np.cumsum(got["counts"])])
    worst = 0.0
    for p in range(n * nl):
        i, li = divmod(p, nl)
        lab = labels[i, li]
        k = int(got["counts"][p])
        if not k:
            continue
        ch = probs[i, int(np.searchsorted(inds, li, side="right"))]
        order = np.argsort(lab.ravel(), kind="stable")
        bounds = np.searchsorted(lab.ravel()[order], np.arange(1, k + 2))
        vals = ch.ravel()[order]
        for l in range(k):
            v = vals[bounds[l]:bounds[l + 1]]
            ref = math.fsum(v.tolist()) / v.size
            err = abs(got["mean_prob"][offs[p] + l] - ref)
            assert err <= v.size * U53 * ref, (i, li, l + 1, err)
            worst = max(worst, err)
    return worst


def device_features(case, annotations):
    from mcb200 import postprocessing as G
    probs, labels, _ = case
    lab = torch.from_numpy(labels).cuda()
    pr = torch.from_numpy(probs).cuda()
    return G.FeatureExtractor().transform(lab, pr, annotations)["features"]


def test_features_with_annotations_match_golden(mcb, cuda, case, golden):
    probs, labels, annotations = case
    got = S.flatten(device_features(case, annotations))
    want = {k[4:]: golden[k] for k in golden.files if k.startswith("ann_")}
    check_flat(got, want, labels, probs)
    assert got["counts"].size == 400


def test_features_without_annotations_match_golden(mcb, cuda, case, golden):
    probs, labels, _ = case
    got = S.flatten(device_features(case, None))
    want = {k[5:]: golden[k] for k in golden.files if k.startswith("none_")}
    check_flat(got, want, labels, probs)
    assert got["iou_none"][got["counts"] > 0].all()


def test_step_chain_lists_and_per_image_functions_match_the_oracle(mcb, cuda, case):
    """the Step chain's per-image numpy lists, get_features_for_image, get_iou_matrix / get_iou and
    get_mask_with_iou against the restatement on images 0 (no annotations), 1 (whole-image annotation) and 2"""
    import pandas as pd
    from mcb200 import postprocessing as G
    probs, labels, annotations = case
    idx = [0, 1, 2]
    got = G.FeatureExtractor().transform([labels[i] for i in idx], [probs[i] for i in idx],
                                         [annotations[i] for i in idx])["features"]
    want = S.feature_extractor([labels[i] for i in idx], [probs[i] for i in idx], [annotations[i] for i in idx])
    for gi, wi in zip(got, want["features"]):
        for a, b in zip(gi, wi):
            pd.testing.assert_frame_equal(a.drop(columns=["mean_prob"]) if len(a) else a,
                                          b.drop(columns=["mean_prob"]) if len(b) else b, check_exact=True)
    anns = annotations[1][100]
    m_got = G.get_iou_matrix(labels[1, 10], anns)
    m_want = S.get_iou_matrix(labels[1, 10], anns)
    assert np.array_equal(np.asarray(m_got), np.asarray(m_want))
    assert G.get_iou_matrix(labels[1, 10], []) is None and G.get_iou(None, 1) is None
    assert all(G.get_iou(m_got, l) == S.get_iou(m_want, l) for l in range(1, labels[1, 10].max() + 1))
    ys = list(G.get_mask_with_iou(10, labels[1, 10], np.cumsum(S.SCORING_LAYERS), {100: anns}, probs[1]))
    assert len(ys) == labels[1, 10].max() and all(np.array_equal(m, labels[1, 10] == l + 1) for l, (m, _, _) in
                                                    enumerate(ys))


def stream(fn, *iterables):
    """make_apply_transformer_stream (src/utils.py:392-405): a generator of fn over the per-image inputs"""
    return (fn(*args) for args in zip(*iterables))


def test_scoring_pipelines_match_the_oracle_chain(mcb, cuda):
    """scoring_model_train then scoring_model_inference, wired as src/pipelines.py:307-392 wires them, after the
    network.  Train runs in stream mode (scoring_model_train sets it): categorize_multilayer_image ->
    label_multilayer_image -> dilate_image reach FeatureExtractor as generators, with the annotations; a
    ScoringRandomForest (the reference's host model, restated in oracle/scoring_oracle.py) is fitted once on the
    oracle's training features.  Inference feeds lists: FeatureExtractor -> that forest -> ScoreImageJoiner ->
    NonMaximumSupression -> create_annotations.  The oracle chain computes its own features and its own NMS and
    annotations; features, scores, scores after NMS and annotations must be equal.  The device and oracle mean_prob
    may differ in the last bits (float64 sums in another order); a forest split would have to fall between them to
    change a score."""
    from mcb200 import postprocessing as G
    from mcb200 import utils as U
    probs, labels, annotations = S.scoring_case(n=5, size=64, seed=11)
    train, test = slice(1, 5), slice(0, 5)

    def mask_chain(pr):                  # mask_postprocessing after mask_resize, erode / dilate 0 as in neptune.yaml
        m = stream(lambda x: G.erode_image(x, 0), stream(G.categorize_multilayer_image, pr))
        return stream(lambda x: G.dilate_image(x, 0), stream(G.label_multilayer_image, m))

    f_train = G.FeatureExtractor().transform(mask_chain(list(probs[train])), (p for p in probs[train]),
                                             annotations[train])["features"]
    o_train = S.feature_extractor(list(labels[train]), list(probs[train]), annotations[train])["features"]
    a, b = S.flatten(f_train), S.flatten(o_train)
    for k in EXACT:
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
    assert (a["iou"] > 0.5).sum() >= 5
    model = S.ScoringRandomForest(0.8, "iou", {"n_estimators": 10, "max_depth": 6, "random_state": 0}).fit(o_train)

    lab_dev = list(mask_chain(list(probs[test])))
    assert all(np.array_equal(x, y) for x, y in zip(lab_dev, labels[test]))
    f_dev = G.FeatureExtractor().transform(lab_dev, list(probs[test]))["features"]
    f_ora = S.feature_extractor(list(labels[test]), list(probs[test]))["features"]
    a, b = S.flatten(f_dev), S.flatten(f_ora)
    for k in EXACT:
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
    s_dev, s_ora = model.transform(f_dev)["scores"], model.transform(f_ora)["scores"]
    assert s_dev == s_ora and sum(len(l) for im in s_dev for l in im) > 20
    j_dev = G.ScoreImageJoiner().transform(lab_dev, s_dev)["images_with_scores"]
    j_ora = S.score_image_joiner(list(labels[test]), s_ora)["images_with_scores"]
    c_dev = G.NonMaximumSupression(0.5).transform(j_dev)["images_with_scores"]
    c_ora = [I.remove_overlapping_masks(*p, iou_threshold=0.5) for p in j_ora]
    assert [sc for _, sc in c_dev] == [sc for _, sc in c_ora]
    assert any(v == 0 for _, sc in c_dev for l in sc for v in l)          # NMS suppressed something
    ids = list(range(len(c_dev)))
    assert U.create_annotations(ids, c_dev, None, [None, 100], [1, 19]) == \
        I.create_annotations(ids, c_ora, [None, 100], [1, 19])


def test_feature_extractor_batches_mixed_sizes(mcb, cuda):
    """lists are consumed in runs of one size: 64 x 64 and 48 x 48 tiles mixed give the per-size results"""
    from mcb200 import postprocessing as G
    p1, l1, a1 = S.scoring_case(n=3, size=64, seed=3)
    p2, l2, a2 = S.scoring_case(n=2, size=48, seed=4)
    order = [(l1[0], p1[0], a1[0]), (l2[0], p2[0], a2[0]), (l1[1], p1[1], a1[1]), (l1[2], p1[2], a1[2]),
             (l2[1], p2[1], a2[1])]
    got = G.FeatureExtractor(batch_size=2).transform(*[[o[k] for o in order] for k in range(3)])["features"]
    want = S.feature_extractor(*[[o[k] for o in order] for k in range(3)])["features"]
    a, b = S.flatten(got), S.flatten(want)
    for k in EXACT:
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
