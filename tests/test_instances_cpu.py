"""CPU tests that pin oracle/instances_oracle.py:
  * COCO RLE (pycocotools is absent): hand-derived known-answer vectors of maskApi.c's rleEncode / rleToString /
    rleToBbox, plus encode -> string -> decode round trips;
  * test-time augmentation: against the outputs of the reference's own functions (tests/golden/live_reference.npz),
    skimage.rotate at quarter turns assumed exact;
  * NMS / features: against the reference's NMS output; the contour-length rule the CUDA kernel uses
    (mask pixels with a 4-neighbour outside) against cv2 itself."""
import json
import os

import numpy as np
import pytest

from oracle import instances_oracle as I
from oracle import synthetic


def test_rle_known_answers():
    # 2x2 [[0,1],[1,1]]: column-major scan 0,1,1,1 -> counts [1,3]; "1" = 49, "3" = 51; the run of ones crosses the
    # column boundary -> full-height bbox
    m = np.array([[0, 1], [1, 1]], np.uint8)
    assert I.rle_encode(m) == [1, 3]
    assert I.rle_to_string([1, 3]) == b"13"
    assert I.rle_to_bbox([1, 3], 2, 2) == [0.0, 0.0, 2.0, 2.0]
    # all background, h=3 w=2 -> one count, empty bbox
    z = np.zeros((3, 2), np.uint8)
    assert I.rle_encode(z) == [6] and I.rle_to_string([6]) == b"6" and I.rle_to_bbox([6], 3, 2) == [0.0] * 4
    # mask that starts with a one: a leading empty run of zeros
    m = np.array([[1, 0], [0, 0]], np.uint8)
    assert I.rle_encode(m) == [0, 1, 3]
    assert I.rle_to_string([0, 1, 3]) == b"013"
    assert I.rle_to_bbox([0, 1, 3], 2, 2) == [0.0, 0.0, 1.0, 1.0]
    # two-character groups and delta coding: 40 = 8 + 32*1 -> (8|0x20)+48='X', 1+48='1'; 4th count 30-2=28:
    # 28 has bit 0x10 set and the rest is 0 != -1 -> continue: (28|0x20)+48='l', then 0 -> '0'
    assert I.rle_to_string([40, 2, 5, 30]) == b"X125l0"
    # negative delta: 3-10 = -7 -> low five bits 25, remainder -1, bit 0x10 set and rest == -1 -> stop: 25+48='I'
    assert I.rle_to_string([5, 10, 7, 3]) == b"5:7I"
    for cnts in ([40, 2, 5, 30], [5, 10, 7, 3], [0, 1, 3], [6], [1000, 3, 70000, 1, 2, 900000]):
        assert I.rle_from_string(I.rle_to_string(cnts)) == cnts


def test_rle_bbox_is_tight_without_column_crossing_runs():
    rs = np.random.RandomState(3)
    for _ in range(20):
        h, w = rs.randint(3, 12), rs.randint(3, 12)
        m = np.zeros((h, w), np.uint8)
        y0, x0 = rs.randint(0, h - 1), rs.randint(0, w - 1)
        y1, x1 = rs.randint(y0 + 1, h + 1), rs.randint(x0 + 1, w + 1)
        m[y0:y1, x0:x1] = 1
        if y0 == 0 and y1 == h and x1 - x0 > 1:
            continue  # full-height boxes cross columns
        cnts = I.rle_encode(m)
        assert sum(cnts) == h * w
        assert I.rle_to_bbox(cnts, h, w) == [float(x0), float(y0), float(x1 - x0), float(y1 - y0)]
        # decode: alternate runs
        flat = np.concatenate([np.full(c, i % 2, np.uint8) for i, c in enumerate(cnts)])
        assert np.array_equal(flat.reshape((w, h)).T, m)


def test_contour_rule_matches_cv2():
    """drawContours(findContours(RETR_TREE, CHAIN_APPROX_NONE), thickness 1) marks exactly the mask pixels that have a
    4-neighbour outside the mask (image border = outside), holes included"""
    cv2 = pytest.importorskip("cv2")
    rs = np.random.RandomState(11)
    for trial in range(12):
        h, w = rs.randint(8, 40), rs.randint(8, 40)
        m, _ = synthetic.rectangles_mask(rs, h, w, n_rect=4, lo=3, hi=12)
        if trial % 3 == 0 and h > 12 and w > 12:
            m[4:9, 4:9] = 1
            m[6, 6] = 0                      # a hole
        if trial % 4 == 1:
            m = (rs.rand(h, w) > 0.45).astype(np.uint8)   # ragged blobs, diagonal contacts
        p = np.pad(m, 1)
        inner = (p[:-2, 1:-1] & p[2:, 1:-1] & p[1:-1, :-2] & p[1:-1, 2:]).astype(bool)
        rule = int(np.count_nonzero(m.astype(bool) & ~inner))
        assert I.get_contour_length(m.astype(bool)) == rule, trial


def test_tta_and_nms_oracles_live_against_reference():
    """against the outputs of the reference's src/loaders.py test-time augmentation and src/postprocessing.py NMS on the
    same seeded inputs (tests/golden/live_reference.npz, oracle/make_golden.py live)"""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "live_reference.npz"))
    specs = I.tta_specs()
    # TestTimeAugmentationGenerator(flip_ud, flip_lr, rotation).transform on two images
    assert json.loads(str(g["tta_params_json"])) == specs * 2 and g["tta_img_ids"].tolist() == [0] * 16 + [1] * 16
    assert len(specs) == 16
    rs = np.random.RandomState(5)
    img = rs.randint(0, 255, (12, 12, 3)).astype(np.uint8)
    preds = []
    for i, p in enumerate(specs):
        assert np.array_equal(g["tta_forward"][i], I.tta_transform(img, p))
        pr = rs.rand(2, 12, 12).astype(np.float32)
        assert np.array_equal(g["tta_inverse"][i], I.tta_inverse(pr, p))
        preds.append(pr)
    for method in ("gmean", "mean", "max", "min"):
        want = I.tta_aggregate(preds * 2, specs * 2, [0] * 16 + [1] * 16, method)
        assert len(want) == len(g["tta_agg_" + method])
        for a, b in zip(g["tta_agg_" + method], want):
            assert np.array_equal(a, b)
    # NMS on two overlapping layers
    lab = np.zeros((2, 20, 20), np.int32)
    lab[0, 2:8, 2:8] = 1
    lab[0, 10:18, 10:18] = 2
    lab[1, 3:8, 2:8] = 1          # IoU 30/36 with layer 0 label 1
    lab[1, 12:14, 12:14] = 2      # small: IoU 4/64
    s1 = [[0.9, 0.5], [0.8, 0.7]]
    s2 = [[0.9, 0.5], [0.8, 0.7]]
    a = g["nms_scores"].tolist()                 # pp.remove_overlapping_masks(lab, s1, 0.5)
    _, b = I.remove_overlapping_masks(lab, s2, 0.5)
    assert a == b == [[0.9, 0.5], [0, 0.7]]
    # features without annotations
    prob = rs.rand(2, 20, 20)
    # (the reference's get_contour unpacks cv2 3's three return values and cannot run on cv2 4; everything else of
    # get_features_for_mask is restated line by line)
    feats = I.instance_features(lab, prob)
    assert feats[0][0]["area"] == 36 and feats[0][0]["bbox_area"] == 36 and feats[0][0]["contour_length"] == 20
