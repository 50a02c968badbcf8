"""COCO evaluation without a GPU: the pycocotools stand-in of oracle/coco_oracle.py pinned by hand-derived vectors,
the oracle's COCOeval restatement and mcb200.evaluation's host accumulate / summarize against the reference's own
output (tests/golden/cocoeval.npz, written by oracle/make_golden_cocoeval.py), and the new C-ABI symbols."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle import coco_oracle as CO
from oracle import instances_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _rle(m):
    m = np.asarray(m, np.uint8)
    return {"size": list(m.shape), "counts": I.rle_to_string(I.rle_encode(m))}


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(GOLDEN, "cocoeval.npz")) as g:
        return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def golden_files(golden, tmp_path_factory):
    """the fixture's ground-truth and result JSON texts as files -> (gt path, dt path)"""
    d = tmp_path_factory.mktemp("cocoeval")
    for k in ("gt_json", "dt_json"):
        (d / (k + ".json")).write_bytes(golden[k].tobytes())
    return str(d / "gt_json.json"), str(d / "dt_json.json")


# ---------------------------------------------------------------------------------------------------------------------
# the stand-in's mask functions: known answers
# ---------------------------------------------------------------------------------------------------------------------
def test_rle_encode_matches_the_scalar_restatement():
    rs = np.random.RandomState(0)
    cases = [np.zeros((4, 5)), np.ones((4, 5)), np.eye(5), (rs.rand(37, 23) > 0.5), (rs.rand(9, 64) > 0.9)]
    for m in cases:
        assert CO.rle_encode(m) == I.rle_encode(m)
        assert np.array_equal(CO.decode(_rle(m)), (np.asarray(m) != 0).astype(np.uint8))


def test_iou_area_and_crowd_rule_known_answers():
    # column-major: d = [[1, 1], [0, 0]] -> pixels 0 and 2; g = [[1, 0], [1, 0]] -> pixels 0 and 1
    d = _rle([[1, 1], [0, 0]])
    g = _rle([[1, 0], [1, 0]])
    assert CO.area(d) == 2 and list(CO.toBbox(d)) == [0.0, 0.0, 2.0, 1.0]
    o = CO.iou([d], [g, g], [0, 1])
    assert o.shape == (1, 2)
    assert o[0, 0] == 1 / 3          # i = 1, u = 2 + 2 - 1
    assert o[0, 1] == 1 / 2          # crowd: u = area of the detection
    # boxes overlap, masks do not: i == 0 -> 0 (u forced to 1)
    assert CO.iou([_rle([[1, 0], [0, 1]])], [_rle([[0, 1], [1, 0]])], [0])[0, 0] == 0.0
    # boxes that touch without overlapping: the box gate gives 0 before any pixel is counted
    a = np.zeros((4, 4)); a[:, :2] = 1
    b = np.zeros((4, 4)); b[:, 2:] = 1
    assert CO.bb_gate_iou(CO.toBbox([_rle(a)]), CO.toBbox([_rle(b)]), [0])[0, 0] == 0.0
    assert CO.iou([_rle(a)], [_rle(b)], [0])[0, 0] == 0.0
    # a crowd ground truth covering the detection: IoU 1 although the union is larger
    assert CO.iou([_rle(a)], [_rle(np.ones((4, 4)))], [1])[0, 0] == 1.0
    assert CO.iou([_rle(a)], [_rle(np.ones((4, 4)))], [0])[0, 0] == 0.5
    # different mask sizes: -1; an empty list: []
    assert CO.iou([_rle(a)], [_rle(np.ones((4, 5)))], [0])[0, 0] == -1
    assert CO.iou([], [_rle(a)], [0]) == []
    # uncompressed RLE through frPyObjects
    assert CO.frPyObjects({"size": [4, 4], "counts": [8, 8]}, 4, 4) == _rle(b)


# ---------------------------------------------------------------------------------------------------------------------
# the fixture and the evaluation against it
# ---------------------------------------------------------------------------------------------------------------------
def test_fixture_holds_the_quirks(golden):
    gt, dt = json.loads(golden["gt_json"].tobytes()), json.loads(golden["dt_json"].tobytes())
    anns = gt["annotations"]
    assert len(gt["images"]) >= 200
    assert any(a["id"] == 0 for a in anns)
    assert any(a["iscrowd"] for a in anns) and any(a["area"] == 196 for a in anns)
    assert any(a["area"] != CO.area(a["segmentation"]) and a["area"] != 196 for a in anns)
    assert any(a["category_id"] != 100 for a in anns)
    assert any(isinstance(a["segmentation"]["counts"], list) for a in anns)
    gt_imgs, dt_imgs = {a["image_id"] for a in anns}, {d["image_id"] for d in dt}
    all_imgs = {im["id"] for im in gt["images"]}
    assert gt_imgs - dt_imgs and dt_imgs - gt_imgs and all_imgs - gt_imgs - dt_imgs
    per_img = np.bincount([d["image_id"] - 1000 for d in dt])
    assert per_img.max() > 100
    scores = [(d["score"], d["image_id"]) for d in dt]
    assert len({s for s, _ in scores}) < len({(s, i) for s, i in scores})     # equal scores in different images


def test_id0_ground_truth_is_matched_in_the_fixture(golden):
    """the id-0 quirk is exercised: some detection's best match is ground truth 0, stored as 'unmatched'"""
    gt, dt = json.loads(golden["gt_json"].tobytes()), json.loads(golden["dt_json"].tobytes())
    c_gt = CO.COCO()
    c_gt.dataset = gt
    c_gt.createIndex()
    ev = CO.COCOevalOracle(c_gt, c_gt.loadRes(dt), golden["image_ids"], golden["category_ids"], 14)
    ev.evaluate()
    e = [x for x in ev.evalImgs[:len(ev.imgIds)] if x is not None and 0 in x["gtIds"]]
    assert e and (e[0]["gtMatches"][:, e[0]["gtIds"].index(0)] > 0).any()


def test_oracle_cocoeval_reproduces_the_reference_bit_for_bit(golden, golden_files):
    c_gt = CO.COCO(golden_files[0])
    ev = CO.COCOevalOracle(c_gt, c_gt.loadRes(golden_files[1]), golden["image_ids"],
                           golden["category_ids"], int(golden["small_annotations_size"]))
    ev.evaluate()
    ev.accumulate()
    ev.summarize()
    tb = CO.flat_tables(ev)
    for k in ("nd", "ng", "present", "dt_scores", "dt_ids", "dt_match", "dt_ignore", "gt_ignore", "iou"):
        assert np.array_equal(tb[k], golden[k]), k
    assert np.array_equal(ev.precision, golden["precision"]) and np.array_equal(ev.recall, golden["recall"])
    assert np.array_equal(ev.stats, golden["stats"])
    assert (ev.stats[0], ev.stats[3]) == tuple(golden["ap_ar"])


def test_host_accumulate_and_summarize_reproduce_the_reference(mcb, golden):
    from mcb200 import evaluation as E
    precision, recall = E.accumulate(golden["nd"], golden["ng"], golden["present"], golden["dt_scores"],
                                     golden["dt_match"], golden["dt_ignore"], golden["gt_ignore"],
                                     len(golden["category_ids"]), len(golden["image_ids"]))
    assert np.array_equal(precision, golden["precision"]) and np.array_equal(recall, golden["recall"])
    stats = E.summarize(precision, recall)
    assert np.array_equal(stats, golden["stats"])
    assert (stats[0], stats[3]) == tuple(golden["ap_ar"])


def test_accumulate_counts_a_match_to_ground_truth_id_0_as_unmatched(mcb):
    """tps = dtm & ~dtIg tests the stored id: one detection matched to ground truth 0 is a false positive"""
    from mcb200 import evaluation as E
    A, T = 3, 10
    for gid, want in ((0, 0.0), (7, 1.0)):
        dm = np.full((A, T, 1), gid, np.int64)
        p, r = E.accumulate([1], [1], [True], np.array([0.9]), dm, np.zeros((A, T, 1), np.uint8),
                            np.zeros((A, 1), np.uint8), 1, 1)
        assert r[0, 0, 0, 2] == want
    # no ground truth at all: -1 everywhere
    p, r = E.accumulate([1], [0], [True], np.array([0.9]), np.zeros((A, T, 1), np.int64),
                        np.zeros((A, T, 1), np.uint8), np.zeros((A, 0), np.uint8), 1, 1)
    assert (p == -1).all() and (r == -1).all()
    assert (E.summarize(p, r) == -1).all()


def test_area_ranges_are_the_references():
    from mcb200 import evaluation as E
    rng = E.area_ranges(14)
    assert rng.tolist() == [[0, 1e10], [0, 196], [196, 1e10]]
    assert np.array_equal(E.IOU_THRS, np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05) + 1), endpoint=True))
    assert np.array_equal(E.REC_THRS, np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01) + 1), endpoint=True))


def test_library_exports_the_evaluation_entry_points(mcb):
    lib = ctypes.CDLL(os.path.join(ROOT, "open-solution-mapping-challenge_b200", "libmcb200.so"))
    for name in ("mcb_rle_pair_iou", "mcb_coco_match"):
        assert hasattr(lib, name), name


def test_polygon_ground_truth_needs_pycocotools(mcb):
    from mcb200 import evaluation as E
    try:
        import pycocotools.mask  # noqa: F401
        pytest.skip("pycocotools is installed: polygons are converted")
    except ImportError:
        pass
    with pytest.raises(NotImplementedError, match="frPyObjects"):
        E.segmentation_counts([[0, 0, 4, 0, 4, 4]], 8, 8)
    cnts, size = E.segmentation_counts({"size": [4, 4], "counts": [8, 8]}, 4, 4)
    assert cnts.tolist() == [8, 8] and size == (4, 4)
