"""CPU pins of the target preparation from COCO polygons: oracle/overlay_oracle.py's rleFrPoly restatement against
vectors derived by hand from pycocotools' maskApi.c and the integer-box property, its overlay_mask_one_image against
the unmodified reference (tests/golden/overlay.npz), and the host side of mcb200.preparation (JSON indexing, the edge
table, the errors raised before any device work)."""
import json
import os

import numpy as np
import pytest

from oracle import make_golden_overlay as MG
from oracle import overlay_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "overlay.npz")

# (polygon, h, w, RLE counts), each worked through rleFrPoly by hand (vertices scaled by 5, edges walked along
# the major axis, column crossings at xd = (u + .5) / 5 - .5 integral, toggles at x * h + y):
KNOWN = [
    # box (0,1)-(1,5), h=3 w=2: crossings at (0, ceil(.6)=1) and (0, clamp(4.6)=h=3): the bottom toggle is the y == h
    # position, row 0 of column 1 -> column 0 rows 1..2
    ([0, 1, 1, 1, 1, 5, 0, 5], 3, 2, [1, 2, 3]),
    # the same box clockwise
    ([0, 5, 1, 5, 1, 1, 0, 1], 3, 2, [1, 2, 3]),
    # the same box with a repeated vertex: the degenerate edge is one point (5, (int)NaN) between equal columns
    ([0, 1, 1, 1, 1, 1, 1, 5, 0, 5], 3, 2, [1, 2, 3]),
    # collinear (0,0)-(2,2): toggles {0, 0, 4, 4} cancel pairwise -> empty
    ([0, 0, 1, 1, 2, 2], 3, 3, [9]),
    # sub-pixel and negative vertices (-.3,-.3)-(1.2,.8) -> scaled (-1,-1)-(6,4); (int)(-.5) = 0 moves the left edge
    # to u = 0, and only column 0 has a crossing (u = 3 going right, u = 2 going left): toggles {0, 1} -> pixel (0, 0)
    ([-.3, -.3, 1.2, -.3, 1.2, .8, -.3, .8], 2, 3, [0, 1, 5]),
    # every vertex beyond every edge: tops clamp to y = 0, bottoms to y = h; {0, 2, 2, 4, 4, 6} -> all ones
    ([-10, -10, 20, -10, 20, 20, -10, 20], 2, 3, [0, 6]),
]


@pytest.mark.parametrize("poly,h,w,counts", KNOWN)
def test_rle_fr_poly_known_answers(poly, h, w, counts):
    assert O.rle_fr_poly(poly, h, w) == counts
    assert np.array_equal(O.decode(counts, h, w), O.polygon_mask(poly, h, w))


def test_integer_boxes_rasterise_to_their_pixels():
    rs = np.random.RandomState(0)
    for _ in range(400):
        h, w = rs.randint(1, 24, 2)
        x0, y0 = rs.randint(-8, w + 4), rs.randint(-8, h + 4)
        x1, y1 = x0 + rs.randint(1, 20), y0 + rs.randint(1, 20)
        box = [x0, y0, x1, y0, x1, y1, x0, y1]
        if rs.rand() < 0.5:
            box = list(np.asarray(box).reshape(4, 2)[::-1].reshape(-1))
        want = np.zeros((h, w), np.uint8)
        want[max(y0, 0):max(min(y1, h), 0), max(x0, 0):max(min(x1, w), 0)] = 1
        assert np.array_equal(O.polygon_mask(box, h, w), want), (box, h, w)


def test_merge_is_the_union_and_encode_inverts_decode():
    rs = np.random.RandomState(1)
    for _ in range(50):
        h, w = rs.randint(5, 40, 2)
        polys = [O.building_polygon(rs, h, w, size=rs.uniform(3, 20)) for _ in range(rs.randint(1, 4))]
        union = np.zeros((h, w), np.uint8)
        for p in polys:
            union |= O.polygon_mask(p, h, w)
        counts = O.ann_to_rle(polys, h, w)
        assert sum(counts) == h * w and np.array_equal(O.decode(counts, h, w), union)


def _golden_case(g, c):
    d = json.loads(g["json_%d" % c].tobytes().decode())
    by_img = {}
    for a in d["annotations"]:
        by_img.setdefault(a["image_id"], []).append(a)
    return d, by_img


@pytest.mark.parametrize("c", range(len(MG.CONFIGS)))
def test_oracle_overlay_matches_the_reference(c):
    g = np.load(GOLDEN)
    erode, dilate, border = MG.CONFIGS[c]
    d, by_img = _golden_case(g, c)
    for i, im in enumerate(d["images"]):
        mask, dist, sizes = O.overlay_mask_one_image(by_img.get(im["id"], []), im["height"], im["width"], (None, 100),
                                                     erode, dilate, border, MG.SMALL)
        for k, got in (("mask", mask), ("dist", dist), ("sizes", sizes)):
            want = g["c%d_i%d_%s" % (c, i, k)]
            assert got.dtype == want.dtype and np.array_equal(got, want), (c, i, k)


def test_golden_covers_the_configured_cases():
    g = np.load(GOLDEN)
    for c, (erode, dilate, border) in enumerate(MG.CONFIGS):
        d, by_img = _golden_case(g, c)
        n = len(d["images"])
        assert any(g["c%d_i%d_sizes" % (c, i)].dtype == np.uint8 for i in range(n))      # an image without buildings
        assert any(g["c%d_i%d_sizes" % (c, i)].dtype == np.int64 for i in range(n))
        if border:
            assert any((g["c%d_i%d_mask" % (c, i)] == 2).any() for i in range(n))
        multi = any(len(a["segmentation"]) > 1 for a in d["annotations"])
        assert multi == (erode == 0)
        if erode:   # instances eroded to nothing: scipy's no-background distance transform enters the distances
            assert sum(O.eroded_to_empty(by_img.get(im["id"], []), im["height"], im["width"], erode)
                       for im in d["images"]) > 0


def test_coco_index_keeps_pycocotools_order(tmp_path, mcb):
    from mcb200.preparation import coco_index
    d = {"images": [{"id": 5, "file_name": "a.jpg"}, {"id": 2, "file_name": "b.jpg"}, {"id": 9, "file_name": "c.jpg"}],
         "annotations": [{"id": 1, "image_id": 2, "x": 0}, {"id": 2, "image_id": 5, "x": 1},
                         {"id": 3, "image_id": 2, "x": 2}]}
    p = tmp_path / "annotation.json"
    p.write_text(json.dumps(d))
    images, anns = coco_index(str(p))
    assert [im["id"] for im in images] == [5, 2, 9]
    assert [a["x"] for a in anns[2]] == [0, 2] and [a["x"] for a in anns[5]] == [1] and anns[9] == []


def _ann(segm, cid=100):
    return {"id": 1, "image_id": 1, "category_id": cid, "segmentation": segm}


def test_multi_polygon_annotations_cannot_be_eroded(mcb):
    from mcb200.preparation import overlay_batch
    two = _ann([[1, 1, 8, 1, 8, 8, 1, 8], [10, 10, 15, 10, 15, 15]])
    with pytest.raises(ValueError):
        O.overlay_mask_one_image([two], 20, 20, erode=3)
    with pytest.raises(ValueError):
        overlay_batch([[two]], 20, 20, erode=3)
    with pytest.raises(ValueError):
        overlay_batch([[_ann([[1, 1, 8, 1, 8, 8]])]], 20, 20, erode=-1)


@pytest.mark.parametrize("segm,form", [([[1, 2, 3, 4]], "bbox"), ([1, 2, 3, 4], "bbox"),
                                       ({"size": [20, 20], "counts": [400]}, "RLE")])
def test_bbox_and_rle_forms_are_not_implemented(mcb, segm, form):
    from mcb200.preparation import overlay_batch
    with pytest.raises(NotImplementedError, match=form):
        O.overlay_mask_one_image([_ann(segm)], 20, 20)
    with pytest.raises(NotImplementedError, match=form):
        overlay_batch([[_ann(segm)]], 20, 20)


@pytest.mark.parametrize("segm", [[[1, 2, 3]], [[1, 2], [1, 2, 3, 4, 5, 6]], []])
def test_segmentations_pycocotools_rejects_are_rejected(mcb, segm):
    from mcb200.preparation import overlay_batch
    with pytest.raises(ValueError):
        O.overlay_mask_one_image([_ann(segm)], 20, 20)
    with pytest.raises(ValueError):
        overlay_batch([[_ann(segm)]], 20, 20)


def test_edge_table_matches_the_oracle_walk(mcb):
    from mcb200.preparation import _edge_table, polygons_csr
    rs = np.random.RandomState(2)
    polys = [O.building_polygon(rs, 30, 40) for _ in range(20)] + [[3.3, 4.4, 3.3, 4.4], []]
    xy, off = polygons_csr(polys)
    edge_xy, edge_pt, edge_plane = _edge_table(xy, off)
    for p, poly in enumerate(polys):
        x, y = O.scaled_vertices(poly)
        rows = edge_plane == p
        assert np.array_equal(edge_xy[rows, 0], x) and np.array_equal(edge_xy[rows, 1], y)
        u, _ = O.boundary_points(poly)
        e = np.nonzero(rows)[0]
        assert (edge_pt[e[-1] + 1] - edge_pt[e[0]] if e.size else 0) == len(u)
    with pytest.raises(ValueError):
        _edge_table(np.array([0.0, 0.0, 5e8, 0.0]), np.array([0, 2]))
