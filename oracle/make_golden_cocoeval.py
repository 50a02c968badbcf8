"""TEST INFRASTRUCTURE — writes tests/golden/cocoeval.npz from the UNMODIFIED reference `src.utils.coco_evaluation`
and its vendored COCOeval (src/cocoeval.py), run on oracle/coco_oracle.py's pycocotools stand-in, which this generator
installs in place of oracle/ref_shim.py's inert pycocotools stub (the other fixtures keep the stub).  The npz holds the
ground-truth and result JSON texts (`gt_json`, `dt_json`, uint8) next to the reference's tables.

    MCB_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_cocoeval

The seeded synthetic case (`synthetic_case`) holds, on 300 x 300 images: overlapping and crowd ground truths, a ground
truth with id 0, JSON areas of exactly 14**2 = 196 and JSON areas unlike the mask's pixel count, a ground truth of a
category outside catIds, images with only ground truths, only detections and neither, score ties across images, an
image with more than 100 detections, boxes that touch without overlapping, and compressed as well as uncompressed RLE
ground truths.  The reference's results carry a bbox (src/utils.py:109-111), so pycocotools' loadRes takes its bbox
branch and a detection's area is its box's w * h; the detections here carry one too.

numpy 2 bridges, for the duration of the run only: `np.float` (removed in numpy 1.24) is set to `float`, and
`np.linspace` gets int(num) (src/cocoeval.py:507-508 passes np.round(...) + 1, a float).
"""
import json
import os
import sys
import tempfile

import numpy as np

from . import coco_oracle as CO
from . import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
SIZE = 300
CAT, OTHER_CAT = 100, 200
SMALL = 14


def _rect(y0, x0, h, w):
    m = np.zeros((SIZE, SIZE), np.uint8)
    m[max(y0, 0):max(y0 + h, 0), max(x0, 0):max(x0 + w, 0)] = 1
    return m


def _blob(rs):
    """a rectangle or an ellipse somewhere in the image"""
    h, w = rs.randint(4, 60), rs.randint(4, 60)
    y0, x0 = rs.randint(0, SIZE - h), rs.randint(0, SIZE - w)
    if rs.rand() < 0.5:
        return _rect(y0, x0, h, w)
    yy, xx = np.mgrid[:SIZE, :SIZE]
    cy, cx = y0 + h / 2., x0 + w / 2.
    return (((yy - cy) / (h / 2.)) ** 2 + ((xx - cx) / (w / 2.)) ** 2 <= 1).astype(np.uint8)


def _rle(m, compressed=True):
    cnts = CO.rle_encode(m)
    if compressed:
        return {"size": [SIZE, SIZE], "counts": CO.I.rle_to_string(cnts).decode("ascii")}
    return {"size": [SIZE, SIZE], "counts": cnts}


def synthetic_case(n_images=240, seed=2024):
    """-> (ground-truth dict, result list, image ids, category ids)"""
    rs = np.random.RandomState(seed)
    images, anns, results = [], [], []
    next_id = 1
    score_levels = np.round(np.linspace(0.05, 1.0, 20), 2)     # coarse levels: ties across images
    for n in range(n_images):
        img_id = 1000 + n
        images.append({"id": img_id, "height": SIZE, "width": SIZE, "file_name": "%d.png" % img_id})
        kind = n % 12
        n_gt = 0 if kind in (3, 7) else rs.randint(1, 9)         # 3: detections only, 7: neither
        n_dt_extra = 0 if kind in (5, 7) else rs.randint(0, 4)  # 5: ground truths only
        gts = []
        for g in range(n_gt):
            m = _blob(rs)
            if g > 0 and rs.rand() < 0.3:                        # overlap the previous ground truth
                prev = gts[-1][0]
                m = np.roll(np.roll(prev, rs.randint(-8, 9), 0), rs.randint(-8, 9), 1)
                m[:, :1] = 0
            crowd = int(rs.rand() < 0.1) if (n, g) != (0, 0) else 0
            pix = int(m.sum())
            r = rs.rand()
            area = 196 if r < 0.08 else (float(pix) * rs.uniform(0.5, 1.5) if r < 0.2 else pix)
            gts.append((m, crowd, area))
        for g, (m, crowd, area) in enumerate(gts):
            if n == 0 and g == 0:
                ann_id = 0                                       # a ground truth with id 0
            else:
                ann_id = next_id
                next_id += 1
            cat = OTHER_CAT if (n % 17 == 4 and g == 0) else CAT
            anns.append({"id": ann_id, "image_id": img_id, "category_id": cat, "iscrowd": crowd, "area": area,
                         "segmentation": _rle(m, compressed=(ann_id % 5 != 2)),
                         "bbox": [float(v) for v in CO.toBbox(_rle(m))]})
        dets = []
        if kind not in (5, 7):
            for m, _, _ in gts:
                if rs.rand() < 0.8:
                    d = np.roll(np.roll(m, rs.randint(-4, 5), 0), rs.randint(-4, 5), 1)
                    if rs.rand() < 0.3:
                        d = d * (rs.rand(SIZE, SIZE) < 0.9)
                    if d.any():
                        dets.append(d)
            for _ in range(n_dt_extra):
                dets.append(_blob(rs))
            if gts and n % 9 == 1:                               # a box that touches a ground truth's box
                bb = CO.toBbox(_rle(gts[0][0]))
                x1 = int(bb[0] + bb[2])
                if x1 + 5 <= SIZE:
                    dets.append(_rect(int(bb[1]), x1, int(bb[3]), 5))
        if n == 0:                                               # a detection that is ground truth 0's mask
            dets.append(gts[0][0].copy())
        if n == 10:                                              # more than 100 detections in one image
            for q in range(120):
                y0, x0 = (q // 11) * 27, (q % 11) * 27
                dets.append(_rect(y0, x0, 12 + q % 7, 10 + q % 5))
        for d in dets:
            rle = _rle(d)
            results.append({"image_id": img_id, "category_id": CAT, "score": float(rs.choice(score_levels)),
                            "segmentation": rle, "bbox": [float(v) for v in CO.toBbox(rle)]})
    gt = {"images": images, "annotations": anns, "categories": [{"id": CAT, "name": "building"},
                                                               {"id": OTHER_CAT, "name": "other"}]}
    return gt, results, [im["id"] for im in images], [CAT]


def run_reference(gt_path, dt_path, image_ids, category_ids, small):
    """-> (the reference's COCOeval instance, (AP, AR)) of src.utils.coco_evaluation"""
    ref_shim.install()
    if "src.utils" in sys.modules:
        raise RuntimeError("the pycocotools stand-in must be installed before src.utils is imported")
    pc = ref_shim._module("pycocotools")
    pc.mask = ref_shim._module("pycocotools.mask", **vars(CO.mask))
    pc.coco = ref_shim._module("pycocotools.coco", COCO=CO.COCO)
    import src.utils as ut
    captured = []

    class _Capture(ut.COCOeval):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            captured.append(self)

    linspace, had_float = np.linspace, hasattr(np, "float")
    ut.COCOeval, np.float = _Capture, float
    np.linspace = lambda start, stop, num=50, **kw: linspace(start, stop, int(num), **kw)
    try:
        ap_ar = ut.coco_evaluation(gt_path, dt_path, image_ids, category_ids, small)
    finally:
        np.linspace = linspace
        if not had_float:
            del np.float
    return captured[0], ap_ar


def main():
    gt, results, image_ids, category_ids = synthetic_case()
    texts = {"gt_json": json.dumps(gt), "dt_json": json.dumps(results)}
    tmp = tempfile.mkdtemp(prefix="mcb_cocoeval_")
    paths = {}
    for k, t in texts.items():
        paths[k] = os.path.join(tmp, k + ".json")
        with open(paths[k], "w") as f:
            f.write(t)
    ev, ap_ar = run_reference(paths["gt_json"], paths["dt_json"], image_ids, category_ids, SMALL)
    tb = CO.flat_tables(ev)
    out = os.path.join(OUT, "cocoeval.npz")
    np.savez_compressed(out, **{k: np.frombuffer(t.encode("ascii"), np.uint8) for k, t in texts.items()},
                        image_ids=np.asarray(image_ids, np.int64),
                        category_ids=np.asarray(category_ids, np.int64), small_annotations_size=SMALL,
                        precision=ev.eval['precision'], recall=ev.eval['recall'], stats=np.asarray(ev.stats),
                        ap_ar=np.asarray(ap_ar, np.float64), **tb)
    print("wrote", out, "AP/AR", ap_ar)


if __name__ == "__main__":
    main()
