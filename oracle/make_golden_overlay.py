"""TEST INFRASTRUCTURE — writes tests/golden/overlay.npz from the UNMODIFIED reference
`src.preparation.overlay_mask_one_image`, imported through oracle/ref_shim.py.  This generator then points the
module's pycocotools (`cocomask.frPyObjects` / `decode`) and skimage (`binary_erosion`, `binary_dilation`,
`rectangle`) names at oracle/overlay_oracle.py, and its `imwrite` / `joblib.dump` at in-memory captures, in its own
process only: the other generators keep oracle/ref_shim.py's inert stubs.

    MCB_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_overlay

Four configurations (erode, dilate, border_width) in CONFIGS, each on its own seeded annotation set (multi-polygon
annotations only where erode == 0, since the reference cannot erode them) of mostly small non-square images and two
of 300 x 300, with images without annotations among them.  Keys: `json_<c>` (the annotation file, uint8), and per
image `c<c>_i<i>_mask`, `_dist`, `_sizes` as the reference wrote them.
"""
import json
import os
import tempfile
import types

import numpy as np

from . import overlay_oracle as O
from . import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "overlay.npz")
CONFIGS = ((0, 0, 0), (3, 0, 0), (3, 2, 0), (0, 0, 2))
SIZES = ((40, 56), (33, 47), (64, 48), (52, 52), (29, 71), (48, 64), (300, 300), (300, 300))
SMALL = 14


def annotation_set(config_index):
    """-> COCO dict of the configuration's seeded synthetic images"""
    erode = CONFIGS[config_index][0]
    rs = np.random.RandomState(1000 + config_index)
    images, anns = [], []
    for i, (h, w) in enumerate(SIZES + SIZES[:2]):
        iid = 10 * i + 7
        images.append({"id": iid, "file_name": "img_%03d.jpg" % i, "height": h, "width": w})
        if i == 2:
            continue                                      # an image without annotations
        nb = rs.randint(10, 30) if h == 300 else rs.randint(2, 9)
        anns += O.synthetic_image_annotations(rs, h, w, nb, iid, 1000 * i + 1, multi_polygon=erode == 0)
    return {"images": images, "annotations": anns, "categories": [{"id": 100, "name": "building"}]}


class _Coco:
    """the three COCO methods overlay_mask_one_image calls, with pycocotools' ordering"""

    def __init__(self, d):
        self.imgs = {im["id"]: im for im in d["images"]}
        self.anns = {a["id"]: a for a in d["annotations"]}
        self.img_to_anns = {}
        for a in d["annotations"]:
            self.img_to_anns.setdefault(a["image_id"], []).append(a)

    def loadImgs(self, i):
        return [self.imgs[i]]

    def getAnnIds(self, imgIds, catIds):
        return [a["id"] for a in self.img_to_anns.get(imgIds, []) if a["category_id"] in catIds]

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]


def main():
    ref_shim.install()
    import src.preparation as prep
    captured = {}
    prep.cocomask = types.SimpleNamespace(frPyObjects=lambda s, h, w: (O.fr_py_objects(s, h, w), h, w),
                                          decode=lambda r: O.decode_stack(*r))
    prep.binary_erosion, prep.binary_dilation, prep.rectangle = O.binary_erosion, O.binary_dilation, O.rectangle
    prep.imwrite = lambda path, m: captured.__setitem__("mask", np.array(m))
    prep.joblib = types.SimpleNamespace(
        dump=lambda a, path: captured.__setitem__("dist" if "/distances/" in path else "sizes", np.array(a)))
    out = {}
    tmp = tempfile.mkdtemp(prefix="mcb_overlay_")
    for c, (erode, dilate, border) in enumerate(CONFIGS):
        d = annotation_set(c)
        out["json_%d" % c] = np.frombuffer(json.dumps(d).encode(), np.uint8)
        coco = _Coco(d)
        for i, im in enumerate(d["images"]):
            captured.clear()
            prep.overlay_mask_one_image(im["id"], "train", tmp, coco, [None, 100], erode, dilate, border, SMALL)
            for k in ("mask", "dist", "sizes"):
                out["c%d_i%d_%s" % (c, i, k)] = captured[k]
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
