"""TEST INFRASTRUCTURE — writes tests/golden/scoring_features.npz from the UNMODIFIED reference
`src.postprocessing.get_features_for_image`, `FeatureExtractor` and `ScoreImageJoiner`, imported through
oracle/ref_shim.py with CATEGORY_LAYERS = [1, 19].

    MCB_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_scoring

Stand-ins, in this process only: pycocotools.mask is oracle/coco_oracle.py's, with `frPyObjects` of a polygon list
taken from oracle/overlay_oracle.py's rleFrPoly restatement (one RLE per polygon, as pycocotools returns them); the
reference's OpenCV 3 unpacking `_, contours, hierarchy = cv2.findContours(...)` gets OpenCV 4's pair with a leading
None, as oracle/instances_oracle.py:226-230 reads it.  The inputs are oracle/scoring_oracle.py's `scoring_case()`
(seeded: 20 images of 300 x 300, 20 layers).  The reference replaces each annotation's polygons by its first polygon's
RLE in place, so every run gets its own deep copy.

Keys: the flat table of oracle/scoring_oracle.py `flatten` (counts, iou_none, dtypes and one array per column) of
get_features_for_image on every image with annotations (`ann_*`) and of FeatureExtractor.transform without annotations
(`none_*`); the generator asserts that FeatureExtractor.transform with annotations equals the per-image run and that
ScoreImageJoiner pairs its inputs.  Regenerating reproduces every array bit for bit.
"""
import copy
import os
import types

import numpy as np

from . import coco_oracle as CO
from . import overlay_oracle as OV
from . import ref_shim
from . import scoring_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "scoring_features.npz")


def _fr_py_objects(segm, h, w):
    if isinstance(segm, (list, tuple)) and OV.segmentation_form(segm) == "polygons":
        return [{"size": [h, w], "counts": c} for c in OV.fr_py_objects(segm, h, w)]
    return CO.frPyObjects(segm, h, w)


def reference_postprocessing():
    """src.postprocessing with the stand-ins and CATEGORY_LAYERS = [1, 19]"""
    import sys
    ref_shim.install()
    if "src.utils" in sys.modules or "src.postprocessing" in sys.modules:
        raise RuntimeError("the pycocotools stand-in must be installed before src.utils is imported")
    pc = ref_shim._module("pycocotools")
    pc.mask = ref_shim._module("pycocotools.mask", **dict(vars(CO.mask), frPyObjects=_fr_py_objects))
    pc.coco = ref_shim._module("pycocotools.coco", COCO=CO.COCO)
    import cv2
    import src.pipeline_config as cfg
    import src.postprocessing as pp
    cfg.CATEGORY_LAYERS = pp.CATEGORY_LAYERS = list(S.SCORING_LAYERS)
    pp.cv2 = types.SimpleNamespace(findContours=lambda *a: (None,) + tuple(cv2.findContours(*a)),
                                   drawContours=cv2.drawContours, RETR_TREE=cv2.RETR_TREE,
                                   CHAIN_APPROX_NONE=cv2.CHAIN_APPROX_NONE)
    return pp


def frames_equal(a, b):
    import pandas as pd
    assert len(a) == len(b)
    for ia, ib in zip(a, b):
        assert len(ia) == len(ib)
        for fa, fb in zip(ia, ib):
            pd.testing.assert_frame_equal(fa, fb, check_exact=True)


def main():
    pp = reference_postprocessing()
    probs, labels, annotations = S.scoring_case()
    per_image = [pp.get_features_for_image(lab, pr, ann)
                 for lab, pr, ann in zip(labels, probs, copy.deepcopy(annotations))]
    fe = pp.FeatureExtractor().transform(list(labels), list(probs), copy.deepcopy(annotations))['features']
    frames_equal(per_image, fe)
    none = pp.FeatureExtractor().transform(list(labels), list(probs))['features']
    scores = [[list(np.arange(len(df)) / 10.) for df in image] for image in none]
    images = list(labels)
    joined = pp.ScoreImageJoiner().transform(images, scores)['images_with_scores']
    assert len(joined) == len(images) and all(a[0] is b and a[1] is s for a, b, s in zip(joined, images, scores))
    out = {}
    for name, feats in (("ann", per_image), ("none", none)):
        out.update({"%s_%s" % (name, k): v for k, v in S.flatten(feats).items()})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "instances", int(out["ann_counts"].sum()))


if __name__ == "__main__":
    main()
