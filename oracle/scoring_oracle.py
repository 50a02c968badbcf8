"""TEST INFRASTRUCTURE — numpy restatement of the reference's second-level scoring features (src/postprocessing.py:18-33,
261-337): get_features_for_image, get_mask_with_iou, get_iou_matrix, get_iou, FeatureExtractor and ScoreImageJoiner.
Only tests/ and scripts/ import this file.

pycocotools is not installed here: `frPyObjects(segm, h, w)[0]` of a polygon segmentation is
oracle/overlay_oracle.py's rleFrPoly restatement of the FIRST polygon, and `cocomask.iou` is oracle/coco_oracle.py's
(decoded masks, pixel counts, with pycocotools' bounding-box gate).  The per-mask features are
oracle/instances_oracle.py's, cv2 contours included.  The restatement is pinned bit for bit against
tests/golden/scoring_features.npz, which oracle/make_golden_scoring.py writes from the unmodified reference.

`scoring_case` makes the seeded inputs the golden and the GPU tests share: float64 probabilities (what the reference's
resize hands to the scoring pipelines), their [1, 19] label layers and COCO polygon annotations: random buildings
(some multi-polygon, some overlapping, one covering the whole image, one image without any) and, from image 3 on,
boxes laid over instances, single or multi-polygon, so that many IoUs are high.  `ScoringRandomForest` restates the
reference's host scoring model (src/models.py:250-282) with a seeded train/validation split.
"""
import numpy as np

from . import coco_oracle as CO
from . import instances_oracle as I
from . import overlay_oracle as OV

CATEGORY_IDS = (None, 100)
SCORING_LAYERS = (1, 19)
COLUMNS = ('iou', 'threshold', 'area', 'mean_prob', 'max_prob', 'bbox_ar', 'bbox_area', 'bbox_fill',
           'min_dist_to_border', 'max_dist_to_border', 'contour_length')


def get_thresholds(category_layers=SCORING_LAYERS):
    thresholds = []
    for n in category_layers:
        step = 1. / (n + 1)
        thresholds.extend(np.arange(step, 1, step))
    return thresholds


def first_segmentation_rle(segm, h, w):
    """`frPyObjects(segm, h, w)[0]` for polygons; an RLE dict as it is"""
    if isinstance(segm, dict):
        return segm
    return {"size": [h, w], "counts": OV.fr_py_objects(segm, h, w)[0]}


def get_iou_matrix(labels, annotations):
    if annotations is None or annotations == []:
        return None
    h, w = labels.shape
    gts = [first_segmentation_rle(a['segmentation'], h, w) for a in annotations]
    dts = [CO.encode((labels == l).astype(np.uint8)) for l in range(1, labels.max() + 1)]
    return CO.iou(dts, gts, [0] * len(gts))


def get_iou(iou_matrix, label_nr):
    if iou_matrix is not None:
        return iou_matrix[label_nr - 1].max()
    return None


def get_features_for_image(image, probabilities, annotations, category_layers=SCORING_LAYERS,
                           category_ids=CATEGORY_IDS):
    """-> [DataFrame per layer], the reference's columns and dtypes"""
    import pandas as pd
    inds = np.cumsum(category_layers)
    thresholds = get_thresholds(category_layers)
    out = []
    for ci, inst in enumerate(image):
        cat = np.searchsorted(inds, ci, side='right')
        iou_matrix = get_iou_matrix(inst, annotations.get(category_ids[cat], []))
        rows = []
        for l in range(1, inst.max() + 1):
            f = I.get_features_for_mask(inst == l, round(thresholds[ci], 2), probabilities[cat])
            f['iou'] = get_iou(iou_matrix, l)
            rows.append(f)
        out.append(pd.DataFrame(rows))
    return out


def feature_extractor(images, probabilities, annotations=None, **kw):
    if annotations is None:
        annotations = [{}] * len(images)
    return {'features': [get_features_for_image(i, p, a, **kw) for i, p, a in zip(images, probabilities, annotations)]}


def score_image_joiner(images, scores):
    return {'images_with_scores': list(zip(images, scores))}


# ---------------------------------------------------------------------------------------------------------------------
# seeded inputs
# ---------------------------------------------------------------------------------------------------------------------
def scoring_case(n=20, size=300, seed=2024, category_layers=SCORING_LAYERS):
    """-> (probabilities float64 (n, 2, size, size), label layers int32 (n, L, size, size), annotations: n dicts
    {None: [], 100: [...]}).  Image 0 has no annotations; image 1 has an annotation covering the whole image; the
    building layers of image 2 are empty above 0.5 (no instances there); every image has instances touching the border."""
    from scipy import ndimage as ndi
    from bench_data import rectangles_mask
    rs = np.random.RandomState(seed)
    probs = np.zeros((n, 2, size, size))
    for i in range(n):
        m, _ = rectangles_mask(rs, size, size, 12)
        m[:, :6] = 1                                                  # a building on the left border
        z = ndi.gaussian_filter(rs.randn(size, size) * 0.5 - 2.0 + 5.0 * m, 2.0)
        p = 1.0 / (1.0 + np.exp(-z))
        if i == 2:
            p = np.minimum(p, 0.45)
        probs[i, 0], probs[i, 1] = 1 - p, p
    inds = np.cumsum(category_layers)
    thr = get_thresholds(category_layers)
    labels = np.zeros((n, len(thr), size, size), np.int32)
    for i in range(n):
        for li, t in enumerate(thr):
            labels[i, li] = ndi.label(probs[i, np.searchsorted(inds, li, side='right')] > t)[0]
    annotations = []
    for i in range(n):
        anns = [] if i == 0 else OV.synthetic_image_annotations(rs, size, size, rs.randint(6, 16), 1000 + i,
                                                                100 * i + 1)
        if i >= 3:
            anns += instance_annotations(rs, labels[i, len(thr) // 2], 1000 + i, 100 * i + 50)
        if i == 1:
            anns.insert(0, {"id": 99, "image_id": 1001, "category_id": 100, "iscrowd": 0, "area": 1.0,
                            "bbox": [0.0, 0.0, 1.0, 1.0],
                            "segmentation": [[-1.0, -1.0, size + 1.0, -1.0, size + 1.0, size + 1.0, -1.0, size + 1.0]]})
        annotations.append({None: [], 100: anns})
    return probs, labels, annotations


def _box(ys, xs, pad):
    y0, y1, x0, x1 = ys.min() - pad, ys.max() + 1 + pad, xs.min() - pad, xs.max() + 1 + pad
    return [float(x0), float(y0), float(x1), float(y0), float(x1), float(y1), float(x0), float(y1)]


def instance_annotations(rs, layer, image_id, first_ann_id, n=6):
    """annotations laid over instances of one label layer, so that IoUs span the whole range: the instance's box
    (grown or shrunk by up to 2 pixels) as a single polygon, as the SECOND polygon after a decoy in an empty corner,
    or as the first polygon followed by a neighbour's box.  Only the first polygon counts (frPyObjects(...)[0]): the
    second and third forms tell that rule from one that merges the polygons."""
    anns = []
    k = int(layer.max())
    for j, l in enumerate(rs.permutation(np.arange(1, k + 1))[:n]):
        ys, xs = np.nonzero(layer == l)
        box = _box(ys, xs, int(rs.randint(-1, 3)))
        form = j % 3
        if form == 0:
            segm = [box]
        elif form == 1:
            segm = [[-3.0, -3.0, 1.5, -3.0, 1.5, 1.5, -3.0, 1.5], box]
        else:
            other = int(rs.randint(1, k + 1))
            oy, ox = np.nonzero(layer == other)
            segm = [box, _box(oy, ox, 0)]
        anns.append({"id": first_ann_id + j, "image_id": image_id, "category_id": 100, "iscrowd": 0, "area": 1.0,
                     "bbox": [0.0, 0.0, 1.0, 1.0], "segmentation": segm})
    return anns


# ---------------------------------------------------------------------------------------------------------------------
# ScoringRandomForest (src/models.py:250-282) and _convert_features_to_df (src/models.py:457-466)
# ---------------------------------------------------------------------------------------------------------------------
def convert_features_to_df(features):
    import pandas as pd
    df_features = []
    for image_features in features:
        for layer_features in image_features[1:]:
            df_features.append(layer_features)
    return pd.concat(df_features)


class ScoringRandomForest:
    def __init__(self, train_size, target, model_params):
        from sklearn.ensemble import RandomForestRegressor
        self.train_size = train_size
        self.target = target
        self.feature_names = []
        self.estimator = RandomForestRegressor(**model_params)

    def fit(self, features, **kwargs):
        from sklearn.model_selection import train_test_split
        df_features = convert_features_to_df(features)
        train_data, val_data = train_test_split(df_features, train_size=self.train_size, random_state=0)
        self.feature_names = list(df_features.columns.drop(self.target))
        self.estimator.fit(train_data[self.feature_names], train_data[self.target])
        return self

    def transform(self, features, **kwargs):
        scores = []
        for image_features in features:
            image_scores = []
            for layer_features in image_features:
                if len(layer_features) > 0:
                    image_scores.append(list(self.estimator.predict(layer_features[self.feature_names])))
                else:
                    image_scores.append([])
            scores.append(image_scores)
        return {'scores': scores}


# ---------------------------------------------------------------------------------------------------------------------
# flat tables of [[DataFrame per layer] per image] (the golden's layout)
# ---------------------------------------------------------------------------------------------------------------------
def flatten(features):
    """-> dict: counts (rows per (image, layer)), iou_none (per (image, layer)), one float64 / int64 array per column
    (iou NaN where None), dtypes (per (image, layer) the column dtypes joined by ',', '' for an empty frame)"""
    counts, none, dtypes, cols = [], [], [], {c: [] for c in COLUMNS}
    for image in features:
        for df in image:
            counts.append(len(df))
            dtypes.append(",".join("%s:%s" % (c, df[c].dtype) for c in df.columns))
            none.append(bool(len(df)) and df['iou'].isna().all() and df['iou'].dtype == object)
            for c in COLUMNS:
                if len(df):
                    v = df[c].to_numpy()
                    cols[c].append(np.asarray([np.nan if x is None else x for x in v], np.float64) if c == 'iou'
                                   else v)
    out = {"counts": np.asarray(counts, np.int64), "iou_none": np.asarray(none, bool),
           "dtypes": np.asarray(dtypes)}
    for c in COLUMNS:
        out[c] = np.concatenate(cols[c]) if cols[c] else np.zeros(0)
    return out
