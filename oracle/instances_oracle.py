"""TEST INFRASTRUCTURE — CPU restatement of the steps either side of the per-pixel chain (SURVEY.md 8f-2 / 8f-3).
Only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this file.

* COCO run-length encoding.  The reference calls pycocotools (`cocomask.encode`, `cocomask.toBbox`,
  src/utils.py:118-124); pycocotools is NOT installed here and is not vendored in the reference
  (requirements.txt: `pycocotools` unpinned, installed from cocodataset/cocoapi PythonAPI, whose C core is
  common/maskApi.c).  The functions below restate maskApi.c's published algorithms — rleEncode (column-major scan,
  alternating run lengths starting with zeros), rleToString (5-bit groups, continuation bit 0x20, sign rule on bit
  0x10, delta coding against the count two places back from the fourth count on, +48), rleFrString, rleToBbox
  (including its full-height rule when a run of ones crosses a column boundary).  Pinned by hand-derived vectors in
  tests/test_instances_cpu.py; no reference output exists to pin against -> "pinned to the published algorithm by
  known-answer vectors".
* Test-time augmentation (src/loaders.py:437-497): pinned against the reference's own functions
  through oracle/ref_shim.py, with `skimage.transform.rotate` at multiples of 90 degrees ASSUMED to be the exact
  quarter-turn permutation (np.rot90) — skimage is not installable here.
* Non-maximum suppression and mask features (src/postprocessing.py:261-386): plain numpy as the
  reference writes them; contour length through cv2 (installed) exactly as the reference calls it.
"""
import numpy as np


# ---------------------------------------------------------------------------------------------------------------------
# maskApi.c
# ---------------------------------------------------------------------------------------------------------------------
def rle_encode(mask):
    """rleEncode on the Fortran-ordered mask -> list of run lengths"""
    m = np.asarray(mask)
    flat = (np.asfortranarray(m) != 0).ravel(order="F")
    cnts, prev, c = [], 0, 0
    for v in flat:
        v = int(v)
        if v != prev:
            cnts.append(c)
            c = 0
            prev = v
        c += 1
    cnts.append(c)
    return cnts


def rle_to_string(cnts):
    """rleToString"""
    out = bytearray()
    for i, x in enumerate(cnts):
        x = int(x)
        if i > 2:
            x -= int(cnts[i - 2])
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            out.append(c + 48)
    return bytes(out)


def rle_from_string(s):
    """rleFrString"""
    if isinstance(s, str):
        s = s.encode("ascii")
    cnts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return cnts


def rle_to_bbox(cnts, h, w):
    """rleToBbox -> [x, y, w, h]"""
    m = (len(cnts) // 2) * 2
    if m == 0:
        return [0.0, 0.0, 0.0, 0.0]
    xs, ys, xe, ye, cc, xp = w, h, 0, 0, 0, 0
    for j in range(m):
        cc += int(cnts[j])
        t = cc - j % 2
        y = t % h
        x = (t - y) // h
        if j % 2 == 0:
            xp = x
        elif xp < x:
            ys, ye = 0, h - 1
        xs, xe, ys, ye = min(xs, x), max(xe, x), min(ys, y), max(ye, y)
    return [float(xs), float(ys), float(xe - xs + 1), float(ye - ys + 1)]


def rle_from_binary(prediction):
    """src/utils.py:118-120"""
    m = np.asarray(prediction)
    return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": rle_to_string(rle_encode(m))}


def bounding_box_from_rle(rle):
    """src/utils.py:123-124"""
    return rle_to_bbox(rle_from_string(rle["counts"]), rle["size"][0], rle["size"][1])


def decompose(labeled):
    """src/utils.py:61-73"""
    nr_true = labeled.max()
    masks = []
    for i in range(1, nr_true + 1):
        msk = labeled.copy()
        msk[msk != i] = 0.
        msk[msk == i] = 255.
        masks.append(msk)
    return masks if masks else [labeled]


def create_annotations(image_ids, predictions, category_ids, category_layers):
    """src/utils.py:76-115 without the logging / saving"""
    annotations = []
    inds = np.cumsum(category_layers)
    for image_id, (prediction, image_scores) in zip(image_ids, predictions):
        for category_ind, (category_instances, category_scores) in enumerate(zip(prediction, image_scores)):
            category_nr = np.searchsorted(inds, category_ind, side='right')
            if category_ids[category_nr] is not None:
                for mask, score in zip(decompose(category_instances), category_scores):
                    rle = rle_from_binary(mask.astype('uint8'))
                    annotations.append({"image_id": int(image_id), "category_id": category_ids[category_nr],
                                        "score": score,
                                        "segmentation": {"size": rle["size"], "counts": rle["counts"].decode("UTF-8")},
                                        "bbox": bounding_box_from_rle(rle)})
    return annotations


# ---------------------------------------------------------------------------------------------------------------------
# test-time augmentation (src/loaders.py:401-517)
# ---------------------------------------------------------------------------------------------------------------------
def skimage_rotate(image, angle, preserve_range=False, **kwargs):
    """ASSUMPTION: skimage.transform.rotate at a multiple of 90 degrees on a square image = exact quarter turns,
    counter-clockwise for positive angles (np.rot90); float64 output like skimage"""
    if angle % 90 != 0:
        raise NotImplementedError("only quarter turns are restated")
    return np.rot90(np.asarray(image, dtype=np.float64), (int(angle) // 90) % 4, axes=(0, 1)).copy()


def tta_specs(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=False):
    from itertools import product
    specs = [{'ud_flip': False, 'lr_flip': False, 'rotation': 0, 'color_shift': False}]
    ud_options = [True, False] if flip_ud else [False]
    lr_options = [True, False] if flip_lr else [False]
    rot_options = [0, 90, 180, 270] if rotation else [0]
    for ud, lr, rot, color in product(ud_options, lr_options, rot_options, [False]):
        if ud is False and lr is False and rot == 0 and color is False:
            continue
        specs.append({'ud_flip': ud, 'lr_flip': lr, 'rotation': rot, 'color_shift': color})
    return specs


def tta_transform(image, p):
    """src/loaders.py:470-480 on an (H, W, C) image"""
    if p['ud_flip']:
        image = np.flipud(image)
    elif p['lr_flip']:
        image = np.fliplr(image)
    return skimage_rotate(image, p['rotation'], preserve_range=True)


def tta_inverse(image, p):
    """src/loaders.py:483-497 on a (C, H, W) prediction"""
    x = np.stack([skimage_rotate(ch, -1 * p['rotation'], preserve_range=True) for ch in image]).astype(image.dtype)
    if p['ud_flip']:
        x = np.stack([np.flipud(ch) for ch in x])
    elif p['lr_flip']:
        x = np.stack([np.fliplr(ch) for ch in x])
    return x


def tta_aggregate(images, tta_params, img_ids, method="gmean"):
    """src/loaders.py:446-467"""
    from scipy.stats import gmean
    agg = {'mean': np.mean, 'max': np.max, 'min': np.min, 'gmean': gmean}[method]
    out = []
    for u in sorted(set(img_ids)):
        preds = [tta_inverse(im, p) for im, p, i in zip(images, tta_params, img_ids) if i == u]
        out.append(agg(np.stack(preds, axis=-1), axis=-1))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# NMS and mask features (src/postprocessing.py:261-386)
# ---------------------------------------------------------------------------------------------------------------------
def get_iou_for_mask_pair(mask1, mask2):
    intersection = np.count_nonzero(mask1 * mask2)
    union = np.count_nonzero(mask1 + mask2)
    return intersection / union


def remove_overlapping_masks(image, scores, iou_threshold=0.5):
    scores_with_labels = []
    for layer_nr, layer_scores in enumerate(scores):
        scores_with_labels.extend([(score, layer_nr, label_nr + 1) for label_nr, score in enumerate(layer_scores)])
    scores_with_labels.sort(key=lambda x: x[0], reverse=True)
    for i, (score_i, layer_nr_i, label_nr_i) in enumerate(scores_with_labels):
        base_mask = image[layer_nr_i] == label_nr_i
        for score_j, layer_nr_j, label_nr_j in scores_with_labels[i + 1:]:
            mask_to_check = image[layer_nr_j] == label_nr_j
            iou = get_iou_for_mask_pair(base_mask, mask_to_check)
            if iou > iou_threshold:
                scores_with_labels.remove((score_j, layer_nr_j, label_nr_j))
                scores[layer_nr_j][label_nr_j - 1] = 0
    return image, scores


def get_bbox(mask):
    rows = np.any(mask, axis=1)
    cols = np.any(mask, axis=0)
    rmin, rmax = np.where(rows)[0][[0, -1]]
    cmin, cmax = np.where(cols)[0][[0, -1]]
    return rmin, rmax + 1, cmin, cmax + 1


def get_contour_length(mask):
    """src/postprocessing.py:340-352 (cv2 >= 4 returns (contours, hierarchy); the reference unpacks cv2 3's triple)"""
    import cv2
    mask_contour = np.zeros_like(mask).astype(np.uint8)
    contours = cv2.findContours(mask.astype(np.uint8), cv2.RETR_TREE, cv2.CHAIN_APPROX_NONE)[-2]
    cv2.drawContours(mask_contour, contours, -1, (255, 255, 255), 1)
    return np.count_nonzero(mask_contour)


def get_features_for_mask(mask, threshold, category_probabilities):
    mask_probabilities = np.where(mask, category_probabilities, 0)
    area = np.count_nonzero(mask)
    bbox = get_bbox(mask)
    bbox_height = bbox[1] - bbox[0]
    bbox_width = bbox[3] - bbox[2]
    d = (bbox[0], mask.shape[0] - bbox[1], bbox[2], mask.shape[1] - bbox[3])
    return {'iou': None, 'threshold': threshold, 'area': area, 'mean_prob': mask_probabilities.sum() / area,
            'max_prob': mask_probabilities.max(), 'bbox_ar': bbox_height / bbox_width,
            'bbox_area': bbox_width * bbox_height, 'bbox_fill': area / (bbox_width * bbox_height),
            'min_dist_to_border': min(d), 'max_dist_to_border': max(d), 'contour_length': get_contour_length(mask)}


def instance_features(labels, probabilities, category_layers=(1, 1)):
    inds = np.cumsum(category_layers)
    thresholds = []
    for n in category_layers:
        step = 1. / (n + 1)
        thresholds.extend(np.arange(step, 1, step))
    out = []
    for li, lab in enumerate(labels):
        ch = np.searchsorted(inds, li, side='right')
        out.append([get_features_for_mask(lab == l, round(thresholds[li], 2), probabilities[ch])
                    for l in range(1, lab.max() + 1)])
    return out
