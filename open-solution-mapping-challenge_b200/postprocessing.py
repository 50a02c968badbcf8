"""Mirror of the reference's per-pixel post-processing (src/postprocessing.py:48-258,
src/utils.py:231-273,328-339) on the GPU.

Two surfaces:
  * module-level functions with the reference's names and signatures, one image in / numpy out — drop-ins for
    `make_apply_transformer(post.<fn>, ...)` in src/pipelines.py:248-304 (each call round-trips the image over PCIe);
  * `MaskPostprocessor`, the batched transformer the fast path uses: the whole batch of probability maps stays on the
    device through resize/crop -> threshold -> erode -> label -> dilate -> score, one launch sequence per batch.

All arithmetic is in libmcb200.so (csrc/postproc.cu); torch only owns the device buffers.  No CPU fallback.
"""
import importlib.util
import itertools
import warnings

import numpy as np
import torch

from . import _lib as L

CATEGORY_LAYERS = [1, 1]  # src/pipeline_config.py:18
CATEGORY_IDS = [None, 100]  # src/pipeline_config.py:17
MEAN = [0.485, 0.456, 0.406]
STD = [0.229, 0.224, 0.225]


def category_config():
    """(CATEGORY_LAYERS, CATEGORY_IDS) of the reference's src/pipeline_config.py when the reference package is
    importable, else this module's [1, 1] / [None, 100].  Read on every call: the scoring workflow edits the reference
    config to [1, 19] (one background layer, 19 building thresholds 0.05 ... 0.95) and the per-image functions,
    get_thresholds, instance_features and FeatureExtractor follow it as the reference's own module does."""
    if importlib.util.find_spec("src") is None:      # no reference package on the path: the defaults
        return list(CATEGORY_LAYERS), list(CATEGORY_IDS)
    try:
        from src import pipeline_config as pc
        return list(pc.CATEGORY_LAYERS), list(pc.CATEGORY_IDS)
    except Exception as e:  # a `src` package whose pipeline_config does not import
        warnings.warn("mcb200: a `src` package is importable but src.pipeline_config is not (%s: %s); using "
                      "CATEGORY_LAYERS %s and CATEGORY_IDS %s" % (type(e).__name__, e, CATEGORY_LAYERS, CATEGORY_IDS),
                      RuntimeWarning, stacklevel=2)
        return list(CATEGORY_LAYERS), list(CATEGORY_IDS)


def _dev():
    if not torch.cuda.is_available():
        raise RuntimeError("mcb200.postprocessing needs a CUDA device; there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _to_dev(a, dtype):
    if isinstance(a, torch.Tensor):
        return a.to(device=_dev(), dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=_dev(), dtype=dtype)


def layer_thresholds(category_layers=None):
    """threshold list and source channel of every output layer (src/postprocessing.py:77-84)"""
    category_layers = category_config()[0] if category_layers is None else category_layers
    thr, chan = [], []
    for c, n_layers in enumerate(category_layers):
        step = 1. / (n_layers + 1)
        for t in np.arange(step, 1, step):
            thr.append(float(t))
            chan.append(c)
    return thr, chan


# ---------------------------------------------------------------------------------------------------------------------
# device-level batched primitives (tensors in, tensors out; leading dims are planes / images)
# ---------------------------------------------------------------------------------------------------------------------
def resize_batch(probs, target_size):
    """probs (N, C, Hi, Wi) float32 cuda -> (N, C, Ho, Wo) float64 cuda"""
    assert probs.dtype == torch.float32 and probs.is_cuda and probs.is_contiguous()
    n, c, hi, wi = probs.shape
    ho, wo = int(target_size[0]), int(target_size[1])
    out = torch.empty((n, c, ho, wo), dtype=torch.float64, device=probs.device)
    ws = torch.empty(2 * n, dtype=torch.float32, device=probs.device)
    L.fcall("mcb_resize_bilinear_f64", probs.data_ptr(), out.data_ptr(), ws.data_ptr(), n, c, hi, wi, ho, wo)
    return out


_THRESHOLD_CONSTS = {}


def threshold_batch(probs, category_layers=None):
    """probs (N, C, H, W) float32|float64 cuda -> (N, L, H, W) uint8 (0/1)"""
    assert probs.is_cuda and probs.is_contiguous() and probs.dtype in (torch.float32, torch.float64)
    n, c, h, w = probs.shape
    thr, chan = layer_thresholds(category_layers)
    assert max(chan) < c
    key = (probs.device, tuple(thr), tuple(chan))
    if key not in _THRESHOLD_CONSTS:   # tiny device constants, created once (and never inside a graph capture)
        _THRESHOLD_CONSTS[key] = (torch.tensor(thr, dtype=torch.float64, device=probs.device),
                                  torch.tensor(chan, dtype=torch.int32, device=probs.device))
    t, ch = _THRESHOLD_CONSTS[key]
    out = torch.empty((n, len(thr), h, w), dtype=torch.uint8, device=probs.device)
    L.fcall("mcb_threshold_layers", probs.data_ptr(), int(probs.dtype == torch.float64), t.data_ptr(), ch.data_ptr(),
            out.data_ptr(), n, c, len(thr), h, w)
    return out


def label_batch(mask, return_counts=False):
    """mask (..., H, W) uint8|int32 cuda -> int32 labels, same shape (scipy.ndimage.label numbering per plane)"""
    assert mask.is_cuda and mask.is_contiguous() and mask.dtype in (torch.uint8, torch.int32, torch.bool)
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    h, w = mask.shape[-2:]
    planes = mask.numel() // (h * w)
    labels = torch.empty(mask.shape, dtype=torch.int32, device=mask.device)
    ws = torch.empty(mask.numel(), dtype=torch.int32, device=mask.device)
    counts = torch.empty(planes, dtype=torch.int32, device=mask.device)
    L.fcall("mcb_ccl_label", mask.data_ptr(), int(mask.dtype == torch.int32), labels.data_ptr(), ws.data_ptr(),
            counts.data_ptr(), planes, h, w)
    return (labels, counts) if return_counts else labels


def morph_batch(x, size, dilation):
    """skimage erosion / dilation with rectangle(size, size) per plane; x (..., H, W) uint8|int32 cuda"""
    assert x.is_cuda and x.is_contiguous() and x.dtype in (torch.uint8, torch.int32)
    h, w = x.shape[-2:]
    out = torch.empty_like(x)
    L.fcall("mcb_morph_rect", x.data_ptr(), out.data_ptr(), int(x.dtype == torch.int32), int(dilation), int(size),
            x.numel() // (h * w), h, w)
    return out


def erode_batch(mask, size):
    """erode_image per plane incl. add_dropped_objects (src/postprocessing.py:135-156); mask uint8 -> uint8"""
    if not size > 0:
        return mask
    assert mask.dtype == torch.uint8
    h, w = mask.shape[-2:]
    planes = mask.numel() // (h * w)
    eroded = morph_batch(mask, size, dilation=False)
    out = torch.empty_like(mask)
    ws = torch.empty(2 * mask.numel(), dtype=torch.int32, device=mask.device)
    L.fcall("mcb_add_dropped_objects", mask.data_ptr(), eroded.data_ptr(), out.data_ptr(), ws.data_ptr(), planes, h, w)
    return out


def scores_batch(labels, probs, counts):
    """labels (P, H, W) int32, probs (P, H, W) float32|float64, counts (P,) int32 (max label per plane)
    -> (scores float64 (sum counts,), offsets (P,) numpy) ; empty instances score NaN"""
    assert labels.is_cuda and labels.is_contiguous() and probs.is_contiguous()
    p, h, w = labels.shape
    counts_h = counts.cpu().numpy().astype(np.int64)
    offsets_h = np.concatenate([[0], np.cumsum(counts_h)[:-1]]).astype(np.int32) if p else np.zeros(0, np.int32)
    total = int(counts_h.sum())
    scores = torch.empty(max(total, 1), dtype=torch.float64, device=labels.device)
    if total > 0:
        offs = torch.from_numpy(offsets_h).to(labels.device)
        sums = torch.empty(total, dtype=torch.float64, device=labels.device)
        cnt = torch.empty(total, dtype=torch.int32, device=labels.device)
        L.fcall("mcb_instance_scores", labels.data_ptr(), probs.data_ptr(), int(probs.dtype == torch.float64),
                offs.data_ptr(), sums.data_ptr(), cnt.data_ptr(), scores.data_ptr(), total, p, h, w)
    return scores[:total], offsets_h, counts_h


def scores_strided(labels, probs, counts, kcap=1024):
    """build_score without a host round trip: labels (P,H,W) int32, probs (P,H,W) f32|f64, counts (P,) int32 (labels per
    plane) -> scores (P, kcap) float64 on the device; entries beyond counts[p] are undefined.  The caller checks
    counts.max() <= kcap after its single device->host copy (else re-run with a larger kcap)."""
    assert labels.is_cuda and labels.is_contiguous() and probs.is_contiguous()
    p, h, w = labels.shape
    scores = torch.empty((p, kcap), dtype=torch.float64, device=labels.device)
    gsum = torch.empty((p, kcap), dtype=torch.float64, device=labels.device)
    gcnt = torch.empty((p, kcap), dtype=torch.int32, device=labels.device)
    L.fcall("mcb_instance_scores_strided", labels.data_ptr(), probs.data_ptr(), int(probs.dtype == torch.float64),
            counts.data_ptr(), scores.data_ptr(), gsum.data_ptr(), gcnt.data_ptr(), int(kcap), p, h, w)
    return scores


# ---------------------------------------------------------------------------------------------------------------------
# reference-signature per-image functions (numpy in / numpy out)
# ---------------------------------------------------------------------------------------------------------------------
def softmax(X, theta=1.0, axis=None):
    """src/utils.py:231-273 for the pipeline's use (2 classes along `axis` of an (N,2,H,W) or (2,H,W) array)"""
    from . import ops
    X = np.asarray(X)
    if theta != 1.0 or X.ndim not in (3, 4) or (axis not in (0, 1)) or X.shape[axis] != 2 or (X.ndim == 3) != (axis == 0):
        raise NotImplementedError("mcb200 softmax implements the pipeline's 2-class channel softmax only")
    x4 = _to_dev(X if X.ndim == 4 else X[None], torch.float32)
    out = ops.softmax2(x4).cpu().numpy()
    return out if X.ndim == 4 else out[0]


def resize_image(image, target_size):
    x = _to_dev(image, torch.float32)
    return resize_batch(x[None], target_size)[0].cpu().numpy()


def categorize_batch(probs):
    """probs (N, C, H, W) float32|float64 cuda -> (N, H, W) int64 cuda: np.argmax over the channel axis"""
    assert probs.is_cuda and probs.dtype in (torch.float32, torch.float64)
    probs = probs.contiguous()
    n, c, h, w = probs.shape
    out = torch.empty((n, h, w), dtype=torch.int64, device=probs.device)
    L.fcall("mcb_argmax_channels", probs.data_ptr(), int(probs.dtype == torch.float64), out.data_ptr(), n, c, h, w)
    return out


def categorize_image(image):
    """src/postprocessing.py:64-74: np.argmax(image, axis=0) (the validation callback's categoriser,
    src/callbacks.py:168-200); (C, H, W) -> (H, W) int64"""
    image = np.asarray(image)
    x = _to_dev(image, torch.float64 if image.dtype == np.float64 else torch.float32)
    return categorize_batch(x[None])[0].cpu().numpy()


def categorize_multilayer_image(image):
    image = np.asarray(image)
    x = _to_dev(image, torch.float64 if image.dtype == np.float64 else torch.float32)
    return threshold_batch(x[None])[0].cpu().numpy().astype(bool)


def label_multiclass_image(mask):
    mask = np.asarray(mask)
    planes = np.stack([(mask == c) for c in range(0, mask.max() + 1)]).astype(np.uint8)
    return label_batch(_to_dev(planes, torch.uint8)).cpu().numpy()


def label_multilayer_image(mask):
    m = np.asarray(mask)
    return label_batch(_to_dev((m != 0).astype(np.uint8), torch.uint8)).cpu().numpy()


def erode_image(mask, erode_selem_size):
    if not erode_selem_size > 0:
        return mask
    m = _to_dev((np.asarray(mask) != 0).astype(np.uint8), torch.uint8)
    return erode_batch(m, erode_selem_size).cpu().numpy()


def dilate_image(mask, dilate_selem_size):
    if not dilate_selem_size > 0:
        return mask
    m = np.asarray(mask)
    if m.dtype == np.int32:
        x = _to_dev(m, torch.int32)
    elif m.dtype in (np.uint8, np.bool_):
        x = _to_dev(m.astype(np.uint8), torch.uint8)
    else:
        raise NotImplementedError("dilate_image: dtype %s (the pipeline dilates int32 label maps)" % m.dtype)
    out = morph_batch(x, dilate_selem_size, dilation=True).cpu().numpy()
    return out.astype(bool) if m.dtype == np.bool_ else out


def build_score(image, probabilities):
    labels = _to_dev(np.asarray(image), torch.int32)
    probs = np.asarray(probabilities)
    p = min(labels.shape[0], probs.shape[0])  # zip() pairing of the reference
    pr = _to_dev(probs[:p], torch.float64 if probs.dtype == np.float64 else torch.float32)
    counts = labels[:p].reshape(p, -1).max(dim=1).values.to(torch.int32)
    scores, offs, cnts = scores_batch(labels[:p].contiguous(), pr, counts)
    s = scores.cpu().numpy()
    total = []
    for i in range(p):
        vals = s[offs[i]:offs[i] + cnts[i]]
        total.append([np.ma.masked if np.isnan(v) else v for v in vals])
    return image, total


def dense_crf_batch(imgs, probs, compat_gaussian=3, sxy_gaussian=1, compat_bilateral=10, sxy_bilateral=1, srgb=50,
                    iterations=5):
    """imgs (N,3,H,W) float32 ImageNet-normalised, probs (N,2,H,W) float32, both cuda -> (N,2,H,W) float32.
    Mismatched shapes, dtypes or devices raise ValueError before anything is launched: the kernels index both buffers
    with probs' shape."""
    if not (isinstance(imgs, torch.Tensor) and isinstance(probs, torch.Tensor)):
        raise ValueError("dense_crf_batch: imgs and probs must be tensors")
    if imgs.dtype != torch.float32 or probs.dtype != torch.float32:
        raise ValueError("dense_crf_batch: imgs and probs must be float32, got %s and %s" % (imgs.dtype, probs.dtype))
    if not (imgs.is_cuda and imgs.device == probs.device):
        raise ValueError("dense_crf_batch: imgs and probs must be on one CUDA device, got %s and %s"
                         % (imgs.device, probs.device))
    if probs.dim() != 4 or imgs.dim() != 4:
        raise ValueError("dense_crf_batch: imgs (N,3,H,W) and probs (N,2,H,W), got %s and %s"
                         % (tuple(imgs.shape), tuple(probs.shape)))
    n, c, h, w = probs.shape
    if c != 2:
        raise NotImplementedError("dense_crf: 2 labels (the reference builds DenseCRF2D(width, height, 2))")
    if tuple(imgs.shape) != (n, 3, h, w):
        raise ValueError("dense_crf_batch: imgs %s does not match probs %s" % (tuple(imgs.shape), tuple(probs.shape)))
    imgs, probs = imgs.contiguous(), probs.contiguous()
    if probs.numel() == 0:
        return torch.empty_like(probs)
    rgb = torch.empty((n, h, w, 3), dtype=torch.uint8, device=probs.device)
    L.fcall("mcb_crf_rgb_from_normalized", imgs.data_ptr(), rgb.data_ptr(), n, h, w)
    out = torch.empty_like(probs)
    ws = torch.empty(3 * probs.numel(), dtype=torch.float32, device=probs.device)
    L.fcall("mcb_dense_crf", probs.data_ptr(), rgb.data_ptr(), out.data_ptr(), ws.data_ptr(), n, h, w,
            float(compat_gaussian), float(sxy_gaussian), float(compat_bilateral), float(sxy_bilateral), float(srgb),
            int(iterations))
    return out


def dense_crf(img, output_probs, compat_gaussian=3, sxy_gaussian=1, compat_bilateral=10, sxy_bilateral=1, srgb=50,
              iterations=5):
    """src/postprocessing.py:183-225 (parity unpinned: pydensecrf is absent; semantics in oracle/post_oracle.py)"""
    x = _to_dev(np.asarray(img), torch.float32)[None]
    p = _to_dev(np.asarray(output_probs), torch.float32)[None]
    return dense_crf_batch(x, p, compat_gaussian, sxy_gaussian, compat_bilateral, sxy_bilateral, srgb,
                           iterations)[0].cpu().numpy()


def watershed_batch(prob, markers, mask, levels=256):
    """prob (P,H,W) float32|float64, markers (P,H,W) int32, mask (P,H,W) uint8|bool, cuda -> int32 labels.
    Not a reference function; semantics = oracle/post_oracle.py::minimax_watershed (parity unpinned).
    Mismatched shapes, dtypes or devices raise ValueError before anything is launched: the kernel indexes all three
    buffers with prob's shape."""
    if not all(isinstance(t, torch.Tensor) for t in (prob, markers, mask)):
        raise ValueError("watershed_batch: prob, markers and mask must be tensors")
    if prob.dtype not in (torch.float32, torch.float64):
        raise ValueError("watershed_batch: prob must be float32 or float64, got %s" % prob.dtype)
    if markers.dtype not in (torch.int32, torch.int64, torch.int16, torch.int8, torch.uint8):
        raise ValueError("watershed_batch: markers must be an integer tensor, got %s" % markers.dtype)
    if mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError("watershed_batch: mask must be bool or uint8, got %s" % mask.dtype)
    if not (prob.is_cuda and markers.device == prob.device and mask.device == prob.device):
        raise ValueError("watershed_batch: prob, markers and mask must be on one CUDA device, got %s, %s and %s"
                         % (prob.device, markers.device, mask.device))
    if prob.dim() != 3 or markers.shape != prob.shape or mask.shape != prob.shape:
        raise ValueError("watershed_batch: prob, markers and mask must all be (P,H,W), got %s, %s and %s"
                         % (tuple(prob.shape), tuple(markers.shape), tuple(mask.shape)))
    if not 2 <= int(levels) <= 65536:
        raise ValueError("watershed_batch: levels %d outside [2, 65536]" % int(levels))
    prob, markers = prob.contiguous(), markers.contiguous().to(torch.int32)
    mask = mask.contiguous()
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    p, h, w = prob.shape
    out = torch.empty((p, h, w), dtype=torch.int32, device=prob.device)
    if out.numel() == 0:
        return out
    ws = torch.empty(3 * p * h * w, dtype=torch.int32, device=prob.device)
    L.fcall("mcb_watershed", prob.data_ptr(), int(prob.dtype == torch.float64), markers.data_ptr(), mask.data_ptr(),
            out.data_ptr(), ws.data_ptr(), p, h, w, int(levels))
    return out


def watershed_split(prob, hi=0.8, lo=0.5, levels=256):
    """instance split of touching buildings: markers = components of prob > hi, flooded over prob > lo"""
    hi_mask = (prob > hi).to(torch.uint8).contiguous()
    markers = label_batch(hi_mask)
    return watershed_batch(prob, markers, (prob > lo).to(torch.uint8), levels)


def crop_image_center_per_class(image, h_crop, w_crop):
    """src/postprocessing.py:239-258 — pure indexing"""
    out = []
    for class_prediction in image:
        h, w = class_prediction.shape[:2]
        h_start, w_start = int((h - h_crop) / 2.), int((w - w_crop) / 2.)
        out.append(class_prediction[h_start:-h_start, w_start:-w_start])
    return np.stack(out)


# ---------------------------------------------------------------------------------------------------------------------
# instance level: non-maximum suppression and scoring-model features (src/postprocessing.py:18-45, 261-386)
# ---------------------------------------------------------------------------------------------------------------------
def pair_intersections(labels_a, labels_b, ka, kb):
    """labels_a / labels_b (H, W) int32 cuda, ka / kb their label counts -> (ka, kb) int32 cuda intersection areas"""
    assert labels_a.is_cuda and labels_a.dtype == torch.int32 and labels_a.shape == labels_b.shape
    h, w = labels_a.shape
    inter = torch.zeros((max(ka, 1), max(kb, 1)), dtype=torch.int32, device=labels_a.device)
    L.fcall("mcb_pair_intersections", labels_a.contiguous().data_ptr(), labels_b.contiguous().data_ptr(),
            inter.data_ptr(), int(ka), int(kb), h, w)
    return inter[:ka, :kb]


def remove_overlapping_masks(image, scores, iou_threshold=0.5):
    """src/postprocessing.py:355-379: instances of all layers sorted by score; an instance whose IoU with a better one
    exceeds the threshold has its score set to 0 (its mask stays).  The reference builds two full-image masks for
    every pair; here areas and the layer-pair intersection tables come from two device passes and the greedy sweep
    runs on the resulting small integer matrices."""
    from . import utils as U
    lab = _to_dev(np.asarray(image).astype(np.int32), torch.int32)
    n_layers = lab.shape[0]
    counts = lab.reshape(n_layers, -1).max(dim=1).values.to(torch.int32)
    geo = U.instance_geometry(lab, counts)
    k = geo["counts"]
    inter = {}
    for a in range(n_layers):
        for b in range(a + 1, n_layers):
            if k[a] and k[b]:
                inter[(a, b)] = pair_intersections(lab[a], lab[b], int(k[a]), int(k[b])).cpu().numpy()

    def area(layer, label):
        return int(geo["area"][geo["offsets"][layer] + label - 1]) if label <= k[layer] else 0

    def iou(i, j):
        (la, a), (lb, b) = i, j
        if la == lb:
            inter_ab = area(la, a) if a == b else 0
        elif a > k[la] or b > k[lb]:
            inter_ab = 0
        else:
            inter_ab = int(inter[(la, lb)][a - 1, b - 1]) if la < lb else int(inter[(lb, la)][b - 1, a - 1])
        union = area(la, a) + area(lb, b) - inter_ab
        return inter_ab / union if union else float("nan")

    scores_with_labels = []
    for layer_nr, layer_scores in enumerate(scores):
        scores_with_labels.extend([(score, layer_nr, label_nr + 1) for label_nr, score in enumerate(layer_scores)])
    scores_with_labels.sort(key=lambda x: x[0], reverse=True)
    i = 0
    while i < len(scores_with_labels):          # the reference mutates the list it iterates; same visiting order
        score_i, layer_nr_i, label_nr_i = scores_with_labels[i]
        for score_j, layer_nr_j, label_nr_j in list(scores_with_labels[i + 1:]):
            if iou((layer_nr_i, label_nr_i), (layer_nr_j, label_nr_j)) > iou_threshold:
                scores_with_labels.remove((score_j, layer_nr_j, label_nr_j))
                scores[layer_nr_j][label_nr_j - 1] = 0
        i += 1
    return image, scores


class NonMaximumSupression:
    """src/postprocessing.py:34-45"""

    def __init__(self, iou_threshold, num_threads=1):
        self.iou_threshold = iou_threshold
        self.num_threads = num_threads

    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)

    def transform(self, images_with_scores):
        return {'images_with_scores': [remove_overlapping_masks(*p, iou_threshold=self.iou_threshold)
                                       for p in images_with_scores]}


def get_thresholds(category_layers=None):
    """src/postprocessing.py:331-337"""
    return layer_thresholds(category_layers)[0]


# ---------------------------------------------------------------------------------------------------------------------
# second-level scoring: instance features and the ground-truth IoU target (src/postprocessing.py:18-33, 261-337)
# ---------------------------------------------------------------------------------------------------------------------
FEATURE_COLUMNS = ('iou', 'threshold', 'area', 'mean_prob', 'max_prob', 'bbox_ar', 'bbox_area', 'bbox_fill',
                   'min_dist_to_border', 'max_dist_to_border', 'contour_length')


def _starts(lengths):
    return np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.int64)


def ground_truth_runs(annotation_groups, height, width):
    """the masks get_iou_matrix compares against (src/postprocessing.py:311-315), as COCO run lists: per annotation the
    FIRST polygon of its segmentation only, `frPyObjects(segm, h, w)[0]`, rasterised on the device exactly as
    pycocotools does; a segmentation that is already an RLE dict (compressed or uncompressed counts,
    mcb200.evaluation.segmentation_counts) is used as is.  The caller's annotations are not modified.
    annotation_groups: list of lists of COCO annotations -> (cnts uint32, starts int64 [G + 1], group offsets int64
    [groups + 1]) on the host, annotations numbered group by group."""
    from . import utils as U
    from .evaluation import segmentation_counts
    from .preparation import polygons_csr, rasterize_polygons, segmentation_polygons
    h, w = int(height), int(width)
    runs, polys, poly_slot = [], [], []
    for anns in annotation_groups:
        for ann in anns:
            segm = ann['segmentation']
            if isinstance(segm, dict):
                c, size = segmentation_counts(segm, h, w)
                if size != (h, w):
                    raise ValueError("an RLE segmentation of size %s on a %d x %d label map" % (size, h, w))
                runs.append(c.astype(np.uint32))
            else:
                polys.append(segmentation_polygons(segm)[0])
                poly_slot.append(len(runs))
                runs.append(None)
    if polys:
        planes = rasterize_polygons(*polygons_csr(polys), h, w).to(torch.int32)
        cnts, starts, _, _ = U.rle_encode_instances(planes, torch.ones(len(polys), dtype=torch.int32,
                                                                       device=planes.device))
        for j, g in enumerate(poly_slot):
            runs[g] = cnts[starts[j]:starts[j + 1]]
    cnts = np.concatenate(runs).astype(np.uint32) if runs else np.zeros(0, np.uint32)
    return cnts, _starts([len(r) for r in runs]), _starts([len(a) for a in annotation_groups])


def pair_iou(dt_cnts, dt_starts, gt_cnts, gt_starts, pair_dt, pair_gt):
    """cocomask.iou(dt, gt, [0] * len(gt)) entries of the listed (dt, gt) pairs: run lists on the host (uint32 counts,
    int64 starts), pairs int arrays -> float64 cuda [pairs]"""
    dev = _dev()
    npairs = len(pair_dt)
    iou = torch.empty(max(npairs, 1), dtype=torch.float64, device=dev)
    if npairs:
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (
            np.asarray(dt_cnts, np.uint32).view(np.int32), np.asarray(dt_starts, np.int64),
            np.asarray(gt_cnts, np.uint32).view(np.int32), np.asarray(gt_starts, np.int64),
            np.zeros(max(len(gt_starts) - 1, 1), np.uint8), np.asarray(pair_dt, np.int32),
            np.asarray(pair_gt, np.int32), np.arange(npairs, dtype=np.int64))]
        L.fcall("mcb_rle_pair_iou", *[x.data_ptr() for x in t], iou.data_ptr(), int(npairs))
    return iou[:npairs]


def scoring_features_batch(labels, probs, annotations=None, category_layers=None, category_ids=None):
    """get_features_for_image (src/postprocessing.py:261-303) for every layer of a batch in one device pass.
    labels (N, L, H, W) int32 cuda (the dilated label maps), probs (N, C, H, W) float32|float64 cuda (the resized
    probabilities), annotations: None or N dicts {category id: [COCO annotations]}.  Layer l reads channel c(l) of
    CATEGORY_LAYERS; with annotations, an instance's `iou` is the max of cocomask.iou against its image's annotations
    of CATEGORY_IDS[c(l)] (get_mask_with_iou / get_iou_matrix / get_iou), NaN where there are none (the reference's
    None).  Read back once per batch -> dict of host arrays per instance slot (slot order = plane-major, label order)
    plus 'counts' (instances per plane), 'has_gt' (per plane) and the shapes."""
    from . import utils as U
    layers, ids = category_config()
    category_layers = layers if category_layers is None else list(category_layers)
    category_ids = ids if category_ids is None else list(category_ids)
    assert labels.is_cuda and labels.dtype == torch.int32 and labels.dim() == 4
    assert probs.is_cuda and probs.dtype in (torch.float32, torch.float64) and probs.dim() == 4
    n, nl, h, w = labels.shape
    thr, chan = layer_thresholds(category_layers)
    if nl != len(thr):
        raise ValueError("%d label layers, but CATEGORY_LAYERS %s give %d" % (nl, category_layers, len(thr)))
    if probs.shape[0] != n or tuple(probs.shape[2:]) != (h, w) or probs.shape[1] <= max(chan):
        raise ValueError("probabilities %s do not pair with label maps %s" % (tuple(probs.shape), tuple(labels.shape)))
    if annotations is not None and len(annotations) != n:
        raise ValueError("%d annotation dicts for %d images" % (len(annotations), n))
    planes = labels.reshape(n * nl, h, w).contiguous()
    counts = planes.reshape(n * nl, -1).amax(dim=1).to(torch.int32) if n * nl else torch.zeros(0, dtype=torch.int32)
    chan_d = torch.tensor(chan, dtype=torch.int64, device=labels.device)
    pr = probs.contiguous().index_select(1, chan_d).reshape(n * nl, h, w)
    geo = U.instance_geometry(planes, counts, pr)
    total = int(geo["counts"].sum())
    if total and (geo["area"] == 0).any():
        s = int(np.flatnonzero(geo["area"] == 0)[0])
        p = int(geo["plane"][s])
        raise ValueError("label %d of layer %d of image %d is empty: get_bbox has no box for it"
                         % (s - int(geo["offsets"][p]) + 1, p % nl, p // nl))
    clen = torch.zeros(max(total, 1), dtype=torch.int32, device=labels.device)
    if total:
        L.fcall("mcb_contour_length", planes.data_ptr(), geo["_offsets"].data_ptr(), geo["_counts"].data_ptr(),
                clen.data_ptr(), n * nl, h, w)
    plane = geo["plane"].astype(np.int64)
    n_cat = len(category_layers)
    ng_group = np.zeros(n * n_cat, np.int64)
    iou = np.full(total, np.nan)
    if annotations is not None:
        groups = [list(annotations[i].get(category_ids[c], []) or []) for i in range(n) for c in range(n_cat)]
        gt_cnts, gt_starts, goff = ground_truth_runs(groups, h, w)
        ng_group = np.diff(goff)
        grp = (plane // nl) * n_cat + np.asarray(chan, np.int64)[plane % nl]
        ng_slot = ng_group[grp]
        row_off = _starts(ng_slot)
        npairs = int(row_off[-1])
        if npairs:
            dt_cnts, dt_starts, _, _ = U.rle_encode_instances(planes, counts, geometry=geo)
            local = np.arange(npairs, dtype=np.int64) - np.repeat(row_off[:-1], ng_slot)
            pair_dt = np.repeat(np.arange(total, dtype=np.int64), ng_slot)
            pair_gt = np.repeat(goff[grp], ng_slot) + local
            iou_pairs = pair_iou(dt_cnts, dt_starts, gt_cnts, gt_starts, pair_dt, pair_gt)
            best = torch.empty(total, dtype=torch.float64, device=labels.device)
            row_off_d = torch.from_numpy(row_off).to(labels.device)
            L.fcall("mcb_iou_row_max", iou_pairs.data_ptr(), row_off_d.data_ptr(), int(total), best.data_ptr())
            iou = best.cpu().numpy()
    has_gt = ng_group.reshape(n, n_cat)[:, chan].reshape(-1) > 0 if n * nl else np.zeros(0, bool)
    return {"n": n, "layers": nl, "h": h, "w": w, "thresholds": thr, "counts": geo["counts"], "plane": plane,
            "area": geo["area"].astype(np.int64), "rmin": geo["rmin"].astype(np.int64),
            "rmax": geo["rmax"].astype(np.int64), "cmin": geo["cmin"].astype(np.int64),
            "cmax": geo["cmax"].astype(np.int64), "psum": geo["psum"], "pmax": geo["pmax"],
            "prob_dtype": np.float64 if probs.dtype == torch.float64 else np.float32,
            "contour_length": clen[:total].cpu().numpy().astype(np.int64), "iou": iou, "has_gt": has_gt}


def _feature_columns(t):
    """the per-slot feature columns of a scoring_features_batch table, with get_features_for_mask's arithmetic"""
    h, w = t["h"], t["w"]
    area = t["area"]
    r0, r1, c0, c1 = t["rmin"], t["rmax"] + 1, t["cmin"], t["cmax"] + 1
    bh, bw = r1 - r0, c1 - c0
    dists = np.stack([r0, h - r1, c0, w - c1])
    with np.errstate(divide='ignore', invalid='ignore'):
        mean = t["psum"] / area
        # np.where(mask, probabilities, 0).max(): the zeros outside the mask take part
        pmax = np.where(area < h * w, np.maximum(t["pmax"], 0.0), t["pmax"])
        cols = {'area': area, 'mean_prob': mean, 'max_prob': pmax.astype(t["prob_dtype"]), 'bbox_ar': bh / bw,
                'bbox_area': bw * bh, 'bbox_fill': area / (bw * bh), 'min_dist_to_border': dists.min(0),
                'max_dist_to_border': dists.max(0), 'contour_length': t["contour_length"]}
    return cols


def feature_frames(table):
    """scoring_features_batch table -> [[DataFrame per layer] per image] with get_features_for_image's columns, column
    order and dtypes (float64 probabilities, which the pipelines feed, give the reference's dtypes exactly); a layer
    without instances is an empty DataFrame, a layer without ground truth has an object `iou` column of None"""
    import pandas as pd
    cols = _feature_columns(table)
    offs = _starts(table["counts"])
    nl = table["layers"]
    thresholds = [round(np.float64(t), 2) for t in table["thresholds"]]
    out = []
    for i in range(table["n"]):
        image_features = []
        for li in range(nl):
            p = i * nl + li
            a, b = int(offs[p]), int(offs[p + 1])
            if a == b:
                image_features.append(pd.DataFrame([]))
                continue
            iou = table["iou"][a:b] if table["has_gt"][p] else np.full(b - a, None, dtype=object)
            d = {'iou': iou, 'threshold': np.full(b - a, thresholds[li], np.float64)}
            d.update({k: v[a:b] for k, v in cols.items()})
            image_features.append(pd.DataFrame(d, columns=list(FEATURE_COLUMNS)))
        out.append(image_features)
    return out


def instance_features(labels, probabilities, category_layers=None):
    """get_features_for_image without ground truth (src/postprocessing.py:261-306): per layer a list of per-instance
    feature dicts {iou: None, threshold, area, mean_prob, max_prob, bbox_ar, bbox_area, bbox_fill, min_dist_to_border,
    max_dist_to_border, contour_length}.  labels (L, H, W) int32, probabilities (C, H, W)."""
    category_layers = category_config()[0] if category_layers is None else category_layers
    lab = _to_dev(np.asarray(labels).astype(np.int32), torch.int32)
    probs = np.asarray(probabilities)
    pr = _to_dev(probs, torch.float64 if probs.dtype == np.float64 else torch.float32)
    t = scoring_features_batch(lab[None], pr[None], None, category_layers)
    cols = _feature_columns(t)
    offs = _starts(t["counts"])
    thresholds = get_thresholds(category_layers)
    out = []
    for li in range(t["layers"]):
        feats = []
        for s in range(int(offs[li]), int(offs[li + 1])):
            f = {'iou': None, 'threshold': round(thresholds[li], 2)}
            f.update({k: v[s].item() for k, v in cols.items()})
            f['max_prob'] = float(t["pmax"][s]) if f['area'] == t["h"] * t["w"] else max(float(t["pmax"][s]), 0.0)
            feats.append(f)
        out.append(feats)
    return out


def get_features_for_image(image, probabilities, annotations):
    """src/postprocessing.py:261-272: [DataFrame per layer] of one image, on the device"""
    return FeatureExtractor().transform([image], [probabilities], [annotations])['features'][0]


def get_iou_matrix(labels, annotations):
    """src/postprocessing.py:306-321: cocomask.iou of every instance of one label layer (rows, label order) against the
    annotations (columns), float64; None without annotations.  The annotations are left as they are (the reference
    replaces their segmentations by the first polygon's RLE)."""
    from . import utils as U
    if annotations is None or annotations == []:
        return None
    lab = _to_dev(np.asarray(labels).astype(np.int32), torch.int32)
    h, w = lab.shape
    k = int(lab.max()) if lab.numel() else 0
    if k == 0:
        return []                 # cocomask.iou of an empty list
    gt_cnts, gt_starts, _ = ground_truth_runs([list(annotations)], h, w)
    g = len(gt_starts) - 1
    dt_cnts, dt_starts, _, _ = U.rle_encode_instances(lab[None], torch.full((1,), k, dtype=torch.int32,
                                                                            device=lab.device))
    pair_dt = np.repeat(np.arange(k), g)
    pair_gt = np.tile(np.arange(g), k)
    return pair_iou(dt_cnts, dt_starts, gt_cnts, gt_starts, pair_dt, pair_gt).cpu().numpy().reshape(k, g)


def get_iou(iou_matrix, label_nr):
    """src/postprocessing.py:324-328"""
    if iou_matrix is not None:
        return iou_matrix[label_nr - 1].max()
    return None


def get_mask_with_iou(category_ind, category_instances, category_layers_inds, annotations, probabilities):
    """src/postprocessing.py:275-283"""
    category_ids = category_config()[1]
    category_nr = np.searchsorted(category_layers_inds, category_ind, side='right')
    category_annotations = annotations.get(category_ids[category_nr], [])
    iou_matrix = get_iou_matrix(category_instances, category_annotations)
    category_probabilities = probabilities[category_nr]
    for label_nr in range(1, category_instances.max() + 1):
        mask = category_instances == label_nr
        yield mask, get_iou(iou_matrix, label_nr), category_probabilities


def _prob_tensor(x):
    """probabilities on the device, float32 kept, anything else as float64 (what skimage's resize hands over)"""
    t = x.to(_dev()) if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).to(_dev())
    return (t if t.dtype in (torch.float32, torch.float64) else t.to(torch.float64)).contiguous()


def _label_tensor(x):
    t = x.to(_dev()) if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).to(_dev())
    return t.to(torch.int32).contiguous()


def image_batches(images, probabilities, annotations, batch_size):
    """(labels (B, L, H, W) int32 cuda, probabilities (B, C, H, W) cuda, [annotations]) for consecutive images, at most
    `batch_size` of one size each.  Two device tensors are sliced; anything else is consumed once, in step, as the
    reference's zip does: per-image lists, or the generators the Step chain passes in stream mode
    (make_apply_transformer_stream, which scoring_model_train switches on)."""
    if isinstance(images, torch.Tensor) and isinstance(probabilities, torch.Tensor):
        n = images.shape[0]
        ann = [{}] * n if annotations is None else list(annotations)
        for b in range(0, n, batch_size):
            yield _label_tensor(images[b:b + batch_size]), _prob_tensor(probabilities[b:b + batch_size]), \
                ann[b:b + batch_size]
        return
    group = []

    def stacked():
        return (torch.stack([g[0] for g in group]), torch.stack([g[1] for g in group]), [g[2] for g in group])

    for im, pr, ann in zip(images, probabilities, itertools.repeat({}) if annotations is None else annotations):
        im, pr = _label_tensor(im), _prob_tensor(pr)
        if group and (len(group) == batch_size or group[0][0].shape != im.shape or group[0][1].shape != pr.shape):
            yield stacked()
            group = []
        group.append((im, pr, ann))
    if group:
        yield stacked()


class _Stateless:
    """BaseTransformer contract (src/steps/base.py:254-269) of a transformer without state"""

    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        self.fit(*args, **kwargs)
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)


class FeatureExtractor(_Stateless):
    """src/postprocessing.py:18-25: transform(images, probabilities, annotations=None) -> {'features': [[DataFrame per
    layer] per image]}.  images: the dilated label maps, a list of (L, H, W) arrays or an (N, L, H, W) device tensor;
    probabilities: the resized probabilities, (C, H, W) arrays or an (N, C, H, W) device tensor (the fast path: nothing
    crosses PCIe but the feature table); annotations: per image {category id: [COCO annotations]}.  Lists and the
    generators of stream mode are consumed once; images go through scoring_features_batch up to `batch_size` of one
    size at a time, so tiles of different sizes may be mixed."""

    def __init__(self, batch_size=20):
        self.batch_size = int(batch_size)

    def transform(self, images, probabilities, annotations=None):
        features = []
        for lab, pr, ann in image_batches(images, probabilities, annotations, self.batch_size):
            features.extend(feature_frames(scoring_features_batch(lab, pr, ann)))
        return {'features': features}


class ScoreImageJoiner(_Stateless):
    """src/postprocessing.py:28-33"""

    def transform(self, images, scores):
        return {'images_with_scores': list(zip(images, scores))}


# ---------------------------------------------------------------------------------------------------------------------
# batched transformer
# ---------------------------------------------------------------------------------------------------------------------
class MaskPostprocessor:
    """mask_postprocessing of src/pipelines.py:248-304 for a whole batch on the device:
    (resize | centre-crop) -> categorize_multilayer_image -> erode_image -> label_multilayer_image -> dilate_image
    -> build_score.  transform() returns {'y_pred': [(labels (L,H,W) int32, [[score, ...], ...]), ...]} like the
    reference's `output` step."""

    def __init__(self, target_size=(300, 300), mode="resize", erode_selem_size=0, dilate_selem_size=0,
                 category_layers=None):
        assert mode in ("resize", "crop")
        self.target_size, self.mode = tuple(target_size), mode
        self.erode, self.dilate = erode_selem_size, dilate_selem_size
        self.category_layers = category_layers or CATEGORY_LAYERS

    # BaseTransformer contract (src/steps/base.py:254-269): stateless, so fit is a no-op and save/load persist nothing
    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        self.fit(*args, **kwargs)
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("_graphs", None)     # captured CUDA graphs and their static buffers are rebuilt on demand
        return state

    def run_device(self, probs, kcap=1024):
        """probs (N, C, S, S) float32 cuda -> (labels int32 (N,L,H,W), scores float64 (N*L, kcap), counts int32 (N*L,),
        probabilities used).  No host synchronisation inside."""
        assert probs.is_cuda and probs.dtype == torch.float32
        probs = probs.contiguous()
        if self.mode == "resize":
            pr = resize_batch(probs, self.target_size)
        else:
            h, w = probs.shape[-2:]
            h0, w0 = int((h - self.target_size[0]) / 2.), int((w - self.target_size[1]) / 2.)
            pr = probs[:, :, h0:h - h0, w0:w - w0].contiguous()
        masks = threshold_batch(pr, self.category_layers)
        masks = erode_batch(masks, self.erode)
        labels, counts = label_batch(masks, return_counts=True)
        if self.dilate > 0:
            labels = morph_batch(labels, self.dilate, dilation=True)
        n, l, h, w = labels.shape
        if l != pr.shape[1]:
            raise NotImplementedError("score pairing needs as many layers as probability channels (CATEGORY_LAYERS=[1,1])")
        scores = scores_strided(labels.view(n * l, h, w), pr.view(n * l, h, w), counts, kcap)
        return labels, scores, counts, pr

    def run_device_graphed(self, probs, kcap=1024):
        """run_device replayed as ONE CUDA graph per (input shape, kcap): the chain is ~10 short launches whose host-side
        launch cost exceeds their device time.  The returned tensors are STATIC buffers overwritten by the next call with
        the same shape -- consume (or clone) them before calling again."""
        key = (tuple(probs.shape), int(kcap))
        cache = self.__dict__.setdefault("_graphs", {})
        ent = cache.get(key)
        if ent is None:
            static_in = probs.clone()
            self.run_device(static_in, kcap)          # eager warm-up (module loading, allocator)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                outs = self.run_device(static_in, kcap)
            ent = cache[key] = (g, static_in, outs)
        g, static_in, outs = ent
        static_in.copy_(probs, non_blocking=True)
        g.replay()
        return outs

    def transform(self, images, **_):
        probs = images if isinstance(images, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.stack(images)))
        probs = probs.to(device=_dev(), dtype=torch.float32)
        kcap = 1024
        while True:
            labels, scores, counts, _pr = self.run_device_graphed(probs, kcap)
            cnt = counts.cpu().numpy()
            if cnt.size == 0 or int(cnt.max()) <= kcap:
                break
            kcap = int(cnt.max())
        lab = labels.cpu().numpy()
        s = scores.cpu().numpy()
        n, l = lab.shape[:2]
        out = []
        for i in range(n):
            sc = []
            for j in range(l):
                vals = s[i * l + j, :cnt[i * l + j]]
                sc.append([np.ma.masked if np.isnan(v) else v for v in vals])
            out.append((lab[i], sc))
        return {"y_pred": out}
