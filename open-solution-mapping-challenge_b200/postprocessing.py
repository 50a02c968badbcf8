"""Mirror of the reference's per-pixel post-processing (src/postprocessing.py:48-258,
src/utils.py:231-273,328-339) on the GPU.

Two surfaces:
  * module-level functions with the reference's names and signatures, one image in / numpy out — drop-ins for
    `make_apply_transformer(post.<fn>, ...)` in src/pipelines.py:248-304 (each call round-trips the image over PCIe);
  * `MaskPostprocessor`, the batched transformer the fast path uses: the whole batch of probability maps stays on the
    device through resize/crop -> threshold -> erode -> label -> dilate -> score, one launch sequence per batch.

All arithmetic is in libmcb200.so (csrc/postproc.cu); torch only owns the device buffers.  No CPU fallback.
"""
import numpy as np
import torch

from . import _lib as L

CATEGORY_LAYERS = [1, 1]  # src/pipeline_config.py:18
MEAN = [0.485, 0.456, 0.406]
STD = [0.229, 0.224, 0.225]


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
    category_layers = CATEGORY_LAYERS if category_layers is None else category_layers
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
    assert len(category_layers or CATEGORY_LAYERS) <= c or max(chan) < c
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
    """imgs (N,3,H,W) float32 ImageNet-normalised, probs (N,2,H,W) float32, both cuda -> (N,2,H,W) float32"""
    assert imgs.is_cuda and probs.is_cuda and imgs.dtype == torch.float32 and probs.dtype == torch.float32
    imgs, probs = imgs.contiguous(), probs.contiguous()
    n, c, h, w = probs.shape
    if c != 2:
        raise NotImplementedError("dense_crf: 2 labels (the reference builds DenseCRF2D(width, height, 2))")
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
    Not a reference function; semantics = oracle/post_oracle.py::minimax_watershed (parity unpinned)."""
    assert prob.is_cuda and prob.dtype in (torch.float32, torch.float64)
    prob, markers = prob.contiguous(), markers.contiguous().to(torch.int32)
    mask = mask.contiguous()
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    p, h, w = prob.shape
    out = torch.empty((p, h, w), dtype=torch.int32, device=prob.device)
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
    """src/postprocessing.py:321-327"""
    return layer_thresholds(category_layers)[0]


def instance_features(labels, probabilities, category_layers=None):
    """get_features_for_image without ground truth (src/postprocessing.py:261-306): per layer a list of per-instance
    feature dicts {iou: None, threshold, area, mean_prob, max_prob, bbox_ar, bbox_area, bbox_fill, min_dist_to_border,
    max_dist_to_border, contour_length}.  labels (L, H, W) int32, probabilities (C, H, W)."""
    from . import utils as U
    category_layers = CATEGORY_LAYERS if category_layers is None else category_layers
    lab = _to_dev(np.asarray(labels).astype(np.int32), torch.int32)
    n_layers, h, w = lab.shape
    inds = np.cumsum(category_layers)
    probs = np.asarray(probabilities)
    chan = [int(np.searchsorted(inds, li, side='right')) for li in range(n_layers)]
    pr = _to_dev(probs[chan], torch.float64 if probs.dtype == np.float64 else torch.float32)
    counts = lab.reshape(n_layers, -1).max(dim=1).values.to(torch.int32)
    geo = U.instance_geometry(lab, counts, pr)
    total = int(geo["counts"].sum())
    clen = torch.zeros(max(total, 1), dtype=torch.int32, device=lab.device)
    if total:
        L.fcall("mcb_contour_length", lab.data_ptr(), geo["_offsets"].data_ptr(), geo["_counts"].data_ptr(),
                clen.data_ptr(), n_layers, h, w)
    clen = clen.cpu().numpy()
    thresholds = get_thresholds(category_layers)
    out = []
    for li in range(n_layers):
        feats = []
        for i in range(int(geo["counts"][li])):
            s = int(geo["offsets"][li]) + i
            area = int(geo["area"][s])
            bbox = (int(geo["rmin"][s]), int(geo["rmax"][s]) + 1, int(geo["cmin"][s]), int(geo["cmax"][s]) + 1)
            bh, bw = bbox[1] - bbox[0], bbox[3] - bbox[2]
            dists = (bbox[0], h - bbox[1], bbox[2], w - bbox[3])
            feats.append({'iou': None, 'threshold': round(thresholds[li], 2), 'area': area,
                          'mean_prob': float(geo["psum"][s]) / area,
                          # np.where(mask, probabilities, 0).max(): the zeros outside the mask take part
                          'max_prob': max(float(geo["pmax"][s]), 0.0) if area < h * w else float(geo["pmax"][s]),
                          'bbox_ar': bh / bw, 'bbox_area': bw * bh, 'bbox_fill': area / (bw * bh),
                          'min_dist_to_border': min(dists), 'max_dist_to_border': max(dists),
                          'contour_length': int(clen[s])})
        out.append(feats)
    return out


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
