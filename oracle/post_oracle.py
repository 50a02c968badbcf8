"""TEST INFRASTRUCTURE — CPU oracle for the per-pixel mask post-processing.  Never imported by the product path.

Restates, in numpy/scipy, the reference functions of src/postprocessing.py:48-258 and
src/utils.py:231-273,324-339.  Each function cites the lines it follows.

Third-party algorithms the reference calls but that are absent from the reference repository and from its pinned environment:
  * scikit-image (unpinned in environment.yml; the April-2018 conda env resolves to 0.13.x/0.14.x):
      skimage.transform.resize, skimage.morphology.{erosion, dilation, rectangle}
    restated below from skimage's published implementation of that era (they are thin wrappers over scipy.ndimage,
    which IS present and is called directly).  ASSUMPTION (could not be re-verified offline): skimage <= 0.17
    semantics, i.e. resize maps mode='constant' to ndimage mode 'constant' (later releases use 'grid-constant').
  * pydensecrf (git master, unpinned): dense CRF mean-field of Kraehenbuehl & Koltun (NIPS 2011).  dense_crf below
    restates the published algorithm with EXACT (windowed) Gaussian filtering instead of the library's permutohedral
    lattice approximation -> "parity unpinned" for this function (no golden vector from the real library exists).
  * watershed: NOT in the reference at all (SURVEY.md 0.4); minimax_watershed below DEFINES the semantics
    -> "parity unpinned".

Pinned parts: scipy.ndimage.label numbering against the reference's only known-answer vector
(src/postprocessing.py:95-111) and every function against the reference's own code executed through
oracle/ref_shim.py (tests/test_oracle_pins.py, fixtures in tests/golden/ made by oracle/make_golden.py).
"""
import numpy as np
from scipy import ndimage as ndi

CATEGORY_LAYERS = [1, 1]  # src/pipeline_config.py:18
MEAN = [0.485, 0.456, 0.406]  # src/pipeline_config.py:19
STD = [0.229, 0.224, 0.225]  # src/pipeline_config.py:20


# --------------------------------------------------------------------------------------------------------------------
# skimage restatements (used by the shim as the reference's `skimage` module, and by the functions below)
# --------------------------------------------------------------------------------------------------------------------
def skimage_resize(image, output_shape, order=1, mode='constant', cval=0, clip=True, preserve_range=False, **_):
    """skimage.transform.resize (0.13/0.14), n-D branch: float64 output sampled with
    ndi.map_coordinates(order=1, mode='constant', cval=0) at coords (i + 0.5) * in/out - 0.5 per axis; no
    anti-aliasing filter when up-sampling (factors <= 1); output clipped to the input range (a no-op for order 1).
    The 2-D `warp` branch (taken only when the LAST axis keeps its size) is not needed by the reference call
    resize((C,H,W) -> (C,Ht,Wt)) unless W == Wt, which src/pipelines.py never does; it is rejected here."""
    image = np.asarray(image)
    output_shape = tuple(int(s) for s in output_shape)
    assert order == 1 and mode == 'constant' and cval == 0
    assert len(output_shape) == image.ndim
    if image.ndim == 3 and output_shape[2] == image.shape[2] and output_shape != image.shape:
        raise NotImplementedError("skimage 2-D warp branch (unchanged last axis) is outside the reference's usage")
    img = image.astype(np.float64)
    factors = np.asarray(image.shape, dtype=float) / np.asarray(output_shape, dtype=float)
    coord_arrays = [factors[i] * (np.arange(d) + 0.5) - 0.5 for i, d in enumerate(output_shape)]
    coord_map = np.array(np.meshgrid(*coord_arrays, sparse=False, indexing='ij'))
    out = ndi.map_coordinates(img, coord_map, order=1, mode='constant', cval=0.0)
    if clip:
        lo, hi = min(img.min(), 0.0), max(img.max(), 0.0)
        np.clip(out, lo, hi, out=out)
    return out


def skimage_rectangle(width, height, dtype=np.uint8):
    """skimage.morphology.rectangle: np.ones((width, height))"""
    return np.ones((width, height), dtype=dtype)


def _pad_even_selem(selem):
    """skimage.morphology.misc._shift_selem with shift_x = shift_y = False: an even-sized axis gets one zero
    row/column prepended so the element has a centre pixel."""
    selem = np.array(selem)
    if selem.ndim != 2:
        return selem
    m, n = selem.shape
    if m % 2 == 0:
        selem = np.vstack((np.zeros((1, n), selem.dtype), selem))
        m += 1
    if n % 2 == 0:
        selem = np.hstack((np.zeros((m, 1), selem.dtype), selem))
    return selem


def skimage_erosion(image, selem=None, out=None):
    """skimage.morphology.erosion: ndi.grey_erosion(image, footprint=padded selem) (border mode 'reflect')"""
    selem = _pad_even_selem(selem)
    image = np.asarray(image)
    if out is None:
        out = np.empty_like(image)
    ndi.grey_erosion(image, footprint=selem, output=out)
    return out


def skimage_dilation(image, selem=None, out=None):
    """skimage.morphology.dilation: the padded selem is flipped ([::-1, ::-1]) to undo the flip scipy's
    grey_dilation applies internally, then ndi.grey_dilation(image, footprint=...)"""
    selem = _pad_even_selem(selem)
    selem = selem[::-1, ::-1]
    image = np.asarray(image)
    if out is None:
        out = np.empty_like(image)
    ndi.grey_dilation(image, footprint=selem, output=out)
    return out


# --------------------------------------------------------------------------------------------------------------------
# reference functions
# --------------------------------------------------------------------------------------------------------------------
def softmax(X, theta=1.0, axis=None):
    """src/utils.py:231-273 — stable softmax along `axis` (dtype follows X: float32 in the pipeline)"""
    y = np.atleast_2d(X)
    if axis is None:
        axis = next(j[0] for j in enumerate(y.shape) if j[1] > 1)
    y = y * float(theta)
    y = y - np.expand_dims(np.max(y, axis=axis), axis)
    y = np.exp(y)
    p = y / np.expand_dims(np.sum(y, axis=axis), axis)
    if len(np.shape(X)) == 1:
        p = p.flatten()
    return p


def resize_image(image, target_size):
    """src/postprocessing.py:48-61"""
    n_channels = image.shape[0]
    return skimage_resize(image, (n_channels,) + tuple(target_size), mode='constant')


def categorize_image(image):
    """src/postprocessing.py:64-74"""
    return np.argmax(image, axis=0)


def layer_thresholds(category_layers=CATEGORY_LAYERS):
    """the threshold list categorize_multilayer_image builds (src/postprocessing.py:79-81), per channel"""
    out = []
    for n_layers in category_layers:
        step = 1. / (n_layers + 1)
        out.append(np.arange(step, 1, step))
    return out


def categorize_multilayer_image(image, category_layers=CATEGORY_LAYERS):
    """src/postprocessing.py:77-84"""
    layers = []
    for category_output, thresholds in zip(image, layer_thresholds(category_layers)):
        for threshold in thresholds:
            layers.append(category_output > threshold)
    return np.stack(layers)


def label(mask):
    """src/utils.py:328-330 — scipy.ndimage.label, default cross structure (4-connectivity in 2-D), int32"""
    labeled, _ = ndi.label(mask)
    return labeled


def label_multiclass_image(mask):
    """src/postprocessing.py:87-124"""
    return np.stack([label(mask == c) for c in range(0, mask.max() + 1)])


def label_multilayer_image(mask):
    """src/postprocessing.py:127-132"""
    return np.stack([label(channel) for channel in mask])


def add_dropped_objects(original, processed):
    """src/utils.py:333-339 — re-add every component of `original` that vanished completely from `processed`"""
    reconstructed = processed.copy()
    labeled = label(original)
    for i in range(1, labeled.max() + 1):
        if not np.any(np.where((labeled == i) & processed)):
            reconstructed += (labeled == i)
    return reconstructed.astype('uint8')


def erode_image(mask, erode_selem_size):
    """src/postprocessing.py:135-156.  The reference's multi-layer branch raises AttributeError on its second
    layer (np.stack inside the loop, SURVEY.md 0.6) and would label across layers in add_dropped_objects; the
    INTENDED per-layer 2-D behaviour is restated here (deviation documented in DESIGN.md)."""
    if not erode_selem_size > 0:
        return mask
    selem = skimage_rectangle(erode_selem_size, erode_selem_size)
    if mask.ndim == 2:
        return add_dropped_objects(mask, skimage_erosion(mask, selem=selem))
    return np.stack([add_dropped_objects(m, skimage_erosion(m, selem=selem)) for m in mask])


def dilate_image(mask, dilate_selem_size):
    """src/postprocessing.py:159-180"""
    if not dilate_selem_size > 0:
        return mask
    selem = skimage_rectangle(dilate_selem_size, dilate_selem_size)
    if mask.ndim == 2:
        return skimage_dilation(mask, selem=selem)
    return np.stack([skimage_dilation(m, selem=selem) for m in mask])


def build_score(image, probabilities):
    """src/postprocessing.py:228-236 — per layer, per instance: mean probability x sqrt(area)"""
    total_score = []
    for category_instances, category_probabilities in zip(image, probabilities):
        score = []
        for label_nr in range(1, category_instances.max() + 1):
            masked_instance = np.ma.masked_array(category_probabilities, mask=category_instances != label_nr)
            score.append(masked_instance.mean() * np.sqrt(np.count_nonzero(category_instances == label_nr)))
        total_score.append(score)
    return image, total_score


def crop_image_center_per_class(image, h_crop, w_crop):
    """src/postprocessing.py:239-258 (the `[h0:-h0]` slice is empty when h0 == 0, as in the reference)"""
    out = []
    for class_prediction in image:
        h, w = class_prediction.shape[:2]
        h_start, w_start = int((h - h_crop) / 2.), int((w - w_crop) / 2.)
        out.append(class_prediction[h_start:-h_start, w_start:-w_start])
    return np.stack(out)


def denormalize_img(image, mean=MEAN, std=STD):
    """src/utils.py:324-325"""
    return image * np.array(std).reshape(3, 1, 1) + np.array(mean).reshape(3, 1, 1)


# --------------------------------------------------------------------------------------------------------------------
# dense CRF (PARITY UNPINNED: restates the published algorithm; the reference's pydensecrf is absent)
# --------------------------------------------------------------------------------------------------------------------
def crf_rgb_image(img):
    """src/postprocessing.py:213-215: de-normalise, x255, HWC, cast to uint8 (C cast: truncation, wrap-around)"""
    org = denormalize_img(img) * 255.
    org = org.transpose(1, 2, 0)
    return np.ascontiguousarray(org, dtype=np.float64).astype(np.int64).astype(np.uint8)


def dense_crf(img, output_probs, compat_gaussian=3, sxy_gaussian=1, compat_bilateral=10, sxy_bilateral=1, srgb=50,
              iterations=5, radius=6):
    """src/postprocessing.py:183-225 with pydensecrf's calls restated:
      unary_from_softmax: U = -log(max(p, 1e-5))                                 (pydensecrf/utils.py)
      DenseCRF2D.addPairwiseGaussian(sxy, compat)  : features (x, y)/sxy
      DenseCRF2D.addPairwiseBilateral(sxy, srgb, rgbim, compat): features (x, y)/sxy, (r, g, b)/srgb
      both with Potts compatibility and NORMALIZE_SYMMETRIC: message = n (.) K (n (.) Q), n = 1/sqrt(K 1 + 1e-20)
      inference(it): Q = softmax(-U); repeat it times: Q = softmax(-U + sum_k compat_k * message_k(Q))
    The Gaussian kernels are evaluated EXACTLY inside a (2*radius+1)^2 window (K(i,i) = 1 included, as the
    lattice blur does); with sxy = 1 the truncated tail is < exp(-radius^2/2) ~ 1.5e-8 at radius 6.
    float32 arithmetic like the library.  Returns (C, H, W) float32."""
    C, H, W = output_probs.shape
    rgb = crf_rgb_image(img).astype(np.float32)  # H, W, 3
    U = -np.log(np.maximum(output_probs.astype(np.float32), np.float32(1e-5)))

    offs = [(dy, dx) for dy in range(-radius, radius + 1) for dx in range(-radius, radius + 1)]

    def shifted(a, dy, dx):
        """a[y+dy, x+dx] with zeros outside; a is (..., H, W)"""
        out = np.zeros_like(a)
        ys0, ys1 = max(0, -dy), min(H, H - dy)
        xs0, xs1 = max(0, -dx), min(W, W - dx)
        out[..., ys0:ys1, xs0:xs1] = a[..., ys0 + dy:ys1 + dy, xs0 + dx:xs1 + dx]
        return out

    rgb_c = rgb.transpose(2, 0, 1)  # 3, H, W
    inside = np.ones((H, W), np.float32)
    kg, kb = [], []
    for dy, dx in offs:
        sp_g = np.float32(np.exp(-0.5 * (dy * dy + dx * dx) / (sxy_gaussian ** 2)))
        sp_b = np.float32(np.exp(-0.5 * (dy * dy + dx * dx) / (sxy_bilateral ** 2)))
        m = shifted(inside, dy, dx)
        d = rgb_c - shifted(rgb_c, dy, dx)
        col = np.exp(np.float32(-0.5) * (d * d).sum(0) / np.float32(srgb * srgb)).astype(np.float32)
        kg.append(sp_g * m)
        kb.append(sp_b * col * m)
    ng = 1.0 / np.sqrt(sum(kg) + np.float32(1e-20))
    nb = 1.0 / np.sqrt(sum(kb) + np.float32(1e-20))

    def message(Q, ks, nrm):
        Qn = Q * nrm
        acc = np.zeros_like(Q)
        for (dy, dx), k in zip(offs, ks):
            acc += k * shifted(Qn, dy, dx)
        return acc * nrm

    def exp_norm(E):
        E = E - E.max(0, keepdims=True)
        P = np.exp(E)
        return (P / P.sum(0, keepdims=True)).astype(np.float32)

    Q = exp_norm(-U)
    for _ in range(iterations):
        E = -U + np.float32(compat_gaussian) * message(Q, kg, ng) + np.float32(compat_bilateral) * message(Q, kb, nb)
        Q = exp_norm(E)
    return Q.reshape(output_probs.shape)


# --------------------------------------------------------------------------------------------------------------------
# watershed (PARITY UNPINNED: not a reference function; this restatement DEFINES the semantics)
# --------------------------------------------------------------------------------------------------------------------
def minimax_watershed(prob, markers, mask, levels=256):
    """Marker-based watershed on the relief -prob (4-connectivity), defined order-independently in three stages so
    that any relaxation schedule reaches the same fixed point:
      level(p) = floor((1 - prob(p)) * (levels - 1))   (quantised relief; high probability = low ground)
      1. cost(p)  = min over paths from any marker pixel to p inside `mask` of the MAX level on the path
                    (marker pixels have cost 0);
      2. dist(p)  = fewest steps from a marker along "tight" moves q->p, i.e. cost(p) == max(cost(q), level(p));
      3. label(p) = smallest marker label reachable through tight moves that also decrease dist by exactly one.
    Pixels outside `mask` or unreachable get 0.  prob: (H, W) float; markers: (H, W) int32 (0 = none);
    mask: (H, W) bool.  Returns int32 (H, W)."""
    H, W = prob.shape
    lev = np.floor((1.0 - prob.astype(np.float64)) * (levels - 1)).astype(np.int64)
    lev = np.clip(lev, 0, levels - 1)
    INF = np.int64(1 << 40)
    mask = mask.astype(bool) | (markers > 0)
    is_m = markers > 0
    cost = np.where(is_m, 0, INF).astype(np.int64)

    def nbrs(a, fill):
        p = np.pad(a, 1, constant_values=fill)
        return [p[:-2, 1:-1], p[2:, 1:-1], p[1:-1, :-2], p[1:-1, 2:]]

    while True:
        cand = np.minimum.reduce(nbrs(cost, INF))
        new = np.where(mask & ~is_m, np.minimum(cost, np.maximum(cand, lev)), cost)
        if np.array_equal(new, cost):
            break
        cost = new
    dist = np.where(is_m, 0, INF).astype(np.int64)
    while True:
        best = np.full((H, W), INF)
        for cq, dq in zip(nbrs(cost, INF), nbrs(dist, INF)):
            tight = (np.maximum(cq, lev) == cost) & (cq < INF)
            best = np.minimum(best, np.where(tight, dq + 1, INF))
        new = np.where(mask & ~is_m & (cost < INF), np.minimum(dist, best), dist)
        if np.array_equal(new, dist):
            break
        dist = new
    lab = np.where(is_m, markers, INF).astype(np.int64)
    while True:
        best = np.full((H, W), INF)
        for cq, dq, lq in zip(nbrs(cost, INF), nbrs(dist, INF), nbrs(lab, INF)):
            ok = (np.maximum(cq, lev) == cost) & (cq < INF) & (dq + 1 == dist)
            best = np.minimum(best, np.where(ok, lq, INF))
        new = np.where(mask & ~is_m & (dist < INF), np.minimum(lab, best), lab)
        if np.array_equal(new, lab):
            break
        lab = new
    return np.where(lab < INF, lab, 0).astype(np.int32)
