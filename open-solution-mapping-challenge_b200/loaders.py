"""Test-time augmentation on the device: mirror of src/loaders.py:401-517
(TestTimeAugmentationGenerator, TestTimeAugmentationAggregator, test_time_augmentation_transform /
_inverse_transform, aggregate_augmentations) for the flip / rot90 variants the pipeline configures
(src/pipeline_config.py:121-127: flip_ud, flip_lr, rotation, no colour shift -> 16 variants per image).

The reference builds every variant on the host (numpy flips + skimage.rotate per image) inside the DataLoader, runs
the network on 16x the images, then inverts every prediction channel by channel and reduces with scipy's gmean in a
thread pool.  Here the variants are index maps: one kernel writes the 16 views of a batch straight from the normalised
device batch, and ONE kernel undoes the maps, takes the class softmax of the raw logits and reduces
(gmean / mean / max / min) without materialising any inverse-transformed prediction (csrc/instances.cu).

Assumption (skimage is not installable here, SURVEY.md 8c): `skimage.transform.rotate(image, angle,
preserve_range=True)` at angle in {0, 90, 180, 270} on a square image is the exact quarter-turn index permutation
(np.rot90, counter-clockwise).  Colour-shift variants (imgaug, random) are out of scope and rejected.
"""
from itertools import product

import numpy as np
import torch

from . import _lib as L
from .postprocessing import _dev, _to_dev

METHODS = {"gmean": 0, "mean": 1, "max": 2, "min": 3}


def tta_specs(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=False):
    """the spec list of TestTimeAugmentationGenerator._get_tta_data (src/loaders.py:413-432) for one image"""
    if color_shift_runs:
        raise NotImplementedError("colour-shift TTA variants are random imgaug transforms; not built on the H100 path")
    original = {'ud_flip': False, 'lr_flip': False, 'rotation': 0, 'color_shift': False}
    specs = [original]
    ud_options = [True, False] if flip_ud else [False]
    lr_options = [True, False] if flip_lr else [False]
    rot_options = [0, 90, 180, 270] if rotation else [0]
    for ud, lr, rot, color in product(ud_options, lr_options, rot_options, [False]):
        if ud is False and lr is False and rot == 0 and color is False:
            continue
        specs.append({'ud_flip': ud, 'lr_flip': lr, 'rotation': rot, 'color_shift': color})
    return specs


def spec_code(spec):
    """k | flip << 2 as consumed by the kernels.  `if ud_flip ... elif lr_flip` (src/loaders.py:471-474, 489-492): a spec
    with both flips set applies the up-down flip only — kept."""
    if spec.get('color_shift'):
        raise NotImplementedError("colour-shift TTA variants are not built on the H100 path")
    rot = int(spec['rotation'])
    if rot % 90 != 0:
        raise NotImplementedError("TTA rotations are multiples of 90 degrees (src/loaders.py:417)")
    k = (rot // 90) % 4
    flip = 1 if spec['ud_flip'] else (2 if spec['lr_flip'] else 0)
    return k | (flip << 2)


class TestTimeAugmentationGenerator:
    """src/loaders.py:401-432: replicates every metadata row once per variant.  transform(X) -> {'X_tta', 'tta_params',
    'img_ids'} exactly like the reference (X_tta stays whatever row container X was: list or DataFrame rows)."""
    __test__ = False

    def __init__(self, **kwargs):
        self.tta_transformations = dict(kwargs)

    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)

    def transform(self, X, **kwargs):
        X_tta_rows, tta_params, img_ids = [], [], []
        specs = tta_specs(**self.tta_transformations)
        rows = X.values if hasattr(X, "values") else X
        for i in range(len(X)):
            tta_params.extend(specs)
            img_ids.extend([i] * len(specs))
            X_tta_rows.extend([rows[i]] * len(specs))
        try:
            import pandas as pd
            X_tta = pd.DataFrame(X_tta_rows)
        except Exception:
            X_tta = X_tta_rows
        return {'X_tta': X_tta, 'tta_params': tta_params, 'img_ids': img_ids}


def test_time_augmentation_transform_batch(X, tta_params, img_ids):
    """device form of test_time_augmentation_transform (src/loaders.py:470-480) for a whole batch: X (N, C, H, W) float32
    cuda (already normalised / padded; flips and quarter turns commute with per-pixel normalisation and with the
    symmetric replicate padding) -> (len(tta_params), C, H, W) float32 cuda, variant v built from image img_ids[v]"""
    assert X.is_cuda and X.dtype == torch.float32
    X = X.contiguous()
    n, c, h, w = X.shape
    codes = np.array([spec_code(s) for s in tta_params], np.int32)
    if h != w and (codes & 1).any():
        raise NotImplementedError("quarter-turn TTA variants need square images")
    ids = np.asarray(img_ids, np.int32)
    nv = len(codes)
    out = torch.empty((nv, c, h, w), dtype=torch.float32, device=X.device)
    ids_d, codes_d = torch.from_numpy(ids).to(X.device), torch.from_numpy(codes).to(X.device)   # kept alive past the launch
    L.fcall("mcb_tta_transform", X.data_ptr(), out.data_ptr(), ids_d.data_ptr(), codes_d.data_ptr(), nv, c, h, w)
    return out


test_time_augmentation_transform_batch.__test__ = False


def aggregate_batch(pred, tta_params, img_ids, method="gmean", from_logits=False):
    """pred (NV, C, H, W) float32 cuda: probabilities (or raw logits with from_logits=True) of every variant
    -> (N_images, C, H, W) float32 cuda, images ordered by sorted unique img_id"""
    assert pred.is_cuda and pred.dtype == torch.float32
    pred = pred.contiguous()
    nv, c, h, w = pred.shape
    codes = np.array([spec_code(s) for s in tta_params], np.int32)
    if h != w and (codes & 1).any():
        raise NotImplementedError("quarter-turn TTA variants need square images")
    ids = np.asarray(img_ids)
    uniq = sorted(set(ids.tolist()))
    order = np.concatenate([np.nonzero(ids == u)[0] for u in uniq]).astype(np.int32)
    var_start = np.concatenate([[0], np.cumsum([int((ids == u).sum()) for u in uniq])]).astype(np.int32)
    dev = pred.device
    out = torch.empty((len(uniq), c, h, w), dtype=torch.float32, device=dev)
    start_d, order_d, codes_d = (torch.from_numpy(a).to(dev) for a in (var_start, order, codes))   # kept alive past the launch
    L.fcall("mcb_tta_aggregate", pred.data_ptr(), int(bool(from_logits)), start_d.data_ptr(), order_d.data_ptr(),
            codes_d.data_ptr(), out.data_ptr(), len(uniq), c, h, w, METHODS[method])
    return out


class TestTimeAugmentationAggregator:
    """src/loaders.py:435-458: transform(images, tta_params, img_ids) -> {'aggregated_prediction': [ (C,H,W) ... ]}.
    `images` are the network's per-variant class probabilities (numpy (NV, C, H, W) or a list of (C, H, W))."""
    __test__ = False

    def __init__(self, method, num_threads=1):
        if method not in METHODS:
            raise KeyError(method)
        self.method = method
        self.num_threads = num_threads   # host threads of the reference's pool; nothing to parallelise here

    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)

    def transform(self, images, tta_params, img_ids, **kwargs):
        if isinstance(images, torch.Tensor):
            pred = images.to(device=_dev(), dtype=torch.float32)
        else:
            pred = _to_dev(np.stack([np.asarray(im) for im in images]) if not isinstance(images, np.ndarray) else images,
                           torch.float32)
        out = aggregate_batch(pred, tta_params, img_ids, self.method).cpu().numpy()
        return {'aggregated_prediction': [a for a in out]}
