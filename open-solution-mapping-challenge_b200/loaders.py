"""Test-time augmentation on the device: mirror of src/loaders.py:307-517 (the inference loaders
ImageSegmentationLoaderInferencePadding[TTA] / ImageSegmentationLoaderResizeTTA, TestTimeAugmentationGenerator,
TestTimeAugmentationAggregator, test_time_augmentation_transform / _inverse_transform, aggregate_augmentations) for the
flip / rot90 variants and the colour-shift variants (src/pipeline_config.py:121-127: flip_ud, flip_lr, rotation,
color_shift_runs).

The reference builds every variant on the host (numpy flips, imgaug's color_seq, skimage.rotate per image) inside the
DataLoader, decoding each tile once per variant, runs the network on 16x the images, then inverts every prediction
channel by channel and reduces with scipy's gmean in a thread pool.  Here the DataLoader workers decode each distinct
file once per pass, ONE kernel writes the uint8 variant rows of a batch (geometry as index maps, colour per pixel),
the existing pad / Pillow-resize and normalise kernels finish them, and ONE kernel undoes the maps, takes the class
softmax of the raw logits and reduces (gmean / mean / max / min) without materialising any inverse-transformed
prediction (csrc/instances.cu).

Colour draws: the reference reseeds color_seq from `int(time.time()) + pid` on every call (src/utils.py:416-426), so
its draws cannot be reproduced at all.  Here every colour-applying row draws its OneOf branch (uniform over the six)
and its Add value (uniform over the integers 0..100) from a seeded numpy Generator: distribution-equal to the
reference, not draw-equal.  The colour itself is bit-exact to cv2 (csrc/instances.cu, DESIGN.md §4.5).

The training loaders of src/loaders.py:225-305 (MetadataImageSegmentationLoader[Distances]{Resize,CropPad}) are at the
bottom: DataLoader workers only decode files, the augmentation and the tensor assembly run on the device
(mcb200.augmentation).

Assumption (skimage is not installable here, SURVEY.md 8c): `skimage.transform.rotate(image, angle,
preserve_range=True)` at angle in {0, 90, 180, 270} on a square image is the exact quarter-turn index permutation
(np.rot90, counter-clockwise).
"""
from itertools import product

import numpy as np
import torch

from . import _lib as L
from .postprocessing import _dev, _to_dev

METHODS = {"gmean": 0, "mean": 1, "max": 2, "min": 3}


def tta_specs(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=False):
    """the spec list of TestTimeAugmentationGenerator._get_tta_data (src/loaders.py:415-435) for one image: the original,
    then product(ud, lr, rot, colour runs 1..N) with nothing else skipped (1 + 16 N specs with every option on)"""
    original = {'ud_flip': False, 'lr_flip': False, 'rotation': 0, 'color_shift': False}
    specs = [original]
    ud_options = [True, False] if flip_ud else [False]
    lr_options = [True, False] if flip_lr else [False]
    rot_options = [0, 90, 180, 270] if rotation else [0]
    color_options = list(range(1, color_shift_runs + 1)) if color_shift_runs else [False]
    for ud, lr, rot, color in product(ud_options, lr_options, rot_options, color_options):
        if ud is False and lr is False and rot == 0 and color is False:
            continue
        specs.append({'ud_flip': ud, 'lr_flip': lr, 'rotation': rot, 'color_shift': color})
    return specs


def spec_code(spec):
    """geometry code k | flip << 2 as consumed by the kernels (colour specs too: their inverse is geometry only,
    src/loaders.py:489-497).  `if ud_flip ... elif lr_flip` (src/loaders.py:478-481, 492-495): a spec with both flips
    set applies the up-down flip only — kept."""
    rot = int(spec['rotation'])
    if rot % 90 != 0:
        raise NotImplementedError("TTA rotations are multiples of 90 degrees (src/loaders.py:421)")
    k = (rot // 90) % 4
    flip = 1 if spec['ud_flip'] else (2 if spec['lr_flip'] else 0)
    return k | (flip << 2)


def applies_colour(spec):
    """`if ud ... elif lr ... elif color_shift` (src/loaders.py:478-484): a flipped colour spec is a plain flip"""
    return bool(spec.get('color_shift')) and not spec['ud_flip'] and not spec['lr_flip']


def draw_colour(rng, m):
    """m draws of color_seq's OneOf([...six children...]) with Add((0, 100)): branch 1-6 (1-3 Add to H, S, V; 4-6 Add
    to R, G, B), value 0..100 -> (branch int32 (m,), value int32 (m,))"""
    branch = rng.integers(1, 7, size=m).astype(np.int32)
    value = rng.integers(0, 101, size=m).astype(np.int32)
    return branch, value


def variant_codes(tta_params, branch=None, value=None):
    """kernel codes of mcb_tta_variants_u8: geometry | branch << 4 | value << 8 (branch 0 = no colour)"""
    codes = np.array([spec_code(s) for s in tta_params], np.int32)
    if branch is not None:
        codes |= (np.asarray(branch, np.int32) << 4) | (np.asarray(value, np.int32) << 8)
    return codes


def tta_variant_batch(tiles, src, codes, resize=None, pad=(0, 0)):
    """the TTA loaders' device chain for one batch: tiles (N, H, W, 3) uint8 (numpy or cuda), src (NV,) tile of each
    row, codes (NV,) from variant_codes -> (NV, 3, H', W') float32 cuda.  Variant rows (geometry + colour, uint8) ->
    Pillow-exact bilinear resize to `resize` (loader_mode 'resize') -> pad (h_pad, w_pad) replicate -> ToTensor ->
    Normalize, the order of MetadataImageSegmentationTTA.__getitem__ (src/loaders.py:94-111)"""
    from .preparation import image_transform_batch, pil_resize_batch
    x = _to_dev(tiles, torch.uint8).contiguous()
    if x.dim() != 4 or x.shape[3] != 3:
        raise ValueError("expected tiles (N, H, W, 3) uint8, got %s" % (tuple(x.shape),))
    n, h, w, _ = x.shape
    codes = np.ascontiguousarray(codes, np.int32)
    src = np.ascontiguousarray(src, np.int32)
    if len(src) != len(codes) or (len(src) and (src.min() < 0 or src.max() >= n)):
        raise ValueError("tta_variant_batch: src must index the %d tiles, one per code" % n)
    if h != w and (codes & 1).any():
        raise NotImplementedError("quarter-turn TTA variants need square images")
    nv = len(codes)
    rows = torch.empty((nv, h, w, 3), dtype=torch.uint8, device=x.device)
    # pinned, asynchronous: a pageable copy would wait for the stream, i.e. for the network's previous batch
    src_d, codes_d = (torch.from_numpy(a).pin_memory().to(x.device, non_blocking=True) for a in (src, codes))
    L.fcall("mcb_tta_variants_u8", x.data_ptr(), rows.data_ptr(), src_d.data_ptr(), codes_d.data_ptr(), nv, h, w)
    if resize is not None:
        rows = pil_resize_batch(rows, resize)
    return image_transform_batch(rows, pad)


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
    if any(applies_colour(s) for s in tta_params):
        raise NotImplementedError("colour-shift variants cannot be built from normalised images: use "
                                  "ImageSegmentationLoaderInferencePaddingTTA / ImageSegmentationLoaderResizeTTA")
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


# ---------------------------------------------------------------------------------------------------------------------
# training loaders (src/loaders.py:114-305) with the augmentation on the device
# ---------------------------------------------------------------------------------------------------------------------
def load_mask(filepath):
    """the mask of src/loaders.py:145-146 (Image.open(...).convert('RGB')) as its single band: the masks are 0/1
    grayscale PNGs, so the RGB image has three equal bands and to_monochrome gives any one of them back"""
    from PIL import Image
    im = Image.open(filepath, 'r')
    if im.mode == 'L':
        return np.array(im)
    rgb = np.array(im.convert('RGB'))
    if not ((rgb[..., 0] == rgb[..., 1]).all() and (rgb[..., 0] == rgb[..., 2]).all()):
        raise ValueError("%s: mask bands differ; the device path carries one mask plane" % filepath)
    return np.ascontiguousarray(rgb[..., 0])


class SegmentationFiles(torch.utils.data.Dataset):
    """what the DataLoader workers do per sample: decode the files and apply the reference's own numpy casts
    (src/loaders.py:140-154).  Returns (image uint8 (H, W, 3)[, mask uint8 (H, W)[, distances, sizes]]), the uint16
    distances / sizes as their int16 view (same bytes; collated and pinned like any int16 tensor)."""

    def __init__(self, X, y=None, distances=False):
        self.X, self.y, self.distances = X, y, distances

    def __len__(self):
        return len(self.X)

    def __getitem__(self, index):
        import os
        from PIL import Image
        Xi = np.array(Image.open(self.X[index], 'r').convert('RGB'))
        if self.y is None:
            return Xi
        mask_filepath = self.y[index]
        Mi = load_mask(mask_filepath)
        if not self.distances:
            return Xi, Mi
        import joblib
        distance_filepath = os.path.splitext(mask_filepath.replace("/masks/", "/distances/"))[0]
        size_filepath = distance_filepath.replace("/distances/", "/sizes/")
        Di = joblib.load(distance_filepath).astype(np.uint16)
        Si = np.sqrt(joblib.load(size_filepath).astype(np.uint16)).astype(np.uint16)
        return Xi, Mi, Di.view(np.int16), Si.view(np.int16)


class DeviceBatches:
    """iterable over a DataLoader of host batches: draws each batch's augmentation parameters, runs the device chain
    (csrc/augment.cu -> [Pillow resize] -> normalise / pad + target) and yields [X, target] cuda float32 tensors
    (X alone without targets).  `last_params` holds the draw of the batch last yielded."""

    def __init__(self, loader, seq, rng, resize=None, pad=(0, 0)):
        self.loader, self.seq, self.rng, self.resize, self.pad = loader, seq, rng, resize, pad
        self.last_params = None

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        from .augmentation import batch_chain, identity_params
        from .preparation import image_transform_batch, pil_resize_batch
        for batch in self.loader:
            if isinstance(batch, torch.Tensor):                     # images only (inference)
                x = batch.to(_dev(), non_blocking=batch.is_pinned())
                if self.resize is not None:
                    x = pil_resize_batch(x, self.resize)
                yield image_transform_batch(x, self.pad)
                continue
            images, masks = batch[0], batch[1]
            distances, sizes = (batch[2], batch[3]) if len(batch) == 4 else (None, None)
            n, h, w = images.shape[:3]
            params = self.seq.draw(self.rng, n, h, w) if self.seq is not None else identity_params(n)
            self.last_params = params
            yield list(batch_chain(images, masks, distances, sizes, params,
                                   crop_size=None if self.seq is None else self.seq.crop_size, resize=self.resize,
                                   pad=self.pad))


class _AugmentedLoader:
    """ImageSegmentationLoaderBasic (src/loaders.py:176-222): transform(X, y, X_valid, y_valid, train_mode) ->
    {'datagen': (flow, steps), 'validation_datagen': (flow, steps)}.  `seed` (optional) makes the augmentation draws
    and the DataLoader's shuffling reproducible; under torch.distributed it is offset by the rank."""
    distances = False
    crop = False

    def __init__(self, loader_params, dataset_params, seed=None):
        self.loader_params = loader_params
        self.dataset_params = dataset_params
        self.seed = seed

    def fit(self, *args, **kwargs):
        return self

    def fit_transform(self, *args, **kwargs):
        return self.transform(*args, **kwargs)

    def load(self, filepath):
        return self

    def save(self, filepath):
        import joblib
        joblib.dump({}, filepath)

    def transform(self, X, y=None, X_valid=None, y_valid=None, train_mode=True):
        if train_mode and y is not None:
            flow, steps = self.get_datagen(X, y, True, self.loader_params['training'])
        else:
            flow, steps = self.get_datagen(X, None, False, self.loader_params['inference'])
        if X_valid is not None and y_valid is not None:
            valid_flow, valid_steps = self.get_datagen(X_valid, y_valid, False, self.loader_params['inference'])
        else:
            valid_flow, valid_steps = None, None
        return {'datagen': (flow, steps), 'validation_datagen': (valid_flow, valid_steps)}

    def _seed(self):
        if self.seed is None:
            return None
        import torch.distributed as dist
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        return int(self.seed) + rank

    def get_datagen(self, X, y, train_mode, loader_params):
        from .augmentation import crop_seq, fast_seq
        seed = self._seed()
        kwargs = dict(loader_params)
        if seed is not None and kwargs.get('shuffle'):
            kwargs['generator'] = torch.Generator().manual_seed(seed)
        loader = torch.utils.data.DataLoader(SegmentationFiles(X, y, self.distances), **kwargs)
        dp = self.dataset_params
        h, w = int(dp['h']), int(dp['w'])
        if self.crop:
            seq = crop_seq((h, w)) if train_mode else None
            flow = DeviceBatches(loader, seq, np.random.default_rng(seed), None,
                                 (0, 0) if train_mode else (int(dp['h_pad']), int(dp['w_pad'])))
        else:
            flow = DeviceBatches(loader, fast_seq if train_mode else None, np.random.default_rng(seed), (h, w))
        return flow, len(loader)


class MetadataImageSegmentationLoaderDistancesCropPad(_AugmentedLoader):
    """src/loaders.py:225-243"""
    distances, crop = True, True


class MetadataImageSegmentationLoaderDistancesResize(_AugmentedLoader):
    """src/loaders.py:246-263"""
    distances, crop = True, False


class MetadataImageSegmentationLoaderCropPad(_AugmentedLoader):
    """src/loaders.py:266-284"""
    distances, crop = False, True


class MetadataImageSegmentationLoaderResize(_AugmentedLoader):
    """src/loaders.py:287-304"""
    distances, crop = False, False


# ---------------------------------------------------------------------------------------------------------------------
# inference loaders (src/loaders.py:307-398) with the variants built on the device
# ---------------------------------------------------------------------------------------------------------------------
def _paths(X):
    """the loader's X (src/utils.py:227-228 squeezes the metadata column to a 1-D array of paths; a DataFrame or a list
    of one-element rows is accepted too) -> list of path strings"""
    rows = X.values if hasattr(X, "values") else X
    return [str(np.asarray(r, dtype=object).reshape(-1)[0]) for r in rows]


class TTABatches:
    """iterable over the batches of MetadataImageSegmentationTTA's DataLoader (shuffle off): the same batch boundaries
    and len(), each batch a float32 cuda (B, 3, H', W') tensor of the variant rows in X order.  Consecutive rows with
    the same path share one decode: the DataLoader runs over the distinct runs of paths, so each file is decoded once
    per pass however many variants it has, and a tile whose variants straddle two batches is kept for the second.
    `last_draws` holds the colour draws of the batch last yielded: {'branch', 'value'} int32 arrays of the batch's
    length (branch 0 where the row applies no colour)."""

    def __init__(self, paths, tta_params, loader_params, rng, resize=None, pad=(0, 0)):
        self.tta_params = list(tta_params) if tta_params is not None else [None] * len(paths)
        if len(self.tta_params) != len(paths):
            raise ValueError("%d tta_params for %d rows" % (len(self.tta_params), len(paths)))
        if loader_params.get('shuffle'):
            raise NotImplementedError("the inference loaders keep X order (shuffle: False, src/pipeline_config.py)")
        self.batch_size = int(loader_params.get('batch_size', 1))
        self.drop_last = bool(loader_params.get('drop_last', False))
        is_start = np.array([i == 0 or paths[i] != paths[i - 1] for i in range(len(paths))], bool)
        starts = np.nonzero(is_start)[0]
        self.run_of = np.cumsum(is_start) - 1
        kwargs = {k: v for k, v in loader_params.items() if k in ('num_workers', 'pin_memory', 'timeout',
                                                                  'worker_init_fn', 'prefetch_factor',
                                                                  'persistent_workers')}
        self.loader = torch.utils.data.DataLoader(SegmentationFiles([paths[b] for b in starts]), batch_size=None,
                                                  shuffle=False, **kwargs)
        self.codes = np.array([spec_code(p) if p is not None else 0 for p in self.tta_params], np.int32)
        self.colour = np.array([p is not None and applies_colour(p) for p in self.tta_params], bool)
        self.rng, self.resize, self.pad = rng, resize, pad
        self.last_draws = None

    def __len__(self):
        return len(self.batch_bounds())

    def batch_bounds(self):
        """[(first row, end row)] of every batch, as the reference's BatchSampler cuts them"""
        n, b = len(self.run_of), self.batch_size
        ends = range(b, n + 1, b) if self.drop_last else range(b, n + b, b)
        return [(e - b, min(e, n)) for e in ends]

    def __iter__(self):
        tiles = iter(self.loader)
        cache, next_run = {}, 0
        for b0, b1 in self.batch_bounds():
            runs = self.run_of[b0:b1]
            first, last = int(runs[0]), int(runs[-1])
            while next_run <= last:
                cache[next_run] = next(tiles)
                next_run += 1
            for r in [r for r in cache if r < first]:
                del cache[r]
            batch = torch.stack([torch.as_tensor(cache[r]) for r in range(first, last + 1)])
            colour = self.colour[b0:b1]
            branch, value = np.zeros(b1 - b0, np.int32), np.zeros(b1 - b0, np.int32)
            branch[colour], value[colour] = draw_colour(self.rng, int(colour.sum()))
            self.last_draws = {'branch': branch, 'value': value}
            codes = self.codes[b0:b1] | (branch << 4) | (value << 8)
            x = batch.pin_memory().to(_dev(), non_blocking=True)
            yield tta_variant_batch(x, runs - first, codes, self.resize, self.pad)


class _InferenceLoader:
    """ImageSegmentationLoaderBasic's inference form (src/loaders.py:307-398): transform(X[, tta_params]) ->
    {'datagen': (flow, steps), 'validation_datagen': (None, None)}; `flow` is a TTABatches over
    loader_params['inference'].  `seed` (optional) makes the colour draws reproducible; under torch.distributed it is
    offset by the rank."""
    resize = False

    def __init__(self, loader_params, dataset_params, seed=None):
        self.loader_params = loader_params
        self.dataset_params = dataset_params
        self.seed = seed

    fit = _AugmentedLoader.fit
    fit_transform = _AugmentedLoader.fit_transform
    load = _AugmentedLoader.load
    save = _AugmentedLoader.save
    _seed = _AugmentedLoader._seed

    def get_datagen(self, X, tta_params, loader_params):
        dp = self.dataset_params
        if self.resize:
            geometry = dict(resize=(int(dp['h']), int(dp['w'])))
        else:
            geometry = dict(pad=(int(dp['h_pad']), int(dp['w_pad'])))
        flow = TTABatches(_paths(X), tta_params, dict(loader_params), np.random.default_rng(self._seed()), **geometry)
        return flow, len(flow)


class ImageSegmentationLoaderInferencePadding(_InferenceLoader):
    """src/loaders.py:307-336: the `crop_and_pad` inference flow (pad (h_pad, w_pad) replicate, no variants)"""

    def transform(self, X, **kwargs):
        flow, steps = self.get_datagen(X, None, self.loader_params['inference'])
        return {'datagen': (flow, steps), 'validation_datagen': (None, None)}


class ImageSegmentationLoaderInferencePaddingTTA(_InferenceLoader):
    """src/loaders.py:339-368: the variant rows of X_tta, padded (h_pad, w_pad) replicate"""

    def transform(self, X, tta_params, **kwargs):
        flow, steps = self.get_datagen(X, tta_params, self.loader_params['inference'])
        return {'datagen': (flow, steps), 'validation_datagen': (None, None)}


class ImageSegmentationLoaderResizeTTA(_InferenceLoader):
    """src/loaders.py:371-398: the variant rows of X_tta, resized to (h, w) with Pillow's bilinear filter"""
    resize = True

    def transform(self, X, tta_params, **kwargs):
        flow, steps = self.get_datagen(X, tta_params, self.loader_params['inference'])
        return {'datagen': (flow, steps), 'validation_datagen': (None, None)}
