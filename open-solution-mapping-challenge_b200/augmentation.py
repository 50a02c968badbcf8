"""The training loaders' random augmentation on the device: mirror of src/augmentation.py:5-10 (fast_seq), :34-37
(crop_seq) and :91-135 (RandomCropFixedSize) as the loaders apply them (src/loaders.py:140-159, ImgAug of
src/steps/pytorch/utils.py:108-129: one deterministic draw per sample, applied to the image, the mask and, in the
distance loaders, the distances and sizes).

The draws happen here, on the host, from a seeded `numpy.random.Generator`; the pixels move in one batched launch of
csrc/augment.cu.  The draws follow the reference's distributions:

    fast_seq = SomeOf((1, 2), [Fliplr(0.5), Flipud(0.5), Affine(rotate=(-10, 10), translate_percent=(-0.1, 0.1))],
                      random_order=True)
      1 or 2 children with probability 1/2 each, every ordered choice of them equally likely; a chosen flip flips with
      probability 1/2; rotation ~ U(-10, 10) degrees; ONE translation fraction t ~ U(-0.1, 0.1) for both axes
      (a tuple translate_percent), int(round(t * W)) / int(round(t * H)) pixels.
    crop_seq(crop_size) = fast_seq, then RandomCropFixedSize: top ~ randint(H - h), left ~ randint(W - w)
      (the last offset is never drawn, H == h raises like numpy's randint(0)).

They are distribution-equal, not draw-equal, to imgaug's random stream: reproducing imgaug's stream needs imgaug, and
nothing here depends on it.  The Affine matrix is built in numpy exactly like imgaug 0.2.5 builds it over
skimage.transform (oracle/augment_oracle.py states the assumptions and tests/test_augmentation_cpu.py pins them).
"""
import math

import numpy as np
import torch

from . import _lib as L
from .postprocessing import MEAN, STD, _dev
from .preparation import PAD_MODES, image_transform_batch, pil_resize_batch

FLIPLR, FLIPUD, AFFINE = 0, 1, 2

# one sample's draw: children in application order (-1 = unused slot), the flip coins of those children, the Affine
# child's rotation (degrees) and translation fraction, the crop offset
PARAMS = np.dtype([('n_children', '<i4'), ('children', '<i4', (2,)), ('coin', '?', (2,)), ('rotate', '<f8'),
                   ('translate', '<f8'), ('top', '<i4'), ('left', '<i4')])
# mcb_augment_row (include/mcb200.h)
ROW = np.dtype([('inv', '<f8', (9,)), ('warp', '<i4'), ('pre_flip', '<i4'), ('post_flip', '<i4'), ('top', '<i4'),
                ('left', '<i4'), ('reserved', '<i4')])
assert ROW.itemsize == 96


class FastSeq:
    """src/augmentation.py:5-10 as a sampler: draw(rng, n, height, width) -> PARAMS[n]"""
    crop_size = None

    def draw(self, rng, n, height, width):
        p = np.zeros(n, PARAMS)
        p['n_children'] = rng.integers(1, 3, n)
        order = rng.permuted(np.tile(np.arange(3, dtype=np.int32), (n, 1)), axis=1)[:, :2]
        p['children'] = np.where(np.arange(2)[None, :] < p['n_children'][:, None], order, -1)
        p['coin'] = rng.random((n, 2)) < 0.5
        p['rotate'] = rng.uniform(-10.0, 10.0, n)
        p['translate'] = rng.uniform(-0.1, 0.1, n)
        return p


class CropSeq(FastSeq):
    """src/augmentation.py:34-37: fast_seq then RandomCropFixedSize(px=crop_size)"""

    def __init__(self, crop_size):
        self.crop_size = (int(crop_size[0]), int(crop_size[1])) if isinstance(crop_size, tuple) else \
            (int(crop_size), int(crop_size))

    def draw(self, rng, n, height, width):
        ch, cw = self.crop_size
        if height - ch <= 0 or width - cw <= 0:
            raise ValueError("RandomCropFixedSize draws randint(H - h): a %dx%d crop of a %dx%d image has no offset "
                             "to draw" % (ch, cw, height, width))
        p = super().draw(rng, n, height, width)
        p['top'] = rng.integers(0, height - ch, n)
        p['left'] = rng.integers(0, width - cw, n)
        return p


fast_seq = FastSeq()


def crop_seq(crop_size):
    return CropSeq(crop_size)


def identity_params(n):
    """no child drawn, no crop: what the inference-mode datasets apply (nothing)"""
    p = np.zeros(n, PARAMS)
    p['children'] = -1
    return p


def affine_matrix(rotate, translate, height, width):
    """imgaug 0.2.5 Affine._augment_images: SimilarityTransform(-shift) + AffineTransform(scale 1, rotation, shear 0,
    translation) + SimilarityTransform(shift), composed as skimage's __add__ does (other.params.dot(self.params)).
    Returns None where imgaug skips the warp (no translation pixels and no rotation)."""
    shift_x, shift_y = width / 2.0 - 0.5, height / 2.0 - 0.5
    tx, ty = int(round(translate * width)), int(round(translate * height))
    if tx == 0 and ty == 0 and rotate == 0:
        return None

    def similarity(t):
        m = np.array([[math.cos(0), -math.sin(0), 0], [math.sin(0), math.cos(0), 0], [0, 0, 1]], np.float64)
        m[0:2, 0:2] *= 1
        m[0:2, 2] = t
        return m

    rot, shear = math.radians(rotate), math.radians(0)
    aff = np.array([[1.0 * math.cos(rot), -1.0 * math.sin(rot + shear), 0],
                    [1.0 * math.sin(rot), 1.0 * math.cos(rot + shear), 0],
                    [0, 0, 1]], np.float64)
    aff[0:2, 2] = (tx, ty)
    return similarity([shift_x, shift_y]).dot(aff.dot(similarity([-shift_x, -shift_y])))


def rows(params, height, width):
    """PARAMS[n] -> ROW[n] (mcb_augment_row): the flips before / after the Affine child, skimage's output -> input map
    (np.linalg.inv of the Affine matrix, like warp(img, matrix.inverse)), the crop offset"""
    out = np.zeros(len(params), ROW)
    for i, p in enumerate(params):
        warped = False
        for k in range(int(p['n_children'])):
            child = int(p['children'][k])
            if child == AFFINE:
                m = affine_matrix(float(p['rotate']), float(p['translate']), height, width)
                if m is not None:
                    out[i]['inv'] = np.linalg.inv(m).reshape(-1)
                    out[i]['warp'] = 1
                    warped = True
            elif p['coin'][k]:
                bit = 1 if child == FLIPLR else 2
                if warped:
                    out[i]['post_flip'] ^= bit
                else:
                    out[i]['pre_flip'] ^= bit
        if not warped:                       # flips only: all of them act on the output index
            out[i]['post_flip'] ^= out[i]['pre_flip']
            out[i]['pre_flip'] = 0
        out[i]['top'], out[i]['left'] = int(p['top']), int(p['left'])
    return out


def _u8(a):
    if isinstance(a, torch.Tensor):
        return a.to(device=_dev(), dtype=torch.uint8, non_blocking=a.is_pinned()).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a, np.uint8)).to(_dev())


def _u16(a):
    """uint16 planes travel as int16 tensors with the same bytes (torch's uint16 support is partial)"""
    if isinstance(a, torch.Tensor):
        if a.dtype not in (torch.int16, torch.uint16):
            raise ValueError("distances / sizes must be uint16 (or their int16 view), got %s" % a.dtype)
        return a.view(torch.int16).to(device=_dev(), non_blocking=a.is_pinned()).contiguous()
    a = np.asarray(a)
    if a.dtype != np.uint16:
        raise ValueError("distances / sizes must be uint16 (the reference's astype(np.uint16)), got %s" % a.dtype)
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).to(_dev())


def augment_batch(images, masks, distances=None, sizes=None, params=None, crop_size=None):
    """fast_seq / crop_seq + to_pil on a batch: images (N, H, W, 3) uint8, masks (N, H, W) uint8 (one band of the
    reference's equal-banded RGB mask), distances / sizes (N, H, W) uint16 or None, params PARAMS[N] (a sampler's
    draw) -> (image uint8 (N, h, w, 3) cuda, targets uint8 (N, h, w, C) cuda) with C = 3 (mask, distances, sizes) or
    1 (mask); (h, w) = crop_size, or (H, W) without a crop.  Inputs may be numpy arrays or (pinned) tensors."""
    x, m = _u8(images), _u8(masks)
    if x.dim() != 4 or x.shape[3] != 3 or tuple(m.shape) != tuple(x.shape[:3]):
        raise ValueError("expected images (N, H, W, 3) and masks (N, H, W), got %s and %s"
                         % (tuple(x.shape), tuple(m.shape)))
    if (distances is None) != (sizes is None):
        raise ValueError("distances and sizes come together")
    n, h, w, _ = x.shape
    d = s = None
    if distances is not None:
        d, s = _u16(distances), _u16(sizes)
        if tuple(d.shape) != (n, h, w) or tuple(s.shape) != (n, h, w):
            raise ValueError("distances / sizes must be (N, H, W) = %s" % ((n, h, w),))
    params = np.asarray(params, PARAMS)
    if params.shape != (n,):
        raise ValueError("one parameter row per sample: %d images, %s rows" % (n, params.shape))
    oh, ow = (h, w) if crop_size is None else (int(crop_size[0]), int(crop_size[1]))
    r = np.ascontiguousarray(rows(params, h, w))
    c = 1 if d is None else 3
    img_out = torch.empty((n, oh, ow, 3), dtype=torch.uint8, device=x.device)
    tgt_out = torch.empty((n, oh, ow, c), dtype=torch.uint8, device=x.device)
    ws = torch.empty((n, 8), dtype=torch.int32, device=x.device)
    L.fcall("mcb_augment_warp", x.data_ptr(), m.data_ptr(), None if d is None else d.data_ptr(),
            None if s is None else s.data_ptr(), r.ctypes.data, n, h, w, oh, ow, ws.data_ptr(), img_out.data_ptr(),
            tgt_out.data_ptr())
    return img_out, tgt_out


def target_u8_batch(planes, pad=(0, 0), pad_method="replicate"):
    """(N, h, w, C) uint8 cuda target planes -> (N, C, h + 2 pad_h, w + 2 pad_w) float32 cuda (to_monochrome,
    to_tensor, cat; padded like the image)"""
    n, h, w, c = planes.shape
    ph, pw = int(pad[0]), int(pad[1])
    out = torch.empty((n, c, h + 2 * ph, w + 2 * pw), dtype=torch.float32, device=planes.device)
    L.fcall("mcb_target_channels_u8", planes.data_ptr(), out.data_ptr(), n, h, w, c, ph, pw, PAD_MODES[pad_method])
    return out


def batch_chain(images, masks, distances=None, sizes=None, params=None, crop_size=None, resize=None, pad=(0, 0),
                pad_method="replicate", mean=MEAN, std=STD):
    """one loader batch on the device: augment_batch -> [Pillow bilinear resize of image and targets (resize mode)] ->
    [pad] + ToTensor + Normalize, target tensor -> (X (N, 3, h', w') float32, target (N, C, h', w') float32)"""
    img, tgt = augment_batch(images, masks, distances, sizes, params, crop_size)
    if resize is not None:
        img, tgt = pil_resize_batch(img, resize), pil_resize_batch(tgt, resize)
    return image_transform_batch(img, pad, pad_method, mean, std), target_u8_batch(tgt, pad, pad_method)
