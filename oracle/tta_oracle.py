"""TEST INFRASTRUCTURE — CPU restatement of the inference loaders' variant rows (src/loaders.py:74-111,307-398,
477-487) with the colour-shift branch of test_time_augmentation_transform (color_seq, src/augmentation.py:12-31).
Only tests/ and scripts/ import this file.

Assumptions, imgaug 0.2.5 being not installable here (stated from its published source):
* `OneOf(children)` applies exactly one child, chosen uniformly; `Sequential([...], random_order=True)` around a single
  child is that child.
* `Add((0, 100))` draws one integer value per image from DiscreteUniform(0, 100) (per_channel=False) and computes
  `clip(image.astype(int32) + value, 0, 255).astype(uint8)`; `WithChannels(c, Add)` applies it to channel c only.  So
  H is clipped at 255, not at 180, and cv2's HSV2RGB then wraps it modulo 180.
* `ChangeColorspace(from_colorspace=RGB, to_colorspace=HSV)` and back is `cv2.cvtColor` with COLOR_RGB2HSV /
  COLOR_HSV2RGB on the uint8 image (alpha 1: the blend returns the converted image unchanged).
* `skimage.transform.rotate` at quarter turns: oracle/instances_oracle.py's assumption (exact np.rot90).

cv2 itself is called for the colour conversions.  Its HSV2RGB on uint8 runs a SIMD body over whole vectors of a row and
a scalar tail over the remaining columns; the two round differently (DESIGN.md §4.5).  `tail=False` runs the same cv2
call on the rows widened to a multiple of 64 columns, so every pixel takes the vector body: the map the device kernel
reproduces."""
import numpy as np

from . import input_oracle as IN
from . import instances_oracle as I

VECTOR_COLUMNS = 64   # a multiple of every vector width cv2 dispatches on x86 (4 x 8 or 4 x 16 float lanes)


def rgb2hsv(rgb):
    """cv2's RGB2HSV_b restated in integer numpy: uint8 (..., 3) -> uint8 (..., 3), H in 0..179"""
    x = np.asarray(rgb).astype(np.int64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    v = x.max(-1)
    diff = v - x.min(-1)
    i = np.arange(1, 256)
    sdiv = np.concatenate([[0], np.rint((255 << 12) / i.astype(np.float64))]).astype(np.int64)
    hdiv = np.concatenate([[0], np.rint((180 << 12) / (6.0 * i))]).astype(np.int64)
    s = (diff * sdiv[v] + 2048) >> 12
    num = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (num * hdiv[diff] + 2048) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def hsv2rgb_cv2(hsv, tail=True):
    """cv2.cvtColor(hsv, COLOR_HSV2RGB); tail=False: every pixel through cv2's vector body"""
    import cv2
    hsv = np.ascontiguousarray(hsv)
    if tail:
        return cv2.cvtColor(hsv, cv2.COLOR_HSV2RGB)
    h, w = hsv.shape[:2]
    wide = np.zeros((h, -(-w // VECTOR_COLUMNS) * VECTOR_COLUMNS, 3), np.uint8)
    wide[:, :w] = hsv
    return np.ascontiguousarray(cv2.cvtColor(wide, cv2.COLOR_HSV2RGB)[:, :w])


def add_clip(channel, value):
    """imgaug 0.2.5 Add on a uint8 channel"""
    return np.clip(channel.astype(np.int32) + int(value), 0, 255).astype(np.uint8)


def color_shift(img, branch, value, tail=True):
    """color_seq with OneOf child `branch` (1-3: HSV channel 0-2 through cv2; 4-6: RGB channel 0-2) and Add `value`,
    on an (H, W, 3) uint8 RGB image"""
    import cv2
    img = np.ascontiguousarray(img, np.uint8)
    if not 1 <= branch <= 6:
        raise ValueError("branch %r" % (branch,))
    if branch >= 4:
        out = img.copy()
        out[..., branch - 4] = add_clip(out[..., branch - 4], value)
        return out
    hsv = cv2.cvtColor(img, cv2.COLOR_RGB2HSV)
    hsv[..., branch - 1] = add_clip(hsv[..., branch - 1], value)
    return hsv2rgb_cv2(hsv, tail)


def applies_colour(spec):
    """`if ud ... elif lr ... elif color_shift` (src/loaders.py:478-484)"""
    return bool(spec['color_shift']) and not spec['ud_flip'] and not spec['lr_flip']


def tta_transform(image, spec, draw=None, tail=True):
    """test_time_augmentation_transform (src/loaders.py:477-487) on an (H, W, 3) uint8 image -> float64 (H, W, 3);
    draw = (branch, value) for a spec that applies colour"""
    if spec['ud_flip']:
        image = np.flipud(image)
    elif spec['lr_flip']:
        image = np.fliplr(image)
    elif spec['color_shift']:
        image = color_shift(image, draw[0], draw[1], tail)
    return I.skimage_rotate(image, spec['rotation'], preserve_range=True)


def tta_loader_row(img, spec, draw=None, mode="crop_and_pad", pad=(0, 0), size=None, tail=True):
    """MetadataImageSegmentationTTA.__getitem__ (src/loaders.py:94-111) with the inference loaders' transforms:
    variant (float64) -> to_pil (astype uint8) -> 'crop_and_pad': PadFixed(pad, replicate) + ToTensor + Normalize
    (src/loaders.py:339-350) | 'resize': Resize(size) + ToTensor + Normalize (src/loaders.py:371-380).
    spec None = no variant (ImageSegmentationLoaderInferencePadding) -> (3, H', W') float32"""
    x = img if spec is None else tta_transform(img, spec, draw, tail)
    x = np.asarray(x).astype(np.uint8)
    if mode == "crop_and_pad":
        return IN.image_transform(x, pad)
    if mode == "resize":
        return IN.image_transform_resize(x, size)
    raise ValueError(mode)
