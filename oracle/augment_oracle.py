"""TEST INFRASTRUCTURE — CPU restatement of the training loaders' augmentation (src/augmentation.py:5-10, 34-37,
91-135 through ImgAug, src/steps/pytorch/utils.py:108-129) and of the rest of the per-sample chain (to_pil, Pillow
resize, to_monochrome, ToTensor, Normalize; src/loaders.py:140-171, 225-305).  Only tests/ import it.

imgaug 0.2.5 and scikit-image are not installable here, so what they compute is restated from their sources.  These are
ASSUMPTIONS, each pinned by a test of its visible consequence in tests/test_augmentation_cpu.py:

 1. Matrix.  imgaug 0.2.5 Affine._augment_images builds, per image of H x W,
      shift = (W / 2 - 0.5, H / 2 - 0.5);  translate_px = (int(round(t * W)), int(round(t * H))) with ONE fraction t
      for both axes (translate_percent is a tuple, not a dict);  rotation = math.radians(angle);
      matrix = SimilarityTransform(translation=-shift) + AffineTransform(scale=(1, 1), rotation, shear=0,
               translation=translate_px) + SimilarityTransform(translation=shift)
    where skimage's ProjectiveTransform.__add__ composes as other.params.dot(self.params) into a ProjectiveTransform,
    and skips the warp entirely when translate_px == (0, 0) and angle == 0.  It then calls
      warp(image, matrix.inverse, order=1, mode='constant', cval=0, preserve_range=True)
    and skimage resolves `matrix.inverse` (a bound method of a homography) to np.linalg.inv(matrix.params), applied to
    every channel of the image.
 2. Sampling.  skimage's _warp_fast in fp64: the affine path when the inverse's last row is exactly (0, 0, 1), else
    the projective one (divide by M20 x + M21 y + M22); c = M00 x + M01 y + M02, r = M10 x + M11 y + M12 for output
    column x, row y; bilinear_interpolation with floor / ceil neighbours, cval for neighbours outside the image,
    top = (1 - dc) tl + dc tr, bottom = (1 - dc) bl + dc br, (1 - dr) top + dr bottom, each operation rounded (the
    compiled C has no FMA).  _clip_warp_output then clips to the input's [min, max] (over all channels), keeping
    pixels that are exactly cval when cval lies outside that range; imgaug casts back with a truncating astype.
 3. Flips are exactly np.fliplr / np.flipud.

A draw is a record with fields n_children, children (application order; 0 Fliplr, 1 Flipud, 2 Affine), coin (the flip
children's outcome), rotate (degrees), translate (fraction), top, left (RandomCropFixedSize offset).
"""
import math

import numpy as np

from . import input_oracle as IO

FLIPLR, FLIPUD, AFFINE = 0, 1, 2


# ------------------------------------------------------------------------------------------------ skimage.transform
def _similarity(translation):
    """SimilarityTransform(translation=...).params"""
    scale, rotation = 1, 0
    p = np.array([[math.cos(rotation), - math.sin(rotation), 0],
                  [math.sin(rotation), math.cos(rotation), 0],
                  [0, 0, 1]])
    p[0:2, 0:2] *= scale
    p[0:2, 2] = translation
    return p


def _affine(scale, rotation, shear, translation):
    """AffineTransform(scale=, rotation=, shear=, translation=).params"""
    sx, sy = scale
    p = np.array([[sx * math.cos(rotation), - sy * math.sin(rotation + shear), 0],
                  [sx * math.sin(rotation), sy * math.cos(rotation + shear), 0],
                  [0, 0, 1]])
    p[0:2, 2] = translation
    return p


def _add(self_params, other_params):
    """ProjectiveTransform.__add__: applies self, then other"""
    return other_params.dot(self_params)


def affine_matrix(angle, t, height, width):
    """imgaug 0.2.5 Affine: the forward matrix params, or None where it skips the warp"""
    shift_x, shift_y = width / 2.0 - 0.5, height / 2.0 - 0.5
    tx, ty = int(round(t * width)), int(round(t * height))
    if tx == 0 and ty == 0 and angle == 0:
        return None
    m = _add(_similarity([-shift_x, -shift_y]), _affine((1.0, 1.0), math.radians(angle), math.radians(0), (tx, ty)))
    return _add(m, _similarity([shift_x, shift_y]))


def _warp_plane(img, inv):
    """_warp_fast of one float64 plane, order 1, mode 'constant', cval 0"""
    rows, cols = img.shape
    ys, xs = np.mgrid[0:rows, 0:cols].astype(np.float64)
    M = inv.reshape(-1)
    if M[6] == 0 and M[7] == 0 and M[8] == 1:
        c = M[0] * xs + M[1] * ys + M[2]
        r = M[3] * xs + M[4] * ys + M[5]
    else:
        z = M[6] * xs + M[7] * ys + M[8]
        c = (M[0] * xs + M[1] * ys + M[2]) / z
        r = (M[3] * xs + M[4] * ys + M[5]) / z
    minr, minc = np.floor(r).astype(np.int64), np.floor(c).astype(np.int64)
    maxr, maxc = np.ceil(r).astype(np.int64), np.ceil(c).astype(np.int64)
    dr, dc = r - minr, c - minc

    def pixel(rr, cc):
        ok = (rr >= 0) & (rr < rows) & (cc >= 0) & (cc < cols)
        out = np.zeros(rr.shape)
        out[ok] = img[rr[ok], cc[ok]]
        return out

    top = (1 - dc) * pixel(minr, minc) + dc * pixel(minr, maxc)
    bottom = (1 - dc) * pixel(maxr, minc) + dc * pixel(maxr, maxc)
    return (1 - dr) * top + dr * bottom


def warp(image, matrix):
    """warp(image, matrix.inverse, order=1, mode='constant', cval=0, preserve_range=True) + imgaug's astype"""
    inv = np.linalg.inv(matrix)
    img = image.astype(np.double)
    if img.ndim == 2:
        out = _warp_plane(img, inv)
    else:
        out = np.dstack([_warp_plane(img[..., k], inv) for k in range(img.shape[2])])
    lo, hi, cval = img.min(), img.max(), 0.0
    preserve_cval = not (lo <= cval <= hi)
    if preserve_cval:
        at_cval = out == cval
    np.clip(out, lo, hi, out=out)
    if preserve_cval:
        out[at_cval] = cval
    return out.astype(image.dtype) if image.dtype != np.float64 else out


# ------------------------------------------------------------------------------------------------ the augmenters
def augment(image, p, crop_size=None):
    """one array through fast_seq (the draw p) and, with crop_size, RandomCropFixedSize"""
    a = image
    h, w = image.shape[:2]
    for k in range(int(p['n_children'])):
        child = int(p['children'][k])
        if child == AFFINE:
            m = affine_matrix(float(p['rotate']), float(p['translate']), h, w)
            if m is not None:
                a = warp(a, m)
        elif p['coin'][k]:
            a = np.fliplr(a) if child == FLIPLR else np.flipud(a)
    if crop_size is not None:
        top, left = int(p['top']), int(p['left'])
        a = a[top:top + crop_size[0], left:left + crop_size[1]]
    return a


def to_pil(a):
    """src/utils.py:284-289"""
    from PIL import Image
    return Image.fromarray(a.astype(np.uint8))


def loader_sample(image, mask_rgb, distances=None, sizes=None, p=None, mode="resize", size=(256, 256), train=True,
                  pad=(10, 10)):
    """one (X, target) pair of the reference's Dataset __getitem__ (src/loaders.py:47-67, 140-169): image uint8
    (H, W, 3), mask_rgb uint8 (H, W, 3) (the RGB image of the mask PNG), distances / sizes uint16 (H, W) after the
    Dataset's casts, or None for the plain-mask loaders.  mode 'resize' | 'crop'; train applies the draw p, otherwise
    the inference augmenter (padding_seq in crop mode, nothing in resize mode).
    -> (X float32 (3, h', w'), target float32 (C, h', w'))"""
    import torchvision.transforms as T
    from PIL import Image
    arrays = [image, mask_rgb] + ([distances, sizes] if distances is not None else [])
    if train:
        arrays = [augment(a, p, size if mode == "crop" else None) for a in arrays]
    elif mode == "crop":
        arrays = [IO.pad_image(a, pad, "replicate") for a in arrays]
    pils = [to_pil(a) for a in arrays]
    if mode == "resize":
        pils = [im.resize((int(size[1]), int(size[0])), Image.BILINEAR) for im in pils]
    x = T.Normalize(mean=IO.MEAN, std=IO.STD)(T.ToTensor()(pils[0])).numpy()
    target = np.stack([np.array(im.convert('L')).astype(np.float32) for im in pils[1:]])
    return x, target


def augmented_planes(image, mask_rgb, distances=None, sizes=None, p=None, crop_size=None):
    """the uint8 arrays right after to_pil (before any resize): image (h, w, 3), then the mask as convert('L') and the
    wrapped distances / sizes stacked as (h, w, C)"""
    arrays = [image, mask_rgb] + ([distances, sizes] if distances is not None else [])
    arrays = [augment(a, p, crop_size).astype(np.uint8) for a in arrays]
    from PIL import Image
    m = np.array(Image.fromarray(arrays[1]).convert('L'))
    return arrays[0], np.stack([m] + arrays[2:], axis=-1)
