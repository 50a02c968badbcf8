"""Input side of the path on the GPU (SURVEY.md 8f-4): mirror of the deterministic parts of
src/loaders.py:141-171,311-317 (image / target tensors of the padded loaders),
src/augmentation.py:40-86 (PadFixed) and src/preparation.py:151-195 (two-nearest
building distances, component-size map).

Both loader modes are covered: `crop_and_pad` (PadFixed) and `resize` (transforms.Resize on the PIL image = Pillow's
8-bit bilinear resampler, restated bit-exactly).  Out of scope: JPEG / PNG decoding, COCO polygon rasterisation
(pycocotools), the random imgaug augmenters.  Everything here is batched device work in libmcb200.so (csrc/input.cu); no
CPU fallback."""
import numpy as np
import torch

from . import _lib as L
from .postprocessing import MEAN, STD, _dev, _to_dev, label_batch

PAD_MODES = {"replicate": 0, "reflect": 1}


def image_transform_batch(images, pad=(0, 0), pad_method="replicate", mean=MEAN, std=STD):
    """images (N, H, W, 3) uint8 (numpy or cuda tensor) -> (N, 3, H + 2 pad_h, W + 2 pad_w) float32 cuda:
    PadFixed(pad, pad_method) -> transforms.ToTensor() -> transforms.Normalize(mean, std), bit-exact"""
    x = _to_dev(images, torch.uint8)
    if x.dim() != 4 or x.shape[3] != 3:
        raise ValueError("expected images (N, H, W, 3) uint8, got %s" % (tuple(x.shape),))
    n, h, w, _ = x.shape
    ph, pw = int(pad[0]), int(pad[1])
    out = torch.empty((n, 3, h + 2 * ph, w + 2 * pw), dtype=torch.float32, device=x.device)
    m = (L.C.c_float * 3)(*[float(np.float32(v)) for v in mean])
    s = (L.C.c_float * 3)(*[float(np.float32(v)) for v in std])
    L.fcall("mcb_image_pad_normalize", x.data_ptr(), out.data_ptr(), n, h, w, ph, pw, PAD_MODES[pad_method], m, s)
    return out


_PIL_PRECISION = 32 - 8 - 2


def pil_bilinear_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the BILINEAR filter (support 1, widened by the scale
    factor when shrinking): -> (coef int32 (out, ksize), bounds int32 (out, 2) = (first source index, taps))"""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    coef = np.zeros((out_size, ksize), np.int32)
    bounds = np.zeros((out_size, 2), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = np.zeros(ksize)
        for x in range(xmax):
            a = abs((x + xmin - center + 0.5) * ss)
            w[x] = 1.0 - a if a < 1.0 else 0.0
        ww = w[:xmax].sum()
        if ww != 0.0:
            w[:xmax] /= ww
        k = w * (1 << _PIL_PRECISION)
        coef[xx] = np.where(w < 0, k - 0.5, k + 0.5).astype(np.int64).astype(np.int32)   # C double -> int: truncation
        bounds[xx] = (xmin, xmax)
    return coef, bounds


_PIL_TABLES = {}


def pil_resize_batch(images, size):
    """transforms.Resize(size) on PIL images (src/loaders.py:287-305): images (N, H, W, C) uint8 -> (N, h, w, C) uint8 cuda,
    bit-identical to Image.resize((w, h), BILINEAR)"""
    x = _to_dev(images, torch.uint8)
    n, h, w, c = x.shape
    oh, ow = int(size[0]), int(size[1])
    key = (x.device, h, w, oh, ow)
    if key not in _PIL_TABLES:
        ch, bh = pil_bilinear_coeffs(w, ow)
        cv, bv = pil_bilinear_coeffs(h, oh)
        _PIL_TABLES[key] = tuple(torch.from_numpy(a).to(x.device) for a in (ch, bh, cv, bv)) + (ch.shape[1], cv.shape[1])
    ch, bh, cv, bv, kh, kv = _PIL_TABLES[key]
    tmp = torch.empty((n, h, ow, c), dtype=torch.uint8, device=x.device)
    out = torch.empty((n, oh, ow, c), dtype=torch.uint8, device=x.device)
    L.fcall("mcb_pil_resize_bilinear_u8", x.data_ptr(), tmp.data_ptr(), out.data_ptr(), ch.data_ptr(), bh.data_ptr(), kh,
            cv.data_ptr(), bv.data_ptr(), kv, n, h, w, c, oh, ow)
    return out


def image_transform_resize_batch(images, size, mean=MEAN, std=STD):
    """the `resize` loader mode's image_transform (src/loaders.py:291-295): Resize -> ToTensor -> Normalize"""
    return image_transform_batch(pil_resize_batch(images, size), (0, 0), "replicate", mean, std)


def two_nearest_distances(instance_masks):
    """update_distances + clean_distances (src/preparation.py:151-168) for ONE image: instance_masks (K, H, W) uint8|bool
    (one non-empty plane per building) -> (distances float16 (H, W) numpy, second_nearest float64 (H, W) numpy)"""
    m = np.asarray(instance_masks)
    if m.ndim != 3:
        raise ValueError("expected (K, H, W) instance masks")
    k, h, w = m.shape
    dev = _dev()
    md = _to_dev((m != 0).astype(np.uint8), torch.uint8) if k else None
    ws = torch.empty(max(k, 1) * h * w, dtype=torch.int32, device=dev)
    dsum = torch.empty((h, w), dtype=torch.float16, device=dev)
    second = torch.empty((h, w), dtype=torch.float64, device=dev)
    L.fcall("mcb_edt_two_nearest", None if md is None else md.data_ptr(), k, h, w, ws.data_ptr(), dsum.data_ptr(),
            second.data_ptr())
    return dsum.cpu().numpy(), second.cpu().numpy()


def get_size_matrix(mask):
    """src/preparation.py:189-195: pixel count of each pixel's 4-connected component of `mask`, 1 on background"""
    m = np.asarray(mask)
    md = _to_dev((m != 0).astype(np.uint8), torch.uint8)[None].contiguous()
    labels, counts = label_batch(md, return_counts=True)
    k = int(counts.item())
    if k == 0:
        return np.ones_like(m)           # the reference returns the untouched np.ones_like(mask) in that case
    area = torch.bincount(labels.reshape(-1), minlength=k + 1)[1:].to(torch.int32).contiguous()
    out = torch.empty(m.shape, dtype=torch.int64, device=md.device)
    L.fcall("mcb_size_matrix", labels.data_ptr(), area.data_ptr(), out.data_ptr(), m.shape[0], m.shape[1])
    return out.cpu().numpy()


def target_batch(masks, distances, sizes, pad=(0, 0), pad_method="replicate"):
    """the (N, 3, H', W') float32 target of MetadataImageSegmentationDatasetDistances (src/loaders.py:141-171) from the
    prepared per-image arrays: masks (N, H, W) uint8 {0,1}, distances (N, H, W) float16, sizes (N, H, W) int64"""
    md = _to_dev(np.asarray(masks).astype(np.uint8), torch.uint8)
    dd = _to_dev(np.asarray(distances).astype(np.float16), torch.float16)
    sd = _to_dev(np.asarray(sizes).astype(np.int64), torch.int64)
    n, h, w = md.shape
    ph, pw = int(pad[0]), int(pad[1])
    out = torch.empty((n, 3, h + 2 * ph, w + 2 * pw), dtype=torch.float32, device=md.device)
    L.fcall("mcb_target_channels", md.data_ptr(), dd.data_ptr(), sd.data_ptr(), out.data_ptr(), n, h, w, ph, pw,
            PAD_MODES[pad_method])
    return out
