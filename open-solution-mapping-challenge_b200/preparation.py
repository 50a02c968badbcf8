"""Input side of the path on the GPU (SURVEY.md 8f-4): mirror of the deterministic parts of
src/loaders.py:141-171,311-317 (image / target tensors of the padded loaders),
src/augmentation.py:40-86 (PadFixed) and src/preparation.py:18-198 (`overlay_masks`: COCO polygons -> the mask,
distance and size files the training loaders read).

Both loader modes are covered: `crop_and_pad` (PadFixed) and `resize` (transforms.Resize on the PIL image = Pillow's
8-bit bilinear resampler, restated bit-exactly).  Polygons are rasterised exactly as pycocotools' frPyObjects +
decode do (csrc/polygon.cu); the bbox and RLE segmentation forms are not.  Out of scope: JPEG / PNG decoding; the
random augmenters of the training loaders are mcb200.augmentation.  Everything here is batched device work in
libmcb200.so (csrc/input.cu, csrc/polygon.cu); no CPU fallback."""
import json
import os
from collections import deque
from concurrent.futures import ThreadPoolExecutor

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


# ---------------------------------------------------------------------------------------------------------------------
# COCO polygons -> training targets (src/preparation.py:18-198)
# ---------------------------------------------------------------------------------------------------------------------
_INT_MIN, _INT_MAX = -2 ** 31, 2 ** 31 - 1
_MAX_PLANES_Y = 65535   # mcb_ccl_label / mcb_add_dropped_objects launch one grid row per plane (gridDim.y)


def segmentation_polygons(segm):
    """the polygons of a COCO segmentation that frPyObjects would rasterise as polygons; the bbox and RLE forms raise
    NotImplementedError naming the form, and what frPyObjects rejects (a first polygon of fewer than 4 coordinates,
    no polygon at all) raises ValueError"""
    if isinstance(segm, dict):
        form = "RLE"
    elif isinstance(segm, (list, tuple)) and len(segm) and isinstance(segm[0], (list, tuple, np.ndarray)):
        if len(segm[0]) < 4:
            raise ValueError("segmentation input type is not supported: the first polygon has %d coordinates"
                             % len(segm[0]))
        form = "bbox" if len(segm[0]) == 4 else "polygons"
    elif isinstance(segm, (list, tuple)) and len(segm) and isinstance(segm[0], dict):
        form = "RLE"
    elif isinstance(segm, (list, tuple)) and len(segm) == 4:
        form = "bbox"
    elif isinstance(segm, (list, tuple)) and not len(segm):
        raise ValueError("segmentation input type is not supported: no polygon")
    else:
        form = "flat polygon"
    if form != "polygons":
        raise NotImplementedError("only COCO polygon segmentations are rasterised, not the %s form" % form)
    return segm


def polygons_csr(polygons):
    """list of flat [x0, y0, x1, y1, ...] polygons -> (xy float64 [2 V], poly_off int64 [P + 1] in vertices); an odd
    trailing coordinate is dropped as rleFrPoly's k = len / 2 does"""
    ks = [len(p) // 2 for p in polygons]
    off = np.concatenate([[0], np.cumsum(ks)]).astype(np.int64)
    xy = np.concatenate([np.asarray(p, np.float64)[:2 * k] for p, k in zip(polygons, ks)]) if polygons else \
        np.zeros(0, np.float64)
    return xy, off


def _edge_table(xy, poly_off):
    """rleFrPoly's vertex scaling (int)(5 x + .5) and the edge rows of csrc/polygon.cu"""
    xy = np.asarray(xy, np.float64).reshape(-1)
    off = np.asarray(poly_off, np.int64)
    v = int(off[-1])
    if xy.size != 2 * v:
        raise ValueError("xy holds %d coordinates, poly_off describes %d vertices" % (xy.size, v))
    if not np.isfinite(xy).all():
        raise ValueError("polygon vertices must be finite")
    s = np.trunc(np.float64(5.0) * xy + 0.5)          # two IEEE operations, C's truncating (int) cast
    if (s < _INT_MIN + 1).any() or (s > _INT_MAX).any():
        raise ValueError("polygon vertex out of range: 5 * coordinate must fit a 32-bit int")
    s = s.astype(np.int64)
    x, y = s[0::2], s[1::2]
    k = np.diff(off)
    plane = np.repeat(np.arange(len(k), dtype=np.int64), k)
    nxt = np.arange(v, dtype=np.int64) + 1
    last = off[1:][k > 0] - 1
    nxt[last] = off[:-1][k > 0]
    edge_xy = np.stack([x, y, x[nxt], y[nxt]], axis=1).astype(np.int32)
    count = np.maximum(np.abs(x[nxt] - x), np.abs(y[nxt] - y)) + 1
    edge_pt = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    return edge_xy, edge_pt, plane.astype(np.int32)


def _rasterize_into(out, xy, poly_off, h, w):
    planes = len(poly_off) - 1
    edge_xy, edge_pt, edge_plane = _edge_table(xy, poly_off)
    e = len(edge_plane)
    dev = out.device
    ex = torch.from_numpy(edge_xy).to(dev) if e else None
    ep = torch.from_numpy(edge_pt).to(dev) if e else None
    epl = torch.from_numpy(edge_plane).to(dev) if e else None
    bits = torch.empty(planes * ((h * w + 31) // 32), dtype=torch.int32, device=dev)
    L.fcall("mcb_rasterize_polygons", L.dp(ex), L.dp(ep), L.dp(epl), e, int(edge_pt[-1]), bits.data_ptr(),
            out.data_ptr(), planes, h, w)


def rasterize_polygons(xy, poly_off, height, width):
    """cocomask.decode(cocomask.frPyObjects(polygons, h, w)) bit for bit, one plane per polygon: xy float64 [2 V],
    poly_off int64 [P + 1] (vertex offsets) -> uint8 (P, h, w) cuda, row-major"""
    h, w = int(height), int(width)
    p = len(poly_off) - 1
    out = torch.empty((p, h, w), dtype=torch.uint8, device=_dev())
    if p:
        _rasterize_into(out, xy, poly_off, h, w)
    return out


def _i32(a, dev):
    """a small int32 device array; the caller keeps it referenced until the launch that reads it is enqueued"""
    a = np.asarray(a, np.int32)
    return torch.from_numpy(a if a.size else np.zeros(1, np.int32)).to(dev)


def _group_offsets(groups, n_groups):
    return np.concatenate([[0], np.cumsum(np.bincount(np.asarray(groups, np.int64), minlength=n_groups))]).astype(
        np.int32)


def _union(planes, index, groups, n_groups, h, w):
    """union of planes[index[j]] per group (index sorted by group) -> uint8 (n_groups, h, w)"""
    dev = planes.device
    out = torch.empty((n_groups, h, w), dtype=torch.uint8, device=dev)
    index_d, off_d = _i32(index, dev), _i32(_group_offsets(groups, n_groups), dev)
    L.fcall("mcb_plane_union", planes.data_ptr(), index_d.data_ptr(), off_d.data_ptr(), n_groups, h, w, out.data_ptr())
    return out


def overlay_batch(annotations_per_image, height, width, category_ids=(None, 100), erode=0, dilate=0, border_width=0,
                  small_annotations_size=14):
    """overlay_mask_one_image (src/preparation.py:44-100) for a batch of equally sized images, on the device.
    annotations_per_image: one list of COCO annotation dicts per image, in file order.
    -> (mask uint8 (N, H, W), distances float16 (N, H, W), sizes int64 (N, H, W) cuda,
        sizes_uint8 bool numpy (N,): the image has no component, so the reference's sizes are np.ones_like(mask), uint8)

    Every polygon is rasterised exactly as pycocotools does.  With erode == 0 each polygon is an instance; otherwise
    each annotation is, must hold one polygon (the reference's reshape raises ValueError), and is eroded with
    rectangle(erode, erode) when its area exceeds small_annotations_size**2, else dilated with rectangle(dilate,
    dilate) when dilate > 0 -- skimage <= 0.17's binary_erosion / binary_dilation (mcb_binary_morph_rect).  Instances
    with no pixel in [2:-2, 2:-2] are dropped.  The distances are the two nearest kept instances (update_distances /
    clean_distances, including the replacement while the accumulated sum is 0), the sizes get_size_matrix of the
    overlaid mask, and border_width > 0 adds the reference's border class."""
    h, w, n = int(height), int(width), len(annotations_per_image)
    if n == 0:
        raise ValueError("overlay_batch needs at least one image")
    cats = [(nr, cid) for nr, cid in enumerate(category_ids) if cid is not None]
    if cats and (erode < 0 or dilate < 0):
        raise ValueError("erode and dilate cannot be negative")
    c_n = max(len(cats), 1)
    if n * c_n > _MAX_PLANES_Y:
        raise ValueError("overlay_batch takes at most %d images x categories per call, got %d" % (_MAX_PLANES_Y, n * c_n))
    polys, group = [], []
    for i, anns in enumerate(annotations_per_image):
        for c, (_, cid) in enumerate(cats):
            for ann in anns:
                if ann["category_id"] != cid:
                    continue
                segm = segmentation_polygons(ann["segmentation"])
                if erode > 0 and len(segm) != 1:
                    raise ValueError("annotation %s has %d polygons; with erode > 0 every annotation is reshaped to "
                                     "one mask, which needs exactly one" % (ann.get("id"), len(segm)))
                polys.extend(segm)
                group.append(np.full(len(segm), i * c_n + c, np.int64))
    group = np.concatenate(group) if group else np.zeros(0, np.int64)
    dev = _dev()
    hw = h * w
    p = len(polys)
    stages = 1 if erode == 0 else (2 if dilate == 0 else 3)
    buf = torch.empty((max(stages * p, 1), h, w), dtype=torch.uint8, device=dev)
    if p:
        xy, off = polygons_csr(polys)
        _rasterize_into(buf[:p], xy, off, h, w)
        if erode > 0:
            L.fcall("mcb_binary_morph_rect", buf.data_ptr(), buf[p:].data_ptr(), 0, int(erode), p, h, w)
            if dilate > 0:
                L.fcall("mcb_binary_morph_rect", buf.data_ptr(), buf[2 * p:].data_ptr(), 1, int(dilate), p, h, w)
        stats_d = torch.empty((stages * p, 4), dtype=torch.int32, device=dev)
        L.fcall("mcb_plane_stats", buf.data_ptr(), stages * p, h, w, 2, stats_d.data_ptr())
        stats = stats_d.cpu().numpy()
    else:
        stats_d, stats = None, np.zeros((0, 4), np.int32)
    idx = np.arange(p, dtype=np.int64)
    kept = stats[:p, 1] != 0
    if erode == 0:
        inst = idx
    else:
        big = stats[:p, 0] > small_annotations_size ** 2
        inst = np.where(big, p + idx, 2 * p + idx if dilate > 0 else idx)
    inst, inst_group = inst[kept], group[kept]

    cat_masks = _union(buf, inst, inst_group, n * c_n, h, w)
    if erode > 0 and dilate == 0:
        full = _union(buf, idx[kept], inst_group, n * c_n, h, w)
        dropped = torch.empty_like(full)
        ws = torch.empty(2 * full.numel(), dtype=torch.int32, device=dev)
        L.fcall("mcb_add_dropped_objects", full.data_ptr(), cat_masks.data_ptr(), dropped.data_ptr(), ws.data_ptr(),
                n * c_n, h, w)
        cat_masks = dropped
    mask = torch.empty((n, h, w), dtype=torch.uint8, device=dev)
    nr = _i32([nr for nr, _ in cats] or [0], dev)
    if cats:
        L.fcall("mcb_category_overlay", cat_masks.data_ptr(), nr.data_ptr(), c_n, n, h, w, mask.data_ptr())
    else:
        L.zero(mask)

    # update_distances replaces the stack while its sum is 0: an image's leading instances that cover it entirely
    # (distance transform 0 everywhere) are dropped
    img = inst_group // c_n
    full_cover = stats[inst, 0] == hw if p else np.zeros(0, bool)
    keep_d = np.ones(len(inst), bool)
    for i in range(n):
        sel = np.nonzero(img == i)[0]
        lead = sel[np.cumprod(full_cover[sel]).astype(bool)] if sel.size else sel
        keep_d[lead] = False
    d_inst, d_img = inst[keep_d], img[keep_d]
    k = len(d_inst)
    dist = torch.empty((n, h, w), dtype=torch.float16, device=dev)
    second = torch.empty((n, h, w), dtype=torch.float64, device=dev)
    ws = torch.empty(max(k * hw, 1), dtype=torch.int32, device=dev)
    d_inst_d, d_off_d = _i32(d_inst, dev), _i32(_group_offsets(d_img, n), dev)
    L.fcall("mcb_edt_two_nearest_batched", buf.data_ptr(), d_inst_d.data_ptr(), d_off_d.data_ptr(), L.dp(stats_d), k,
            n, h, w, ws.data_ptr(), dist.data_ptr(), second.data_ptr())

    labels, counts = label_batch(mask, return_counts=True)
    sizes = torch.empty((n, h, w), dtype=torch.int64, device=dev)
    area = torch.empty((n, h, w), dtype=torch.int32, device=dev)
    L.fcall("mcb_size_matrix_batched", labels.data_ptr(), area.data_ptr(), sizes.data_ptr(), n, h, w)
    if border_width > 0:
        L.fcall("mcb_border_class", mask.data_ptr(), second.data_ptr(), n, h, w, float(border_width))
    return mask, dist, sizes, counts.cpu().numpy() == 0


def coco_index(annotation_file):
    """pycocotools COCO's indexing of an annotation file: -> (images in getImgIds order, {image id: [annotations in
    file order]})"""
    with open(annotation_file) as f:
        dataset = json.load(f)
    imgs = {}
    for im in dataset.get("images", []):
        imgs[im["id"]] = im
    anns = {i: [] for i in imgs}
    for a in dataset.get("annotations", []):
        anns.setdefault(a["image_id"], []).append(a)
    return list(imgs.values()), anns


OVERLAY_CHUNK = 128   # images per device batch: 128 x 40 buildings of 300 x 300 keep the workspaces near 3 GB
OVERLAY_IN_FLIGHT = 2  # chunks whose host arrays may wait for the writers (about 127 MB each at 300 x 300)


def _write_targets(target_dir, dataset, image, mask, dist, sizes):
    import joblib
    from PIL import Image
    stem = os.path.splitext(image["file_name"])[0]
    paths = [os.path.join(target_dir, dataset, sub, stem) for sub in ("masks", "distances", "sizes")]
    for pth in paths:
        os.makedirs(os.path.dirname(pth), exist_ok=True)
    Image.fromarray(mask, mode="L").save(paths[0] + ".png")
    joblib.dump(dist, paths[1])
    joblib.dump(sizes, paths[2])


def overlay_masks(data_dir, dataset, target_dir, category_ids, erode=0, dilate=0, is_small=False, num_threads=1,
                  border_width=0, small_annotations_size=14):
    """drop-in for src/preparation.py:18-41: reads <data_dir>/<dataset>/annotation{-small}.json and writes, per image,
    <target_dir>/<dataset>/masks/<stem>.png (uint8 grayscale), distances/<stem> (joblib, float16) and sizes/<stem>
    (joblib, int64; uint8 ones for an image without buildings).  Images are batched by size on the device; a pool of
    num_threads host threads encodes and writes one batch while the device prepares the next; at most
    OVERLAY_IN_FLIGHT batches wait for the writers, so host memory stays bounded however large the dataset."""
    suffix = "-small" if is_small else ""
    images, anns = coco_index(os.path.join(data_dir, dataset, "annotation{}.json".format(suffix)))
    by_size = {}
    for im in images:
        by_size.setdefault((int(im["height"]), int(im["width"])), []).append(im)
    with ThreadPoolExecutor(max(1, min(int(num_threads), max(len(images), 1)))) as pool:
        pending = deque()   # one list of write futures per chunk
        for (h, w), ims in by_size.items():
            for c0 in range(0, len(ims), OVERLAY_CHUNK):
                chunk = ims[c0:c0 + OVERLAY_CHUNK]
                mask, dist, sizes, ones_u8 = overlay_batch([anns.get(im["id"], []) for im in chunk], h, w,
                                                           category_ids, erode, dilate, border_width,
                                                           small_annotations_size)
                mask, dist, sizes = mask.cpu().numpy(), dist.cpu().numpy(), sizes.cpu().numpy()
                while len(pending) >= OVERLAY_IN_FLIGHT:
                    for f in pending.popleft():
                        f.result()
                pending.append([pool.submit(_write_targets, target_dir, dataset, im, mask[j], dist[j],
                                            sizes[j].astype(np.uint8) if ones_u8[j] else sizes[j])
                                for j, im in enumerate(chunk)])
        for fs in pending:
            for f in fs:
                f.result()
