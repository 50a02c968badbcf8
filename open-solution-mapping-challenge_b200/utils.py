"""Instance emission: mirror of src/utils.py:61-127 (decompose, create_annotations, rle_from_binary,
bounding_box_from_rle) on the GPU.

The reference turns every labelled instance into a full-image uint8 mask on the host and hands it to pycocotools
(`cocomask.encode` on the Fortran-ordered mask, `cocomask.toBbox`), twice per instance.  Here one device pass computes
area / bounding box of every instance of a batch of label planes, one warp per (instance, column) run-length encodes the mask
inside its bounding box (csrc/instances.cu), and only the run lengths come back to the host, where the LEB128-like
COCO string of pycocotools' rleToString is produced with vectorised numpy.  No pycocotools, no CPU fallback for the
pixel work.

`rle_from_binary` / `bounding_box_from_rle` keep the reference's per-mask signatures (dict with 'size' and 'counts'
bytes, list [x, y, w, h] of floats)."""
import json
import os

import numpy as np
import torch

from . import _lib as L
from .postprocessing import _dev, _to_dev

_INT_MAX = 2 ** 31 - 1


# ---------------------------------------------------------------------------------------------------------------------
# device level
# ---------------------------------------------------------------------------------------------------------------------
def _offsets(counts):
    """counts (P,) int32 cuda -> (offsets cuda int32 (P,), counts host, offsets host, total)"""
    counts_h = counts.cpu().numpy().astype(np.int64)
    offs_h = np.concatenate([[0], np.cumsum(counts_h)[:-1]]).astype(np.int32) if counts_h.size else np.zeros(0, np.int32)
    total = int(counts_h.sum())
    return torch.from_numpy(offs_h).to(counts.device), counts_h, offs_h, total


def instance_geometry(labels, counts, probs=None):
    """labels (P, H, W) int32 cuda, counts (P,) int32 cuda (labels per plane), probs (P, H, W) float32|float64 or None
    -> dict of host arrays per instance slot: area, rmin, rmax, cmin, cmax [, psum (float64), pmax (float32)],
    plus 'offsets', 'counts', 'plane' (slot -> plane)."""
    assert labels.is_cuda and labels.dtype == torch.int32 and labels.is_contiguous() and labels.dim() == 3
    p, h, w = labels.shape
    counts = counts.to(torch.int32).contiguous()
    offs_d, counts_h, offs_h, total = _offsets(counts)
    geo = torch.empty((max(total, 1), 5), dtype=torch.int32, device=labels.device)
    geo[:, 0] = 0
    geo[:, 1] = _INT_MAX
    geo[:, 2] = -1
    geo[:, 3] = _INT_MAX
    geo[:, 4] = -1
    psum = pmax = None
    if probs is not None:
        assert probs.shape == labels.shape and probs.is_cuda and probs.is_contiguous()
        psum = torch.zeros(max(total, 1), dtype=torch.float64, device=labels.device)
        # order-preserving integer image of float32 -inf
        pmax = torch.full((max(total, 1),), int(np.array(-np.inf, np.float32).view(np.int32)) ^ 0x7FFFFFFF,
                          dtype=torch.int32, device=labels.device)
    if total > 0:
        L.fcall("mcb_instance_geometry", labels.data_ptr(), None if probs is None else probs.data_ptr(),
                int(probs is not None and probs.dtype == torch.float64), offs_d.data_ptr(), counts.data_ptr(),
                geo.data_ptr(), None if psum is None else psum.data_ptr(), None if pmax is None else pmax.data_ptr(),
                p, h, w)
    g = geo[:total].cpu().numpy()
    out = {"area": g[:, 0], "rmin": g[:, 1], "rmax": g[:, 2], "cmin": g[:, 3], "cmax": g[:, 4], "offsets": offs_h,
           "counts": counts_h, "plane": np.repeat(np.arange(p, dtype=np.int32), counts_h), "_geo": geo,
           "_offsets": offs_d, "_counts": counts}
    if probs is not None:
        out["psum"] = psum[:total].cpu().numpy()
        pm = pmax[:total].cpu().numpy()
        out["pmax"] = np.where(pm >= 0, pm, pm ^ 0x7FFFFFFF).astype(np.int32).view(np.float32)
    return out


def rle_encode_instances(labels, counts, geometry=None):
    """COCO run lengths of every instance of a batch of label planes.
    -> (cnts uint32 host (concatenated), starts int64 host (total + 1,), spans bool host (total,), geometry dict)
    instance `slot` owns cnts[starts[slot]:starts[slot + 1]] (pycocotools RLE counts of its column-major mask)."""
    geo = geometry if geometry is not None else instance_geometry(labels, counts)
    p, h, w = labels.shape
    total = int(geo["counts"].sum())
    if total == 0:
        return np.zeros(0, np.uint32), np.zeros(1, np.int64), np.zeros(0, bool), geo
    dev = labels.device
    inst_plane = torch.from_numpy(geo["plane"]).to(dev)
    # one task per (instance, bounding-box column): columns are independent, so the image-sized background instance of
    # every plane is walked by 300 warps instead of one
    width = np.where(geo["area"] > 0, geo["cmax"] - geo["cmin"] + 1, 0).astype(np.int64)
    ntasks = int(width.sum())
    task_slot_h = np.repeat(np.arange(total, dtype=np.int32), width)
    first = np.concatenate([[0], np.cumsum(width)[:-1]])
    task_x_h = (np.arange(ntasks, dtype=np.int64) - np.repeat(first, width) + np.repeat(geo["cmin"].astype(np.int64), width)).astype(np.int32)
    task_slot, task_x = torch.from_numpy(task_slot_h).to(dev), torch.from_numpy(task_x_h).to(dev)
    task_n = torch.zeros(max(ntasks, 1), dtype=torch.int32, device=dev)
    L.fcall("mcb_rle_walk", labels.data_ptr(), geo["_offsets"].data_ptr(), geo["_geo"].data_ptr(), inst_plane.data_ptr(),
            task_slot.data_ptr(), task_x.data_ptr(), None, task_n.data_ptr(), None, None, ntasks, h, w, 0)
    task_n_h = task_n[:ntasks].cpu().numpy().astype(np.int64)
    task_start_h = np.concatenate([[0], np.cumsum(task_n_h)[:-1]]).astype(np.int32) if ntasks else np.zeros(0, np.int32)
    n_changes_total = int(task_n_h.sum())
    n_h = np.bincount(task_slot_h, weights=task_n_h, minlength=total).astype(np.int64)      # changes per instance
    out_start_h = np.concatenate([[0], np.cumsum(n_h)[:-1]]).astype(np.int32)
    task_start = torch.from_numpy(task_start_h).to(dev)
    nchanges = torch.from_numpy(n_h.astype(np.int32)).to(dev)
    out_start = torch.from_numpy(out_start_h).to(dev)
    changes = torch.empty(max(n_changes_total, 1), dtype=torch.int32, device=dev)
    spans = torch.zeros(total, dtype=torch.int32, device=dev)
    L.fcall("mcb_rle_walk", labels.data_ptr(), geo["_offsets"].data_ptr(), geo["_geo"].data_ptr(), inst_plane.data_ptr(),
            task_slot.data_ptr(), task_x.data_ptr(), task_start.data_ptr(), task_n.data_ptr(), changes.data_ptr(),
            spans.data_ptr(), ntasks, h, w, 1)
    total_counts = n_changes_total + total
    slot_of_count = torch.from_numpy(np.repeat(np.arange(total, dtype=np.int32), n_h + 1)).to(dev)
    cnts = torch.empty(total_counts, dtype=torch.int32, device=dev)
    L.fcall("mcb_rle_counts", changes.data_ptr(), nchanges.data_ptr(), out_start.data_ptr(), slot_of_count.data_ptr(),
            cnts.data_ptr(), total_counts, h * w)
    starts = np.concatenate([[0], np.cumsum(n_h + 1)]).astype(np.int64)
    return cnts.cpu().numpy().view(np.uint32), starts, spans.cpu().numpy().astype(bool), geo


# ---------------------------------------------------------------------------------------------------------------------
# pycocotools string / bbox formats (host, vectorised; a few thousand small integers per batch)
# ---------------------------------------------------------------------------------------------------------------------
def rle_counts_to_string(cnts):
    """pycocotools rleToString: counts (with the third and later ones delta-coded against the count two places back)
    in 5-bit groups, least significant first, bit 5 = continuation, + 48 -> ASCII bytes"""
    c = np.asarray(cnts, dtype=np.int64)
    x = c.copy()
    if c.size > 3:
        x[3:] -= c[1:-2]
    out = np.zeros((c.size, 13), np.uint8)   # 64-bit values need at most 13 groups
    alive = np.ones(c.size, bool)
    length = np.zeros(c.size, np.int64)
    for g in range(13):
        if not alive.any():
            break
        ch = x & 0x1f
        x = x >> 5
        more = np.where((ch & 0x10) != 0, x != -1, x != 0)
        ch = np.where(more, ch | 0x20, ch) + 48
        out[alive, g] = ch[alive]
        length[alive] += 1
        alive &= more
    mask = np.arange(13)[None, :] < length[:, None]
    return out[mask].tobytes()


def rle_to_bbox(cnts, h, w):
    """pycocotools rleToBbox -> [x, y, w, h] (floats), including its full-height rule for runs that cross a column"""
    c = np.asarray(cnts, dtype=np.int64)
    m = (c.size // 2) * 2
    if m == 0:
        return [0.0, 0.0, 0.0, 0.0]
    cc = np.cumsum(c[:m])
    j = np.arange(m)
    t = cc - (j % 2)
    y = t % h
    x = (t - y) // h
    xs, xe, ys, ye = x.min(), x.max(), y.min(), y.max()
    if (x[0::2] < x[1::2]).any():
        ys, ye = 0, h - 1
    return [float(xs), float(ys), float(xe - xs + 1), float(ye - ys + 1)]


def rle_from_binary(prediction):
    """src/utils.py:118-120: cocomask.encode(np.asfortranarray(prediction)) -> {'size': [h, w], 'counts': bytes}"""
    m = np.asarray(prediction)
    if m.ndim != 2:
        raise ValueError("rle_from_binary expects one 2-D mask")
    lab = _to_dev((m != 0).astype(np.int32), torch.int32)[None].contiguous()
    one = torch.ones(1, dtype=torch.int32, device=lab.device)
    cnts, starts, _, _ = rle_encode_instances(lab, one)
    return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": rle_counts_to_string(cnts[starts[0]:starts[1]])}


def rle_string_to_counts(s):
    """inverse of rle_counts_to_string (pycocotools rleFrString)"""
    if isinstance(s, str):
        s = s.encode("ascii")
    cnts = []
    p = 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return cnts


def bounding_box_from_rle(rle):
    """src/utils.py:123-124: list(cocomask.toBbox(rle))"""
    h, w = rle["size"]
    return rle_to_bbox(rle_string_to_counts(rle["counts"]), h, w)


def decompose(labeled):
    """src/utils.py:61-73 (host helper kept for signature parity; create_annotations below does not use it)"""
    nr_true = labeled.max()
    masks = []
    for i in range(1, nr_true + 1):
        msk = labeled.copy()
        msk[msk != i] = 0.
        msk[msk == i] = 255.
        masks.append(msk)
    return masks if masks else [labeled]


def create_annotations(meta, predictions, logger, category_ids, category_layers, save=False, experiment_dir='./'):
    """src/utils.py:76-115.  predictions: per image (labels (L, H, W) int32, [[score, ...] per layer]).  All instances
    of all images and layers are encoded in one device batch."""
    annotations = []
    if logger is not None:
        logger.info('Creating annotations')
    category_layers_inds = np.cumsum(category_layers)
    if isinstance(meta, (list, tuple, np.ndarray)):
        image_ids = list(meta)                       # plain ids (tests / callers without a metadata frame)
    else:
        ids = meta["ImageId"]                        # the reference's pd.DataFrame (src/utils.py:97)
        image_ids = list(getattr(ids, "values", ids))
    planes, owners = [], []
    for image_id, (prediction, image_scores) in zip(image_ids, predictions):
        for category_ind, (category_instances, category_scores) in enumerate(zip(prediction, image_scores)):
            category_nr = int(np.searchsorted(category_layers_inds, category_ind, side='right'))
            if category_ids[category_nr] is not None:
                planes.append(np.asarray(category_instances))
                owners.append((image_id, category_ids[category_nr], category_scores))
    if planes:
        shapes = {p.shape for p in planes}
        if len(shapes) != 1:
            raise NotImplementedError("create_annotations batches equally sized label maps")
        lab = _to_dev(np.stack(planes).astype(np.int32), torch.int32)
        counts = lab.reshape(lab.shape[0], -1).max(dim=1).values.to(torch.int32)
        cnts, starts, _, geo = rle_encode_instances(lab, counts)
        h, w = planes[0].shape
        for pi, (image_id, cat_id, scores) in enumerate(owners):
            k = int(geo["counts"][pi])
            if k == 0:
                # decompose() of an empty layer returns the layer itself: one all-background "mask" (src/utils.py:70-71)
                k_iter = [(None, s) for s in list(scores)[:1]]
            else:
                k_iter = [(int(geo["offsets"][pi]) + i, s) for i, s in zip(range(k), scores)]
            for slot, score in k_iter:
                c = cnts[starts[slot]:starts[slot + 1]] if slot is not None else np.array([h * w], np.uint32)
                annotations.append({"image_id": int(image_id), "category_id": cat_id, "score": score,
                                    "segmentation": {"size": [int(h), int(w)],
                                                     "counts": rle_counts_to_string(c).decode("UTF-8")},
                                    "bbox": rle_to_bbox(c, h, w)})
    if save:
        submission_filepath = os.path.join(experiment_dir, 'submission.json')
        with open(submission_filepath, "w") as fp:
            fp.write(str(json.dumps(annotations)))
        if logger is not None:
            logger.info("Submission saved to {}".format(submission_filepath))
        return True
    return annotations
