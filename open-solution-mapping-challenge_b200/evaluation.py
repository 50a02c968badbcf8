"""COCO segmentation evaluation (src/cocoeval.py, driven by src/utils.py:308-321) with its per-pair and per-image work
on the device.

`DeviceCOCOEvaluator` holds the ground truth of one evaluation as device tables of COCO run lists, built once.
`add_batch` takes the device label maps and scores of a batch of predictions, run-length encodes every instance
(`mcb200.utils.rle_encode_instances`), computes the mask IoU of every (detection, ground truth) pair whose bounding
boxes overlap (`mcb_rle_pair_iou`) and runs COCOeval.evaluateImg for every (image, area range)
(`mcb_coco_match`, csrc/evaluation.cu); the small match tables stay on the device.  `result()` copies them once and
runs COCOeval.accumulate / summarize (src/cocoeval.py:322-494) on the host in numpy.

`coco_evaluation` keeps the reference's signature and return value for `main.py evaluate` users: ground-truth and
prediction JSON files in, (AP at IoU 0.5, AR at IoU 0.5) out.

Parameters are the reference's (src/cocoeval.py:503-511 with the area ranges of src/utils.py:314-316): IoU thresholds
.50:.05:.95, 101 recall thresholds, maxDets 1 / 10 / 100, area ranges all / small / large with both bounds inclusive.
"""
import json

import numpy as np
import torch

from . import _lib as L
from .utils import rle_encode_instances, rle_string_to_counts, rle_to_bbox

IOU_THRS = np.linspace(.5, 0.95, 10, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, 101, endpoint=True)
MAX_DETS = (1, 10, 100)
AREA_LABELS = ('all', 'small', 'large')
CATEGORY_IDS = (None, 100)      # src/pipeline_config.py:17: output layer 0 is background, layer 1 buildings
CATEGORY_LAYERS = (1, 1)        # src/pipeline_config.py:18


def area_ranges(small_annotations_size):
    """src/utils.py:314-315"""
    s = small_annotations_size
    return np.array([[0 ** 2, 1e5 ** 2], [0 ** 2, s ** 2], [s ** 2, 1e5 ** 2]], dtype=np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# annotations -> run lists
# ---------------------------------------------------------------------------------------------------------------------
def segmentation_counts(segm, h, w):
    """COCO.annToRLE + the decoding of its counts -> (run lengths int64, (height, width)).  Compressed and uncompressed
    RLE are read here; polygons go through pycocotools.mask.frPyObjects / merge, the reference's own dependency."""
    if isinstance(segm, list):
        try:
            from pycocotools import mask as mask_utils
        except ImportError as e:
            raise NotImplementedError("polygon segmentations need pycocotools.mask.frPyObjects, which is not "
                                      "importable (%s); give the annotations as RLE" % e)
        segm = mask_utils.merge(mask_utils.frPyObjects(segm, h, w))
    counts = segm['counts']
    cnts = counts if isinstance(counts, list) else rle_string_to_counts(counts)
    return np.asarray(cnts, dtype=np.int64), (int(segm['size'][0]), int(segm['size'][1]))


GT_RLE_CHUNK = 4096   # polygon annotations rasterised per device batch


def ground_truth_rle(gt):
    """a copy of a COCO ground truth (dict or JSON path) whose polygon segmentations are replaced by the uncompressed
    RLE {'size': [h, w], 'counts': [...]} of COCO.annToRLE, merge(frPyObjects(polygons, h, w)): the union of the
    annotation's polygons, rasterised on the device exactly as pycocotools does (mcb200.preparation).  The result
    feeds DeviceCOCOEvaluator / coco_evaluation without pycocotools."""
    import copy
    from .preparation import polygons_csr, rasterize_polygons, segmentation_polygons
    from .postprocessing import _dev
    if not isinstance(gt, dict):
        with open(gt) as f:
            gt = json.load(f)
    out = copy.deepcopy(gt)
    size = {im["id"]: (int(im["height"]), int(im["width"])) for im in out.get("images", [])}
    by_size = {}
    for a in out.get("annotations", []):
        if isinstance(a.get("segmentation"), list):
            by_size.setdefault(size[a["image_id"]], []).append(a)
    for (h, w), anns in by_size.items():
        for c0 in range(0, len(anns), GT_RLE_CHUNK):
            chunk = anns[c0:c0 + GT_RLE_CHUNK]
            polys, group = [], []
            for j, a in enumerate(chunk):
                segm = segmentation_polygons(a["segmentation"])
                polys.extend(segm)
                group.extend([j] * len(segm))
            dev = _dev()
            planes = rasterize_polygons(*polygons_csr(polys), h, w)
            union = torch.empty((len(chunk), h, w), dtype=torch.uint8, device=dev)
            goff = np.concatenate([[0], np.cumsum(np.bincount(group, minlength=len(chunk)))]).astype(np.int32)
            index = torch.arange(max(len(polys), 1), dtype=torch.int32, device=dev)
            goff_d = torch.from_numpy(goff).to(dev)
            L.fcall("mcb_plane_union", planes.data_ptr() if len(polys) else index.data_ptr(), index.data_ptr(),
                    goff_d.data_ptr(), len(chunk), h, w, union.data_ptr())
            labels = union.to(torch.int32)
            cnts, starts, _, _ = rle_encode_instances(labels, torch.ones(len(chunk), dtype=torch.int32, device=dev))
            for j, a in enumerate(chunk):
                a["segmentation"] = {"size": [h, w], "counts": cnts[starts[j]:starts[j + 1]].astype(np.int64).tolist()}
    return out


def _rle_area(cnts):
    return int(np.asarray(cnts, dtype=np.int64)[1::2].sum())


def _starts(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def _dev_tensor(a, dtype, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dtype)


# ---------------------------------------------------------------------------------------------------------------------
# COCOeval.accumulate / summarize on flat per-unit tables
# ---------------------------------------------------------------------------------------------------------------------
def accumulate(nd, ng, present, dt_scores, dt_match, dt_ignore, gt_ignore, n_cats, n_imgs, iou_thrs=IOU_THRS,
               rec_thrs=REC_THRS, max_dets=MAX_DETS):
    """src/cocoeval.py:322-427.  Unit u = k * n_imgs + i is (category k, image i) in sorted id order; it holds nd[u]
    detections (score order, at most max_dets[-1]) and ng[u] ground truths, stored back to back in unit order:
    dt_scores [sum nd], dt_match int [A][T][sum nd] (matched ground-truth id, 0 = none), dt_ignore [A][T][sum nd],
    gt_ignore [A][sum ng].  present[u] is False where evaluateImg returned None.  -> (precision [T,R,K,A,M],
    recall [T,K,A,M]).  The precision envelope is np.maximum.accumulate over the reversed array, which is the reference's
    backward max loop exactly."""
    nd, ng = np.asarray(nd, np.int64), np.asarray(ng, np.int64)
    T, R, A, M = len(iou_thrs), len(rec_thrs), dt_match.shape[0], len(max_dets)
    precision = -np.ones((T, R, n_cats, A, M))
    recall = -np.ones((T, n_cats, A, M))
    doff, goff = _starts(nd), _starts(ng)
    for k in range(n_cats):
        units = np.arange(k * n_imgs, (k + 1) * n_imgs)
        units = units[np.asarray(present, bool)[units]]
        if units.size == 0:
            continue
        g_cols = np.concatenate([np.arange(goff[u], goff[u + 1]) for u in units])
        for a in range(A):
            npig = np.count_nonzero(gt_ignore[a][g_cols] == 0)
            for m, max_det in enumerate(max_dets):
                if npig == 0:
                    continue
                cols = np.concatenate([np.arange(doff[u], doff[u] + min(nd[u], max_det)) for u in units])
                inds = np.argsort(-dt_scores[cols], kind='mergesort')
                dtm = dt_match[a][:, cols][:, inds]
                dtig = dt_ignore[a][:, cols][:, inds].astype(bool)
                tps = np.logical_and(dtm, np.logical_not(dtig))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtig))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                n = tp_sum.shape[1]
                rc = tp_sum / npig
                pr = tp_sum / (fp_sum + tp_sum + np.spacing(1))
                recall[:, k, a, m] = rc[:, -1] if n else 0
                if n:
                    pr = np.maximum.accumulate(pr[:, ::-1], axis=1)[:, ::-1]
                for t in range(T):
                    ri = np.searchsorted(rc[t], rec_thrs, side='left')
                    q = np.zeros((R,))
                    ok = ri < n
                    q[ok] = pr[t, ri[ok]]
                    precision[t, :, k, a, m] = q
    return precision, recall


def summarize(precision, recall, iou_thrs=IOU_THRS, max_dets=MAX_DETS, area_labels=AREA_LABELS):
    """src/cocoeval.py:429-473 (segm): stats[0..2] = AP at IoU .5 for all / small / large, stats[3..5] = AR likewise,
    all at maxDets[2]"""
    def _summarize(ap, iou_thr, area_rng='all', max_det=100):
        aind = [i for i, a in enumerate(area_labels) if a == area_rng]
        mind = [i for i, m in enumerate(max_dets) if m == max_det]
        t = np.where(iou_thr == iou_thrs)[0]
        if ap == 1:
            s = precision[t]
            s = s[:, :, :, aind, mind]
        else:
            s = recall[t]
            s = s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    stats = np.zeros((6,))
    stats[0] = _summarize(1, .5, max_det=max_dets[2])
    stats[1] = _summarize(1, .5, 'small', max_dets[2])
    stats[2] = _summarize(1, .5, 'large', max_dets[2])
    stats[3] = _summarize(0, .5, max_det=max_dets[2])
    stats[4] = _summarize(0, .5, 'small', max_dets[2])
    stats[5] = _summarize(0, .5, 'large', max_dets[2])
    return stats


# ---------------------------------------------------------------------------------------------------------------------
# device evaluator
# ---------------------------------------------------------------------------------------------------------------------
class DeviceCOCOEvaluator:
    """COCOeval (iouType 'segm', useCats 1) of one ground truth against predictions added batch by batch.

    gt: COCO annotation dict or JSON path; image_ids / category_ids: what is evaluated (the reference passes the
    validation metadata's ImageId and CATEGORY_IDS[1:]); ground truths of other images or categories are ignored.
    layer_category_ids / category_layers map the label layers of `add_batch` to categories as create_annotations does
    (src/utils.py:76-115; None = layer not emitted).  Every image is added at most once."""

    def __init__(self, gt, image_ids, category_ids, small_annotations_size=14, layer_category_ids=CATEGORY_IDS,
                 category_layers=CATEGORY_LAYERS, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("DeviceCOCOEvaluator needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if isinstance(gt, str):
            with open(gt) as f:
                gt = json.load(f)
        self.img_ids = [int(i) for i in np.unique(np.asarray(image_ids))]
        self.cat_ids = [int(c) for c in np.unique(np.asarray(category_ids))]
        self.area_rng = area_ranges(small_annotations_size)
        self.layer_category_ids = list(layer_category_ids)
        self.category_layers = list(category_layers)
        self._img_index = {i: n for n, i in enumerate(self.img_ids)}
        self._cat_index = {c: n for n, c in enumerate(self.cat_ids)}
        self.image_sizes = {int(im['id']): (int(im['height']), int(im['width'])) for im in gt.get('images', [])}
        I, K = len(self.img_ids), len(self.cat_ids)
        self.n_units = I * K
        per_unit = [[] for _ in range(self.n_units)]
        for ann in gt['annotations']:      # getAnnIds(imgIds, catIds) + loadAnns: file order within an image
            i, k = self._img_index.get(ann['image_id']), self._cat_index.get(ann['category_id'])
            if i is not None and k is not None:
                per_unit[k * I + i].append(ann)
        ids, crowd, area, cnts, sizes, bboxes, ng = [], [], [], [], [], [], []
        for u, anns in enumerate(per_unit):
            ng.append(len(anns))
            for ann in anns:
                h, w = self.image_sizes.get(int(ann['image_id']), (None, None))
                c, size = segmentation_counts(ann['segmentation'], h, w)
                ids.append(int(ann['id']))
                crowd.append(1 if ann.get('iscrowd', 0) else 0)   # _prepare: ignore = iscrowd
                area.append(float(ann['area']))
                cnts.append(c)
                sizes.append(size)
                bboxes.append(rle_to_bbox(c, *size))
        self.gt_ng = np.asarray(ng, np.int64)
        self.gt_off = _starts(self.gt_ng)
        self.gt_id = np.asarray(ids, np.int64)
        self.gt_crowd = np.asarray(crowd, np.uint8)
        self.gt_area = np.asarray(area, np.float64)
        self.gt_size = np.asarray(sizes, np.int64).reshape(-1, 2)
        self.gt_bbox = np.asarray(bboxes, np.float64).reshape(-1, 4)
        self.gt_starts = _starts([len(c) for c in cnts])
        dev = self.device
        self._gt_cnts = _dev_tensor(np.concatenate(cnts) if cnts else np.zeros(1, np.int64), torch.int32, dev)
        self._gt_starts = _dev_tensor(self.gt_starts, torch.int64, dev)
        self._gt_crowd = _dev_tensor(self.gt_crowd if ids else np.zeros(1, np.uint8), torch.uint8, dev)
        self._thr = _dev_tensor(IOU_THRS, torch.float64, dev)
        self._rng = _dev_tensor(self.area_rng, torch.float64, dev)
        self.reset()

    def reset(self):
        self._batches = []
        self._seen = set()
        self._next_id = 1

    # ---- detections
    def add_batch(self, labels, scores, image_ids, counts=None):
        """labels (N, L, H, W) int32 cuda (label maps per layer, 0 = background); scores (N * L, kcap) float64 cuda,
        entry [n * L + l, j] = score of label j + 1 of layer l of image n (MaskPostprocessor.run_device /
        postprocessing.scores_strided); counts (N * L,) int32 cuda = labels per plane (derived when None)."""
        assert labels.is_cuda and labels.dtype == torch.int32 and labels.dim() == 4
        n, nl, h, w = labels.shape
        if len(image_ids) != n:
            raise ValueError("add_batch: %d label maps for %d image ids" % (n, len(image_ids)))
        planes = labels.reshape(n * nl, h, w).contiguous()
        if counts is None:
            counts = planes.reshape(n * nl, -1).amax(dim=1).to(torch.int32)
        cnts, starts, spans, geo = rle_encode_instances(planes, counts.to(torch.int32).contiguous())
        total = int(geo["counts"].sum())
        plane = geo["plane"].astype(np.int64)
        local = np.arange(total, dtype=np.int64) - np.repeat(geo["offsets"].astype(np.int64), geo["counts"])
        kcap = scores.shape[-1]
        if total and int(local.max()) >= kcap:
            raise ValueError("add_batch: a plane has more labels than the score table's %d columns" % kcap)
        sc = scores.reshape(-1)[_dev_tensor(plane * kcap + local, torch.int64, self.device)].cpu().numpy() \
            if total else np.zeros(0)
        # rleToBbox: x = first column, width = columns spanned; rows likewise unless a run of ones crosses a column
        x0 = geo["cmin"].astype(np.float64)
        bw = (geo["cmax"] - geo["cmin"] + 1).astype(np.float64)
        y0 = np.where(spans, 0, geo["rmin"]).astype(np.float64)
        bh = np.where(spans, h, geo["rmax"] - geo["rmin"] + 1).astype(np.float64)
        bbox = np.stack([x0, y0, bw, bh], axis=1)
        layer_inds = np.cumsum(self.category_layers)
        layer_cat = [self.layer_category_ids[int(np.searchsorted(layer_inds, li, side='right'))] for li in range(nl)]
        img_of = np.asarray([int(i) for i in image_ids], np.int64)[plane // nl]
        cat_of = np.asarray([layer_cat[li] if layer_cat[li] is not None else -1 for li in range(nl)], np.int64)[plane % nl]
        emitted = np.asarray([c is not None for c in layer_cat], bool)[plane % nl]
        # the reference's results carry a bbox, so COCO.loadRes takes its bbox branch: area = w * h of the box
        self._add(img_of[emitted], cat_of[emitted], sc[emitted], cnts, starts, np.flatnonzero(emitted),
                  (bbox[:, 2] * bbox[:, 3])[emitted], bbox[emitted], np.tile([h, w], (int(emitted.sum()), 1)),
                  image_ids)

    def _add(self, img, cat, score, cnts, starts, rle_index, area, bbox, size, batch_image_ids):
        """detections in result-file order: image / category ids, score, run list cnts[starts[r]:starts[r + 1]] with
        r = rle_index[j], area (what loadRes sets), rleToBbox box, mask size (h, w)"""
        for i in batch_image_ids:
            if int(i) in self._seen:
                raise ValueError("image %d was added twice" % int(i))
            self._seen.add(int(i))
        nres = len(img)
        det_id = np.arange(self._next_id, self._next_id + nres, dtype=np.int64)   # loadRes: id = index + 1
        self._next_id += nres
        I = len(self.img_ids)
        iu = np.asarray([self._img_index.get(int(i), -1) for i in img], np.int64)
        ku = np.asarray([self._cat_index.get(int(c), -1) for c in cat], np.int64)
        keep = (iu >= 0) & (ku >= 0)
        unit = (ku * I + iu)[keep]
        sel = np.flatnonzero(keep)
        # computeIoU / evaluateImg: stable mergesort by descending score inside each unit, cut to maxDets[-1]
        order = sel[np.lexsort((-np.asarray(score, np.float64)[sel], unit))]
        unit_sorted = (ku * I + iu)[order]
        first = np.searchsorted(unit_sorted, unit_sorted, side='left')
        rank = np.arange(order.size) - first
        order = order[rank < MAX_DETS[-1]]
        units_all = np.asarray(sorted(set(int(i) for i in
                                          [self._img_index[int(x)] for x in batch_image_ids
                                           if int(x) in self._img_index])), np.int64)
        batch_units = (np.arange(len(self.cat_ids))[:, None] * I + units_all[None, :]).reshape(-1)
        batch_units.sort()
        d_unit = (ku * I + iu)[order]
        nd = np.bincount(np.searchsorted(batch_units, d_unit), minlength=batch_units.size).astype(np.int64)
        ng = self.gt_ng[batch_units]
        dt_off = _starts(nd)
        self._batches.append(self._run(batch_units, nd, ng, dt_off, order, score, det_id, area, bbox, size, cnts,
                                       starts, rle_index))

    def _run(self, units, nd, ng, dt_off, order, score, det_id, area, bbox, size, cnts, starts, rle_index):
        """the two kernels for one set of units; returns host bookkeeping plus the device tables"""
        dev = self.device
        A, T = len(self.area_rng), len(IOU_THRS)
        npair = nd * ng
        iou_off = _starts(npair)
        n_tab = int(iou_off[-1])
        d_total, g_total = int(dt_off[-1]), int(ng.sum())
        g_glob = np.concatenate([np.arange(self.gt_off[u], self.gt_off[u + 1]) for u in units]) \
            if units.size else np.zeros(0, np.int64)
        # every entry of every unit's D x G table, then the bounding-box gate
        pu = np.repeat(np.arange(units.size), npair)
        loc = np.arange(n_tab, dtype=np.int64) - np.repeat(iou_off[:-1], npair)
        ngp = np.maximum(ng[pu], 1)
        pd_batch = dt_off[pu] + loc // ngp                    # detection (score order) within the batch
        g_local = _starts(ng)[pu] + loc % ngp                  # ground truth within the batch
        pg = g_glob[g_local]
        det = order[pd_batch]
        gate = np.zeros(n_tab, bool)
        if n_tab:
            db, gb = bbox[det], self.gt_bbox[pg]
            w = np.minimum(db[:, 2] + db[:, 0], gb[:, 2] + gb[:, 0]) - np.maximum(db[:, 0], gb[:, 0])
            h = np.minimum(db[:, 3] + db[:, 1], gb[:, 3] + gb[:, 1]) - np.maximum(db[:, 1], gb[:, 1])
            gate = (w > 0) & (h > 0)
            if (gate & np.any(size[det] != self.gt_size[pg], axis=1)).any():
                raise ValueError("a detection and a ground truth of one image have different mask sizes")
        iou = torch.empty(max(n_tab, 1), dtype=torch.float64, device=dev)
        L.zero(iou)
        sel = np.flatnonzero(gate)
        if sel.size:
            dt_cnts = _dev_tensor(cnts.view(np.int32) if cnts.dtype == np.uint32 else cnts, torch.int32, dev)
            dt_starts = _dev_tensor(starts, torch.int64, dev)
            p_dt = _dev_tensor(rle_index[det[sel]], torch.int32, dev)
            p_gt = _dev_tensor(pg[sel], torch.int32, dev)
            p_out = _dev_tensor(sel, torch.int64, dev)
            L.fcall("mcb_rle_pair_iou", dt_cnts.data_ptr(), dt_starts.data_ptr(), self._gt_cnts.data_ptr(),
                    self._gt_starts.data_ptr(), self._gt_crowd.data_ptr(), p_dt.data_ptr(), p_gt.data_ptr(),
                    p_out.data_ptr(), iou.data_ptr(), int(sel.size))
        d_ids = det_id[order] if d_total else np.zeros(1, np.int64)
        d_area = np.asarray(area, np.float64)[order] if d_total else np.zeros(1)
        g_src = g_glob if g_total else np.zeros(1, np.int64)
        t = {k: _dev_tensor(v, dt, dev) for k, (v, dt) in {
            "iou_off": (iou_off[:-1] if units.size else np.zeros(1, np.int64), torch.int64),
            "nd": (nd if units.size else np.zeros(1), torch.int32), "ng": (ng if units.size else np.zeros(1), torch.int32),
            "dt_off": (dt_off[:-1] if units.size else np.zeros(1, np.int64), torch.int64),
            "dt_id": (d_ids, torch.int64), "dt_area": (d_area, torch.float64),
            "gt_off": (_starts(ng)[:-1] if units.size else np.zeros(1, np.int64), torch.int64),
            "gt_id": (self.gt_id[g_src] if g_total else np.zeros(1, np.int64), torch.int64),
            "gt_crowd": (self.gt_crowd[g_src] if g_total else np.zeros(1, np.uint8), torch.uint8),
            "gt_area": (self.gt_area[g_src] if g_total else np.zeros(1), torch.float64)}.items()}
        dt_match = torch.empty((A, T, max(d_total, 1)), dtype=torch.int64, device=dev)
        dt_ignore = torch.empty((A, T, max(d_total, 1)), dtype=torch.uint8, device=dev)
        gt_ignore = torch.empty((A, max(g_total, 1)), dtype=torch.uint8, device=dev)
        taken = torch.empty((A, T, max(g_total, 1)), dtype=torch.uint8, device=dev)
        L.zero(taken)
        L.fcall("mcb_coco_match", iou.data_ptr(), t["iou_off"].data_ptr(), t["nd"].data_ptr(), t["ng"].data_ptr(),
                t["dt_off"].data_ptr(), t["dt_id"].data_ptr(), t["dt_area"].data_ptr(), t["gt_off"].data_ptr(),
                t["gt_id"].data_ptr(), t["gt_crowd"].data_ptr(), t["gt_area"].data_ptr(), self._rng.data_ptr(),
                self._thr.data_ptr(), int(units.size), A, T, d_total, g_total, dt_match.data_ptr(),
                dt_ignore.data_ptr(), gt_ignore.data_ptr(), taken.data_ptr())
        return {"units": units, "nd": nd, "ng": ng, "scores": np.asarray(score, np.float64)[order],
                "iou": iou[:n_tab], "iou_off": iou_off, "dt_match": dt_match[:, :, :d_total],
                "dt_ignore": dt_ignore[:, :, :d_total], "gt_ignore": gt_ignore[:, :g_total]}

    # ---- result
    def tables(self):
        """per-unit tables of every unit, in unit order (unit u = k * len(image_ids) + i), on the host:
        dict nd, ng, present, dt_scores, dt_match, dt_ignore, gt_ignore (accumulate's inputs) plus iou / iou_off"""
        covered = np.zeros(self.n_units, bool)
        for b in self._batches:
            covered[b["units"]] = True
        rest = np.flatnonzero(~covered)
        batches = list(self._batches)
        if rest.size:       # units never added: no detections, their ground truths still count
            empty = np.zeros(0, np.int64)
            nd = np.zeros(rest.size, np.int64)
            batches.append(self._run(rest, nd, self.gt_ng[rest], _starts(nd), empty, np.zeros(0), empty,
                                     np.zeros(0), np.zeros((0, 4)), np.zeros((0, 2), np.int64),
                                     np.zeros(1, np.int32), np.zeros(1, np.int64), empty))
        units = np.concatenate([b["units"] for b in batches])
        nd = np.concatenate([b["nd"] for b in batches])
        ng = np.concatenate([b["ng"] for b in batches])
        dm = torch.cat([b["dt_match"] for b in batches], dim=2).cpu().numpy()
        di = torch.cat([b["dt_ignore"] for b in batches], dim=2).cpu().numpy()
        gi = torch.cat([b["gt_ignore"] for b in batches], dim=1).cpu().numpy()
        iou = torch.cat([b["iou"] for b in batches]).cpu().numpy()
        scores = np.concatenate([b["scores"] for b in batches])
        # batch order -> unit order
        pos = np.empty(self.n_units, np.int64)
        pos[units] = np.arange(units.size)
        doff, goff, toff = _starts(nd), _starts(ng), _starts(nd * ng)
        d_idx = np.concatenate([np.arange(doff[p], doff[p + 1]) for p in pos]) if nd.sum() else np.zeros(0, np.int64)
        g_idx = np.concatenate([np.arange(goff[p], goff[p + 1]) for p in pos]) if ng.sum() else np.zeros(0, np.int64)
        t_idx = np.concatenate([np.arange(toff[p], toff[p + 1]) for p in pos]) if toff[-1] else np.zeros(0, np.int64)
        nd_u, ng_u = nd[pos], ng[pos]
        return {"nd": nd_u, "ng": ng_u, "present": (nd_u + ng_u) > 0, "dt_scores": scores[d_idx],
                "dt_match": dm[:, :, d_idx], "dt_ignore": di[:, :, d_idx], "gt_ignore": gi[:, g_idx],
                "iou": iou[t_idx], "iou_off": _starts(nd_u * ng_u)}

    def result(self):
        """-> dict precision [T,R,K,A,M], recall [T,K,A,M], stats (6,), ap_ar (stats[0], stats[3])"""
        tb = self.tables()
        precision, recall = accumulate(tb["nd"], tb["ng"], tb["present"], tb["dt_scores"], tb["dt_match"],
                                       tb["dt_ignore"], tb["gt_ignore"], len(self.cat_ids), len(self.img_ids))
        stats = summarize(precision, recall)
        return {"precision": precision, "recall": recall, "stats": stats, "ap_ar": (stats[0], stats[3])}

    def add_results(self, anns):
        """detections as COCO result annotations (a `loadRes` list): every image they name counts as added"""
        if not anns:
            return
        bbox_branch = 'bbox' in anns[0] and not anns[0]['bbox'] == []
        cnts, sizes, areas, bboxes = [], [], [], []
        for ann in anns:
            h, w = self.image_sizes.get(int(ann['image_id']), (None, None))
            if 'segmentation' not in ann:
                raise NotImplementedError("results without a segmentation (box-only) are not evaluated as masks")
            c, size = segmentation_counts(ann['segmentation'], h, w)
            cnts.append(c)
            sizes.append(size)
            box = rle_to_bbox(c, *size)
            bboxes.append(box)
            # COCO.loadRes: with a bbox on the first result, area = w * h of each result's bbox; else the RLE area
            areas.append(ann['bbox'][2] * ann['bbox'][3] if bbox_branch else _rle_area(c))
        starts = _starts([len(c) for c in cnts])
        self._add(np.asarray([a['image_id'] for a in anns], np.int64),
                  np.asarray([a['category_id'] for a in anns], np.int64),
                  np.asarray([a['score'] for a in anns], np.float64),
                  np.concatenate(cnts).astype(np.int64), starts, np.arange(len(anns)), np.asarray(areas, np.float64),
                  np.asarray(bboxes, np.float64), np.asarray(sizes, np.int64),
                  sorted(set(int(a['image_id']) for a in anns)))


def coco_evaluation(gt_filepath, prediction_filepath, image_ids, category_ids, small_annotations_size):
    """src/utils.py:308-321 -> (stats[0], stats[3]): AP and AR at IoU 0.5, all areas, 100 detections"""
    with open(prediction_filepath) as f:
        anns = json.load(f)
    ev = DeviceCOCOEvaluator(gt_filepath, image_ids, category_ids, small_annotations_size)
    ev.add_results(anns)
    res = ev.result()
    return res["stats"][0], res["stats"][3]
