"""TEST INFRASTRUCTURE — a pycocotools stand-in and a numpy restatement of the vendored COCOeval (src/cocoeval.py).

pycocotools is not installed here.  `mask` restates the RLE functions of its C core (common/maskApi.c, published with
cocodataset/cocoapi) that the evaluation calls: rleEncode (vectorised, pinned against instances_oracle.rle_encode),
rleDecode, rleArea, rleToBbox, rleFrString / rleToString (instances_oracle), and rleIou with its bounding-box gate
bbIou.  The mask IoU here decodes both masks and counts pixels (an independent route from the run-list walk of
csrc/evaluation.cu).  `COCO` restates createIndex, getImgIds, getCatIds, getAnnIds, loadAnns, loadRes and annToRLE
for RLE segmentations (polygons raise).  All of it is pinned by hand-derived vectors in tests/test_evaluation_cpu.py.

`COCOevalOracle` restates COCOeval.evaluate / accumulate / summarize (src/cocoeval.py:128-494) loop for loop, so that
tests on a machine without the reference have an oracle of the whole evaluation.

oracle/make_golden_cocoeval.py runs the unmodified reference on top of this stand-in.  The vendored cocoeval.py does not run on numpy 2 as written: it uses `np.float` and passes a
float `num` to `np.linspace`; the generator bridges both (np.float = float, linspace with int(num)) for the duration of
its run only.
"""
import copy
import json
import types
from collections import defaultdict

import numpy as np

from . import instances_oracle as I


# ---------------------------------------------------------------------------------------------------------------------
# pycocotools.mask
# ---------------------------------------------------------------------------------------------------------------------
def rle_encode(mask):
    """rleEncode of one (h, w) mask, column-major, run lengths alternating from zeros"""
    flat = (np.asarray(mask) != 0).ravel(order="F")
    if flat.size == 0:
        return [0]
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    cnts = np.diff(np.concatenate([[0], change, [flat.size]]))
    if flat[0]:
        cnts = np.concatenate([[0], cnts])
    return [int(c) for c in cnts]


def _counts(rle):
    c = rle["counts"]
    return list(c) if isinstance(c, list) else I.rle_from_string(c)


def decode_flat(rle):
    """rleDecode -> column-major flat bool mask"""
    c = np.asarray(_counts(rle), dtype=np.int64)
    return np.repeat((np.arange(c.size) % 2).astype(bool), c)


def encode(bimask):
    """one (h, w) mask -> RLE dict with compressed counts"""
    m = np.asarray(bimask)
    return {"size": [m.shape[0], m.shape[1]], "counts": I.rle_to_string(rle_encode(m))}


def decode(rle):
    h, w = rle["size"]
    return decode_flat(rle).reshape((h, w), order="F").astype(np.uint8)


def area(rle):
    return int(np.asarray(_counts(rle), dtype=np.int64)[1::2].sum())


def toBbox(rle):
    if isinstance(rle, list):
        return np.array([toBbox(r) for r in rle]).reshape(-1, 4)
    return np.array(I.rle_to_bbox(_counts(rle), rle["size"][0], rle["size"][1]))


def frPyObjects(pyobj, h, w):
    """one RLE dict: uncompressed counts (a list) become compressed ones; polygons and boxes are not restated"""
    if not (isinstance(pyobj, dict) and "counts" in pyobj and "size" in pyobj):
        raise NotImplementedError("only RLE input is restated")
    if isinstance(pyobj["counts"], list):
        return {"size": list(pyobj["size"]), "counts": I.rle_to_string(pyobj["counts"])}
    return pyobj


def bb_gate_iou(db, gb, iscrowd):
    """bbIou: (m, 4) x (n, 4) [x, y, w, h] -> (m, n)"""
    out = np.zeros((len(db), len(gb)))
    for g in range(len(gb)):
        G = gb[g]
        ga = G[2] * G[3]
        for d in range(len(db)):
            D = db[d]
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            out[d, g] = i / (da if iscrowd[g] else da + ga - i)
    return out


def iou(dt, gt, iscrowd):
    """rleIou as maskUtils.iou(d, g, iscrowd) returns it: (m, n) fp64, [] when either list is empty.  Pairs whose
    boxes do not overlap get 0; integer intersection i and union u (u = detection area for a crowd ground truth),
    o = i / u, 0 when i == 0; -1 where the mask sizes differ."""
    if len(dt) == 0 or len(gt) == 0:
        return []
    iscrowd = [int(c) for c in iscrowd]
    o = bb_gate_iou(toBbox(dt), toBbox(gt), iscrowd)
    dm = [decode_flat(d) for d in dt]
    gm = [decode_flat(g) for g in gt]
    rows, cols = np.nonzero(o > 0)
    if rows.size == 0:
        return o
    dmat = np.stack([m.astype(np.float32) for m in dm]) if len({m.size for m in dm}) == 1 else None
    gmat = np.stack([m.astype(np.float32) for m in gm]) if len({m.size for m in gm}) == 1 else None
    inter = dmat @ gmat.T if dmat is not None and gmat is not None and dmat.shape[1] == gmat.shape[1] else None
    for d, g in zip(rows, cols):
        if list(dt[d]["size"]) != list(gt[g]["size"]):
            o[d, g] = -1
            continue
        i = int(inter[d, g]) if inter is not None else int(np.count_nonzero(dm[d] & gm[g]))   # exact: < 2**24
        da, ga = int(dm[d].sum()), int(gm[g].sum())
        if i == 0:
            u = 1
        elif iscrowd[g]:
            u = da
        else:
            u = da + ga - i
        o[d, g] = i / u
    return o


mask = types.SimpleNamespace(encode=encode, decode=decode, area=area, toBbox=toBbox, frPyObjects=frPyObjects, iou=iou)


# ---------------------------------------------------------------------------------------------------------------------
# pycocotools.coco
# ---------------------------------------------------------------------------------------------------------------------
def _is_array_like(obj):
    return hasattr(obj, '__iter__') and hasattr(obj, '__len__')


class COCO:
    def __init__(self, annotation_file=None):
        self.dataset, self.anns, self.imgs, self.imgToAnns = {}, {}, {}, defaultdict(list)
        if annotation_file is not None:
            with open(annotation_file) as f:
                self.dataset = json.load(f)
            self.createIndex()

    def createIndex(self):
        """anns, imgs and imgToAnns (file order per image); the category indexes are not used by COCOeval"""
        self.anns, self.imgs, self.imgToAnns = {}, {}, defaultdict(list)
        for ann in self.dataset.get('annotations', []):
            self.imgToAnns[ann['image_id']].append(ann)
            self.anns[ann['id']] = ann
        for img in self.dataset.get('images', []):
            self.imgs[img['id']] = img

    def getAnnIds(self, imgIds=[], catIds=[], areaRng=[], iscrowd=None):
        imgIds = imgIds if _is_array_like(imgIds) else [imgIds]
        catIds = catIds if _is_array_like(catIds) else [catIds]
        if len(imgIds) == len(catIds) == len(areaRng) == 0:
            anns = self.dataset['annotations']
        else:
            if not len(imgIds) == 0:
                lists = [self.imgToAnns[imgId] for imgId in imgIds if imgId in self.imgToAnns]
                anns = [a for lst in lists for a in lst]
            else:
                anns = self.dataset['annotations']
            anns = anns if len(catIds) == 0 else [ann for ann in anns if ann['category_id'] in catIds]
            anns = anns if len(areaRng) == 0 else [ann for ann in anns if areaRng[0] < ann['area'] < areaRng[1]]
        if iscrowd is not None:
            return [ann['id'] for ann in anns if ann['iscrowd'] == iscrowd]
        return [ann['id'] for ann in anns]

    def getCatIds(self):
        return [cat['id'] for cat in self.dataset.get('categories', [])]

    def getImgIds(self):
        return list(self.imgs.keys())

    def loadAnns(self, ids=[]):
        return [self.anns[i] for i in ids] if _is_array_like(ids) else [self.anns[ids]]

    def loadRes(self, resFile):
        res = COCO()
        res.dataset['images'] = [img for img in self.dataset['images']]
        if isinstance(resFile, str):
            with open(resFile) as f:
                resFile = json.load(f)
        anns = resFile
        annsImgIds = [ann['image_id'] for ann in anns]
        assert set(annsImgIds) == (set(annsImgIds) & set(self.getImgIds())), \
            'Results do not correspond to current coco set'
        # the bbox branch comes first: with a box on the first result, area = w * h of each result's box
        bbox_branch = 'bbox' in anns[0] and not anns[0]['bbox'] == []
        if not all('segmentation' in ann for ann in anns):
            raise NotImplementedError("box-only, caption and keypoint results are not restated")
        res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
        for id, ann in enumerate(anns):
            if bbox_branch:
                ann['area'] = ann['bbox'][2] * ann['bbox'][3]
            else:
                ann['area'] = area(ann['segmentation'])
                ann.setdefault('bbox', toBbox(ann['segmentation']))
            ann['id'] = id + 1
            ann['iscrowd'] = 0
        res.dataset['annotations'] = anns
        res.createIndex()
        return res

    def annToRLE(self, ann):
        t = self.imgs[ann['image_id']]
        return frPyObjects(ann['segmentation'], t['height'], t['width'])   # polygons raise there


# ---------------------------------------------------------------------------------------------------------------------
# COCOeval (iouType 'segm', useCats 1), loop for loop
# ---------------------------------------------------------------------------------------------------------------------
IOU_THRS = np.linspace(.5, 0.95, 10, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, 101, endpoint=True)


class COCOevalOracle:
    def __init__(self, cocoGt, cocoDt, imgIds, catIds, small_annotations_size=14):
        s = small_annotations_size
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.imgIds = list(np.unique(imgIds))
        self.catIds = list(np.unique(catIds))
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, s ** 2], [s ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'small', 'large']
        self.maxDets = [1, 10, 100]
        self.iouThrs, self.recThrs = IOU_THRS, REC_THRS

    def evaluate(self):
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=self.imgIds, catIds=self.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=self.imgIds, catIds=self.catIds))
        for ann in gts:
            ann['segmentation'] = self.cocoGt.annToRLE(ann)
        for ann in dts:
            ann['segmentation'] = self.cocoDt.annToRLE(ann)
        for gt in gts:
            gt['ignore'] = 'iscrowd' in gt and gt['iscrowd']
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        for gt in gts:
            self._gts[gt['image_id'], gt['category_id']].append(gt)
        for dt in dts:
            self._dts[dt['image_id'], dt['category_id']].append(dt)
        self.ious = {(i, c): self.computeIoU(i, c) for i in self.imgIds for c in self.catIds}
        self.evalImgs = [self.evaluateImg(i, c, a, self.maxDets[-1])
                         for c in self.catIds for a in self.areaRng for i in self.imgIds]

    def computeIoU(self, imgId, catId):
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds][:self.maxDets[-1]]
        return mask.iou([d['segmentation'] for d in dt], [g['segmentation'] for g in gt],
                        [int(o['iscrowd']) for o in gt])

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        gt, dt = self._gts[imgId, catId], self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g['_ignore'] = 1 if (g['ignore'] or g['area'] < aRng[0] or g['area'] > aRng[1]) else 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[imgId, catId]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(self.iouThrs), len(gt), len(dt)
        gtm, dtm, dtIg = np.zeros((T, G)), np.zeros((T, D)), np.zeros((T, D))
        gtIg = np.array([g['_ignore'] for g in gt])
        if not len(ious) == 0:
            for tind, t in enumerate(self.iouThrs):
                for dind, d in enumerate(dt):
                    best, m = min([t, 1 - 1e-10]), -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < best:
                            continue
                        best, m = ious[dind, gind], gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < aRng[0] or d['area'] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'image_id': imgId, 'category_id': catId, 'aRng': aRng, 'maxDet': maxDet,
                'dtIds': [d['id'] for d in dt], 'gtIds': [g['id'] for g in gt], 'dtMatches': dtm, 'gtMatches': gtm,
                'dtScores': [d['score'] for d in dt], 'gtIgnore': gtIg, 'dtIgnore': dtIg}

    def accumulate(self):
        T, R, K, A, M = len(self.iouThrs), len(self.recThrs), len(self.catIds), len(self.areaRng), len(self.maxDets)
        precision, recall = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M))
        I0, A0 = len(self.imgIds), len(self.areaRng)
        for k in range(K):
            for a in range(A):
                for m, maxDet in enumerate(self.maxDets):
                    E = [self.evalImgs[k * A0 * I0 + a * I0 + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind='mergesort')
                    dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        for ri, pi in enumerate(np.searchsorted(rc, self.recThrs, side='left')):
                            if pi >= nd:
                                break
                            q[ri] = pr[pi]
                        precision[t, :, k, a, m] = np.array(q)
        self.precision, self.recall = precision, recall

    def summarize(self):
        def _summarize(ap, iouThr, areaRng='all', maxDets=100):
            aind = [i for i, r in enumerate(self.areaRngLbl) if r == areaRng]
            mind = [i for i, d in enumerate(self.maxDets) if d == maxDets]
            t = np.where(iouThr == self.iouThrs)[0]
            s = self.precision[t][:, :, :, aind, mind] if ap == 1 else self.recall[t][:, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        md = self.maxDets[2]
        self.stats = np.array([_summarize(1, .5, maxDets=md), _summarize(1, .5, 'small', md),
                               _summarize(1, .5, 'large', md), _summarize(0, .5, maxDets=md),
                               _summarize(0, .5, 'small', md), _summarize(0, .5, 'large', md)], dtype=np.float64)


def flat_tables(ev):
    """an evaluated COCOevalOracle (or the reference's COCOeval) -> the flat per-unit tables of
    mcb200.evaluation.accumulate, plus the IoU tables (unit order, each row-major [D][G] in computeIoU's order)"""
    imgIds, catIds = list(np.unique(ev.params.imgIds if hasattr(ev, 'params') else ev.imgIds)), \
        list(np.unique(ev.params.catIds if hasattr(ev, 'params') else ev.catIds))
    A = len(ev.params.areaRng if hasattr(ev, 'params') else ev.areaRng)
    I0, K = len(imgIds), len(catIds)
    nd, ng, present, scores, dm, di, gi, ious, dids = [], [], [], [], [], [], [], [], []
    for k in range(K):
        for i in range(I0):
            e0 = ev.evalImgs[k * A * I0 + i]
            iou = ev.ious[imgIds[i], catIds[k]]
            present.append(e0 is not None)
            if e0 is None:
                nd.append(0)
                ng.append(0)
                continue
            nd.append(len(e0['dtIds']))
            ng.append(len(e0['gtIds']))
            scores.extend(e0['dtScores'])
            dids.extend(e0['dtIds'])
            ious.append(np.asarray(iou, np.float64).reshape(-1) if len(iou) else np.zeros(0))
            dm.append(np.stack([ev.evalImgs[k * A * I0 + a * I0 + i]['dtMatches'] for a in range(A)]))
            di.append(np.stack([ev.evalImgs[k * A * I0 + a * I0 + i]['dtIgnore'] for a in range(A)]))
            gi.append(np.stack([ev.evalImgs[k * A * I0 + a * I0 + i]['gtIgnore'] for a in range(A)]))
    T = 10
    cat = lambda xs, shape: np.concatenate(xs, axis=-1) if xs else np.zeros(shape)  # noqa: E731
    return {"nd": np.asarray(nd, np.int64), "ng": np.asarray(ng, np.int64), "present": np.asarray(present, bool),
            "dt_scores": np.asarray(scores, np.float64), "dt_ids": np.asarray(dids, np.int64),
            "dt_match": cat(dm, (A, T, 0)).astype(np.int64), "dt_ignore": cat(di, (A, T, 0)).astype(np.uint8),
            "gt_ignore": cat([g.reshape(A, -1) for g in gi], (A, 0)).astype(np.uint8),
            "iou": np.concatenate(ious) if ious else np.zeros(0)}
