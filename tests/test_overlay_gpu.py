"""The target preparation on the device (csrc/polygon.cu, mcb200.preparation, mcb200.evaluation.ground_truth_rle)
against oracle/overlay_oracle.py and the unmodified reference (tests/golden/overlay.npz), bit for bit."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import coco_oracle as CO
from oracle import input_oracle as IO
from oracle import make_golden_overlay as MG
from oracle import overlay_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "overlay.npz")


def _random_polygons(rs, n, h, w):
    polys = []
    for i in range(n):
        r = rs.rand()
        if r < 0.05:                                              # far outside: long edge walks
            polys.append(list(rs.uniform(-3000, 3000, 2 * rs.randint(3, 7))))
        elif r < 0.1:
            polys.append([round(float(v)) for v in rs.uniform(-5, max(h, w) + 5, 2 * rs.randint(2, 6))])
        elif r < 0.13:
            p = O.building_polygon(rs, h, w)
            polys.append(p[:2] + p + p[-2:])                      # repeated vertices
        elif r < 0.15:
            x0, y0, dx, dy = rs.uniform(0, w), rs.uniform(0, h), rs.uniform(-9, 9), rs.uniform(-9, 9)
            polys.append([x0, y0, x0 + dx, y0 + dy, x0 + 2 * dx, y0 + 2 * dy])   # collinear
        else:
            polys.append(O.building_polygon(rs, h, w))
    return polys


@pytest.mark.parametrize("h,w,n", [(300, 300, 3000), (37, 61, 1200), (64, 23, 1200)])
def test_rasterize_polygons_equals_the_oracle(mcb, cuda, h, w, n):
    from mcb200.preparation import polygons_csr, rasterize_polygons
    rs = np.random.RandomState(h * 1000 + w)
    polys = _random_polygons(rs, n, h, w)
    got = rasterize_polygons(*polygons_csr(polys), h, w).cpu().numpy()
    for i, p in enumerate(polys):
        want = O.polygon_mask(p, h, w)
        assert np.array_equal(got[i], want), (i, p)
    assert got.any(axis=(1, 2)).sum() > n // 2


def test_binary_morphology_equals_scipy_at_every_size(mcb, cuda):
    from mcb200 import _lib as L
    rs = np.random.RandomState(5)
    planes = (rs.rand(6, 37, 53) < 0.6).astype(np.uint8)
    planes[2] = 1                                               # all ones: the erosion's border_value=True
    planes[3] = 0
    x = torch.from_numpy(planes).to(cuda)
    for size in range(1, 7):
        for dil in (0, 1):
            out = torch.empty_like(x)
            L.fcall("mcb_binary_morph_rect", x.data_ptr(), out.data_ptr(), dil, size, 6, 37, 53)
            op = O.binary_dilation if dil else O.binary_erosion
            want = np.stack([op(p, O.rectangle(size, size)).astype(np.uint8) for p in planes])
            assert np.array_equal(out.cpu().numpy(), want), (size, dil)


def test_two_nearest_distances_of_an_empty_instance_is_scipys(mcb, cuda):
    from mcb200.preparation import two_nearest_distances
    m = np.zeros((3, 29, 41), np.uint8)
    m[0, 5:9, 7:20] = 1
    m[2, 20:22, 30:33] = 1
    for planes in (m, m[1:2], m[1:]):
        got_sum, got_second = two_nearest_distances(planes)
        want_sum, want_second = IO.two_nearest_distances(planes)
        assert np.array_equal(got_sum, want_sum) and np.array_equal(got_second, want_second)


def _golden(g, c):
    d = json.loads(g["json_%d" % c].tobytes().decode())
    by_img = {}
    for a in d["annotations"]:
        by_img.setdefault(a["image_id"], []).append(a)
    return d, by_img


@pytest.mark.parametrize("c", range(len(MG.CONFIGS)))
def test_overlay_batch_equals_the_reference(mcb, cuda, c):
    from mcb200.preparation import overlay_batch
    g = np.load(GOLDEN)
    erode, dilate, border = MG.CONFIGS[c]
    d, by_img = _golden(g, c)
    groups = {}
    for i, im in enumerate(d["images"]):
        groups.setdefault((im["height"], im["width"]), []).append(i)
    for (h, w), idx in groups.items():
        mask, dist, sizes, ones_u8 = overlay_batch([by_img.get(d["images"][i]["id"], []) for i in idx], h, w,
                                                   (None, 100), erode, dilate, border, MG.SMALL)
        mask, dist, sizes = mask.cpu().numpy(), dist.cpu().numpy(), sizes.cpu().numpy()
        for j, i in enumerate(idx):
            want_sizes = g["c%d_i%d_sizes" % (c, i)]
            assert np.array_equal(mask[j], g["c%d_i%d_mask" % (c, i)]), (c, i)
            assert np.array_equal(dist[j], g["c%d_i%d_dist" % (c, i)]), (c, i)
            assert ones_u8[j] == (want_sizes.dtype == np.uint8) and np.array_equal(sizes[j], want_sizes), (c, i)


def _scale_images(seed, n, h=300, w=300, multi_polygon=True):
    rs = np.random.RandomState(seed)
    return [O.synthetic_image_annotations(rs, h, w, rs.randint(10, 41), i, 100 * i, multi_polygon) for i in range(n)]


@pytest.mark.parametrize("erode,dilate,border,n", [(0, 0, 0, 256), (3, 2, 3, 256), (2, 0, 0, 48), (4, 4, 1, 48)])
def test_overlay_batch_at_scale_equals_the_oracle(mcb, cuda, erode, dilate, border, n):
    from mcb200.preparation import overlay_batch
    images = _scale_images(7 + erode, n, multi_polygon=erode == 0)
    if erode:
        assert sum(O.eroded_to_empty(a, 300, 300, erode) for a in images) > 0
    mask, dist, sizes, ones_u8 = overlay_batch(images, 300, 300, (None, 100), erode, dilate, border, 14)
    mask, dist, sizes = mask.cpu().numpy(), dist.cpu().numpy(), sizes.cpu().numpy()
    for i, anns in enumerate(images):
        wm, wd, ws = O.overlay_mask_one_image(anns, 300, 300, (None, 100), erode, dilate, border, 14)
        assert np.array_equal(mask[i], wm) and np.array_equal(dist[i], wd), i
        assert ones_u8[i] == (ws.dtype == np.uint8) and np.array_equal(sizes[i], ws), i


def test_overlay_masks_files_feed_the_loaders(mcb, cuda, tmp_path):
    from mcb200.loaders import SegmentationFiles
    from mcb200.preparation import overlay_masks, target_batch
    from PIL import Image
    rs = np.random.RandomState(3)
    images, anns = [], []
    shapes = [(300, 300)] * 5 + [(40, 56)] * 3
    for i, (h, w) in enumerate(shapes):
        images.append({"id": 50 + i, "file_name": "tile_%02d.jpg" % i, "height": h, "width": w})
        if i != 1:
            anns += O.synthetic_image_annotations(rs, h, w, rs.randint(2, 20), 50 + i, 1000 * i)
    os.makedirs(tmp_path / "data" / "train")
    (tmp_path / "data" / "train" / "annotation-small.json").write_text(json.dumps({"images": images, "annotations": anns}))
    for im in images:
        Image.fromarray(np.zeros((im["height"], im["width"], 3), np.uint8)).save(tmp_path / im["file_name"])
    overlay_masks(str(tmp_path / "data"), "train", str(tmp_path / "out"), [None, 100], is_small=True, num_threads=3)
    for i, im in enumerate(images):
        stem = os.path.splitext(im["file_name"])[0]
        mask_path = str(tmp_path / "out" / "train" / "masks" / (stem + ".png"))
        assert Image.open(mask_path).mode == "L"
        _, m, dd, ss = SegmentationFiles([str(tmp_path / im["file_name"])], [mask_path], distances=True)[0]
        wm, wd, ws = O.overlay_mask_one_image([a for a in anns if a["image_id"] == im["id"]], im["height"], im["width"])
        assert np.array_equal(m, wm)
        import joblib
        assert joblib.load(mask_path.replace("/masks/", "/sizes/")[:-4]).dtype == ws.dtype
        got = target_batch(m[None], dd.view(np.uint16)[None].astype(np.float16), ss.view(np.uint16)[None] ** 2)
        want = IO.target(wm, wd, ws)
        assert np.array_equal(got[0].cpu().numpy(), want), i


def test_ground_truth_rle_feeds_the_evaluator_like_the_oracle(mcb, cuda, monkeypatch):
    from mcb200 import evaluation as E
    from mcb200.preparation import polygons_csr, rasterize_polygons
    n, size = 24, 300
    images = _scale_images(11, n)
    rs = np.random.RandomState(12)
    anns = []
    for i, im_anns in enumerate(images):
        for a in im_anns:
            anns.append(dict(a, id=len(anns) + 1, iscrowd=int(rs.rand() < 0.05)))
    gt = {"images": [{"id": i, "height": size, "width": size} for i in range(n)], "annotations": anns,
          "categories": [{"id": 100}]}
    conv = E.ground_truth_rle(gt)
    want_gt = json.loads(json.dumps(gt))
    for a in want_gt["annotations"]:
        a["segmentation"] = {"size": [size, size], "counts": O.ann_to_rle(a["segmentation"], size, size)}
    for a, b in zip(conv["annotations"], want_gt["annotations"]):
        assert np.array_equal(O.decode(a["segmentation"]["counts"], size, size),
                              O.decode(b["segmentation"]["counts"], size, size))
    assert gt["annotations"][0]["segmentation"] is not conv["annotations"][0]["segmentation"]
    # detections: every ground truth's own polygons, shifted, as label planes with scores
    labels = np.zeros((n, 2, size, size), np.int32)
    scores = np.zeros((2 * n, 64), np.float32)
    for i, im_anns in enumerate(images):
        k = 0
        for a in im_anns[:60]:
            m = O.polygon_mask(a["segmentation"][0], size, size)
            m = np.roll(m, (rs.randint(-2, 3), rs.randint(-2, 3)), axis=(0, 1)).astype(bool) & (labels[i, 1] == 0)
            if not m.any():
                continue
            k += 1
            labels[i, 1][m] = k
        scores[2 * i + 1, :k] = np.round(rs.rand(k), 3)
    ev = E.DeviceCOCOEvaluator(conv, np.arange(n), [100], 14)
    ev.add_batch(torch.from_numpy(labels).to(cuda), torch.from_numpy(scores).to(cuda), list(range(n)))
    res = ev.result()
    from oracle import instances_oracle as I
    monkeypatch.setattr(I, "rle_encode", CO.rle_encode)
    results = I.create_annotations(list(range(n)), [(labels[i], [[], [float(v) for v in scores[2 * i + 1, :labels[i, 1].max()]]])
                                                    for i in range(n)], [None, 100], [1, 1])
    c_gt = CO.COCO()
    c_gt.dataset = want_gt
    c_gt.createIndex()
    want = CO.COCOevalOracle(c_gt, c_gt.loadRes(json.loads(json.dumps(results))), np.arange(n), [100], 14)
    want.evaluate()
    want.accumulate()
    want.summarize()
    assert np.array_equal(res["stats"], want.stats) and 0 < res["stats"][0] < 1


def test_overlay_masks_bounds_the_batches_waiting_for_the_writers(mcb, cuda, tmp_path, monkeypatch):
    import time
    from mcb200 import preparation as P
    rs = np.random.RandomState(4)
    images = [{"id": i, "file_name": "t%02d.jpg" % i, "height": 40, "width": 56} for i in range(14)]
    anns = [a for i in range(14) for a in O.synthetic_image_annotations(rs, 40, 56, 3, i, 100 * i)]
    os.makedirs(tmp_path / "d" / "train")
    (tmp_path / "d" / "train" / "annotation.json").write_text(json.dumps({"images": images, "annotations": anns}))
    monkeypatch.setattr(P, "OVERLAY_CHUNK", 2)
    produced, written, ahead = [0], [0], []
    write, batch = P._write_targets, P.overlay_batch

    def slow_write(*a):
        time.sleep(0.05)
        write(*a)
        written[0] += 1

    def counted_batch(anns_per_image, *a):
        ahead.append(produced[0] - written[0])
        produced[0] += len(anns_per_image)
        return batch(anns_per_image, *a)
    monkeypatch.setattr(P, "_write_targets", slow_write)
    monkeypatch.setattr(P, "overlay_batch", counted_batch)
    P.overlay_masks(str(tmp_path / "d"), "train", str(tmp_path / "o"), [None, 100], num_threads=1)
    assert written[0] == 14 and len(ahead) == 7
    assert max(ahead) <= P.OVERLAY_IN_FLIGHT * P.OVERLAY_CHUNK
