"""COCO evaluation on the H100 (csrc/evaluation.cu through mcb200.evaluation / mcb200.callbacks) against the
reference's own output (tests/golden/cocoeval.npz) and, at scale and end to end, against oracle/coco_oracle.py's
COCOeval restatement.  Every comparison is exact."""
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import coco_oracle as CO
from oracle import instances_oracle as I
from oracle import post_oracle as P

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(GOLDEN, "cocoeval.npz")) as g:
        return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def golden_files(golden, tmp_path_factory):
    """the fixture's ground-truth and result JSON texts as files -> (gt path, dt path)"""
    d = tmp_path_factory.mktemp("cocoeval")
    for k in ("gt_json", "dt_json"):
        (d / (k + ".json")).write_bytes(golden[k].tobytes())
    return str(d / "gt_json.json"), str(d / "dt_json.json")


@pytest.fixture(scope="module")
def golden_tables(mcb, cuda, golden, golden_files):
    from mcb200 import evaluation as E
    ev = E.DeviceCOCOEvaluator(golden_files[0], golden["image_ids"], golden["category_ids"],
                               int(golden["small_annotations_size"]))
    ev.add_results(json.loads(golden["dt_json"].tobytes()))
    return ev, ev.tables()


def test_pair_iou_equals_the_golden_tables(golden_tables, golden):
    _, tb = golden_tables
    for k in ("nd", "ng", "present"):
        assert np.array_equal(tb[k], golden[k]), k
    assert tb["iou"].dtype == np.float64 and np.array_equal(tb["iou"], golden["iou"])
    assert (golden["iou"] > 0).sum() > 500 and ((golden["iou"] > 0) & (golden["iou"] < 1)).any()


def test_coco_match_equals_the_golden_tables(golden_tables, golden):
    _, tb = golden_tables
    assert np.array_equal(tb["dt_scores"], golden["dt_scores"])
    for k in ("dt_match", "dt_ignore", "gt_ignore"):
        assert np.array_equal(tb[k], golden[k]), k


def test_coco_evaluation_returns_the_golden_result(golden_tables, golden, golden_files):
    from mcb200 import evaluation as E
    res = golden_tables[0].result()
    assert np.array_equal(res["precision"], golden["precision"]) and np.array_equal(res["recall"], golden["recall"])
    assert np.array_equal(res["stats"], golden["stats"])
    ap_ar = E.coco_evaluation(golden_files[0], golden_files[1], golden["image_ids"], golden["category_ids"],
                              int(golden["small_annotations_size"]))
    assert ap_ar == tuple(golden["ap_ar"])


# ---------------------------------------------------------------------------------------------------------------------
# at scale: 1000 images, ~20 instances each, through add_batch
# ---------------------------------------------------------------------------------------------------------------------
def _scale_case(n_images=1000, size=300, seed=5):
    """label maps (n, 2, size, size) int32 (layer 0 empty), scores (n * 2, kcap), ground truth dict"""
    rs = np.random.RandomState(seed)
    labels = np.zeros((n_images, 2, size, size), np.int32)
    kcap = 32
    scores = np.zeros((n_images * 2, kcap))
    anns, next_id = [], 1
    for n in range(n_images):
        k = 0
        for q in range(rs.randint(15, 26)):
            h, w = rs.randint(6, 40), rs.randint(6, 40)
            y, x = rs.randint(0, size - h), rs.randint(0, size - w)
            if labels[n, 1, y:y + h, x:x + w].any():
                continue
            k += 1
            labels[n, 1, y:y + h, x:x + w] = k
        scores[2 * n + 1, :k] = np.round(rs.rand(k), 3)          # rounded: ties inside and across images
        for l in range(1, k + 1):
            if rs.rand() < 0.15:
                continue
            m = np.roll(labels[n, 1] == l, (rs.randint(-3, 4), rs.randint(-3, 4)), axis=(0, 1))
            if rs.rand() < 0.3:                                 # a second, overlapping ground truth
                m2 = np.roll(m, (2, 2), axis=(0, 1))
                anns.append({"id": next_id, "image_id": n, "category_id": 100, "iscrowd": 0,
                             "area": int(m2.sum()), "segmentation": CO.encode(m2.astype(np.uint8))})
                next_id += 1
            crowd = int(rs.rand() < 0.05)
            anns.append({"id": next_id, "image_id": n, "category_id": 100, "iscrowd": crowd,
                         "area": int(m.sum()) if rs.rand() < 0.9 else 196, "segmentation": CO.encode(m.astype(np.uint8))})
            next_id += 1
    for a in anns:
        a["segmentation"]["counts"] = a["segmentation"]["counts"].decode("ascii")
    gt = {"images": [{"id": n, "height": size, "width": size} for n in range(n_images)], "annotations": anns,
          "categories": [{"id": 100}]}
    return labels, scores, gt


def _oracle_ap(gt, results, image_ids, small=14):
    c_gt = CO.COCO()
    c_gt.dataset = json.loads(json.dumps(gt))
    c_gt.createIndex()
    ev = CO.COCOevalOracle(c_gt, c_gt.loadRes(json.loads(json.dumps(results))), image_ids, [100], small)
    ev.evaluate()
    ev.accumulate()
    ev.summarize()
    return ev


def _annotations(image_ids, labels, scores_per_image, monkeypatch):
    """instances_oracle.create_annotations with the vectorised (pinned-equal) RLE encoder"""
    monkeypatch.setattr(I, "rle_encode", CO.rle_encode)
    return I.create_annotations(image_ids, list(zip(labels, scores_per_image)), [None, 100], [1, 1])


def test_device_evaluator_equals_the_oracle_at_scale(mcb, cuda, monkeypatch):
    from mcb200 import evaluation as E
    labels, scores, gt = _scale_case()
    n = labels.shape[0]
    ev = E.DeviceCOCOEvaluator(gt, np.arange(n), [100], 14)
    batch = 64
    for s in range(0, n, batch):
        ev.add_batch(torch.from_numpy(labels[s:s + batch]).to(cuda), torch.from_numpy(scores[2 * s:2 * (s + batch)]).to(cuda),
                     list(range(s, min(s + batch, n))))
    tb = ev.tables()
    res = ev.result()
    per_image = [[[], list(scores[2 * i + 1, :int(labels[i, 1].max())])] for i in range(n)]
    want = _oracle_ap(gt, _annotations(list(range(n)), labels, per_image, monkeypatch), np.arange(n))
    wt = CO.flat_tables(want)
    assert (tb["nd"] * tb["ng"]).max() >= 4 * 32 * 4          # several warps' worth of pairs per image
    for k in ("nd", "ng", "present", "dt_scores", "dt_match", "dt_ignore", "gt_ignore", "iou"):
        assert np.array_equal(tb[k], wt[k]), k
    assert np.array_equal(res["precision"], want.precision) and np.array_equal(res["recall"], want.recall)
    assert np.array_equal(res["stats"], want.stats) and 0 < res["stats"][0] < 1


# ---------------------------------------------------------------------------------------------------------------------
# end to end: the validation callback over a seeded UNetResNet-34
# ---------------------------------------------------------------------------------------------------------------------
def test_validation_monitor_ap_equals_the_oracle_chain(mcb, cuda, tmp_path, monkeypatch):
    import pandas as pd
    import bench
    from mcb200 import ops
    from mcb200.callbacks import ValidationMonitorSegmentation
    from mcb200.models import PyTorchUNet
    from oracle import synthetic
    from oracle import unet_oracle as O

    model = PyTorchUNet(**bench.unet_config("ResNet34"))
    model.model.load_state_dict(O.make_reference_like_state_dict(34, seed=21))
    model._to_device()
    net = model.model
    net.eval()
    batches = [torch.from_numpy(synthetic.train_batch(4, 256, seed=100 + b, n_rect=6)[0]) for b in range(6)]
    with torch.no_grad():     # centre the class margin so that both classes form instances
        margin = torch.cat([net(x.to(cuda)) for x in batches])
        shift = float((margin[:, 1] - margin[:, 0]).median())
        net.final.bias.data[1] -= shift
        net.refresh_operands()
        logits = torch.cat([net(x.to(cuda)) for x in batches])
    probs = ops.softmax2(logits.contiguous()).cpu().numpy()
    ids = list(range(500, 500 + len(probs)))
    preds = []
    for p in probs:
        r = P.resize_image(p, (300, 300))
        lab = P.label_multiclass_image(P.categorize_image(r))
        preds.append(P.build_score(lab, r))
    results = _annotations(ids, [p[0] for p in preds], [p[1] for p in preds], monkeypatch)
    assert len(results) > 20
    anns = []
    for j, a in enumerate(results[::2]):       # every other detection is a ground truth, some of them crowds
        anns.append({"id": j + 1, "image_id": a["image_id"], "category_id": 100, "iscrowd": int(j % 7 == 3),
                     "area": CO.area(a["segmentation"]), "segmentation": dict(a["segmentation"])})
    gt = {"images": [{"id": i, "height": 300, "width": 300} for i in ids], "annotations": anns,
          "categories": [{"id": 100}]}
    os.makedirs(tmp_path / "val")
    with open(tmp_path / "val" / "annotation.json", "w") as f:
        json.dump(gt, f)
    want = _oracle_ap(gt, results, ids)

    got = []
    for run in range(2):
        mon = ValidationMonitorSegmentation(data_dir=str(tmp_path), small_annotations_size=14, validate_with_map=True,
                                            epoch_every=1)
        transformer = types.SimpleNamespace(model=net, optimizer=None, loss_function=None,
                                            output_names=['multichannel_map'], validation_loss={})
        mon.set_params(transformer, validation_datagen=(batches, None), meta_valid=pd.DataFrame({'ImageId': ids}))
        mon.on_train_begin()
        mon.on_epoch_end()
        stored = transformer.validation_loss[0]['sum']
        res = mon.evaluator().result()
        assert res["stats"][0] == want.stats[0] and np.array_equal(res["precision"], want.precision)
        assert stored.shape == (1,) and stored.item() == torch.tensor([want.stats[0]], dtype=torch.float32).item()
        got.append((stored.clone(), res["precision"]))
    assert torch.equal(got[0][0], got[1][0]) and np.array_equal(got[0][1], got[1][1])
    assert 0 < want.stats[0] < 1
