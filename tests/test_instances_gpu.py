"""GPU parity of the instance-level steps (csrc/instances.cu through mcb200.utils / mcb200.loaders /
mcb200.postprocessing) against oracle/instances_oracle.py: integer outputs bit-exact, float reductions to 1e-6."""
import numpy as np
import pytest
import torch

from oracle import instances_oracle as I
from oracle import post_oracle as P
from oracle import synthetic

pytestmark = pytest.mark.gpu


def _label_planes(n, s, seed):
    probs = synthetic.probability_maps(n, s, seed=seed, n_rect=max(6, s // 12))
    return np.stack([P.label_multilayer_image(P.categorize_multilayer_image(p)) for p in probs]), probs


def test_categorize_image_is_numpy_argmax(mcb, cuda):
    from mcb200 import postprocessing as pp
    rs = np.random.RandomState(0)
    for dt in (np.float32, np.float64):
        x = rs.rand(3, 37, 41).astype(dt)
        x[1, 5, 5] = x[0, 5, 5] = 0.75          # tie -> first index
        x[2, 9, 9] = np.nan                      # NaN wins like numpy
        got = pp.categorize_image(x)
        assert got.dtype == np.int64 and np.array_equal(got, np.argmax(x, axis=0))


def test_rle_and_bbox_bit_exact(mcb, cuda):
    from mcb200 import utils as U
    # known answers first (tests/test_instances_cpu.py derives them by hand)
    assert U.rle_from_binary(np.array([[0, 1], [1, 1]], np.uint8)) == {"size": [2, 2], "counts": b"13"}
    assert U.rle_from_binary(np.array([[1, 0], [0, 0]], np.uint8))["counts"] == b"013"
    assert U.rle_counts_to_string([40, 2, 5, 30]) == b"X125l0" and U.rle_counts_to_string([5, 10, 7, 3]) == b"5:7I"
    assert U.rle_string_to_counts(b"X125l0") == [40, 2, 5, 30]
    # edge cases: empty, full, last pixel set, full-height instance, single pixel, 1-wide, 1-tall planes
    cases = [np.zeros((5, 7), np.uint8), np.ones((5, 7), np.uint8), np.eye(6, dtype=np.uint8)]
    m = np.zeros((9, 4), np.uint8); m[:, 1:3] = 1; cases.append(m)            # full height, crosses columns
    m = np.zeros((9, 4), np.uint8); m[8, 3] = 1; cases.append(m)              # last pixel only
    m = np.zeros((1, 40), np.uint8); m[0, 3:9] = 1; m[0, 39] = 1; cases.append(m)
    m = np.zeros((70, 1), np.uint8); m[3:40, 0] = 1; cases.append(m)          # > 32 rows: several ballot chunks
    rs = np.random.RandomState(1)
    cases += [(rs.rand(67, 45) > 0.5).astype(np.uint8), (rs.rand(33, 64) > 0.2).astype(np.uint8)]
    for m in cases:
        want = I.rle_from_binary(m)
        got = U.rle_from_binary(m)
        assert got == want, (m.shape, got, want)
        assert U.bounding_box_from_rle(got) == I.bounding_box_from_rle(want)


@pytest.mark.parametrize("s", [64, 300])
def test_create_annotations_matches_oracle(mcb, cuda, s):
    from mcb200 import utils as U
    labels, probs = _label_planes(3, s, seed=7)
    preds = []
    for lab, p in zip(labels, probs):
        _, sc = P.build_score(lab, p)
        preds.append((lab, sc))
    want = I.create_annotations([11, 12, 13], preds, [None, 100], [1, 1])
    got = U.create_annotations([11, 12, 13], preds, None, [None, 100], [1, 1])
    assert len(got) == len(want) and len(got) > 3
    for a, b in zip(got, want):
        assert a["image_id"] == b["image_id"] and a["category_id"] == b["category_id"]
        assert a["segmentation"] == b["segmentation"], (a["segmentation"], b["segmentation"])
        assert a["bbox"] == b["bbox"]
        assert a["score"] == b["score"]


def test_tta_transform_and_aggregate(mcb, cuda):
    from mcb200 import loaders as lo
    specs = lo.tta_specs()
    assert specs == I.tta_specs() and len(specs) == 16
    rs = np.random.RandomState(2)
    x = rs.randn(3, 3, 24, 24).astype(np.float32)
    params, ids = specs * 3, sum(([i] * 16 for i in range(3)), [])
    got = lo.test_time_augmentation_transform_batch(torch.from_numpy(x).to(cuda), params, ids).cpu().numpy()
    for v, (p, i) in enumerate(zip(params, ids)):
        want = I.tta_transform(x[i].transpose(1, 2, 0), p).transpose(2, 0, 1)
        assert np.array_equal(got[v], want.astype(np.float32)), (v, p)
    # aggregator on probabilities (the reference contract) ...
    logits = rs.randn(48, 2, 24, 24).astype(np.float32) * 2
    e = np.exp(logits - logits.max(1, keepdims=True))
    probs = (e / e.sum(1, keepdims=True)).astype(np.float32)
    for method in ("gmean", "mean", "max", "min"):
        agg = lo.TestTimeAugmentationAggregator(method, 2).transform(probs, params, ids)["aggregated_prediction"]
        want = I.tta_aggregate(list(probs), params, ids, method)
        for a, b in zip(agg, want):
            assert a.shape == b.shape and np.abs(a - b).max() < 2e-6, method
    # ... and fused with the softmax, from raw logits
    fused = lo.aggregate_batch(torch.from_numpy(logits).to(cuda), params, ids, "gmean", from_logits=True).cpu().numpy()
    want = np.stack(I.tta_aggregate(list(probs), params, ids, "gmean"))
    assert np.abs(fused - want).max() < 2e-6
    # shuffled variant order and non-contiguous image ids
    perm = rs.permutation(48)
    ids2 = [ids[j] * 5 + 2 for j in perm]
    agg = lo.TestTimeAugmentationAggregator("mean").transform(probs[perm], [params[j] for j in perm], ids2)
    want = I.tta_aggregate(list(probs), params, ids, "mean")
    for a, b in zip(agg["aggregated_prediction"], want):
        assert np.abs(a - b).max() < 2e-6


def test_nms_and_features(mcb, cuda):
    from mcb200 import postprocessing as pp
    labels, probs = _label_planes(2, 96, seed=3)
    rs = np.random.RandomState(4)
    for lab, p in zip(labels, probs):
        lab = lab.copy()
        lab[1] = lab[0] * (rs.rand(*lab[0].shape) > 0.15)           # layer 1 overlaps layer 0 heavily
        lab[1] = P.label_multilayer_image(lab[1][None] > 0)[0]
        sc = [[float(v) for v in rs.rand(int(l.max()))] for l in lab]
        import copy
        _, want = I.remove_overlapping_masks(lab, copy.deepcopy(sc), 0.5)
        _, got = pp.remove_overlapping_masks(lab, copy.deepcopy(sc), 0.5)
        assert got == want and any(v == 0 for layer in got for v in layer)
        res = pp.NonMaximumSupression(0.5).transform([(lab, copy.deepcopy(sc))])["images_with_scores"][0][1]
        assert res == want
        pr = P.resize_image(p, lab.shape[1:])
        f_got = pp.instance_features(lab, pr)
        f_want = I.instance_features(lab, pr)
        for lg, lw in zip(f_got, f_want):
            assert len(lg) == len(lw)
            for a, b in zip(lg, lw):
                for k in ("threshold", "area", "bbox_area", "min_dist_to_border", "max_dist_to_border",
                          "contour_length", "max_prob"):
                    assert a[k] == b[k], (k, a[k], b[k])
                for k in ("mean_prob", "bbox_ar", "bbox_fill"):
                    assert abs(a[k] - b[k]) <= 1e-9 * max(1.0, abs(b[k])), (k, a[k], b[k])


def test_tta_inference_pipeline_end_to_end(mcb, cuda):
    """unet_tta (src/pipelines.py:94-155) on the device: generator -> 16 index-map variants of the batch -> network ->
    ONE aggregation kernel on the raw logits (softmax + inverse maps + gmean) -> centre crop -> MaskPostprocessor ->
    create_annotations.  The fused aggregation must equal the reference's chain (numpy softmax per variant, per-channel
    inverse transforms, scipy gmean) applied to the SAME network outputs, and the emitted RLEs must decode back to the
    label maps."""
    import bench
    from mcb200 import loaders as lo, ops, postprocessing as pp, utils as U
    from mcb200.models import PyTorchUNet
    from oracle import unet_oracle as O
    sd = O.make_reference_like_state_dict(34, seed=11)
    model = PyTorchUNet(**bench.unet_config("ResNet34"))
    model.model.load_state_dict(sd)
    model._to_device()
    net = model.model
    net.eval()
    x, _ = synthetic.train_batch(2, 64, seed=4, n_rect=5)
    gen = lo.TestTimeAugmentationGenerator(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=False)
    meta = gen.transform([["a"], ["b"]])
    params, ids = meta["tta_params"], meta["img_ids"]
    assert len(params) == 32
    X = torch.from_numpy(x).to(cuda)
    Xv = lo.test_time_augmentation_transform_batch(X, params, ids)
    with torch.no_grad():
        logits = net(Xv)
    fused = lo.aggregate_batch(logits.contiguous(), params, ids, "gmean", from_logits=True).cpu().numpy()
    probs = ops.softmax2(logits.contiguous()).cpu().numpy()
    want = np.stack(I.tta_aggregate(list(probs), params, ids, "gmean"))
    assert fused.shape == (2, 2, 64, 64) and np.abs(fused - want).max() < 2e-6
    # a flip-equivariance sanity check of the index maps: the variant-0 prediction is the plain prediction
    with torch.no_grad():
        plain = ops.softmax2(net(X).contiguous()).cpu().numpy()
    assert np.abs(probs[0] - plain[0]).max() < 1e-6 and np.abs(probs[16] - plain[1]).max() < 1e-6
    # downstream: crop -> chain -> annotations; RLEs decode to the label maps
    out = pp.MaskPostprocessor((56, 56), "crop", 0, 0).transform(torch.from_numpy(fused))["y_pred"]
    ann = U.create_annotations([7, 8], out, None, [None, 100], [1, 1])
    k = 0
    for image_id, (labels, scores) in zip([7, 8], out):
        for l in range(1, int(labels[1].max()) + 1):
            a = ann[k]
            k += 1
            assert a["image_id"] == image_id and a["category_id"] == 100
            cnts = U.rle_string_to_counts(a["segmentation"]["counts"])
            flat = np.concatenate([np.full(c, i % 2, np.uint8) for i, c in enumerate(cnts)])
            assert np.array_equal(flat.reshape(56, 56).T.astype(bool), labels[1] == l)
    assert k == len(ann)
