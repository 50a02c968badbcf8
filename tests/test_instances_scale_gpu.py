"""The instance layer (csrc/instances.cu through mcb200.utils / mcb200.postprocessing / mcb200.loaders) at the inference
batch size, on inputs made the way the reference makes them.

Inputs.  64 seeded 256x256 probability maps go through the device MaskPostprocessor((300, 300), 'resize', erode 2,
dilate 2) and through the device resize (float32 256^2 -> float64 300^2, skimage's resize), as bench.py --workload
infer and the reference's scoring pipelines do.  The resize samples the cval-0 border, so the first and last rows and
columns of its output are 0, and the 2x2 grey dilation only spreads up and left: in that chain no building reaches the
bottom or right border and no label can vanish.  Eight 320x320 maps cropped to 300x300 (bench.py's --size 320 path,
identity-sized resize) supply those cases: buildings on every border, one spanning all 300 rows (pycocotools
rleToBbox's full-height rule), one covering the last pixel, and top-row / left-column single pixels whose diagonal
neighbours carry larger labels, so that the dilation swallows them (gaps in 1..K).

Bars, all derived a priori:
  * annotations, NMS scores, integer features, box ratios, TTA index maps, max / min TTA over probabilities: exact;
  * max_prob: exact (==) in the probabilities' own precision;
  * mean_prob: |got - fsum / area| <= area * 2^-53 * (fsum / area): float64 summation of `area` non-negative terms in
    any order is off by at most (area - 1) * 2^-53 relative, plus half an ulp for the division; the reference's own
    numpy value is held to the same bar, so the bar is known to be fair;
  * mean / gmean TTA over probabilities: 1e-7 absolute (float64 accumulation rounded once to float32: <= 2^-25);
  * TTA from logits: 1e-6 absolute (the fused softmax is float32: expf <= 2 ulp plus the divide, ~2.4e-7 relative on
    values <= 1; the rest is float64);
  * TTA against the scipy oracle (float32 probabilities, scipy.stats.gmean): 2e-6, as in test_instances_gpu.py.
The CPU oracles are O(instances x image) or worse, so they run on fixed subsets; the device always runs the full batch.
"""
import copy
import math

import numpy as np
import pytest
import torch

from oracle import coco_oracle as CO
from oracle import instances_oracle as I
from oracle import post_oracle as P
from oracle import synthetic

pytestmark = pytest.mark.gpu

N = 64
S = 300
U53 = 2.0 ** -53


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def resize_inputs():
    """64 maps of 256x256 [1 - p, p] float32; image 3 has no building, 0 has buildings reaching the top and left
    borders through the dilation"""
    probs = synthetic.probability_maps(N, 256, seed=2024)
    p = probs[:, 1].copy()
    p[0, 0:12, 40:70] = 0.97
    p[0, 100:130, 0:10] = 0.97
    p[3] = 0.03
    probs[:, 1], probs[:, 0] = p, 1 - p
    return probs


def crop_inputs():
    """8 maps of 320x320 centre-cropped to 300x300 (bench.py's --size 320 path), float32"""
    probs = np.ascontiguousarray(synthetic.probability_maps(8, 320, seed=99)[:, :, 10:310, 10:310])
    p = probs[:, 1].copy()
    p[0, 280:, 20:60] = 0.97                        # bottom border
    p[0, 100:140, 285:] = 0.97                      # right border
    p[0, :, 150:160] = 0.97                         # all 300 rows
    p[1, 270:, 265:] = 0.97                         # the last pixel
    # single pixels on the top row / left column, each with larger-labelled diagonal neighbours: the up-left 2x2
    # dilation replaces every pixel they would reach
    p[2, :3, :] = 0.03
    p[2, :, :3] = 0.03
    p[2, 0, 11:60:2] = 0.97
    p[2, 1, 10:61:2] = 0.97
    p[2, 11:60:2, 0] = 0.97
    p[2, 10:61:2, 1] = 0.97
    probs[:, 1], probs[:, 0] = p, 1 - p
    return probs


def _nan_scores(scores):
    return [[math.nan if v is np.ma.masked else float(v) for v in layer] for layer in scores]


@pytest.fixture(scope="module")
def G(mcb, cuda):
    from mcb200 import postprocessing
    return postprocessing


@pytest.fixture(scope="module")
def chain(G, cuda):
    pp = G.MaskPostprocessor((S, S), "resize", erode_selem_size=2, dilate_selem_size=2)
    r_in, c_in = resize_inputs(), crop_inputs()
    y_r = pp.transform(r_in)["y_pred"]
    y_c = pp.transform(c_in)["y_pred"]
    pr = G.resize_batch(torch.from_numpy(r_in).to(cuda), (S, S)).cpu().numpy()
    pr_c = G.resize_batch(torch.from_numpy(c_in).to(cuda), (S, S)).cpu().numpy()
    preds = [(lab, _nan_scores(sc)) for lab, sc in y_r + y_c]
    labels = np.stack([lab for lab, _ in preds])
    # the cases the file is about are really in the batch
    k = labels.reshape(len(preds), 2, -1).max(-1)
    b = labels[:, 1]
    vanished = [(i, l) for i in range(len(preds)) for l in range(1, k[i, 1] + 1) if not (b[i] == l).any()]
    assert k[3, 1] == 0 and len(vanished) >= 10 and all(i >= N for i, _ in vanished)
    assert (b[:, 0] > 0).any() and (b[:, -1] > 0).any() and (b[:, :, 0] > 0).any() and (b[:, :, -1] > 0).any()
    assert b[N + 1, -1, -1] > 0
    full = b[N][:, 155]
    assert full.min() > 0 and (full == full[0]).all()
    assert not np.array_equal(pr.astype(np.float32).astype(np.float64), pr)    # values a float32 copy cannot hold
    return dict(preds=preds, labels=labels, pr=np.concatenate([pr, pr_c]), vanished=vanished,
                ids=[1000 + 7 * i for i in range(len(preds))])


# ---------------------------------------------------------------------------------------------------------------------
# A. annotations
# ---------------------------------------------------------------------------------------------------------------------
def test_create_annotations_equal_the_reference(chain, monkeypatch):
    from mcb200 import utils as U
    preds, ids = chain["preds"], chain["ids"]
    got = U.create_annotations(ids, preds, None, [None, 100], [1, 1])
    monkeypatch.setattr(I, "rle_encode", CO.rle_encode)
    want = I.create_annotations(ids, preds, [None, 100], [1, 1])
    assert len(got) == len(want) == sum(len(sc[1]) for _, sc in preds)
    for j, (a, b) in enumerate(zip(got, want)):
        assert a["image_id"] == b["image_id"] and a["category_id"] == b["category_id"], j
        assert a["segmentation"] == b["segmentation"], (j, a["image_id"])
        assert a["bbox"] == b["bbox"], (j, a["bbox"], b["bbox"])
        sa, sb = a["score"], b["score"]
        assert sa == sb or (math.isnan(sa) and math.isnan(sb)), (j, sa, sb)
    # a vanished label is decompose()'s all-zero mask: one run of h*w zeros, box [0, 0, 0, 0], score NaN
    empty = [a for a in got if a["bbox"] == [0.0, 0.0, 0.0, 0.0]]
    assert len(empty) == len(chain["vanished"])
    assert all(a["segmentation"]["counts"] == I.rle_to_string([S * S]).decode() and math.isnan(a["score"]) for a in empty)
    assert any(a["bbox"][1] == 0.0 and a["bbox"][3] == float(S) for a in got)      # rleToBbox's full-height rule


# ---------------------------------------------------------------------------------------------------------------------
# B. features
# ---------------------------------------------------------------------------------------------------------------------
EXACT_FEATURES = ("threshold", "area", "bbox_area", "bbox_ar", "bbox_fill", "min_dist_to_border", "max_dist_to_border",
                  "contour_length")


def check_features(got, want, labels, probs, category_layers, numpy_fair=True):
    inds = np.cumsum(category_layers)
    n = 0
    assert len(got) == len(want) == labels.shape[0]
    for li, (lg, lw) in enumerate(zip(got, want)):
        assert len(lg) == len(lw) == labels[li].max()
        ch = probs[int(np.searchsorted(inds, li, side="right"))]
        for l, (a, b) in enumerate(zip(lg, lw), start=1):
            for k in EXACT_FEATURES:
                assert a[k] == b[k], (li, l, k, a[k], b[k])
            assert a["max_prob"] == b["max_prob"], (li, l, a["max_prob"], b["max_prob"], a["max_prob"] - b["max_prob"])
            vals = ch[labels[li] == l].astype(np.float64)
            ref = math.fsum(vals.tolist()) / vals.size
            bar = vals.size * U53 * ref
            assert abs(a["mean_prob"] - ref) <= bar, (li, l, a["mean_prob"], ref)
            if numpy_fair:
                assert abs(float(b["mean_prob"]) - ref) <= bar, (li, l, b["mean_prob"], ref)
            n += 1
    return n


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_features_two_layers(G, chain, dtype):
    """[1, 1] on every 256 -> 300 image and on the crop-path images without vanished labels (the reference's get_bbox
    fails on an empty mask); float64 is what the reference's scoring pipelines feed"""
    images = list(range(N)) + [i for i in range(N, len(chain["preds"])) if i not in {v[0] for v in chain["vanished"]}]
    n = 0
    for i in images:
        lab, pr = chain["labels"][i], chain["pr"][i].astype(dtype)
        got = G.instance_features(lab, pr, [1, 1])
        want = I.instance_features(lab, pr, (1, 1))
        n += check_features(got, want, lab, pr, (1, 1), numpy_fair=dtype == np.float64)
    assert n > 1500


def test_features_multi_threshold_stack(G, chain):
    """[1, 19]: the background layer plus label(p > t) at t = 0.05 ... 0.95 -- nested instances of every size"""
    thr = P.layer_thresholds((1, 19))
    n = 0
    for i in (0, 5, 17, 63):
        pr = chain["pr"][i]
        lab = np.stack([P.label(pr[0] > thr[0][0])] + [P.label(pr[1] > t) for t in thr[1]]).astype(np.int32)
        got = G.instance_features(lab, pr, [1, 19])
        want = I.instance_features(lab, pr, (1, 19))
        n += check_features(got, want, lab, pr, (1, 19))
    assert n > 1000


# ---------------------------------------------------------------------------------------------------------------------
# C. non-maximum suppression
# ---------------------------------------------------------------------------------------------------------------------
def nms_case(pr, seed):
    """label(p > t) at three thresholds (nested instances, IoUs either side of 0.5) plus two constructed layers:
    A1 / B1 with IoU exactly 100/200 (kept: the test is `>`), A2 / B2 with IoU 101/200 (suppressed), a vanished
    label B3; scores rounded to 0.1 (ties everywhere) and A1 / A2 tied at the top"""
    rs = np.random.RandomState(seed)
    layers = [P.label(pr[1] > t).astype(np.int32) for t in (0.3, 0.5, 0.7)]
    la, lb = np.zeros((S, S), np.int32), np.zeros((S, S), np.int32)
    la[2:12, 270:290] = 1
    la[20:30, 270:290] = 2
    lb[2:12, 270:280] = 1
    lb[20:30, 270:280] = 2
    lb[20, 280] = 2
    lb[40:45, 270:275] = 4                            # label 3 has no pixel
    image = np.stack(layers + [la, lb])
    scores = [[round(float(v), 1) for v in rs.rand(int(l.max()))] for l in layers] + [[9.0, 9.0], [8.0, 8.0, 0.7, 0.3]]
    return image, scores


def test_nms_equals_the_reference(G, chain):
    n_zero = 0
    for i in (0, 1, 3, 5, 9, 13, 17, 21, 29, 33, 41, 50, 55, 58, 61, 63):
        image, scores = nms_case(chain["pr"][i], seed=i)
        _, want = I.remove_overlapping_masks(image, copy.deepcopy(scores), 0.5)
        _, got = G.remove_overlapping_masks(image, copy.deepcopy(scores), 0.5)
        assert got == want, i
        assert got[-1][:3] == [8.0, 0, 0.7], (i, got[-1])      # IoU 0.5 kept, 101/200 suppressed, vanished kept
        n_zero += sum(v == 0 for layer in got[:3] for v in layer)
    assert n_zero > 20


# ---------------------------------------------------------------------------------------------------------------------
# D. test-time augmentation at the network's inference shapes
# ---------------------------------------------------------------------------------------------------------------------
def forward_ref(x, spec):
    """test_time_augmentation_transform on NCHW: the up-down flip wins over left-right, then quarter turns"""
    if spec["ud_flip"]:
        x = x.flip(2)
    elif spec["lr_flip"]:
        x = x.flip(3)
    return torch.rot90(x, spec["rotation"] // 90, dims=(2, 3))


def inverse_ref(x, spec):
    x = torch.rot90(x, -(spec["rotation"] // 90), dims=(2, 3))
    if spec["ud_flip"]:
        x = x.flip(2)
    elif spec["lr_flip"]:
        x = x.flip(3)
    return x


def shuffled_variants(seed):
    """16 variants of 64 images in a shuffled order -> (specs per variant, image index per variant)"""
    from mcb200 import loaders as lo
    specs = lo.tta_specs()
    perm = np.random.RandomState(seed).permutation(N * 16)
    return [specs[j % 16] for j in perm], [int(j // 16) for j in perm]


@pytest.mark.parametrize("s", [256, 320])
def test_tta_transform_is_the_index_map(mcb, cuda, s):
    from mcb200 import loaders as lo
    params, img = shuffled_variants(s)
    g = torch.Generator(device=cuda).manual_seed(s)
    x = torch.randn((N, 3, s, s), generator=g, device=cuda)
    got = lo.test_time_augmentation_transform_batch(x, params, img)
    assert got.shape == (N * 16, 3, s, s)
    img_t = torch.tensor(img, device=cuda)
    for spec in lo.tta_specs():
        idx = torch.tensor([v for v, p in enumerate(params) if p == spec], device=cuda)
        assert torch.equal(got[idx], forward_ref(x[img_t[idx]], spec)), spec
    for v, (p, i) in enumerate(zip(params, img)):
        if i in (0, N - 1):
            want = I.tta_transform(x[i].cpu().numpy().transpose(1, 2, 0), p).transpose(2, 0, 1)
            assert np.array_equal(got[v].cpu().numpy(), want.astype(np.float32)), (v, p)


def tta_logits(s, cuda, params, img, seed):
    """per-variant 2-class logits (NV, 2, s, s) float32: each image has a gap map up to +-120 (cubed uniform, so most
    gaps are small), every variant sees it through its own transform plus N(0, 0.5) noise.  Probabilities of gaps
    beyond ~87 are float32 denormals, beyond ~104 exact zeros."""
    g = torch.Generator(device=cuda).manual_seed(seed)
    gap = (torch.rand((N, 1, s, s), generator=g, device=cuda) * 2 - 1) ** 3 * 120
    base = torch.cat([gap / 2, -gap / 2], dim=1)
    out = torch.empty((len(params), 2, s, s), device=cuda)
    img_t = torch.tensor(img, device=cuda)
    for spec in I.tta_specs():
        idx = torch.tensor([v for v, p in enumerate(params) if p == spec], device=cuda)
        out[idx] = forward_ref(base[img_t[idx]], spec)
    return (out + 0.5 * torch.randn(out.shape, generator=g, device=cuda)).contiguous()


def aggregate_ref(p64, params, img, method):
    """float64 restatement of TestTimeAugmentationAggregator.transform: inverse maps, then the reduction over each
    image's variants; images in sorted id order"""
    inv = torch.empty_like(p64)
    for spec in I.tta_specs():
        idx = torch.tensor([v for v, p in enumerate(params) if p == spec], device=p64.device)
        inv[idx] = inverse_ref(p64[idx], spec)
    order = torch.from_numpy(np.argsort(np.asarray(img), kind="stable")).to(p64.device)
    inv = inv[order].view(N, 16, *p64.shape[1:])
    if method == "mean":
        return inv.mean(1)
    if method == "max":
        return inv.amax(1)
    if method == "min":
        return inv.amin(1)
    return torch.exp(torch.log(inv).mean(1))


@pytest.mark.parametrize("from_logits", [False, True])
@pytest.mark.parametrize("s", [256, 320])
def test_tta_aggregate_against_float64(mcb, cuda, s, from_logits):
    from mcb200 import loaders as lo
    params, img = shuffled_variants(s + 1)
    ids = [3 + 7 * i for i in img]                               # non-contiguous ids; sorted order = image order
    logits = tta_logits(s, cuda, params, img, seed=s)
    p64 = torch.softmax(logits.double(), dim=1)
    probs32 = p64.float()                                        # the network's float32 probabilities
    assert int((probs32 == 0).sum()) > 0 and int(((probs32 > 0) & (probs32 < 1.1754944e-38)).sum()) > 0
    if not from_logits:
        p64 = probs32.double()
    for method in ("gmean", "mean", "max", "min"):
        pred = logits if from_logits else probs32
        got = lo.aggregate_batch(pred, params, ids, method, from_logits=from_logits)
        ref = aggregate_ref(p64, params, img, method)
        err = float((got.double() - ref).abs().max())
        if from_logits:
            assert err <= 1e-6, (method, err)
        elif method in ("max", "min"):
            assert torch.equal(got.double(), ref), (method, err)
        else:
            assert err <= 1e-7, (method, err)
        del got, ref
    # the scipy oracle on two images (from the float32 probabilities in both cases)
    sub = [v for v, i in enumerate(img) if i in (0, N - 1)]
    p_sub = probs32[sub].cpu().numpy()
    pred_sub = (logits if from_logits else probs32)[sub].contiguous()
    for method in ("gmean", "mean", "max", "min"):
        got = lo.aggregate_batch(pred_sub, [params[v] for v in sub], [ids[v] for v in sub], method,
                                 from_logits=from_logits).cpu().numpy()
        want = I.tta_aggregate(list(p_sub), [params[v] for v in sub], [ids[v] for v in sub], method)
        assert np.abs(got - np.stack(want)).max() < 2e-6, method


# ---------------------------------------------------------------------------------------------------------------------
# E. more planes than gridDim.y holds
# ---------------------------------------------------------------------------------------------------------------------
def test_planes_beyond_grid_y(mcb, cuda, monkeypatch):
    """70 000 label planes of 6x5 (sparse labels 1..3 with gaps, every 97th plane empty) through one
    create_annotations batch, instance_geometry with float64 probabilities and mcb_contour_length"""
    from mcb200 import _lib as L
    from mcb200 import utils as U
    n, h, w = 70000, 6, 5
    rs = np.random.RandomState(70000)
    lab = np.where(rs.rand(n, h, w) < 0.15, rs.randint(1, 4, (n, h, w)), 0).astype(np.int32)
    lab[::97] = 0
    prob = rs.rand(n, h, w)
    counts = lab.reshape(n, -1).max(1)
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    total = int(counts.sum())
    pl, y, x = np.nonzero(lab)
    slot = offs[pl] + lab[pl, y, x] - 1
    assert slot.max() == total - 1 and np.bincount(slot, minlength=total).min() == 0    # gaps present

    lab_d = torch.from_numpy(lab).to(cuda)
    geo = U.instance_geometry(lab_d, torch.from_numpy(counts.astype(np.int32)).to(cuda),
                              torch.from_numpy(prob).to(cuda))
    area = np.bincount(slot, minlength=total)
    rmin, rmax = np.full(total, 2 ** 31 - 1), np.full(total, -1)
    cmin, cmax = np.full(total, 2 ** 31 - 1), np.full(total, -1)
    pmax = np.full(total, -np.inf)
    np.minimum.at(rmin, slot, y)
    np.maximum.at(rmax, slot, y)
    np.minimum.at(cmin, slot, x)
    np.maximum.at(cmax, slot, x)
    np.maximum.at(pmax, slot, prob[pl, y, x])
    for k, ref in (("area", area), ("rmin", rmin), ("rmax", rmax), ("cmin", cmin), ("cmax", cmax), ("pmax", pmax)):
        assert np.array_equal(geo[k], ref), k
    order = np.argsort(slot, kind="stable")
    bounds = np.searchsorted(slot[order], np.arange(total + 1))
    vals = prob[pl, y, x][order].tolist()
    psum = np.array([math.fsum(vals[bounds[s]:bounds[s + 1]]) for s in range(total)])
    assert (np.abs(geo["psum"] - psum) <= area * U53 * psum).all()

    clen = torch.zeros(total, dtype=torch.int32, device=cuda)
    L.fcall("mcb_contour_length", lab_d.data_ptr(), geo["_offsets"].data_ptr(), geo["_counts"].data_ptr(),
            clen.data_ptr(), n, h, w)
    padded = np.pad(lab, ((0, 0), (1, 1), (1, 1)), constant_values=-1)
    v = lab[pl, y, x]
    edge = ((padded[pl, y, x + 1] != v) | (padded[pl, y + 2, x + 1] != v) | (padded[pl, y + 1, x] != v) |
            (padded[pl, y + 1, x + 2] != v))
    assert np.array_equal(clen.cpu().numpy(), np.bincount(slot[edge], minlength=total))

    # one annotation per label of every plane; an empty plane's single score meets decompose()'s [labeled]
    preds = [(lab[i][None], [[0.5]] if counts[i] == 0 else [[float(s) for s in np.arange(1, counts[i] + 1) / 4]])
             for i in range(n)]
    got = U.create_annotations(list(range(n)), preds, None, [100], [1])
    monkeypatch.setattr(I, "rle_encode", CO.rle_encode)
    want = I.create_annotations(list(range(n)), preds, [100], [1])
    assert len(got) == len(want) == total + int((counts == 0).sum())
    assert got == want
