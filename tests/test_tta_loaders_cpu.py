"""The TTA inference loaders' host side without a GPU (src/loaders.py:307-487): spec lists and the non-colour transform
against the unmodified reference (tests/golden/tta_loaders.npz, oracle/make_golden_tta.py), the colour oracle's
consequences against cv2, the colour draws, the batch boundaries and the loader surface src/pipelines.py uses."""
import inspect
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import instances_oracle as I
from oracle import tta_oracle as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tta_loaders.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _combos():
    from itertools import product
    return [(ud, lr, rot, runs) for ud, lr, rot in product((True, False), repeat=3) for runs in (False, 1, 2)]


def _tag(ud, lr, rot, runs):
    return "ud%d_lr%d_rot%d_runs%d" % (ud, lr, rot, int(runs))


def test_spec_lists_and_generator_equal_the_reference(mcb, golden):
    from mcb200 import loaders as lo
    X = [["tiles/a.png"], ["tiles/b.png"]]
    for ud, lr, rot, runs in _combos():
        t = _tag(ud, lr, rot, runs)
        want = json.loads(str(golden["specs_" + t]))
        opts = dict(flip_ud=ud, flip_lr=lr, rotation=rot, color_shift_runs=runs)
        assert lo.tta_specs(**opts) * 2 == want, t
        got = lo.TestTimeAugmentationGenerator(**opts).transform(X)
        assert got["tta_params"] == want and got["img_ids"] == golden["ids_" + t].tolist(), t
        assert np.asarray(got["X_tta"].values).reshape(-1).tolist() == json.loads(str(golden["xtta_" + t])), t
    assert len(lo.tta_specs(color_shift_runs=2)) == 1 + 16 * 2


def test_non_colour_transforms_equal_the_reference(mcb, golden):
    from mcb200 import loaders as lo
    img = golden["transform_img"]
    specs = json.loads(str(golden["transform_specs"]))
    assert len(specs) == 25 and any(s["color_shift"] for s in specs)     # flipped colour specs are plain flips
    for s, want in zip(specs, golden["transform_out"]):
        assert not lo.applies_colour(s) and not T.applies_colour(s)
        assert np.array_equal(T.tta_transform(img, s), want), s
        assert np.array_equal(I.tta_transform(img, s), want), s


def test_spec_code_and_the_float_path(mcb):
    from mcb200 import loaders as lo
    specs = lo.tta_specs(color_shift_runs=1)
    plain = {(s['ud_flip'], s['lr_flip'], s['rotation']): lo.spec_code(s) for s in lo.tta_specs()}
    for s in specs:
        assert lo.spec_code(s) == plain.get((s['ud_flip'], s['lr_flip'], s['rotation']), 0)
    assert sum(lo.applies_colour(s) for s in specs) == 4
    with pytest.raises(NotImplementedError, match="ImageSegmentationLoaderResizeTTA"):
        lo.test_time_augmentation_transform_batch(torch.zeros(1, 3, 4, 4), specs, [0] * len(specs))


def test_colour_oracle_consequences():
    import cv2
    rs = np.random.RandomState(3)
    img = rs.randint(0, 256, (40, 70, 3)).astype(np.uint8)
    hsv = cv2.cvtColor(img, cv2.COLOR_RGB2HSV)
    # branch 1: H is clipped at 255 (not 180), then cv2 wraps it modulo 180: H 200 is H 20
    for value in (0, 37, 100):
        h = np.clip(hsv[..., 0].astype(np.int32) + value, 0, 255)
        assert (h > 179).any() or value == 0
        want = hsv.copy()
        want[..., 0] = h
        assert np.array_equal(T.color_shift(img, 1, value), cv2.cvtColor(want, cv2.COLOR_HSV2RGB))
    wrapped = np.array([[[200, 180, 200]]], np.uint8)
    assert np.array_equal(cv2.cvtColor(wrapped, cv2.COLOR_HSV2RGB),
                          cv2.cvtColor(np.array([[[20, 180, 200]]], np.uint8), cv2.COLOR_HSV2RGB))
    # branches 4-6: a plain add and clip on R, G or B
    for branch in (4, 5, 6):
        got = T.color_shift(img, branch, 60)
        c = branch - 4
        assert np.array_equal(got[..., c], np.minimum(img[..., c].astype(np.int32) + 60, 255))
        assert np.array_equal(np.delete(got, c, axis=2), np.delete(img, c, axis=2))
    # value 0 on branches 1-3 is the (lossy) cv2 round trip, never skipped
    trip = cv2.cvtColor(hsv, cv2.COLOR_HSV2RGB)
    assert not np.array_equal(trip, img)
    for branch in (1, 2, 3):
        assert np.array_equal(T.color_shift(img, branch, 0), trip)


def test_rgb2hsv_restatement_equals_cv2_on_all_colours():
    import cv2
    idx = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([idx >> 16, (idx >> 8) & 255, idx & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(T.rgb2hsv(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2HSV))


def test_vector_body_oracle_differs_from_cv2_only_in_the_tail_columns():
    rs = np.random.RandomState(4)
    hsv = rs.randint(0, 256, (50, 300, 3)).astype(np.uint8)
    d = (T.hsv2rgb_cv2(hsv, tail=True) != T.hsv2rgb_cv2(hsv, tail=False)).any(2)
    assert d.any() and d[:, :300 - T.VECTOR_COLUMNS].sum() == 0


def test_colour_draws(mcb):
    from mcb200 import loaders as lo
    a = lo.draw_colour(np.random.default_rng(5), 1000)
    b = lo.draw_colour(np.random.default_rng(5), 1000)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    branch, value = lo.draw_colour(np.random.default_rng(6), 60_000)
    freq = np.bincount(branch, minlength=7)[1:] / 60_000
    assert set(np.unique(branch)) == set(range(1, 7)) and np.abs(freq - 1 / 6).max() < 0.02 / 6
    assert set(np.unique(value)) == set(range(101))


def _flow(lo, n_tiles, specs, batch_size, drop_last=False, seed=0):
    paths = sum(([f"t{i}.png"] * len(specs) for i in range(n_tiles)), [])
    return lo.TTABatches(paths, specs * n_tiles, {'batch_size': batch_size, 'shuffle': False, 'drop_last': drop_last,
                                                  'num_workers': 0}, np.random.default_rng(seed), pad=(10, 10))


@pytest.mark.parametrize("batch_size,drop_last", [(20, False), (16, False), (7, True), (1, False), (500, False)])
def test_steps_and_batch_bounds_equal_the_dataloader(mcb, batch_size, drop_last):
    from mcb200 import loaders as lo
    specs = lo.tta_specs(color_shift_runs=2)
    flow = _flow(lo, 6, specs, batch_size, drop_last)
    ref = torch.utils.data.DataLoader(list(range(6 * len(specs))), batch_size=batch_size, shuffle=False,
                                      drop_last=drop_last)
    assert len(flow) == len(ref)
    assert [list(range(b0, b1)) for b0, b1 in flow.batch_bounds()] == [b.tolist() for b in ref]
    assert flow.colour.sum() == 6 * 8 and not flow.colour[flow.codes >> 2 != 0].any()


def test_flip_rows_take_no_draw(mcb):
    from mcb200 import loaders as lo
    specs = lo.tta_specs(color_shift_runs=1)
    flow = _flow(lo, 2, specs, 20)
    flipped = np.array([s['ud_flip'] or s['lr_flip'] for s in specs * 2])
    assert flipped.sum() == 2 * 12 and not flow.colour[flipped].any()
    assert flow.colour[~flipped].sum() == 2 * 4


def test_loader_surface_of_the_reference_pipelines(mcb):
    """src/pipelines.py uses nine names of its `loaders` module; mcb200.loaders has all of them, with the reference's
    constructor and transform signatures"""
    from mcb200 import loaders as lo
    names = ["MetadataImageSegmentationLoaderCropPad", "MetadataImageSegmentationLoaderResize",
             "MetadataImageSegmentationLoaderDistancesCropPad", "MetadataImageSegmentationLoaderDistancesResize",
             "ImageSegmentationLoaderInferencePadding", "ImageSegmentationLoaderInferencePaddingTTA",
             "ImageSegmentationLoaderResizeTTA", "TestTimeAugmentationGenerator", "TestTimeAugmentationAggregator"]
    for n in names:
        assert hasattr(lo, n), n
    sig = lambda cls: list(inspect.signature(cls.transform).parameters)
    assert sig(lo.ImageSegmentationLoaderInferencePadding) == ["self", "X", "kwargs"]
    assert sig(lo.ImageSegmentationLoaderInferencePaddingTTA) == ["self", "X", "tta_params", "kwargs"]
    assert sig(lo.ImageSegmentationLoaderResizeTTA) == ["self", "X", "tta_params", "kwargs"]
    for n in names[4:7]:
        assert list(inspect.signature(getattr(lo, n).__init__).parameters)[:3] == ["self", "loader_params",
                                                                                  "dataset_params"]
    params = {'inference': {'batch_size': 20, 'shuffle': False, 'num_workers': 0, 'pin_memory': False}}
    dp = {'h': 256, 'w': 256, 'h_pad': 10, 'w_pad': 10}
    specs = lo.tta_specs(color_shift_runs=2)
    X = np.array(sum(([f"t{i}.png"] * len(specs) for i in range(6)), []))
    out = lo.ImageSegmentationLoaderResizeTTA(params, dp, seed=1).transform(X, specs * 6)
    flow, steps = out['datagen']
    assert out['validation_datagen'] == (None, None) and steps == math.ceil(6 * 33 / 20) == len(flow) == 10
    assert flow.resize == (256, 256)
    flow, steps = lo.ImageSegmentationLoaderInferencePadding(params, dp).transform(X[::33])['datagen']
    assert steps == 1 and flow.pad == (10, 10) and flow.resize is None
