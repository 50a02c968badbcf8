"""The training augmentation's host side without a GPU: the samplers of mcb200.augmentation against the reference's
distributions (src/augmentation.py:5-10, 34-37, 91-135), and the oracle's restatement of imgaug / skimage
(oracle/augment_oracle.py, assumptions 1-3) against what those assumptions visibly imply."""
import math

import numpy as np
import pytest
from scipy import ndimage as ndi
from scipy import stats

from oracle import augment_oracle as AO

N_DRAWS = 200_000


def _chi2_ok(counts):
    counts = np.asarray(counts, np.float64)
    return stats.chisquare(counts).pvalue > 1e-4


@pytest.fixture(scope="module")
def draws(mcb):
    from mcb200 import augmentation as A
    return A.crop_seq((256, 256)).draw(np.random.default_rng(1234), N_DRAWS, 300, 300)


def test_child_count_and_ordered_subsets(draws):
    k = draws['n_children']
    assert set(np.unique(k)) == {1, 2}
    assert abs((k == 1).mean() - 0.5) < 5 * math.sqrt(0.25 / N_DRAWS)
    singles = draws['children'][k == 1, 0]
    assert (draws['children'][k == 1, 1] == -1).all()
    assert _chi2_ok(np.bincount(singles, minlength=3))
    pairs = draws['children'][k == 2]
    assert (pairs[:, 0] != pairs[:, 1]).all() and (pairs >= 0).all()
    codes = pairs[:, 0] * 3 + pairs[:, 1]
    counts = np.bincount(codes, minlength=9)[[1, 2, 3, 5, 6, 7]]
    assert counts.sum() == len(pairs) and _chi2_ok(counts)


def test_flip_coin_rotation_and_translation_distributions(draws):
    coin = draws['coin'].reshape(-1)
    assert abs(coin.mean() - 0.5) < 5 * math.sqrt(0.25 / coin.size)
    assert stats.kstest(draws['rotate'], 'uniform', args=(-10, 20)).pvalue > 1e-4
    assert stats.kstest(draws['translate'], 'uniform', args=(-0.1, 0.2)).pvalue > 1e-4
    assert draws['rotate'].min() >= -10 and draws['rotate'].max() < 10


def test_one_translation_fraction_for_both_axes(mcb):
    """translate_percent=(-0.1, 0.1) is a tuple: one draw moves x by round(t W) and y by round(t H) pixels"""
    from mcb200 import augmentation as A
    for t, h, w in ((0.0731, 300, 300), (-0.0312, 300, 300), (0.05, 200, 300), (0.0999, 64, 37)):
        m = A.affine_matrix(0.0, t, h, w)
        assert (m[0, 2], m[1, 2]) == (int(round(t * w)), int(round(t * h)))
    assert A.affine_matrix(0.0, 0.001, 300, 300) is None       # 0 px, 0 degrees: imgaug skips the warp


def test_crop_offsets_uniform_and_full_size_crop_raises(draws, mcb):
    from mcb200 import augmentation as A
    for f in ('top', 'left'):
        v = draws[f]
        assert v.min() == 0 and v.max() == 300 - 256 - 1       # randint(H - h): the last offset is never drawn
        assert _chi2_ok(np.bincount(v, minlength=44))
    with pytest.raises(ValueError):
        A.crop_seq((300, 300)).draw(np.random.default_rng(0), 4, 300, 300)
    with pytest.raises(ValueError):
        A.crop_seq(320).draw(np.random.default_rng(0), 4, 300, 300)


def test_same_seed_same_parameters(mcb):
    from mcb200 import augmentation as A
    for seq in (A.fast_seq, A.crop_seq((256, 256))):
        a = seq.draw(np.random.default_rng(7), 64, 300, 300)
        b = seq.draw(np.random.default_rng(7), 64, 300, 300)
        c = seq.draw(np.random.default_rng(8), 64, 300, 300)
        assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()
        assert np.array_equal(A.rows(a, 300, 300), A.rows(b, 300, 300))


def test_package_matrix_equals_oracle_restatement(mcb):
    from mcb200 import augmentation as A
    rng = np.random.default_rng(3)
    for _ in range(200):
        angle, t = rng.uniform(-10, 10), rng.uniform(-0.1, 0.1)
        h, w = (300, 300) if rng.random() < 0.5 else (int(rng.integers(20, 400)), int(rng.integers(20, 400)))
        a, b = A.affine_matrix(angle, t, h, w), AO.affine_matrix(angle, t, h, w)
        assert a.tobytes() == b.tobytes()


def test_rows_place_flips_around_the_warp(mcb):
    from mcb200 import augmentation as A
    p = A.identity_params(4)
    p['n_children'] = [2, 2, 1, 2]
    p['children'] = [[A.FLIPLR, A.AFFINE], [A.AFFINE, A.FLIPUD], [A.FLIPUD, -1], [A.FLIPLR, A.FLIPUD]]
    p['coin'] = True
    p['rotate'], p['translate'] = 3.0, 0.05
    r = A.rows(p, 300, 300)
    assert list(r['warp']) == [1, 1, 0, 0]
    assert list(r['pre_flip']) == [1, 0, 0, 0] and list(r['post_flip']) == [0, 2, 2, 3]
    assert np.array_equal(r['inv'][0].reshape(3, 3), np.linalg.inv(AO.affine_matrix(3.0, 0.05, 300, 300)))


# ------------------------------------------------------------------------------------------------ oracle sanity
def test_integer_translation_is_a_zero_filled_shift():
    rng = np.random.default_rng(0)
    img = rng.integers(1, 256, (40, 50, 3)).astype(np.uint8)     # min > 0: the exact-zero fill survives the clip
    t = 0.1                                                       # 5 px right, 4 px down
    m = AO.affine_matrix(0.0, t, 40, 50)
    got = AO.warp(img, m)
    want = np.zeros_like(img)
    want[4:, 5:] = img[:-4, :-5]
    assert np.array_equal(got, want)


def test_warp_agrees_with_map_coordinates():
    """same bilinear maths as scipy's order-1 spline, in a different operation order"""
    rng = np.random.default_rng(1)
    plane = rng.random((61, 47))
    plane[0, 0] = 0.0                                              # cval inside the input range: the clip is inert
    for angle, t in ((7.3, 0.061), (-9.9, -0.083), (0.4, 0.0)):
        m = AO.affine_matrix(angle, t, 61, 47)
        got = AO.warp(plane, m)
        inv = np.linalg.inv(m)
        ys, xs = np.mgrid[0:61, 0:47].astype(np.float64)
        c = inv[0, 0] * xs + inv[0, 1] * ys + inv[0, 2]
        r = inv[1, 0] * xs + inv[1, 1] * ys + inv[1, 2]
        want = ndi.map_coordinates(plane, [r, c], order=1, mode='grid-constant', cval=0.0)
        assert np.abs(got - want).max() < 1e-12
        inside = (r >= 0) & (r <= 60) & (c >= 0) & (c <= 46)
        want_c = ndi.map_coordinates(plane, [r, c], order=1, mode='constant', cval=0.0)
        assert np.abs(got - want_c)[inside].max() < 1e-12


def test_warp_clips_to_the_input_range_and_keeps_cval():
    """assumption 2's _clip_warp_output: an image whose minimum is above cval = 0 keeps exact zeros outside and
    never shows a blend below its minimum along the border"""
    rng = np.random.default_rng(2)
    img = rng.integers(40, 200, (50, 50)).astype(np.uint8)
    out = AO.warp(img, AO.affine_matrix(8.0, 0.07, 50, 50))
    assert (out == 0).any() and out[out > 0].min() >= 40 and out.max() <= 199


def test_projective_path_when_the_inverse_is_not_exactly_affine():
    m = AO.affine_matrix(6.1, 0.03, 300, 300)
    inv = np.linalg.inv(m)
    plane = np.random.default_rng(4).integers(0, 256, (300, 300)).astype(np.float64)
    a = AO._warp_plane(plane, inv)
    inv2 = inv.copy()
    inv2[2] = (0.0, 0.0, 1.0)
    b = AO._warp_plane(plane, inv2)
    assert np.abs(a - b).max() < 1e-6          # the divide changes rounding only


def test_flips_are_numpy_flips():
    img = np.arange(24, dtype=np.uint8).reshape(2, 4, 3)
    p = {'n_children': 2, 'children': (AO.FLIPLR, AO.FLIPUD), 'coin': (True, True), 'rotate': 0.0, 'translate': 0.0,
         'top': 0, 'left': 0}
    assert np.array_equal(AO.augment(img, p), np.flipud(np.fliplr(img)))
    p['coin'] = (False, True)
    assert np.array_equal(AO.augment(img, p), np.flipud(img))


@pytest.mark.parametrize("mode", ["resize", "crop"])
def test_three_band_mask_path_equals_one_band_path(mode):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (120, 110, 3)).astype(np.uint8)
    m1 = (rng.random((120, 110)) > 0.6).astype(np.uint8)
    d = rng.integers(0, 900, (120, 110)).astype(np.uint16)
    s = rng.integers(1, 300, (120, 110)).astype(np.uint16)
    p = {'n_children': 2, 'children': (AO.AFFINE, AO.FLIPLR), 'coin': (False, True), 'rotate': -6.5,
         'translate': 0.04, 'top': 7, 'left': 3}
    size = (100, 100) if mode == "crop" else (64, 80)
    x3, t3 = AO.loader_sample(img, np.dstack([m1] * 3), d, s, p, mode, size)
    x1, t1 = AO.loader_sample(img, m1, d, s, p, mode, size)
    assert np.array_equal(x3, x1) and np.array_equal(t3, t1)
    assert t3.shape == (3,) + size and (t3[1] != d[:size[0], :size[1]] % 256).any()
