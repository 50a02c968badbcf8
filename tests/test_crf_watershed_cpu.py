"""CPU pins of the dense-CRF and watershed references in oracle/crf_watershed_checks.py, which the GPU tests of
csrc/crf.cu and csrc/watershed.cu compare against:
  * crf_f64 (float64 torch) is one mean-field step away from post_oracle.dense_crf (float32 numpy) at every iteration,
    within the float32 rounding bound of the oracle's arithmetic;
  * the 13x13 window stays within TRUNCATION_BAR of a full-window filter up to the refusal bound sxy = 1.2329;
  * watershed_ref_batched equals post_oracle.minimax_watershed bit for bit, plane by plane, on every generator;
  * minimax_watershed's relief is clipped in float64 before the cast, with an explicit rule for NaN and +-Inf."""
import math

import numpy as np
import pytest
import torch

from oracle import crf_watershed_checks as K
from oracle import post_oracle as P


# ------------------------------------------------------------------------------------------------------------ dense CRF
def _crf_case(n, h, w, seed):
    rgb = K.dark_border_images(n, h, w, seed)
    imgs = K.normalised_from_rgb(rgb)
    probs = K.soft_probs(n, h, w, seed)
    return rgb, imgs, probs


def test_normalised_images_convert_back_to_their_colours():
    rgb, imgs, _ = _crf_case(2, 11, 13, 0)
    assert np.array_equal(K.crf_rgb_ref(imgs).numpy(), rgb)
    for i in range(2):
        assert np.array_equal(P.crf_rgb_image(imgs[i].numpy()), rgb[i])
    x = torch.from_numpy(np.random.RandomState(1).uniform(-20, 20, (2, 3, 7, 9)).astype(np.float32))
    assert np.array_equal(K.crf_rgb_ref(x).numpy(), np.stack([P.crf_rgb_image(v) for v in x.numpy()]))


CRF_PARAMS = [
    dict(),
    dict(srgb=3.0),
    dict(srgb=1e4, compat_gaussian=1.0, compat_bilateral=5.0),
    dict(sxy_gaussian=0.5, sxy_bilateral=0.5),
    dict(sxy_gaussian=K.SXY_OK, sxy_bilateral=K.SXY_OK),
]


@pytest.mark.parametrize("kw", CRF_PARAMS, ids=lambda kw: "-".join("%s=%g" % x for x in kw.items()) or "default")
@pytest.mark.parametrize("h,w", [(18, 21), (9, 5)])
def test_crf_f64_is_one_step_from_the_float32_oracle(kw, h, w):
    """post_oracle.dense_crf with k iterations against one float64 step from its own k - 1 iterations"""
    params = K.crf_params(**kw)
    rgb, imgs, probs = _crf_case(2, h, w, seed=h * w)
    probs[0, 1, :3, :4], probs[0, 0, :3, :4] = 0.0, 1.0      # exact 0 and 1: the 1e-5 clip
    probs[1, 1, -2:] = 0.3                                     # channels that do not sum to one
    rgb_t, p_t = torch.from_numpy(rgb), torch.from_numpy(probs)
    worst = 0.0
    for i in range(2):
        prev = None
        for k in range(1, 4):
            got = P.dense_crf(imgs[i].numpy(), probs[i], iterations=k, **params).astype(np.float64)
            ref, bar = K.crf_one_step(rgb_t[i:i + 1], p_t[i:i + 1], params, prev, model=K.ORACLE_F32)
            dev = np.abs(got - ref[0].numpy())
            assert (dev <= bar[0].numpy()).all(), (i, k, dev.max(), (dev / bar[0].numpy()).max())
            worst = max(worst, float((dev / bar[0].numpy()).max()))
            prev = torch.from_numpy(got)[None]
    assert worst > 0.0


def test_crf_f64_iterates_its_one_step():
    params = K.crf_params()
    rgb, _, probs = _crf_case(1, 14, 17, seed=3)
    rgb_t, p_t = torch.from_numpy(rgb), torch.from_numpy(probs)
    q2 = K.crf_f64(rgb_t, p_t, params, 2)
    q1 = K.crf_f64(rgb_t, p_t, params, 1)
    assert torch.allclose(K.crf_f64(rgb_t, p_t, params, 1, q0=q1), q2, rtol=0, atol=1e-14)
    step, _ = K.crf_one_step(rgb_t, p_t, params, q1)
    assert torch.allclose(step, q2, rtol=0, atol=1e-14)


@pytest.mark.parametrize("sxy", [0.5, 1.0, K.SXY_OK])
def test_crf_window_truncation_claim(sxy):
    """crf.cu: at sxy up to the refusal bound the 13x13 window stays within TRUNCATION_BAR of a full-window filter after
    5 iterations at the default compatibilities, on noise images"""
    params = K.crf_params(sxy_gaussian=sxy, sxy_bilateral=sxy)
    rs = np.random.RandomState(7)
    rgb = torch.from_numpy(rs.randint(0, 256, (3, 40, 40, 3)).astype(np.uint8))
    p1 = rs.rand(3, 40, 40).astype(np.float32)
    probs = torch.from_numpy(np.stack([1 - p1, p1], axis=1))
    win = K.crf_f64(rgb, probs, params, 5)
    full = K.crf_f64(rgb, probs, params, 5, radius=12)
    assert float((win - full).abs().max()) <= K.TRUNCATION_BAR


# ------------------------------------------------------------------------------------------------------------ watershed
def _ws_equal(prob, markers, mask, levels=256):
    got = K.watershed_ref_batched(torch.from_numpy(prob), torch.from_numpy(markers), torch.from_numpy(mask), levels)
    got = got.numpy()
    for i in range(prob.shape[0]):
        ref = P.minimax_watershed(prob[i], markers[i], mask[i], levels)
        assert np.array_equal(got[i], ref), (i, int((got[i] != ref).sum()))
    return got


def test_relief_levels_clip_before_the_cast():
    prob = np.array([-1e30, -10.0, -1.0, 0.0, 0.5, 1.0, 2.0, 1e30, np.nan, np.inf, -np.inf], np.float64)
    for levels in (2, 3, 256, 65536):
        lev = P.relief_levels(prob, levels)
        top = levels - 1
        want = [top, top, top, top, int(math.floor(0.5 * top)), 0, 0, 0, 0, 0, top]
        assert lev.tolist() == want, (levels, lev.tolist())
        assert K.watershed_levels(torch.from_numpy(prob), levels).tolist() == want
    # finite values inside [0, 1] keep the plain formula
    p = np.random.RandomState(0).rand(1000)
    assert np.array_equal(P.relief_levels(p, 256), np.floor((1.0 - p) * 255).astype(np.int64))


def test_minimax_watershed_known_answers():
    """a 1 x 7 row: markers 1 (left) and 9 (right); the ridge at x = 3 sends the middle to the lower side"""
    prob = np.array([[1.0, 0.8, 0.8, 0.2, 0.7, 0.7, 1.0]], np.float32)
    markers = np.array([[1, 0, 0, 0, 0, 0, 9]], np.int32)
    assert P.minimax_watershed(prob, markers, np.ones((1, 7), bool)).tolist() == [[1, 1, 1, 1, 9, 9, 9]]
    # a NaN pixel is lowest ground, a -Inf pixel a wall at the top level: both still flood, -Inf last
    prob = np.array([[1.0, np.nan, 0.5, -np.inf, 0.5, 1.0]], np.float32)
    markers = np.array([[4, 0, 0, 0, 0, 2]], np.int32)
    assert P.minimax_watershed(prob, markers, np.ones((1, 6), bool)).tolist() == [[4, 4, 4, 2, 2, 2]]


def test_watershed_ref_batched_generators():
    cases = []
    m, order = K.serpentine(40, 37, period=2)
    rs = np.random.RandomState(0)
    n = order.max() + 1
    rise = np.where(m, 1.0 - order / n, 0.0)
    fall = np.where(m, order / n, 0.0)
    noise = np.where(m, 0.3 + 0.7 * rs.rand(*m.shape), 0.0)
    for prob in (rise, fall, noise):
        mk = np.zeros(m.shape, np.int32)
        mk[order == 0], mk[order == n - 1] = 3, 2
        cases.append((prob, mk, m))
    s, sorder = np.zeros(m.shape, bool), np.full(m.shape, -1, np.int64)
    s[:32, :32], sorder[:32, :32] = K.spiral(32)               # inside the plane's first tile
    assert sorder.max() + 1 > 4 * 32
    mk = np.zeros(m.shape, np.int32)
    mk[sorder == 0] = 7
    cases.append((np.where(s, 0.6, 0.0), mk, s))
    mk = np.zeros(m.shape, np.int32)
    mk[sorder == sorder.max()], mk[sorder == 0] = 5, 6
    cases.append((np.where(s, 0.2 + 0.6 * rs.rand(*m.shape), 0.0), mk, s))
    prob, mk, mask = K.plateau_with_markers(40, 37, {(3, 3): 2 ** 31 - 1, (3, 5): 1, (30, 30): 40, (20, 2): 9})
    cases.append((prob, mk, mask))
    prob = K.blob_map(rs, 40, 37, 2.5)
    cases.append((prob, P.label(prob > 0.7).astype(np.int32), prob > 0.35))
    prob = np.stack([c[0] for c in cases]).astype(np.float32)
    markers = np.stack([c[1] for c in cases])
    mask = np.stack([c[2] for c in cases])
    _ws_equal(prob, markers, mask)
    _ws_equal(prob.astype(np.float64), markers, mask, levels=65536)


@pytest.mark.parametrize("levels", [2, 3, 256, 65536])
def test_watershed_ref_batched_values_and_markers(levels):
    rs = np.random.RandomState(levels)
    prob = np.stack([K.blob_map(rs, 33, 31, 2.0) for _ in range(6)]).astype(np.float64)
    prob = prob * 20.0 - 10.0 if levels == 3 else prob
    prob[1, rs.rand(33, 31) < 0.05] = np.nan
    prob[1, rs.rand(33, 31) < 0.05] = np.inf
    prob[1, rs.rand(33, 31) < 0.05] = -np.inf
    markers = np.stack([P.label(p > 0.7) for p in prob]).astype(np.int32)
    markers[2, rs.rand(33, 31) < 0.05] = -3                    # negative values are no markers
    markers[3, 0, :] = np.arange(1, 32)                         # adjacent markers on the border
    markers[4] = 0                                              # no marker: all zeros
    mask = prob > 0.3
    mask[5] = False                                             # markers outside the mask
    got = _ws_equal(prob, markers, mask, levels)
    assert (got[4] == 0).all()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 20), (20, 1), (33, 31)])
def test_watershed_ref_batched_shapes(h, w):
    rs = np.random.RandomState(h * w)
    prob = rs.rand(3, h, w).astype(np.float32)
    markers = np.where(rs.rand(3, h, w) < 0.2, rs.randint(1, 5, (3, h, w)), 0).astype(np.int32)
    markers[2] = rs.randint(1, 9, (h, w))                       # every pixel a marker
    _ws_equal(prob, markers, rs.rand(3, h, w) < 0.8)
