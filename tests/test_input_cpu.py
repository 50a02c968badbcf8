"""CPU pins of oracle/input_oracle.py against the libraries the reference itself calls (cv2, torchvision, scipy) and
against the outputs of the reference's src/preparation.py (tests/golden/live_reference.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import input_oracle as IO
from oracle import synthetic


def test_pad_and_normalize_match_cv2_and_torchvision():
    cv2 = pytest.importorskip("cv2")
    from torchvision import transforms
    from PIL import Image
    rs = np.random.RandomState(0)
    img = rs.randint(0, 256, (37, 41, 3)).astype(np.uint8)
    for method, flag in (("replicate", cv2.BORDER_REPLICATE), ("reflect", cv2.BORDER_REFLECT_101)):
        want_pad = cv2.copyMakeBorder(img.copy(), 10, 10, 7, 7, flag)
        assert np.array_equal(IO.pad_image(img, (10, 7), method), want_pad)
        tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=IO.MEAN, std=IO.STD)])
        want = tf(Image.fromarray(want_pad)).numpy()
        got = IO.image_transform(img, (10, 7), method)
        assert got.dtype == np.float32 and np.array_equal(got, want)


def test_distances_and_sizes_live_against_reference():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "live_reference.npz"))
    rs = np.random.RandomState(1)
    masks = []
    for _ in range(5):
        m, _ = synthetic.rectangles_mask(rs, 40, 52, n_rect=1, lo=4, hi=10)
        masks.append(m)
    masks = np.stack(masks)
    want_sum, want_second = g["prep_dist_sum"], g["prep_dist_second"]   # prep.update_distances / clean_distances
    got_sum, got_second = IO.two_nearest_distances(masks)
    assert got_sum.dtype == np.float16 and np.array_equal(got_sum, want_sum) and np.array_equal(got_second, want_second)
    one_sum, one_second = IO.two_nearest_distances(masks[:1])
    assert np.array_equal(one_sum, (2 * one_second).astype(np.float16))
    overlay = (masks.sum(0) > 0).astype(np.uint8)
    assert np.array_equal(IO.get_size_matrix(overlay), g["prep_size_matrix"])
