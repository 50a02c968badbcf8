"""GPU parity of the device JPEG decode (csrc/jpeg.cu through mcb200.jpeg): the file matrix of tests/test_jpeg_cpu.py
against Pillow bit for bit and stage by stage against oracle/jpeg_oracle.py, the training and inference batch sizes
with mixed files in one launch, and a truncated file reported for its own image only."""
import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as O

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (8, 8), (16, 16), (9, 17), (17, 9), (257, 255), (256, 256), (300, 300)]
SAMPLINGS = ["444", "422", "420", "440"]


def _encode(img, sampling, quality=75, **kw):
    if sampling == "440" or kw.get("restart"):
        return O.encode_cv2(img, quality, sampling, **kw)
    return O.encode_pil(img, quality, sampling, **kw)


def _matrix():
    """{(h, w): [blob, ...]}: every size x sampling (gray too), every quality x sampling at 300x300, restart intervals
    1 and 4, optimised Huffman tables, 16-bit quantisation tables, saturated content and an IDCT far outside the sample
    range"""
    cases = {}

    def add(blob):
        h, w = O.pillow_rgb(blob).shape[:2]
        cases.setdefault((h, w), []).append(blob)
    for size in SIZES:
        for s in SAMPLINGS + ["gray"]:
            add(_encode(O.content(*size, seed=size[0] * 1000 + size[1]), s))
    for q in (1, 50, 75, 95, 100):
        for s in SAMPLINGS + ["gray"]:
            add(_encode(O.content(300, 300, seed=q), s, q))
    for r in (1, 4):
        for s in SAMPLINGS:
            add(_encode(O.content(300, 300, seed=r), s, 80, restart=r))
    for s in ("444", "420", "gray"):
        add(O.encode_pil(O.content(300, 300, seed=3), 90, s, optimize=True))
    q16 = [[min(1 + 9 * i, 1000) for i in range(64)], [min(2 + 11 * i, 700) for i in range(64)]]
    for s in ("444", "422", "420"):
        add(O.encode_pil(O.content(300, 300, seed=5), None, s, qtables=q16))
    for kind in ("primaries", "checker"):
        for s in SAMPLINGS:
            for q in (75, 95, 100):
                add(_encode(O.content(300, 300, seed=7, kind=kind), s, q))
        add(O.scale_qtables(O.encode_pil(O.content(64, 64, seed=1, kind=kind), 100, "444"), 4))
    return cases


def _oracle_blocks(rec):
    """oracle coefficients and planes in pack_batch's block order"""
    rgb, coefs, planes = O.decode(rec, stages=True)
    cb = np.concatenate([c.reshape(-1, 64) for c in coefs])
    pb = np.concatenate([p.reshape(p.shape[0] // 8, 8, p.shape[1] // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)
                         for p in planes])
    return rgb, cb, pb


def test_matrix_equals_pillow_and_every_stage_the_oracle(mcb, cuda):
    from mcb200 import jpeg as J
    total = 0
    for size, blobs in _matrix().items():
        recs = [J.load(b, "case%d" % i) for i, b in enumerate(blobs)]
        out, coef, planes, st = J.decode_records(recs, cuda)
        assert not st.any()
        out, coef, planes = out.cpu().numpy(), coef.cpu().numpy(), planes.cpu().numpy()
        at = 0
        for i, (b, r) in enumerate(zip(blobs, recs)):
            rgb, cb, pb = _oracle_blocks(r)
            np.testing.assert_array_equal(coef[at:at + len(cb)], cb, err_msg="coefficients %s #%d" % (size, i))
            np.testing.assert_array_equal(planes[at:at + len(cb)], pb, err_msg="IDCT %s #%d" % (size, i))
            np.testing.assert_array_equal(out[i], rgb, err_msg="upsample / colour %s #%d" % (size, i))
            np.testing.assert_array_equal(out[i], O.pillow_rgb(b), err_msg="Pillow %s #%d" % (size, i))
            at += len(cb)
            total += 1
    assert total > 100


@pytest.mark.parametrize("n", [20, 64])
def test_training_and_inference_batch_sizes_with_mixed_files(mcb, cuda, n):
    """one launch over n 300x300 tiles of mixed quality, sampling and restart interval"""
    from mcb200 import jpeg as J
    rng = np.random.default_rng(n)
    blobs = []
    for i in range(n):
        q = int(rng.choice([60, 75, 90, 95]))
        s = ["444", "420", "422", "440", "gray"][i % 5]
        r = [0, 0, 1, 4, 7][(i // 5) % 5] if s != "gray" else 0
        blobs.append(_encode(O.content(300, 300, seed=100 + i), s, q, **({"restart": r} if r else {})))
    out = J.decode_jpeg_batch(blobs, cuda).cpu().numpy()
    assert out.shape == (n, 300, 300, 3)
    for i, b in enumerate(blobs):
        np.testing.assert_array_equal(out[i], O.pillow_rgb(b), err_msg="tile %d" % i)


def test_truncated_file_fails_alone(mcb, cuda):
    from mcb200 import jpeg as J
    blobs = [O.encode_pil(O.content(300, 300, seed=i), 85, "420") for i in range(5)]
    blobs[2] = blobs[2][:len(blobs[2]) // 2]
    recs = [J.load(b, "tile%d.jpg" % i) for i, b in enumerate(blobs)]
    out, _, _, st = J.decode_records(recs, cuda)
    assert st[2] == 1 and not np.delete(st, 2).any()
    out = out.cpu().numpy()
    for i in (0, 1, 3, 4):
        np.testing.assert_array_equal(out[i], O.pillow_rgb(blobs[i]))
    with pytest.raises(ValueError, match="tile2.jpg"):
        J.decode_jpeg_batch(recs, cuda)
    torch.cuda.synchronize()
