"""The JPEG decode restatement (oracle/jpeg_oracle.py) against Pillow (libjpeg-turbo) bit for bit, and the host parser of
mcb200.jpeg: the forms it takes, the ones it names and refuses, malformed files, and the C ABI symbols of csrc/jpeg.cu."""
import ctypes
import io
import os

import numpy as np
import pytest

from oracle import jpeg_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (8, 8), (16, 16), (9, 17), (17, 9), (257, 255), (256, 256), (300, 300)]
SAMPLINGS = ["444", "422", "420", "440"]


def _encode(img, sampling, quality=75, **kw):
    """Pillow writes 4:4:4 / 4:2:2 / 4:2:0 and grayscale; cv2 writes 4:4:0 and restart intervals"""
    if sampling == "440" or kw.get("restart"):
        return O.encode_cv2(img, quality, sampling, **kw)
    return O.encode_pil(img, quality, sampling, **kw)


def _check(blob):
    got = O.decode(blob)
    want = O.pillow_rgb(blob)
    assert got.shape == want.shape and got.dtype == np.uint8
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("sampling", SAMPLINGS + ["gray"])
def test_oracle_equals_pillow_at_every_size(mcb, size, sampling):
    _check(_encode(O.content(*size, seed=size[0] * 1000 + size[1]), sampling))


@pytest.mark.parametrize("quality", [1, 50, 75, 95, 100])
@pytest.mark.parametrize("sampling", SAMPLINGS + ["gray"])
def test_oracle_equals_pillow_at_every_quality(mcb, quality, sampling):
    _check(_encode(O.content(300, 300, seed=quality), sampling, quality))


@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("restart", [1, 4])
def test_oracle_equals_pillow_with_restart_intervals(mcb, sampling, restart):
    blob = _encode(O.content(61, 77, seed=restart), sampling, 80, restart=restart)
    from mcb200 import jpeg as J
    rec = J.load(blob)
    assert rec.restart == restart and len(rec.segments) > 1
    _check(blob)


@pytest.mark.parametrize("sampling", ["444", "420", "gray"])
def test_oracle_equals_pillow_with_optimised_tables(mcb, sampling):
    _check(O.encode_pil(O.content(255, 257, seed=3), 90, sampling, optimize=True))


@pytest.mark.parametrize("sampling", ["444", "422", "420"])
def test_oracle_equals_pillow_with_16_bit_quantisation_tables(mcb, sampling):
    """qtables with entries > 255 are written as 16-bit DQT in an SOF1 (extended sequential) frame"""
    from mcb200 import jpeg as J
    q = [[min(1 + 9 * i, 1000) for i in range(64)], [min(2 + 11 * i, 700) for i in range(64)]]
    blob = O.encode_pil(O.content(64, 48, seed=5), None, sampling, qtables=q)
    marks = [blob[i + 1] for i in range(len(blob) - 1) if blob[i] == 0xFF]
    assert 0xC1 in marks
    rec = J.load(blob)
    assert rec.qt.max() > 255
    _check(blob)


@pytest.mark.parametrize("kind", ["primaries", "checker"])
@pytest.mark.parametrize("sampling", SAMPLINGS)
@pytest.mark.parametrize("quality", [75, 95, 100])
def test_oracle_equals_pillow_on_saturated_content(mcb, kind, sampling, quality):
    """pure primaries and 1-pixel checkerboards push the IDCT outside the sample range: the limit decides those pixels"""
    from mcb200 import jpeg as J
    blob = _encode(O.content(120, 136, seed=7, kind=kind), sampling, quality)
    if kind == "checker" and quality < 100:
        rec = J.load(blob)
        coefs = O.entropy_decode(rec)
        assert any(_idct_out_of_range(coefs[ci], rec.qt[ci], margin=1) for ci in range(len(rec.comps)))
    _check(blob)


def _idct_out_of_range(coef, q, margin=10):
    """does any IDCT output of these blocks fall more than `margin` outside [-128, 127] (float IDCT)"""
    from scipy.fft import idctn
    x = coef.reshape(-1, 8, 8).astype(np.float64) * np.asarray(q, np.float64).reshape(8, 8)
    y = idctn(x, axes=(1, 2), norm="ortho")
    return bool((y > 127 + margin).any() or (y < -128 - margin).any())


@pytest.mark.parametrize("kind", ["primaries", "checker"])
def test_oracle_equals_pillow_far_outside_the_sample_range(mcb, kind):
    """quantisation tables scaled by 4 after encoding push the IDCT beyond +-512, where jidctint.c's range-limit table
    would wrap and libjpeg-turbo's AVX2 path (Pillow on x86) saturates: the restatement saturates"""
    from mcb200 import jpeg as J
    blob = O.scale_qtables(O.encode_pil(O.content(64, 64, seed=1, kind=kind), 100, "444"), 4)
    rec = J.load(blob)
    coefs = O.entropy_decode(rec)
    assert any(_idct_out_of_range(coefs[ci], rec.qt[ci], margin=384) for ci in range(3))
    _check(blob)


def test_range_limit_saturates():
    x = np.array([-100000, -1153, -513, -512, -129, -128, -1, 0, 127, 128, 511, 512, 1029, 100000])
    want = [0, 0, 0, 0, 0, 0, 127, 128, 255, 255, 255, 255, 255, 255]
    np.testing.assert_array_equal(O.range_limit(x), want)


def _cmyk_jpeg():
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.zeros((16, 16, 4), np.uint8), "CMYK").save(b, "JPEG")
    return b.getvalue()


def _partial_scan_jpeg():
    """a 3-component frame whose first scan holds only the luma component (a multi-scan sequential file)"""
    blob = bytearray(O.encode_pil(O.content(16, 16), 75, "444"))
    p = blob.index(b"\xff\xda")
    ns = blob[p + 4]
    assert ns == 3
    hdr = bytes(blob[p + 5:p + 5 + 2 * ns])
    new = b"\xff\xda" + (2 + 1 + 2 + 3).to_bytes(2, "big") + b"\x01" + hdr[:2] + bytes(blob[p + 5 + 2 * ns:p + 8 + 2 * ns])
    return bytes(blob[:p]) + new + bytes(blob[p + 8 + 2 * ns:])


@pytest.mark.parametrize("make,form", [
    (lambda: O.encode_cv2(O.content(32, 32), 75, "420", progressive=True), "progressive"),
    (lambda: O.encode_cv2(O.content(32, 32), 75, "411"), "sampling factors"),
    (_cmyk_jpeg, "CMYK"),
    (_partial_scan_jpeg, "multi-scan"),
], ids=["progressive", "411", "cmyk", "multi-scan"])
def test_parser_names_unsupported_forms(mcb, make, form):
    from mcb200 import jpeg as J
    blob = make()
    with pytest.raises(NotImplementedError, match=form):
        J.parse_jpeg(blob, "tile.jpg")
    assert O.pillow_rgb(blob).ndim == 3          # Pillow reads them: they reach the loaders' host path


def test_read_jpeg_leaves_other_files_to_the_host(mcb, tmp_path):
    from PIL import Image
    from mcb200 import jpeg as J
    png = tmp_path / "a.png"
    Image.fromarray(O.content(8, 8)).save(png)
    prog = tmp_path / "p.jpg"
    prog.write_bytes(O.encode_cv2(O.content(32, 32), 75, "420", progressive=True))
    base = tmp_path / "b.jpg"
    base.write_bytes(O.encode_pil(O.content(32, 32)))
    assert J.read_jpeg(str(png)) is None and J.read_jpeg(str(prog)) is None
    rec = J.read_jpeg(str(base))
    assert isinstance(rec, J.JpegRecord) and rec.name == str(base)
    import pickle
    np.testing.assert_array_equal(O.decode(pickle.loads(pickle.dumps(rec))), O.pillow_rgb(base.read_bytes()))


def test_truncated_file_parses_and_the_decode_reports_it(mcb):
    """a file cut inside its entropy data parses (the device decode reports it); the oracle fails the same way"""
    from mcb200 import jpeg as J
    blob = O.encode_pil(O.content(64, 64, seed=1), 90)
    cut = blob[:len(blob) * 2 // 3]
    rec = J.parse_jpeg(cut, "cut.jpg")
    with pytest.raises(ValueError, match="ends inside"):
        O.entropy_decode(rec)


@pytest.mark.parametrize("where", ["header", "marker-length", "dqt", "dht", "sof", "sos", "soi"])
def test_malformed_headers_raise_value_error(mcb, where):
    from mcb200 import jpeg as J
    blob = bytearray(O.encode_pil(O.content(32, 32), 75))

    def at(marker):
        return blob.index(marker)
    if where == "header":
        bad = bytes(blob[:at(b"\xff\xc4") + 10])                  # ends before the scan
    elif where == "marker-length":
        p = at(b"\xff\xdb")
        blob[p + 2:p + 4] = (len(blob)).to_bytes(2, "big")
        bad = bytes(blob)
    elif where == "dqt":
        p = at(b"\xff\xdb")
        blob[p + 4] = 0x27                                         # precision 2
        bad = bytes(blob)
    elif where == "dht":
        p = at(b"\xff\xc4")
        blob[p + 5:p + 21] = bytes([255] * 16)                     # more symbols than the marker holds
        bad = bytes(blob)
    elif where == "sof":
        p = at(b"\xff\xc0")
        blob[p + 2:p + 4] = (20).to_bytes(2, "big")                # length disagrees with the component count
        bad = bytes(blob)
    elif where == "sos":
        p = at(b"\xff\xda")
        blob[p + 6] = 0x77                                         # Huffman table ids 7
        bad = bytes(blob)
    else:
        bad = b"\x00\x00" + bytes(blob[2:])
    with pytest.raises(ValueError):
        J.parse_jpeg(bad, "bad.jpg")


def test_batch_of_mixed_sizes_is_refused(mcb):
    from mcb200 import jpeg as J
    a = J.load(O.encode_pil(O.content(16, 16)))
    b = J.load(O.encode_pil(O.content(16, 24)))
    with pytest.raises(ValueError, match="one size"):
        J.pack_batch([a, b])


def test_pack_batch_layout(mcb):
    """the per-image / per-segment tables that csrc/jpeg.cu reads"""
    from mcb200 import jpeg as J
    r1 = J.load(O.encode_pil(O.content(20, 20), 75, "420"))
    r2 = J.load(O.encode_cv2(O.content(20, 20), 75, "444", restart=2))
    pk = J.pack_batch([r1, r2])
    im, sg = pk["images"], pk["segments"]
    assert im.shape == (2, J.IMAGE_WORDS) and sg.shape[1] == J.SEGMENT_WORDS
    assert list(im[0, :6]) == [3, 2, 2, 2, 0, 1] and list(im[1, :6]) == [3, 3, 1, 1, 1, 5]
    assert list(im[0, 6:10]) == [2, 2, 4, 4] and im[0, 10] == 0 and im[0, 20] == 16 and im[0, 30] == 20
    assert im[1, 10] == 24 and pk["n_blocks"] == 24 + 27
    assert (sg[:, 0] == [0] + [1] * 5).all() and sg[1:, 4].tolist() == [2, 2, 2, 2, 1]
    assert (np.diff(sg[:, 1]) == sg[:-1, 2]).all()


def test_jpeg_abi_symbols_are_exported(mcb):
    lib = ctypes.CDLL(os.path.join(ROOT, "open-solution-mapping-challenge_b200", "libmcb200.so"))
    for name in ("mcb_jpeg_entropy_decode", "mcb_jpeg_idct", "mcb_jpeg_upsample_rgb"):
        assert hasattr(lib, name), name
