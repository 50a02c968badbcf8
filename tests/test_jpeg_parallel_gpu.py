"""The parallel entropy decode (mcb_jpeg_entropy_decode_parallel) against the one-thread-per-segment kernel and
oracle/jpeg_oracle.py: coefficients bit for bit on every image that decodes, status equal on every image, over long
scans, scan lengths at a subsequence boundary, restart intervals, grayscale, flat tiles (whose periodic stream can lock
onto a wrong phase), one-length Huffman tables that resynchronise poorly, planted errors at and between subsequence
boundaries, truncation inside one restart interval, and a CUDA graph replay.  The speculation counters show that both
the held and the corrected branches run, with correction chains longer than one subsequence."""
import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as O
from oracle import jpeg_reencode as R

pytestmark = pytest.mark.gpu

SAMPLINGS = ["444", "422", "420", "440", "gray"]


def _sub_bytes():
    from mcb200 import _lib as L
    return L.lib.mcb_jpeg_subsequence_bits() // 8


def _encode(img, sampling, quality=75, **kw):
    if sampling == "440" or kw.get("restart"):
        return O.encode_cv2(img, quality, sampling, **kw)
    return O.encode_pil(img, quality, sampling, **kw)


def _noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _both(recs, cuda):
    """(parallel coef, status, counters), (serial coef, status), block ranges of the images"""
    from mcb200 import jpeg as J
    pk = J.pack_batch(recs)
    b = J.DeviceBatch(pk, cuda)
    b.entropy_decode()
    par = (b.coef.cpu().numpy(), b.status.cpu().numpy(), b.counters())
    b.entropy_decode_serial()
    ser = (b.coef.cpu().numpy(), b.status.cpu().numpy())
    first = list(pk["images"][:, 10]) + [pk["n_blocks"]]
    return par, ser, [(first[i], first[i + 1]) for i in range(len(recs))]


def _check(recs, cuda, oracle=False, what=""):
    """parallel == serial (== oracle) on every status-0 image, statuses equal; returns (status, counters)"""
    (cp, sp, cnt), (cs, ss), ranges = _both(recs, cuda)
    np.testing.assert_array_equal(sp, ss, err_msg="status %s" % what)
    for i, (a, b) in enumerate(ranges):
        if sp[i]:
            continue
        np.testing.assert_array_equal(cp[a:b], cs[a:b], err_msg="coefficients %s #%d (%s)" % (what, i, recs[i].name))
        if oracle:
            ref = np.concatenate([c.reshape(-1, 64) for c in O.entropy_decode(recs[i])])
            np.testing.assert_array_equal(cp[a:b], ref, err_msg="oracle %s #%d" % (what, i))
    return sp, cnt


def test_long_scans_thousands_of_subsequences(mcb, cuda):
    """2048x2048 quality-100 noise: one segment of tens of thousands of subsequences per image"""
    from mcb200 import jpeg as J
    recs = [J.load(O.encode_pil(_noise(2048, 2048, s), 100, sampling), "noise%s" % sampling)
            for s, sampling in enumerate(("444", "420"))]
    assert min(len(r.segments[0]) for r in recs) > 2000 * _sub_bytes()
    st, cnt = _check(recs, cuda, what="noise")
    assert not st.any()
    assert cnt[0] > 2000


def test_scan_lengths_around_a_subsequence_multiple(mcb, cuda):
    """segments of k * subsequence bytes - 1, + 0 and + 1, long enough to be split"""
    from mcb200 import jpeg as J
    sub = _sub_bytes()
    found = {}
    for seed in range(4000):
        s = SAMPLINGS[seed % 5]
        blob = _encode(_noise(64, 64 + seed % 24, seed), s, 60 + seed % 40)
        r = J.load(blob, "len%d" % seed)
        n = len(r.segments[0])
        d = (n + 1) % sub - 1
        if n > (J.SPLIT_MIN_SUBSEQUENCES + 1) * sub and d in (-1, 0, 1) and (d, r.height, r.width) not in found:
            found[(d, r.height, r.width)] = r
        if len({k[0] for k in found}) == 3 and len(found) >= 6:
            break
    assert {k[0] for k in found} == {-1, 0, 1}
    by_size = {}
    for (d, h, w), r in found.items():
        by_size.setdefault((h, w), []).append(r)
    for recs in by_size.values():
        st, _ = _check(recs, cuda, oracle=True, what="boundary lengths")
        assert not st.any()


@pytest.mark.parametrize("restart", [1, 4, 7])
def test_restart_intervals(mcb, cuda, restart):
    """restart segments shorter than one subsequence (smooth content) and longer (quality-100 noise), in one batch"""
    from mcb200 import jpeg as J
    recs = []
    for i, s in enumerate(SAMPLINGS[:4]):
        recs.append(J.load(_encode(O.content(300, 300, seed=i), s, 80, restart=restart), "smooth%s" % s))
        recs.append(J.load(_encode(_noise(300, 300, i), s, 100, restart=restart), "noise%s" % s))
    sub = _sub_bytes()
    lens = [len(x) for r in recs for x in r.segments]
    assert min(lens) < sub and max(lens) > sub
    st, _ = _check(recs, cuda, oracle=restart == 7, what="restart %d" % restart)
    assert not st.any()


def test_grayscale(mcb, cuda):
    from mcb200 import jpeg as J
    recs = [J.load(O.encode_pil(_noise(300, 300, q) if q == 100 else O.content(300, 300, seed=q), q, "gray"),
                   "gray%d" % q) for q in (50, 90, 100)]
    st, _ = _check(recs, cuda, oracle=True, what="gray")
    assert not st.any()


def test_flat_tiles_every_sampling(mcb, cuda):
    """blocks of 'DC diff 0 + EOB': a periodic stream a misaligned guess can follow for ever"""
    from mcb200 import jpeg as J
    for s in SAMPLINGS:
        recs = [J.load(_encode(np.full((600, 600, 3), v, np.uint8), s, q), "flat%s_%d" % (s, v))
                for v, q in ((128, 75), (37, 95), (250, 50))]
        st, _ = _check(recs, cuda, oracle=True, what="flat %s" % s)
        assert not st.any()


def test_one_length_huffman_tables(mcb, cuda):
    """files re-encoded with every DC code of one length and every AC code of another: Pillow decodes them to the
    original pixels, and the device decode must still equal the serial one where the guesses fail"""
    from mcb200 import jpeg as J
    held = corrected = chain = 0
    for s in SAMPLINGS:
        for shared in (True, False):
            blobs = [O.encode_pil(O.content(256, 256, seed=3), 90, s) if s != "440" else
                     O.encode_cv2(O.content(256, 256, seed=3), 90, s),
                     O.encode_pil(_noise(256, 256, 4), 95, "444" if s == "440" else s)]
            recs = []
            for i, b in enumerate(blobs):
                nb = R.reencode(b, shared=shared)
                np.testing.assert_array_equal(O.pillow_rgb(nb), O.pillow_rgb(b))
                recs.append(J.load(nb, "oneLength%s_%d_%d" % (s, shared, i)))
            st, cnt = _check(recs, cuda, oracle=True, what="one-length %s" % s)
            assert not st.any()
            held, corrected, chain = held + cnt[0], corrected + cnt[1], max(chain, cnt[2])
    assert held > 0 and corrected > 0, (held, corrected)
    assert chain >= 2, chain


def test_planted_errors_at_and_between_boundaries(mcb, cuda):
    """status 2 (invalid code), 3 (index past 63) and 1 (data ends) planted at every subsequence boundary and in the
    middle of subsequences of one scan, each in its own image of one batch"""
    from mcb200 import jpeg as J
    bits = 8 * _sub_bytes()
    base = O.encode_pil(O.content(256, 256, seed=9), 95, "420")
    nbits = 8 * len(J.load(base).segments[0])
    positions = sorted({k * bits + off for k in range(1, nbits // bits) for off in (0, bits // 2)})[:24]
    recs, want = [], []
    for p in positions:
        for kind in (2, 3):
            recs.append(J.load(R.reencode(base, shared=False, corrupt={p: kind}), "kind%d@%d" % (kind, p)))
            want.append(kind)
        r = J.load(R.reencode(base, shared=False), "cut@%d" % p)
        r.segments = [r.segments[0][:p // 8]]
        recs.append(r)
        want.append(1)
    recs.append(J.load(base, "intact"))
    want.append(0)
    st, _ = _check(recs, cuda, what="planted errors")
    assert st.tolist() == want


def test_truncation_inside_one_restart_segment(mcb, cuda):
    from mcb200 import jpeg as J
    recs = [J.load(_encode(_noise(300, 300, i), "420", 100, restart=4), "rst%d" % i) for i in range(3)]
    mid = len(recs[1].segments) // 2
    recs[1].segments[mid] = recs[1].segments[mid][:len(recs[1].segments[mid]) // 2]
    st, _ = _check(recs, cuda, what="truncated restart segment")
    assert st.tolist() == [0, 1, 0]


def test_graph_capture_and_replay(mcb, cuda):
    """the three launches captured into a CUDA graph, replayed once: the same coefficients as the serial kernel"""
    from mcb200 import jpeg as J
    recs = [J.load(_encode(O.content(300, 300, seed=i), s, 90, **({"restart": 5} if i == 2 else {})), "g%d" % i)
            for i, s in enumerate(["444", "420", "422", "gray"])]
    pk = J.pack_batch(recs)
    b = J.DeviceBatch(pk, cuda)
    b.entropy_decode_serial()
    ref = b.coef.clone()
    s = torch.cuda.Stream(cuda)
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        b.coef.fill_(-1)
        with torch.cuda.graph(g, stream=s):
            b.entropy_decode()
    torch.cuda.current_stream().wait_stream(s)
    b.coef.fill_(-1)
    b.status.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    assert not b.status.cpu().numpy().any()
    assert torch.equal(b.coef, ref)
