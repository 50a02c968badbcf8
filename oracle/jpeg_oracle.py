"""numpy restatement of the device JPEG decode (csrc/jpeg.cu, mcb200.jpeg) in the C semantics the kernels use, stage by
stage, so that a mismatch can be put down to one of them:

  entropy_decode(rec) -> per component int16 (blocks_h, blocks_w, 64) coefficients in natural order, padding blocks
                         included (ITU T.81 F.2.2: canonical Huffman codes, EXTEND, DC prediction reset per restart
                         interval)
  idct(rec, coefs)    -> per component uint8 (blocks_h * 8, blocks_w * 8) planes: libjpeg's "islow" integer IDCT
                         (Loeffler-Ligtenberg-Moschytz with 13-bit constants, 2 extra bits between passes, descale by
                         rounding shift) with the dequantisation folded in (the table entry read as a 16-bit signed
                         multiplier, the product and every later sum in 64 bits, the pass-1 result stored as int32), and
                         the result saturated to the sample range as the AVX2 path does
  to_rgb(rec, planes) -> uint8 (H, W, 3): libjpeg-turbo's "fancy" triangle upsampling of every half-resolution component
                         (h2v1, h2v2: 3/4 nearer + 1/4 farther sample, alternating +1/+2 or +7/+8 rounding biases; h1v2:
                         +1 above, +2 below), edge samples replicated, box replication for a component at most two
                         samples wide, then the JFIF YCbCr -> RGB conversion with 16-bit fixed-point tables

decode(path_or_bytes) runs the three.  The restatement is pinned against Pillow (libjpeg-turbo) bit for bit in
tests/test_jpeg_cpu.py.
"""
import numpy as np

from mcb200 import jpeg as J

CONST_BITS, PASS1_BITS = 13, 2
FIX = {name: int(round(v * (1 << CONST_BITS))) for name, v in (
    ("0_298631336", 0.298631336), ("0_390180644", 0.390180644), ("0_541196100", 0.541196100),
    ("0_765366865", 0.765366865), ("0_899976223", 0.899976223), ("1_175875602", 1.175875602),
    ("1_501321110", 1.501321110), ("1_847759065", 1.847759065), ("1_961570560", 1.961570560),
    ("2_053119869", 2.053119869), ("2_562915447", 2.562915447), ("3_072711026", 3.072711026))}


class _Bits:
    def __init__(self, seg):
        self.bits = np.unpackbits(np.asarray(seg, np.uint8)).tolist()
        self.pos = 0

    def get(self, n):
        if self.pos + n > len(self.bits):
            raise ValueError("entropy data ends inside a segment")
        v = 0
        for b in self.bits[self.pos:self.pos + n]:
            v = (v << 1) | b
        self.pos += n
        return v

    def decode(self, t):
        maxcode, valoff, vals = t[512:530], t[530:548], t[548:]
        code = 0
        for length in range(1, 17):
            code = (code << 1) | self.get(1)
            if code <= maxcode[length]:
                return int(vals[valoff[length] + code])
        raise ValueError("invalid Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(rec):
    comps = rec.comps
    out = [np.zeros((rec.mcuy * c["v"], rec.mcux * c["h"], 64), np.int16) for c in comps]
    mcu = 0
    for seg, count in zip(rec.segments, rec.seg_mcus):
        bits = _Bits(seg)
        pred = [0] * len(comps)
        for m in range(mcu, mcu + count):
            my, mx = divmod(m, rec.mcux)
            for ci, c in enumerate(comps):
                dc, ac = rec.huff[(0, c["td"])], rec.huff[(1, c["ta"])]
                for v in range(c["v"]):
                    for h in range(c["h"]):
                        blk = out[ci][my * c["v"] + v, mx * c["h"] + h]
                        s = bits.decode(dc)
                        pred[ci] += _extend(bits.get(s), s) if s else 0
                        blk[0] = np.int32(pred[ci]).astype(np.int16)
                        k = 1
                        while k < 64:
                            rs = bits.decode(ac)
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                if k > 63:
                                    raise ValueError("coefficient index past 63")
                                blk[J.ZIGZAG[k]] = _extend(bits.get(s), s)
                                k += 1
                            elif r == 15:
                                k += 16
                            else:
                                break
        mcu += count
    return out


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(s):
    """one islow pass over axis 1 of s (int64 (nb, 8, 8)); returns the 8 outputs before descaling, as a list"""
    c = lambda i: s[:, i]   # noqa: E731
    z2, z3 = c(2), c(6)
    z1 = (z2 + z3) * FIX["0_541196100"]
    tmp2 = z1 + z3 * -FIX["1_847759065"]
    tmp3 = z1 + z2 * FIX["0_765366865"]
    z2, z3 = c(0), c(4)
    tmp0 = (z2 + z3) << CONST_BITS
    tmp1 = (z2 - z3) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = c(7), c(5), c(3), c(1)
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * FIX["1_175875602"]
    tmp0 = tmp0 * FIX["0_298631336"]
    tmp1 = tmp1 * FIX["2_053119869"]
    tmp2 = tmp2 * FIX["3_072711026"]
    tmp3 = tmp3 * FIX["1_501321110"]
    z1 = z1 * -FIX["0_899976223"]
    z2 = z2 * -FIX["2_562915447"]
    z3 = z3 * -FIX["1_961570560"] + z5
    z4 = z4 * -FIX["0_390180644"] + z5
    tmp0 += z1 + z3
    tmp1 += z2 + z4
    tmp2 += z2 + z3
    tmp3 += z1 + z4
    return [tmp10 + tmp3, tmp11 + tmp2, tmp12 + tmp1, tmp13 + tmp0, tmp13 - tmp0, tmp12 - tmp1, tmp11 - tmp2,
            tmp10 - tmp3]


def range_limit(x):
    """the sample limit of libjpeg-turbo's AVX2 islow IDCT (what Pillow runs on x86): signed saturation to [-128, 127],
    then + 128.  jidctint.c's range-limit table agrees inside [-512, 511] and wraps beyond it; the SIMD path does not."""
    return (np.clip(x, -128, 127) + 128).astype(np.uint8)


def idct_blocks(coef, q):
    """coef int16 (nb, 64) natural order, q (64,) quantisation table -> uint8 (nb, 8, 8)"""
    x = coef.reshape(-1, 8, 8).astype(np.int64)
    qm = np.asarray(q, np.int64).astype(np.int16).astype(np.int64).reshape(8, 8)   # ISLOW_MULT_TYPE is 16-bit
    deq = x * qm[None]
    # pass 1: columns (the row index is the frequency), result kept as int32 like libjpeg's workspace
    cols = _idct_1d(deq)                       # each (nb, 8): [:, column]
    ws = np.stack([_descale(v, CONST_BITS - PASS1_BITS) for v in cols], 1).astype(np.int32).astype(np.int64)
    # pass 2: rows; ws[:, r, c] = output row r, column-frequency c
    rows = _idct_1d(ws.transpose(0, 2, 1))
    out = np.stack([_descale(v, CONST_BITS + PASS1_BITS + 3).astype(np.int32) for v in rows], 2)
    return range_limit(out.astype(np.int64))


def idct(rec, coefs):
    planes = []
    for ci, c in enumerate(rec.comps):
        bh, bw = coefs[ci].shape[:2]
        blk = idct_blocks(coefs[ci].reshape(-1, 64), rec.qt[ci]).reshape(bh, bw, 8, 8)
        planes.append(blk.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    return planes


def upsample(plane, cw, ch, rx, ry, width, height):
    """component plane (its first ch rows and cw columns are the image's samples) -> (height, width) int64"""
    s = plane[:ch, :cw].astype(np.int64)
    if rx == 1 and ry == 1:
        return s[:height, :width]
    y = np.arange(height)
    x = np.arange(width)
    if ry == 2:
        i = y >> 1
        near = np.clip(np.where(y & 1, i + 1, i - 1), 0, ch - 1)
    if rx == 2 and cw <= 2:                      # libjpeg-turbo takes the box filter for so narrow a component
        rows = s[y >> 1] if ry == 2 else s[y]
        return rows[:, x >> 1]
    if rx == 1:                                   # h1v2
        bias = np.where(y & 1, 2, 1)[:, None]
        return (3 * s[i] + s[near] + bias) >> 2
    j = x >> 1
    nj = np.clip(np.where(x & 1, j + 1, j - 1), 0, cw - 1)
    hb = np.where(x & 1, 1, 0)[None]
    if ry == 1:                                   # h2v1
        rows = s[y]
        return (3 * rows[:, j] + rows[:, nj] + 1 + hb) >> 2
    colsum = 3 * s[i] + s[near]                   # h2v2
    return (3 * colsum[:, j] + colsum[:, nj] + 8 - hb) >> 4


def to_rgb(rec, planes):
    h, w = rec.height, rec.width
    ups = [upsample(p, c["cw"], c["ch"], rec.hmax // c["h"], rec.vmax // c["v"], w, h)
           for p, c in zip(planes, rec.comps)]
    if len(ups) == 1:
        g = ups[0].astype(np.uint8)
        return np.stack([g, g, g], -1)
    t = J.ycc_tables().astype(np.int64)
    y, cb, cr = ups
    r = y + t[0][cr]
    g = y + ((t[3][cb] + t[2][cr]) >> 16)
    b = y + t[1][cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(src, stages=False):
    rec = src if isinstance(src, J.JpegRecord) else J.load(src)
    coefs = entropy_decode(rec)
    planes = idct(rec, coefs)
    rgb = to_rgb(rec, planes)
    return (rgb, coefs, planes) if stages else rgb


# ---------------------------------------------------------------------------------------------------------------------
# fixtures: JPEG files made at test time by the deterministic encoders of Pillow and cv2
# ---------------------------------------------------------------------------------------------------------------------
PIL_SAMPLING = {"444": 0, "422": 1, "420": 2}
CV2_SAMPLING = {"444": "IMWRITE_JPEG_SAMPLING_FACTOR_444", "422": "IMWRITE_JPEG_SAMPLING_FACTOR_422",
                "420": "IMWRITE_JPEG_SAMPLING_FACTOR_420", "440": "IMWRITE_JPEG_SAMPLING_FACTOR_440",
                "411": "IMWRITE_JPEG_SAMPLING_FACTOR_411"}


def content(h, w, seed=0, kind="smooth"):
    """uint8 (h, w, 3) test content: 'smooth' gradients + noise, 'primaries' 4x4-pixel patches of pure colours,
    'checker' a 1-pixel black / white checkerboard with pure-colour bars"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    if kind == "smooth":
        img = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), ((x + y) * 7) % 256], -1)
        return np.clip(img + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)
    if kind == "primaries":
        pal = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 255], [0, 0, 0], [255, 255, 0],
                        [0, 255, 255], [255, 0, 255]], np.uint8)
        return pal[rng.integers(0, 8, (-(-h // 4), -(-w // 4)))].repeat(4, 0).repeat(4, 1)[:h, :w]
    c = (((x + y) & 1) * 255).astype(np.uint8)
    img = np.stack([c, c, c], -1)
    img[(x // 3) % 5 == 0] = [255, 0, 0]
    img[(y // 5) % 7 == 0] = [0, 0, 255]
    return img


def encode_pil(img, quality=75, sampling="420", **kw):
    import io
    from PIL import Image
    b = io.BytesIO()
    im = Image.fromarray(img)
    if sampling == "gray":
        im = im.convert("L")
    else:
        kw["subsampling"] = PIL_SAMPLING[sampling]
    if quality is not None:                  # (custom qtables are written as given only without a quality)
        kw["quality"] = quality
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def encode_cv2(img, quality=75, sampling="420", restart=0, progressive=False):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
              getattr(cv2, CV2_SAMPLING[sampling])]
    if restart:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if progressive:
        params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(img[..., ::-1]), params)
    assert ok
    return buf.tobytes()


def pillow_rgb(blob):
    import io
    from PIL import Image
    return np.array(Image.open(io.BytesIO(blob)).convert("RGB"))


def scale_qtables(blob, factor):
    """the file with every 8-bit DQT entry multiplied by `factor` (clipped at 255), the entropy data unchanged: the
    dequantised coefficients grow by that factor, so the IDCT reaches far outside the sample range"""
    b = bytearray(blob)
    p = b.index(b"\xff\xdb")
    end = p + 2 + ((b[p + 2] << 8) | b[p + 3])
    q = p + 4
    while q < end:
        assert b[q] >> 4 == 0, "8-bit tables only"
        for k in range(64):
            b[q + 1 + k] = min(255, b[q + 1 + k] * factor)
        q += 65
    return bytes(b)
