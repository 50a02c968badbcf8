"""JPEG tiles decoded on the device: this module hides the file format.

The host parses the markers (SOI, APPn, DQT, DHT, SOF0/SOF1, DRI, SOS, EOI), checks every length and index, removes
the byte stuffing, splits the entropy-coded data at its restart markers into independent segments and builds the
canonical Huffman lookup tables.  `decode_jpeg_batch` packs a batch into one byte buffer plus per-image and per-segment
tables and runs the three stages of csrc/jpeg.cu: entropy decode (parallel inside each long segment: speculate,
resolve, emit), libjpeg's islow IDCT, and libjpeg-turbo's fancy upsampling + YCbCr -> RGB.  The result is what
`np.array(Image.open(f).convert('RGB'))` returns, bit for bit.

Supported: sequential Huffman JPEG (SOF0 / SOF1) with 8-bit samples, one scan holding every component, grayscale or
YCbCr (JFIF or Adobe transform 1), each component sampled at 1 or 1/2 of the largest factor in either direction (4:4:4,
4:2:2, 4:2:0, 4:4:0), any restart interval, 8- or 16-bit quantisation tables, any image size.  Every other form raises
NotImplementedError naming it; a malformed file raises ValueError.
"""
import os

import numpy as np

# natural (row-major) position of the k-th coefficient of the zigzag sequence
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
    47, 55, 62, 63], np.int32)

LOOKAHEAD = 9
# int32 words of one Huffman table: [0, 512) lookahead (length << 8 | symbol, 0 for longer codes),
# [512, 530) maxcode by length (index 17 is a sentinel), [530, 548) value offset by length, [548, 804) symbols
HUFF_WORDS = (1 << LOOKAHEAD) + 18 + 18 + 256
# int32 words of one image row, one segment row (see include/mcb200.h, mcb_jpeg_* )
IMAGE_WORDS = 6 + 3 * 10
SEGMENT_WORDS = 5

_SOF_NAMES = {0xC2: "progressive JPEG (SOF2)", 0xC3: "lossless JPEG (SOF3)", 0xC5: "differential sequential JPEG (SOF5)",
              0xC6: "differential progressive JPEG (SOF6)", 0xC7: "differential lossless JPEG (SOF7)",
              0xC9: "arithmetic-coded JPEG (SOF9)", 0xCA: "arithmetic-coded progressive JPEG (SOF10)",
              0xCB: "arithmetic-coded lossless JPEG (SOF11)", 0xCD: "arithmetic-coded JPEG (SOF13)",
              0xCE: "arithmetic-coded JPEG (SOF14)", 0xCF: "arithmetic-coded JPEG (SOF15)"}


class JpegRecord:
    """a parsed, supported JPEG file: everything the device decode needs, picklable (DataLoader workers can return it)"""
    __slots__ = ("name", "height", "width", "comps", "hmax", "vmax", "mcux", "mcuy", "qt", "huff", "restart",
                 "segments", "seg_mcus")

    def __getstate__(self):
        return {k: getattr(self, k) for k in self.__slots__}

    def __setstate__(self, state):
        for k, v in state.items():
            setattr(self, k, v)


def _u16(b, p):
    return (int(b[p]) << 8) | int(b[p + 1])


def build_huffman(counts, symbols, name, is_dc):
    """canonical Huffman code (ITU T.81 Annex C) -> int32 table of HUFF_WORDS words"""
    t = np.zeros(HUFF_WORDS, np.int32)
    look, maxcode, valoff, vals = (t[:512], t[512:530], t[530:548], t[548:])
    vals[:len(symbols)] = symbols
    if is_dc and any(s > 15 for s in symbols):
        raise ValueError("%s: DC Huffman symbol > 15" % name)
    code, k = 0, 0
    maxcode[:] = -1
    for length in range(1, 17):
        n = counts[length - 1]
        if n:
            valoff[length] = k - code
            for _ in range(n):
                if length <= LOOKAHEAD:
                    shift = LOOKAHEAD - length
                    look[code << shift:(code + 1) << shift] = (length << 8) | symbols[k]
                code += 1
                k += 1
            maxcode[length] = code - 1
        if code > (1 << length):
            raise ValueError("%s: Huffman code lengths overflow the code space" % name)
        code <<= 1
    maxcode[17] = 0x7FFFFFFF
    return t


def _unstuff(data, name):
    """scan bytes (from the first entropy byte) -> (segments split at RSTn with FF 00 -> FF, offset of the marker that
    ended the scan or len(data) when the file ends inside it)"""
    ff = np.flatnonzero(data[:-1] == 0xFF)
    nxt = data[ff + 1]
    marker = ff[(nxt != 0x00) & (nxt != 0xFF)]
    rst = (data[marker + 1] >= 0xD0) & (data[marker + 1] <= 0xD7)
    ends = np.flatnonzero(~rst)
    end = int(marker[ends[0]]) if len(ends) else len(data)
    rst_at = marker[rst]
    rst_at = rst_at[rst_at < end]
    # fill bytes (FF FF ...) before a marker and the 00 of every stuffed FF 00 are dropped
    drop = np.zeros(len(data), bool)
    drop[ff[nxt == 0x00] + 1] = True
    drop[ff[nxt == 0xFF]] = True
    keep = ~drop
    bounds = [0] + [int(p) for p in rst_at] + [end]
    segments = []
    for i in range(len(bounds) - 1):
        a = bounds[i] + (2 if i else 0)
        b = bounds[i + 1]
        seg = data[a:b][keep[a:b]]
        segments.append(np.ascontiguousarray(seg))
    for i, p in enumerate(rst_at):
        if int(data[p + 1]) != 0xD0 + (i % 8):
            raise ValueError("%s: restart markers out of sequence" % name)
    return segments, end


def parse_jpeg(blob, name="<bytes>"):
    """bytes of one JPEG file -> JpegRecord.  NotImplementedError names an unsupported form, ValueError a malformed
    file (a file that ends inside its entropy-coded data parses: the device decode reports it)."""
    b = np.frombuffer(bytes(blob), np.uint8)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise ValueError("%s: not a JPEG file (no SOI marker)" % name)
    p = 2
    qt = {}
    huff = {}
    sof = None
    restart = 0
    jfif = False
    adobe = None
    rec = None
    while True:
        if p >= n:
            if rec is not None:
                return rec
            raise ValueError("%s: truncated before the scan" % name)
        if b[p] != 0xFF:
            raise ValueError("%s: expected a marker at byte %d" % (name, p))
        while p < n and b[p] == 0xFF:
            p += 1
        if p >= n:
            raise ValueError("%s: truncated marker" % name)
        m = int(b[p])
        p += 1
        if m == 0xD9:
            if rec is None:
                raise ValueError("%s: EOI before any scan" % name)
            return rec
        if 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if p + 2 > n:
            raise ValueError("%s: truncated marker length" % name)
        length = _u16(b, p)
        if length < 2 or p + length > n:
            raise ValueError("%s: marker 0x%02X length %d runs past the end of the file" % (name, m, length))
        seg = b[p + 2:p + length]
        p += length
        if m in _SOF_NAMES:
            raise NotImplementedError("%s: %s is not supported" % (name, _SOF_NAMES[m]))
        if m == 0xCC:
            raise NotImplementedError("%s: arithmetic-coded JPEG (DAC) is not supported" % name)
        if m == 0xE0 and len(seg) >= 5 and bytes(seg[:5]) == b"JFIF\0":
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
            adobe = int(seg[11])
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = int(seg[q]) >> 4, int(seg[q]) & 15
                if pq > 1 or tq > 3:
                    raise ValueError("%s: bad DQT precision %d / id %d" % (name, pq, tq))
                size = 64 * (pq + 1)
                if q + 1 + size > len(seg):
                    raise ValueError("%s: DQT runs past its marker" % name)
                raw = seg[q + 1:q + 1 + size]
                vals = raw.astype(np.int32) if pq == 0 else (raw[0::2].astype(np.int32) << 8) | raw[1::2]
                table = np.zeros(64, np.int32)
                table[ZIGZAG] = vals
                qt[tq] = table
                q += 1 + size
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    raise ValueError("%s: DHT runs past its marker" % name)
                tc, th = int(seg[q]) >> 4, int(seg[q]) & 15
                if tc > 1 or th > 3:
                    raise ValueError("%s: bad DHT class %d / id %d" % (name, tc, th))
                counts = [int(c) for c in seg[q + 1:q + 17]]
                total = sum(counts)
                if total > 256 or q + 17 + total > len(seg):
                    raise ValueError("%s: DHT symbol count %d runs past its marker" % (name, total))
                symbols = [int(s) for s in seg[q + 17:q + 17 + total]]
                huff[(tc, th)] = build_huffman(counts, symbols, name, tc == 0)
                q += 17 + total
        elif m in (0xC0, 0xC1):
            if sof is not None:
                raise ValueError("%s: two SOF markers" % name)
            if len(seg) < 6:
                raise ValueError("%s: SOF too short" % name)
            prec, hgt, wid, nc = int(seg[0]), _u16(seg, 1), _u16(seg, 3), int(seg[5])
            if prec != 8:
                raise NotImplementedError("%s: %d-bit JPEG is not supported" % (name, prec))
            if len(seg) != 6 + 3 * nc:
                raise ValueError("%s: SOF length does not match its %d components" % (name, nc))
            if hgt == 0:
                raise NotImplementedError("%s: JPEG with its height in a DNL marker is not supported" % name)
            if wid == 0:
                raise ValueError("%s: image width 0" % name)
            if nc == 4:
                raise NotImplementedError("%s: 4-component (CMYK / YCCK) JPEG is not supported" % name)
            if nc not in (1, 3):
                raise NotImplementedError("%s: %d-component JPEG is not supported" % (name, nc))
            comps = []
            for i in range(nc):
                cid, hv, tq = int(seg[6 + 3 * i]), int(seg[7 + 3 * i]), int(seg[8 + 3 * i])
                h, v = hv >> 4, hv & 15
                if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
                    raise ValueError("%s: bad SOF component %d (sampling %dx%d, table %d)" % (name, cid, h, v, tq))
                if any(c["id"] == cid for c in comps):
                    raise ValueError("%s: duplicate component id %d" % (name, cid))
                comps.append(dict(id=cid, h=h, v=v, tq=tq))
            sof = (hgt, wid, comps)
        elif m == 0xDD:
            if len(seg) != 2:
                raise ValueError("%s: DRI length" % name)
            restart = _u16(seg, 0)
        elif m == 0xDA:
            if sof is None:
                raise ValueError("%s: SOS before SOF" % name)
            if rec is not None:
                raise NotImplementedError("%s: multi-scan sequential JPEG is not supported" % name)
            rec, p = _scan(b, p, seg, sof, qt, huff, restart, jfif, adobe, name)
            if p >= n:
                return rec                       # file ends inside the scan: the device decode reports it
        elif m == 0xDC:
            raise NotImplementedError("%s: DNL marker is not supported" % name)


def _scan(b, p, seg, sof, qt, huff, restart, jfif, adobe, name):
    hgt, wid, comps = sof
    if len(seg) < 1:
        raise ValueError("%s: SOS too short" % name)
    ns = int(seg[0])
    if len(seg) != 4 + 2 * ns:
        raise ValueError("%s: SOS length does not match its %d components" % (name, ns))
    if ns != len(comps):
        raise NotImplementedError("%s: multi-scan sequential JPEG (a scan of %d of %d components) is not supported"
                                  % (name, ns, len(comps)))
    ss, se, ahl = int(seg[1 + 2 * ns]), int(seg[2 + 2 * ns]), int(seg[3 + 2 * ns])
    if ss != 0 or se != 63 or ahl != 0:
        raise ValueError("%s: sequential scan with Ss=%d Se=%d Ah/Al=0x%02X" % (name, ss, se, ahl))
    out = []
    for i in range(ns):
        cs, tdta = int(seg[1 + 2 * i]), int(seg[2 + 2 * i])
        if cs != comps[i]["id"]:
            raise NotImplementedError("%s: scan component order differs from the frame's" % name)
        c = dict(comps[i], td=tdta >> 4, ta=tdta & 15)
        if c["td"] > 3 or c["ta"] > 3:
            raise ValueError("%s: bad Huffman table selector" % name)
        for key in ((0, c["td"]), (1, c["ta"])):
            if key not in huff:
                raise ValueError("%s: component %d uses undefined Huffman table %s" % (name, c["id"], key))
        if c["tq"] not in qt:
            raise ValueError("%s: component %d uses undefined quantisation table %d" % (name, c["id"], c["tq"]))
        out.append(c)
    if len(out) == 3:
        ids = [c["id"] for c in out]
        if not jfif and (adobe == 0 or (adobe is None and ids == [82, 71, 66])):
            raise NotImplementedError("%s: RGB-coded JPEG (no YCbCr transform) is not supported" % name)
        hmax, vmax = max(c["h"] for c in out), max(c["v"] for c in out)
        for c in out:
            if hmax % c["h"] or vmax % c["v"] or hmax // c["h"] > 2 or vmax // c["v"] > 2:
                raise NotImplementedError("%s: sampling factors %s are not supported"
                                          % (name, ",".join("%dx%d" % (d["h"], d["v"]) for d in out)))
        if sum(c["h"] * c["v"] for c in out) > 10:
            raise ValueError("%s: more than 10 blocks per MCU" % name)
    else:
        # a single-component scan is not interleaved: its MCU is one block whatever the declared factors
        out[0]["h"] = out[0]["v"] = 1
        hmax = vmax = 1
    for c in out:
        c["cw"] = -(-wid * c["h"] // hmax)              # downsampled size (jdinput.c initial_setup)
        c["ch"] = -(-hgt * c["v"] // vmax)
    mcux, mcuy = -(-wid // (8 * hmax)), -(-hgt // (8 * vmax))
    data = b[p:]
    segments, end = _unstuff(np.ascontiguousarray(data), name)
    total = mcux * mcuy
    if restart:
        nseg = -(-total // restart)
        if len(segments) > nseg:
            raise ValueError("%s: %d restart intervals for %d MCUs" % (name, len(segments), total))
        # missing trailing intervals are empty segments: their decode reports the truncation
        segments += [np.zeros(0, np.uint8)] * (nseg - len(segments))
        seg_mcus = [min(restart, total - i * restart) for i in range(nseg)]
    else:
        if len(segments) != 1:
            raise ValueError("%s: restart markers without a restart interval" % name)
        seg_mcus = [total]
    rec = JpegRecord()
    rec.name, rec.height, rec.width, rec.comps = name, hgt, wid, out
    rec.hmax, rec.vmax, rec.mcux, rec.mcuy = hmax, vmax, mcux, mcuy
    rec.qt = np.stack([qt[c["tq"]] for c in out]).astype(np.int32)
    rec.huff = {k: v for k, v in huff.items() if k in {(0, c["td"]) for c in out} | {(1, c["ta"]) for c in out}}
    rec.restart, rec.segments, rec.seg_mcus = restart, segments, seg_mcus
    return rec, p + end


def read_jpeg(path):
    """the host share of decoding a file, as a DataLoader worker would run it: a JpegRecord for a supported JPEG, None for
    any other file (PNG, or a JPEG form the device decoder does not take).  A malformed JPEG raises ValueError."""
    with open(path, "rb") as f:
        blob = f.read()
    if blob[:2] != b"\xff\xd8":
        return None
    try:
        return parse_jpeg(blob, str(path))
    except NotImplementedError:
        return None


def load(blob, name="<bytes>"):
    """bytes (or a path) -> JpegRecord"""
    if isinstance(blob, (str, os.PathLike)):
        name = str(blob)
        with open(blob, "rb") as f:
            blob = f.read()
    return parse_jpeg(blob, name)


def ycc_tables():
    """jdcolor.c build_ycc_rgb_table: int32 (4, 256) Cr->R, Cb->B, Cr->G, Cb->G (SCALEBITS 16, ONE_HALF rounding)"""
    x = np.arange(256, dtype=np.int64) - 128
    fix = lambda v: int(v * 65536 + 0.5)   # noqa: E731
    half = 1 << 15
    crr = (fix(1.40200) * x + half) >> 16
    cbb = (fix(1.77200) * x + half) >> 16
    crg = -fix(0.71414) * x
    cbg = -fix(0.34414) * x + half
    return np.stack([crr, cbb, crg, cbg]).astype(np.int32)


def pack_batch(records):
    """records of one image size -> dict of host arrays laid out as csrc/jpeg.cu reads them:
    data uint8 (all segments), segments int32 (nseg, SEGMENT_WORDS) = [image, byte offset, byte count, first MCU,
    MCU count], images int32 (n, IMAGE_WORDS) = [ncomp, mcux, hmax, vmax, first segment, segment count, then per component: h, v, blocks_w,
    blocks_h, coef block offset, cw, ch, dc table slot, ac table slot, 0], huff int32 (n * 8, HUFF_WORDS),
    qt int32 (n, 3, 64), n_blocks (coefficient blocks of the whole batch)"""
    if not records:
        raise ValueError("empty JPEG batch")
    h, w = records[0].height, records[0].width
    for r in records:
        if (r.height, r.width) != (h, w):
            raise ValueError("all images of a JPEG batch must have one size: %s is %dx%d, %s is %dx%d"
                             % (records[0].name, h, w, r.name, r.height, r.width))
    n = len(records)
    images = np.zeros((n, IMAGE_WORDS), np.int32)
    huff = np.zeros((n * 8, HUFF_WORDS), np.int32)
    qt = np.zeros((n, 3, 64), np.int32)
    segs, chunks = [], []
    off, block = 0, 0
    for i, r in enumerate(records):
        images[i, :6] = (len(r.comps), r.mcux, r.hmax, r.vmax, len(segs), len(r.segments))
        for (tc, th), t in r.huff.items():
            huff[i * 8 + tc * 4 + th] = t
        for c, comp in enumerate(r.comps):
            bw, bh = r.mcux * comp["h"], r.mcuy * comp["v"]
            images[i, 6 + 10 * c:16 + 10 * c] = (comp["h"], comp["v"], bw, bh, block, comp["cw"], comp["ch"],
                                                 i * 8 + comp["td"], i * 8 + 4 + comp["ta"], 0)
            block += bw * bh
            qt[i, c] = r.qt[c]
        first = 0
        for s, m in zip(r.segments, r.seg_mcus):
            segs.append((i, off, len(s), first, m))
            chunks.append(s)
            off += len(s)
            first += m
    if block * 64 >= 2 ** 31 or off >= 2 ** 31:
        raise ValueError("JPEG batch too large for 32-bit offsets")
    data = np.concatenate(chunks + [np.zeros(8, np.uint8)])
    return dict(data=data, segments=np.array(segs, np.int32).reshape(-1, SEGMENT_WORDS), images=images, huff=huff,
                qt=qt, n_blocks=block, height=h, width=w)


# A segment of at most this many subsequences is decoded whole by one thread, as the serial kernel does: the parallel
# path's critical path is about four subsequence decodes long even when every guess holds (warm-up, speculation, the
# exact last subsequence, emission), and a short periodic stream (a flat tile) can hold every guess at a wrong phase.
SPLIT_MIN_SUBSEQUENCES = 16


def subsequence_table(pk, bits):
    """subsequences of `bits` unstuffed bits per segment of a packed batch (a segment of at most
    SPLIT_MIN_SUBSEQUENCES of them is one) -> (sub_first int32 (nseg + 1,): first subsequence of each segment, the most
    subsequences of one image)"""
    nbytes = pk["segments"][:, 2].astype(np.int64)
    if len(nbytes) and nbytes.max() >= 2 ** 28:
        raise ValueError("JPEG entropy segment of %d bytes: the device decode takes less than 2^28" % nbytes.max())
    counts = -(-nbytes * 8 // bits)
    counts[counts <= SPLIT_MIN_SUBSEQUENCES] = 1
    sub_first = np.concatenate([[0], np.cumsum(counts)])
    if sub_first[-1] >= 2 ** 31 // 16:
        raise ValueError("JPEG batch too large: %d subsequences" % sub_first[-1])
    im = pk["images"]
    per_image = sub_first[im[:, 4] + im[:, 5]] - sub_first[im[:, 4]]
    return sub_first.astype(np.int32), int(per_image.max())


class DeviceBatch:
    """a packed batch on the device: the tables csrc/jpeg.cu reads, uploaded from pinned memory on the current stream"""

    def __init__(self, pk, dev):
        import torch
        from . import _lib as L

        def up(a):
            return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)
        self.n, self.n_blocks, self.nseg = len(pk["images"]), pk["n_blocks"], len(pk["segments"])
        sub_first, self.max_image_subs = subsequence_table(pk, L.lib.mcb_jpeg_subsequence_bits())
        self.data, self.segs, self.images, self.huff, self.qt, self.sub_first = (
            up(a) for a in (pk["data"], pk["segments"], pk["images"], pk["huff"], pk["qt"], sub_first))
        self.workspace = torch.empty(16 + 16 * int(sub_first[-1]), dtype=torch.int32, device=dev)
        self.coef = torch.empty((self.n_blocks, 64), dtype=torch.int16, device=dev)
        self.status = torch.empty(self.n, dtype=torch.int32, device=dev)

    def entropy_decode(self):
        """the parallel entropy decode into self.coef / self.status (three launches on the current stream)"""
        from . import _lib as L
        L.fcall("mcb_jpeg_entropy_decode_parallel", self.data.data_ptr(), self.segs.data_ptr(), self.nseg,
                self.images.data_ptr(), self.huff.data_ptr(), self.n, self.sub_first.data_ptr(), self.max_image_subs,
                self.workspace.data_ptr(), self.coef.data_ptr(), self.status.data_ptr())

    def entropy_decode_serial(self):
        """the one-thread-per-segment entropy decode into self.coef / self.status, as a reference"""
        from . import _lib as L
        L.fcall("mcb_jpeg_entropy_decode", self.data.data_ptr(), self.segs.data_ptr(), self.nseg,
                self.images.data_ptr(), self.huff.data_ptr(), self.n, self.coef.data_ptr(), self.status.data_ptr())

    def counters(self):
        """speculation counters of the last parallel decode: entry states that held, were corrected, the longest run of
        consecutive corrections, exact re-decodes of a segment's error or last block (synchronises)"""
        return self.workspace[:4].cpu().numpy()


def decode_records(records, device=None):
    """JpegRecords of one size -> (rgb uint8 cuda (n, H, W, 3), coefficients int16 cuda (blocks, 64), IDCT planes uint8
    cuda (blocks, 8, 8), status int32 numpy (n,)), blocks in pack_batch's order.  Five launches on the current stream,
    then one read of the status words; an image with a non-zero status has undefined pixels, the others are exact."""
    import torch
    from . import _lib as L
    pk = pack_batch(records)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    n, hgt, wid = len(records), pk["height"], pk["width"]

    with torch.cuda.device(dev):
        b = DeviceBatch(pk, dev)
        tables = torch.from_numpy(ycc_tables()).pin_memory().to(dev, non_blocking=True)
        coef, status, qt, images = b.coef, b.status, b.qt, b.images
        planes = torch.empty((pk["n_blocks"], 8, 8), dtype=torch.uint8, device=dev)
        out = torch.empty((n, hgt, wid, 3), dtype=torch.uint8, device=dev)
        b.entropy_decode()
        L.fcall("mcb_jpeg_idct", coef.data_ptr(), qt.data_ptr(), images.data_ptr(), n, pk["n_blocks"],
                planes.data_ptr())
        L.fcall("mcb_jpeg_upsample_rgb", planes.data_ptr(), images.data_ptr(), tables.data_ptr(), n, hgt, wid,
                out.data_ptr())
        st = status.cpu().numpy()
    return out, coef, planes, st


def decode_jpeg_batch(blobs, device=None):
    """JPEG files (bytes, paths or JpegRecords) of one size -> uint8 cuda (n, H, W, 3), equal bit for bit to
    `np.array(Image.open(f).convert('RGB'))`.  A file whose entropy data is truncated or corrupt raises ValueError
    naming it."""
    records = [r if isinstance(r, JpegRecord) else load(r) for r in blobs]
    out, _, _, st = decode_records(records, device)
    bad = np.flatnonzero(st)
    if len(bad):
        raise ValueError("corrupt or truncated JPEG entropy data in %s"
                         % ", ".join("%s (%s)" % (records[i].name, STATUS.get(int(st[i]), int(st[i]))) for i in bad))
    return out


# per-image status words written by the entropy decode kernel
STATUS = {1: "data ends inside a segment", 2: "invalid Huffman code", 3: "coefficient index past 63"}
