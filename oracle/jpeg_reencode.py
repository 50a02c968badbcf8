"""Baseline JPEG entropy re-encoder: a file's quantised coefficients (from jpeg_oracle.entropy_decode) written again
with chosen Huffman tables, every other marker kept.  Pillow decodes the result to the original's pixels.

`reencode(blob, shared=True)` gives all 12 DC symbols one code length (4 bits) and all 162 AC symbols one code length
(8 bits), the all-ones code left free.  Codes of a single length do not resynchronise after a misaligned start the way
the encoders' variable-length tables do, and with `shared` one DC and one AC table serve every component, so the
position within the MCU cannot be recovered from the codes either: the worst case for a decoder that guesses where
symbols start.

`corrupt` plants errors the decoder must report: {bit position: kind}; the first block starting at or after each
position is written as an invalid Huffman code (kind 2) or as AC runs that take the coefficient index past 63
(kind 3)."""
import numpy as np

from mcb200 import jpeg as J
from oracle import jpeg_oracle as O

_RUN_PAST_63 = 0xF1        # run 15, size 1: four of them reach index 64


def _category(v):
    return int(abs(int(v))).bit_length()


def _bits(v, s):
    return int(v) if v >= 0 else int(v) + (1 << s) - 1


DC_SYMBOLS = list(range(12))
AC_SYMBOLS = [0x00, 0xF0] + [r << 4 | s for r in range(16) for s in range(1, 11)]


def one_length_table(symbols):
    """DHT counts / symbols giving every symbol the same code length, the shortest that leaves the all-ones code
    unused (a decoder must reject it)"""
    counts = [0] * 16
    counts[len(symbols).bit_length() - 1] = len(symbols)
    return counts, list(symbols)


def _codes(counts, symbols):
    code, k, out = 0, 0, {}
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            out[symbols[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


class _Writer:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0
        self.pos = 0

    def put(self, v, n):
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        self.pos += n
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 0xFF
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0x00)
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        return bytes(self.out)


def _headers(blob):
    """the file's marker segments before SOS, DHT and DRI dropped, and the SOS component ids"""
    b = bytes(blob)
    p, keep = 2, [b"\xff\xd8"]
    while True:
        while b[p] == 0xFF:
            p += 1
        m = b[p]
        length = (b[p + 1] << 8) | b[p + 2]
        seg = b[p - 1:p + 1 + length]
        if m == 0xDA:
            ns = b[p + 3]
            return b"".join(keep), [b[p + 4 + 2 * i] for i in range(ns)]
        if m not in (0xC4, 0xDD):
            keep.append(seg)
        p += 1 + length


def reencode(blob, shared=True, corrupt=None):
    """a baseline file without restart markers -> the same coefficients under one-length Huffman tables (see the
    module docstring); corrupt = {bit position in the entropy data: 2 or 3}"""
    rec = J.load(blob)
    coefs = O.entropy_decode(rec)
    comps = rec.comps
    groups = [list(range(len(comps)))] if shared else [[0], list(range(1, len(comps)))] if len(comps) > 1 else [[0]]
    tables = {}
    dht = bytearray()
    for t, members in enumerate(groups):
        for cls, syms in ((0, DC_SYMBOLS), (1, AC_SYMBOLS)):
            counts, symbols = one_length_table(syms)
            dht += bytes([cls << 4 | t]) + bytes(counts) + bytes(symbols)
            for i in members:
                tables[(cls, i)] = _codes(counts, symbols)
    head, ids = _headers(blob)
    out = bytearray(head)
    out += b"\xff\xc4" + (2 + len(dht)).to_bytes(2, "big") + dht
    sel = [next(t for t, m in enumerate(groups) if i in m) for i in range(len(comps))]
    sos = bytes([len(comps)]) + b"".join(bytes([ids[i], sel[i] << 4 | sel[i]]) for i in range(len(comps))) + \
        bytes([0, 63, 0])
    out += b"\xff\xda" + (2 + len(sos)).to_bytes(2, "big") + sos
    w = _Writer()
    pending = sorted((corrupt or {}).items())
    pred = [0] * len(comps)
    for m in range(rec.mcux * rec.mcuy):
        my, mx = divmod(m, rec.mcux)
        for ci, c in enumerate(comps):
            dct, act = tables[(0, ci)], tables[(1, ci)]
            for v in range(c["v"]):
                for h in range(c["h"]):
                    zz = coefs[ci][my * c["v"] + v, mx * c["h"] + h][J.ZIGZAG].astype(np.int64)
                    kind = 0
                    if pending and w.pos >= pending[0][0]:
                        kind = pending.pop(0)[1]
                    if kind == 2:                      # the unused all-ones code of the DC table
                        length = dct[0][1]
                        w.put((1 << length) - 1, length)
                        continue
                    diff = int(zz[0]) - pred[ci]
                    pred[ci] = int(zz[0])
                    s = _category(diff)
                    w.put(*dct[s])
                    if s:
                        w.put(_bits(diff, s), s)
                    if kind == 3:
                        for _ in range(4):
                            w.put(*act[_RUN_PAST_63])
                            w.put(1, 1)
                        continue
                    k = 1
                    for i in np.flatnonzero(zz[1:]) + 1:
                        r = int(i) - k
                        while r > 15:
                            w.put(*act[0xF0])
                            r -= 16
                        s = _category(zz[i])
                        w.put(*act[(r << 4) | s])
                        w.put(_bits(int(zz[i]), s), s)
                        k = int(i) + 1
                    if k < 64:
                        w.put(*act[0x00])
    out += w.flush() + b"\xff\xd9"
    return bytes(out)
