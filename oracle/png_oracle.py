"""Python / numpy restatement of the PNG label-map path (TEST INFRASTRUCTURE): inflate (RFC 1951, with zlib's checks),
PNG unfiltering and unpacking as csrc/png.cu does them, and the loader's label transform as csrc/input_pipe.cu's
label_preprocess_kernel does it.  Slow and plain on purpose: it is what the device code is checked against."""
import numpy as np

from lanedetection_end2end_b200 import png
from lanedetection_end2end_b200.input_pipeline import nearest_table

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0] + [(d - 2) // 2 for d in range(2, 30)]
CLEN_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class Corrupt(ValueError):
    pass


class _Bits:
    def __init__(self, data, pos):
        self.d, self.pos, self.bit = data, pos, 0     # next bit = bit `bit` of byte `pos`

    def get(self, n):
        v = 0
        for k in range(n):
            if self.pos >= len(self.d):
                raise Corrupt("stream ends before its final block")
            v |= ((self.d[self.pos] >> self.bit) & 1) << k
            self.bit += 1
            if self.bit == 8:
                self.bit, self.pos = 0, self.pos + 1
        return v

    def align(self):
        if self.bit:
            self.bit, self.pos = 0, self.pos + 1


def _code(lens, single_ok):
    """(count, symbols by (length, value)) of a canonical code, with zlib's over-subscribed / incomplete rules"""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    left, maxlen = 1, 0
    for l in range(1, 16):
        left = (left << 1) - count[l]
        if left < 0:
            raise Corrupt("over-subscribed code")
        if count[l]:
            maxlen = l
    if maxlen and left > 0 and not (single_ok and maxlen == 1):
        raise Corrupt("incomplete code")
    if not maxlen and not single_ok:
        raise Corrupt("empty code")
    syms = sorted((l, s) for s, l in enumerate(lens) if l)
    return count, [s for _, s in syms]


def _decode(br, code):
    count, syms = code
    c = first = index = 0
    for l in range(1, 16):
        c |= br.get(1)
        n = count[l]
        if c - n < first:
            return syms[index + c - first]
        index += n
        first = (first + n) << 1
        c <<= 1
    raise Corrupt("invalid code")


def inflate(z, total):
    """Inflate the zlib stream `z` (2-byte header, DEFLATE data, Adler-32) that must hold exactly `total` bytes."""
    br = _Bits(z, 2)
    out = bytearray()
    stats = {"stored": 0, "fixed": 0, "dynamic": 0}
    while True:
        final, btype = br.get(1), br.get(2)
        if btype == 0:
            br.align()
            ln, nln = br.get(16), br.get(16)
            if ln != (~nln & 0xFFFF):
                raise Corrupt("stored block length")
            if br.pos + ln > len(z) or len(out) + ln > total:
                raise Corrupt("stored block overruns")
            out += z[br.pos:br.pos + ln]
            br.pos += ln
            stats["stored"] += 1
        elif btype == 3:
            raise Corrupt("block type 3")
        else:
            if btype == 1:
                lit = _code([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, True)
                dist = _code([5] * 32, True)
                stats["fixed"] += 1
            else:
                hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                if hlit > 286 or hdist > 30:
                    raise Corrupt("too many length or distance symbols")
                cl = [0] * 19
                for k in range(hclen):
                    cl[CLEN_ORDER[k]] = br.get(3)
                clc = _code(cl, False)
                lens = []
                while len(lens) < hlit + hdist:
                    s = _decode(br, clc)
                    if s < 16:
                        lens.append(s)
                        continue
                    if s == 16:
                        if not lens:
                            raise Corrupt("repeat with no length")
                        val, rep = lens[-1], 3 + br.get(2)
                    elif s == 17:
                        val, rep = 0, 3 + br.get(3)
                    else:
                        val, rep = 0, 11 + br.get(7)
                    if len(lens) + rep > hlit + hdist:
                        raise Corrupt("too many lengths")
                    lens += [val] * rep
                if lens[256] == 0:
                    raise Corrupt("no end-of-block code")
                lit, dist = _code(lens[:hlit], True), _code(lens[hlit:], True)
                stats["dynamic"] += 1
            while True:
                s = _decode(br, lit)
                if s < 256:
                    if len(out) >= total:
                        raise Corrupt("output too long")
                    out.append(s)
                elif s == 256:
                    break
                else:
                    if s > 285:
                        raise Corrupt("invalid length symbol")
                    ln = LEN_BASE[s - 257] + br.get(LEN_EXTRA[s - 257])
                    d = _decode(br, dist)
                    if d > 29:
                        raise Corrupt("invalid distance symbol")
                    dd = DIST_BASE[d] + br.get(DIST_EXTRA[d])
                    if dd > len(out):
                        raise Corrupt("distance too far back")
                    if len(out) + ln > total:
                        raise Corrupt("output too long")
                    src = bytes(out[len(out) - dd:])
                    out += (src * (ln // dd + 1))[:ln]
        if final:
            break
    if len(out) != total:
        raise Corrupt("output too short")
    br.align()
    if br.pos + 4 > len(z):
        raise Corrupt("no Adler-32")
    if int.from_bytes(z[br.pos:br.pos + 4], "big") != adler32(out):
        raise Corrupt("Adler-32 mismatch")
    return bytes(out), stats


def adler32(data):
    a = np.frombuffer(bytes(data), np.uint8).astype(np.int64)
    n = len(a)
    s1 = (1 + int(a.sum())) % 65521
    s2 = (n + int(((n - np.arange(n, dtype=np.int64)) * a).sum())) % 65521
    return (s2 << 16) | s1


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def unfilter(raw, H, rowbytes):
    """PNG filters with a 1-byte filter unit -> uint8 [H, rowbytes]; returns (rows, filter types used)"""
    rows = np.frombuffer(raw, np.uint8).reshape(H, rowbytes + 1)
    out = np.zeros((H, rowbytes), np.uint8)
    prev = np.zeros(rowbytes, np.int64)
    used = set()
    for y in range(H):
        ft, x = int(rows[y, 0]), rows[y, 1:].astype(np.int64)
        used.add(ft)
        if ft == 0:
            cur = x
        elif ft == 1:
            cur = np.cumsum(x) % 256
        elif ft == 2:
            cur = (x + prev) % 256
        elif ft in (3, 4):
            cur = np.zeros(rowbytes, np.int64)
            a = c = 0
            for i in range(rowbytes):
                b = int(prev[i])
                pr = (a + b) >> 1 if ft == 3 else _paeth(a, b, c)
                a = cur[i] = (int(x[i]) + pr) & 255
                c = b
        else:
            raise Corrupt("filter type %d" % ft)
        out[y] = cur
        prev = cur.astype(np.int64)
    return out, used


def unpack(rows, W, depth):
    """1/2/4/8-bit samples, most significant bits first -> uint8 [H, W]"""
    if depth == 8:
        return rows[:, :W].copy()
    bits = np.unpackbits(rows, axis=1).reshape(rows.shape[0], -1, depth)
    vals = (bits * (1 << np.arange(depth - 1, -1, -1, dtype=np.uint8))).sum(-1).astype(np.uint8)
    return vals[:, :W]


def decode(data):
    """Label map of one PNG file as the device decodes it: uint8 [H, W] (gray values or palette indices)."""
    h = png.parse(data)
    rowbytes = (h.width * h.depth + 7) // 8
    raw, stats = inflate(h.zdata, h.height * (rowbytes + 1))
    rows, used = unfilter(raw, h.height, rowbytes)
    stats["filters"] = sorted(used)
    return unpack(rows, h.width, h.depth), stats


def label_transform(m, resize, nclasses, flip, crop_rows=640):
    """The reference loader's gt from a decoded uint8 map [H, W]: int64 [1, resize, 2*resize]"""
    H, W = m.shape
    ys = nearest_table(crop_rows, resize) + (H - crop_rows)
    xs = nearest_table(W, 2 * resize)
    v0 = m[ys][:, xs].astype(np.int64)
    v = v0[:, ::-1].copy() if flip else v0.copy()
    if nclasses < 3:
        v[(v == 3) | (v == 4)] = 0
    if flip:
        one, two = v == 1, v == 2
        v[one], v[two] = 2, 1
        v[v0 == 3], v[v0 == 4] = 4, 3
    return v[None]
