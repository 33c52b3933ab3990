"""Restatement of the GPU baseline JPEG encoder (csrc/jpeg_enc.cu) and of its lane-point circles (lf_draw_lane_points) in
numpy, TEST INFRASTRUCTURE.  Every stage follows the libjpeg-turbo that Pillow ships, stated on whole arrays:

  quality_tables   jcparam.c jpeg_set_quality / jpeg_add_quant_table (force_baseline): the Annex K tables scaled
  headers          SOI, APP0 JFIF 1.01, DQT per table, SOF0, DHT (DC, AC per table in scan order), SOS, as jcmarker.c
  colour           jccolor.c rgb_ycc_convert: 16-bit fixed point, 0.5 - epsilon rounding of Cb / Cr
  planes           jcprepct.c / jcsample.c: right and bottom edge replication, h2v2 averaging with the 1, 2, 1, 2 bias
  fdct_islow       jfdctint.c (CONST_BITS 13, PASS1_BITS 2), output scaled by 8
  quantise         jcdctmgr.c compute_reciprocal + quantize (16-bit DCTELEM, the SIMD build's arithmetic)
  dummy blocks     jccoefct.c compress_data: DC-only blocks that copy a neighbour's DC in partial 4:2:0 MCUs
  entropy          jchuff.c encode_one_block with the standard tables, 1-bit padding, 0xFF -> 0xFF 0x00 stuffing

    data = encode(a, quality=75, subsampling="4:2:0")
    data == Image.fromarray(a).save(buf, "JPEG", quality=75, subsampling="4:2:0") bytes

circle_halfwidths / draw_lane_points restate cv2.circle(img, centre, radius, colour, thickness=-1) (LINE_8, shift 0:
drawing.cpp Circle with fill) and the reference's drawing order (BP/test.py:115-119)."""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural index

# ITU-T T.81 Annex K.1, natural order
STD_LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                       49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_Q = np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                         47, 66, 99, 99] + [99] * 36, np.int64)

# ITU-T T.81 Annex K.3: DHT payloads (16 code counts, then the symbols): DC luma, AC luma, DC chroma, AC chroma
STD_HUFF = [bytes.fromhex(h) for h in (
    "00010501010101010100000000000000000102030405060708090a0b",
    "0002010303020403050504040000017d01020300041105122131410613516107227114328191a1082342b1c11552d1f024336272"
    "82090a161718191a25262728292a3435363738393a434445464748494a535455565758595a636465666768696a73747576777879"
    "7a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8"
    "d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa",
    "00030101010101010101010000000000000102030405060708090a0b",
    "00020102040403040705040400010277000102031104052131061241510761711322328108144291a1b1c109233352f0156272d1"
    "0a162434e125f11718191a262728292a35363738393a434445464748494a535455565758595a636465666768696a737475767778"
    "797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6"
    "d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")]

SUBSAMPLINGS = ("4:2:0", "4:4:4")


def quality_tables(quality, ncomp=3):
    """[1 or 2, 64] natural-order quantisation tables of jpeg_set_quality(cinfo, quality, TRUE)."""
    if not (isinstance(quality, (int, np.integer)) and 1 <= quality <= 100):
        raise ValueError("quality must be an integer in 1..100, got %r" % (quality,))
    scale = 5000 // quality if quality < 50 else 200 - quality * 2
    bases = (STD_LUMA_Q, STD_CHROMA_Q)[:2 if ncomp == 3 else 1]
    return np.stack([np.clip((b * scale + 50) // 100, 1, 255) for b in bases])


def huffman_codes(payload):
    """(code, size) per symbol of one DHT payload (jchuff.c jpeg_make_c_derived_tbl); size 0 = no code."""
    bits, vals = payload[:16], payload[16:]
    code_of, size_of = np.zeros(256, np.int64), np.zeros(256, np.int64)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            code_of[vals[k]], size_of[vals[k]] = code, l
            code += 1
            k += 1
        code <<= 1
    return code_of, size_of


def _seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body


def headers(W, H, ncomp, subsampling, qt):
    """Everything before the entropy-coded segment, as Pillow writes it."""
    out = b"\xff\xd8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(len(qt)):
        out += _seg(0xDB, bytes([t]) + bytes(int(v) for v in qt[t][ZIGZAG]))
    hv = 0x22 if subsampling == "4:2:0" else 0x11        # Pillow sets 2x2 on a grayscale component too
    comps = bytes([1, hv, 0]) + (bytes([2, 0x11, 1, 3, 0x11, 1]) if ncomp == 3 else b"")
    out += _seg(0xC0, bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([ncomp]) + comps)
    for t in range(1 if ncomp == 1 else 2):
        out += _seg(0xC4, bytes([0x00 | t]) + STD_HUFF[2 * t]) + _seg(0xC4, bytes([0x10 | t]) + STD_HUFF[2 * t + 1])
    scan = bytes([1, 0x00]) + (bytes([2, 0x11, 3, 0x11]) if ncomp == 3 else b"")
    return out + _seg(0xDA, bytes([ncomp]) + scan + b"\x00\x3f\x00")


def _fix(x):
    return int(x * 65536 + 0.5)


def rgb_to_ycc(a):
    r, g, b = (a[..., c].astype(np.int64) for c in range(3))
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def _pad(p, h, w):
    return np.pad(p, ((0, h - p.shape[0]), (0, w - p.shape[1])), mode="edge")


def h2v2_downsample(p):
    """p [2h, 2w] -> [h, w]: (sum of the 2x2 + bias) >> 2, bias 1, 2, 1, 2, ... along each output row."""
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return (s + bias) >> 2


def planes(a, subsampling):
    """Component planes padded to whole MCUs, and the MCU grid (mcux, mcuy)."""
    H, W = a.shape[:2]
    if a.ndim == 2 or subsampling == "4:4:4":
        mcux, mcuy = -(-W // 8), -(-H // 8)
        comps = [a.astype(np.int64)] if a.ndim == 2 else list(rgb_to_ycc(a))
        return [_pad(c, 8 * mcuy, 8 * mcux) for c in comps], mcux, mcuy
    mcux, mcuy = -(-W // 16), -(-H // 16)
    y, cb, cr = rgb_to_ycc(a)
    out = [_pad(y, 16 * mcuy, 16 * mcux)]
    for c in (cb, cr):
        # odd last row replicated into the row pair, columns to whole chroma blocks; then the last downsampled row
        out.append(_pad(h2v2_downsample(_pad(c, 2 * (-(-H // 2)), 16 * mcux)), 8 * mcuy, 8 * mcux))
    return out, mcux, mcuy


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    """one jpeg_fdct_islow pass along the last axis; first = the row pass (PASS1_BITS up), else the column pass"""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    n = 11 if first else 15
    o = [None] * 8
    o[0] = (t10 + t11) << 2 if first else _descale(t10 + t11, 2)
    o[4] = (t10 - t11) << 2 if first else _descale(t10 - t11, 2)
    z1 = (t12 + t13) * 4433
    o[2] = _descale(z1 + t13 * 6270, n)
    o[6] = _descale(z1 - t12 * 15137, n)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
    z1, z2 = z1 * -7373, z2 * -20995
    z3, z4 = z3 * -16069 + z5, z4 * -3196 + z5
    o[7] = _descale(t4 + z1 + z3, n)
    o[5] = _descale(t5 + z2 + z4, n)
    o[3] = _descale(t6 + z2 + z3, n)
    o[1] = _descale(t7 + z1 + z4, n)
    return np.stack(o, -1)


def fdct_islow(blocks):
    """[n, 8, 8] samples - 128 -> [n, 8, 8] DCT coefficients scaled by 8"""
    d = _fdct_1d(blocks.astype(np.int64), True)
    return np.swapaxes(_fdct_1d(np.swapaxes(d, -1, -2), False), -1, -2)


def reciprocals(q):
    """compute_reciprocal of the divisors q * 8 (16-bit DCTELEM): (reciprocal, correction, shift) per entry"""
    rec, cor, sh = [], [], []
    for d in (np.asarray(q, np.int64) * 8).tolist():
        b = d.bit_length() - 1
        r = 16 + b
        fq, fr = (1 << r) // d, (1 << r) % d
        c = d // 2
        if fr == 0:
            fq >>= 1
            r -= 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        rec.append(fq)
        cor.append(c)
        sh.append(r - 16)
    return np.array(rec, np.int64), np.array(cor, np.int64), np.array(sh, np.int64)


def quantise(coef, q):
    """[n, 64] natural-order DCT outputs -> quantised coefficients, as jcdctmgr.c quantize rounds them"""
    rec, cor, sh = reciprocals(q)
    a = np.abs(coef)
    v = ((a + cor) * rec) >> (sh + 16)
    return np.where(coef < 0, -v, v)


def _blocks(p):
    h, w = p.shape
    return p.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)       # [by, bx, 8, 8]


def coefficients(a, quality=75, subsampling="4:2:0"):
    """Quantised coefficients in MCU order [nblocks, 64] (natural order), the component of each block, and the tables."""
    if subsampling not in SUBSAMPLINGS:
        raise ValueError("subsampling must be one of %s" % (SUBSAMPLINGS,))
    ncomp = 1 if a.ndim == 2 else 3
    qt = quality_tables(quality, ncomp)
    pl, mcux, mcuy = planes(a, subsampling)
    q = []
    for c, p in enumerate(pl):
        b = _blocks(p)
        q.append(quantise(fdct_islow(b - 128).reshape(-1, 64), qt[min(c, 1)]).reshape(b.shape[0], b.shape[1], 64))
    H, W = a.shape[:2]
    if ncomp == 3 and subsampling == "4:2:0":
        y = q[0]
        wb, hb = -(-W // 8), -(-H // 8)
        if wb % 2:                      # right-edge dummy: DC of the block to its left
            y[:, wb] = 0
            y[:, wb, 0] = y[:, wb - 1, 0]
        if hb % 2:                      # bottom dummy row: both blocks take the DC of the MCU's block 1
            dc = y[hb - 1, 1::2, 0].copy()
            y[hb] = 0
            y[hb, 0::2, 0] = dc
            y[hb, 1::2, 0] = dc
        y4 = y.reshape(mcuy, 2, mcux, 2, 64).transpose(0, 2, 1, 3, 4).reshape(mcuy, mcux, 4, 64)
        mcu = np.concatenate([y4, q[1][:, :, None], q[2][:, :, None]], 2)
        comp = np.array([0, 0, 0, 0, 1, 2])
    else:
        mcu = np.stack(q, 2)
        comp = np.arange(ncomp)
    return mcu.reshape(-1, 64), np.tile(comp, mcux * mcuy), qt


def _nbits(v):
    a = np.abs(v)
    n = np.zeros_like(a)
    while (a >> n).any():
        n += (a >> n) > 0
    return n


def _vbits(v, n):
    return np.where(v < 0, v - 1, v) & ((1 << n) - 1)


def entropy(coef, comp):
    """Huffman-coded, padded and stuffed scan of [nblocks, 64] natural-order coefficients in MCU order."""
    tabs = [huffman_codes(t) for t in STD_HUFF]
    nblk = coef.shape[0]
    tsel = np.minimum(comp, 1)                                   # table set of each block: 0 luma, 1 chroma
    dc = coef[:, 0]
    diff = dc.copy()
    for c in np.unique(comp):
        idx = np.nonzero(comp == c)[0]
        diff[idx[1:]] = dc[idx[1:]] - dc[idx[:-1]]
    keys, vals, lens = [], [], []
    n = _nbits(diff)
    dcc = np.where(tsel == 0, tabs[0][0][n], tabs[2][0][n])
    dcs = np.where(tsel == 0, tabs[0][1][n], tabs[2][1][n])
    keys.append(np.arange(nblk) * 4096)
    vals.append((dcc << n) | _vbits(diff, n))
    lens.append(dcs + n)
    zz = coef[:, ZIGZAG[1:]]                                     # [nblk, 63] AC in zig-zag order
    b, k = np.nonzero(zz)
    v = zz[b, k]
    prev = np.r_[-1, k[:-1]]
    prev[np.r_[True, b[1:] != b[:-1]]] = -1                     # previous nonzero of the same block, or -1
    run = k - prev - 1
    s = _nbits(v)
    sym = ((run & 15) << 4) | s
    act = [tabs[1], tabs[3]]
    t = tsel[b]
    code = np.where(t == 0, act[0][0][sym], act[1][0][sym])
    size = np.where(t == 0, act[0][1][sym], act[1][1][sym])
    keys.append(b * 4096 + (k + 1) * 32 + 16)
    vals.append((code << s) | _vbits(v, s))
    lens.append(size + s)
    nz = run >> 4                                               # ZRL symbols before the coefficient
    rb = np.repeat(b, nz)
    rk = np.repeat(k, nz)
    rj = np.arange(int(nz.sum())) - np.repeat(np.cumsum(nz) - nz, nz)
    rt = tsel[rb]
    keys.append(rb * 4096 + (rk + 1) * 32 + rj)
    vals.append(np.where(rt == 0, act[0][0][0xF0], act[1][0][0xF0]))
    lens.append(np.where(rt == 0, act[0][1][0xF0], act[1][1][0xF0]))
    last = np.full(nblk, -1)
    last[b] = k                                                  # nonzero order is ascending in k per block
    eb = np.nonzero(last < 62)[0]
    keys.append(eb * 4096 + 64 * 32)
    vals.append(np.where(tsel[eb] == 0, act[0][0][0], act[1][0][0]))
    lens.append(np.where(tsel[eb] == 0, act[0][1][0], act[1][1][0]))
    keys, vals, lens = (np.concatenate(x).astype(np.int64) for x in (keys, vals, lens))
    o = np.argsort(keys, kind="stable")
    vals, lens = vals[o], lens[o]
    total = int(lens.sum())
    start = np.cumsum(lens) - lens
    rv, rl = np.repeat(vals, lens), np.repeat(lens, lens)
    pos = np.arange(total) - np.repeat(start, lens)
    bits = ((rv >> (rl - 1 - pos)) & 1).astype(np.uint8)
    bits = np.concatenate([bits, np.ones(-total % 8, np.uint8)])  # 1-bit padding to a whole byte
    return np.packbits(bits), total


def stuff(by):
    out = np.repeat(by, np.where(by == 0xFF, 2, 1))
    ff = np.nonzero(by == 0xFF)[0]
    out[ff + np.arange(1, len(ff) + 1)] = 0
    return out


def encode(a, quality=75, subsampling="4:2:0"):
    """Baseline JPEG bytes of uint8 [H, W, 3] RGB or [H, W] grayscale, equal to Pillow's."""
    a = np.asarray(a)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] != 3) or min(a.shape[:2]) < 1:
        raise ValueError("expected uint8 [H, W, 3] or [H, W], got %s %s" % (a.dtype, a.shape))
    if a.shape[0] > 65535 or a.shape[1] > 65535:
        raise ValueError("JPEG dimensions are limited to 65535")
    coef, comp, qt = coefficients(a, quality, subsampling)
    packed, _ = entropy(coef, comp)
    H, W = a.shape[:2]
    return headers(W, H, 1 if a.ndim == 2 else 3, subsampling, qt) + stuff(packed).tobytes() + b"\xff\xd9"


def circle_halfwidths(radius):
    """Half-width of cv2's filled integer circle (drawing.cpp Circle, fill, LINE_8, shift 0) on rows 0..radius below or
    above the centre: the stamp covers (x, y) with |x - cx| <= hw[|y - cy|]."""
    if radius < 0:
        raise ValueError("radius must be >= 0")
    hw = [-1] * (radius + 1)
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    while dx >= dy:
        hw[dy] = max(hw[dy], dx)        # spans on rows cy -+ dy from cx - dx to cx + dx
        hw[dx] = max(hw[dx], dy)        # spans on rows cy -+ dx from cx - dy to cx + dy
        dy += 1
        err += plus
        plus += 2
        mask = (err <= 0) - 1
        err -= minus & mask
        dx += mask
        minus -= mask & 2
    return hw


def draw_lane_points(img, lanes, h_samples, colors, radius=3):
    """Stamp the circles of one frame in place: img uint8 [H, W, 3], lanes [L, S] int (-2 = no point), h_samples [S],
    colors [L] RGB triples; lane by lane, point by point, so the last stamp wins where they overlap."""
    H, W = img.shape[:2]
    hw = circle_halfwidths(radius)
    for l, lane in enumerate(np.asarray(lanes).tolist()):
        for x, y in zip(lane, np.asarray(h_samples).tolist()):
            if x == -2:
                continue
            for dy in range(-radius, radius + 1):
                yy, h = y + dy, hw[abs(dy)]
                if 0 <= yy < H and h >= 0:
                    x0, x1 = max(x - h, 0), min(x + h, W - 1)
                    if x0 <= x1:
                        img[yy, x0:x1 + 1] = colors[l]
    return img
