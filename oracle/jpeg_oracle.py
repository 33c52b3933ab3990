"""Restatement of the GPU JPEG decoder (csrc/jpeg.cu) in Python / numpy, TEST INFRASTRUCTURE: the Huffman decode is a
plain sequential Python loop over the unstuffed bitstream (libjpeg jdhuff.c decode_mcu), dequantisation + ISLOW IDCT
(jidctint.c), fancy upsampling (jdsample.c; replication for chroma at most 2 samples wide) and YCbCr->RGB (jdcolor.c) are vectorised.  Headers come from the product's
marker parser (lanedetection_end2end_b200/jpeg.py), which the CPU tests check against Pillow separately.

    rgb, stats = decode(data)     # uint8 [H,W,3] == np.asarray(Image.open(BytesIO(data)).convert('RGB'))
    stats["symbols"]              # Huffman symbols decoded: the length of the serial dependency chain without restarts"""
import numpy as np

from lanedetection_end2end_b200.jpeg import _ZIGZAG, parse


def _codes(bits, vals):
    """canonical Huffman code -> symbol, keyed by (length, code)"""
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[(l, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return out


def _unstuff(ecs):
    """entropy-coded bytes -> list of restart intervals (bytes), FF00 -> FF, RSTn markers split the intervals"""
    parts, cur, i, n = [], bytearray(), 0, len(ecs)
    while i < n:
        b = ecs[i]
        if b == 0xFF:
            nx = ecs[i + 1] if i + 1 < n else None
            if nx == 0:
                cur.append(0xFF)
                i += 2
                continue
            if nx is not None and 0xD0 <= nx <= 0xD7:
                parts.append(bytes(cur))
                cur = bytearray()
                i += 2
                continue
            i += 1
            continue
        cur.append(b)
        i += 1
    parts.append(bytes(cur))
    return parts


def _decode_interval(data, nblocks, blk_tabs, coef, first_block, stats):
    bits = int.from_bytes(data, "big") if data else 0
    nbits = len(data) * 8
    p = 0

    def get(k):
        nonlocal p
        if k == 0:
            return 0
        if p + k <= nbits:
            v = (bits >> (nbits - p - k)) & ((1 << k) - 1)
        else:   # past the end: zero bits, as libjpeg inserts after a marker
            have = max(0, nbits - p)
            v = ((bits & ((1 << have) - 1)) << (k - have)) if have else 0
        p += k
        return v

    def huff(tab):
        code = 0
        for l in range(1, 17):
            code = (code << 1) | get(1)
            s = tab.get((l, code))
            if s is not None:
                return s
        raise ValueError("invalid Huffman code")

    def extend(v, s):
        return v - (1 << s) + 1 if v < (1 << (s - 1)) else v

    nat = _ZIGZAG
    for j in range(nblocks):
        dct, act = blk_tabs[j]
        blk = coef[first_block + j]
        s = huff(dct)
        stats["symbols"] += 1
        blk[0] = extend(get(s), s) if s else 0
        k = 1
        while k < 64:
            rs = huff(act)
            stats["symbols"] += 1
            r, s = rs >> 4, rs & 15
            if s:
                k += r
                blk[nat[min(k, 63)]] = extend(get(s), s)
            elif r != 15:
                break
            else:
                k += 15
            k += 1


def entropy_decode(data, h=None):
    """coefficients [nblocks][64] int32 (natural order, DC values), in scan order; and the block layout"""
    h = h or parse(data)
    W, H = h.width, h.height
    if h.ncomp == 1:
        mcux, mcuy, layout = -(-W // 8), -(-H // 8), [(0, 0, 0)]
    else:
        hs, vs = [c[1] for c in h.comps], [c[2] for c in h.comps]
        mcux, mcuy = -(-W // (8 * max(hs))), -(-H // (8 * max(vs)))
        layout = [(c, dx, dy) for c in range(3) for dy in range(vs[c]) for dx in range(hs[c])]
    bpm, nmcu = len(layout), mcux * mcuy
    tabs = [(_codes(*[list(x) for x in h.dc_tables[h.scan[c][1]]]), _codes(*[list(x) for x in h.ac_tables[h.scan[c][2]]]))
            for c, _, _ in layout]
    coef = np.zeros((nmcu * bpm, 64), np.int64)
    parts = _unstuff(bytes(data[h.ecs_off:h.ecs_off + h.ecs_len]))
    R = h.restart or nmcu
    stats = {"symbols": 0, "intervals": len(parts)}
    for k, part in enumerate(parts):
        m0, m1 = k * R, min((k + 1) * R, nmcu)
        if m0 >= nmcu:
            break
        _decode_interval(part, (m1 - m0) * bpm, [tabs[j % bpm] for j in range(m0 * bpm, m1 * bpm)], coef, m0 * bpm, stats)
        # DC differences -> values, per component, reset at every interval
        for c in range(h.ncomp):
            idx = [m * bpm + j for m in range(m0, m1) for j in range(bpm) if layout[j][0] == c]
            coef[idx, 0] = np.cumsum(coef[idx, 0])
    return coef, layout, (mcux, mcuy), h, stats


_C = dict(F_0_298=2446, F_0_390=3196, F_0_541=4433, F_0_765=6270, F_0_899=7373, F_1_175=9633, F_1_501=12299, F_1_847=15137,
          F_1_961=16069, F_2_053=16819, F_2_562=20995, F_3_072=25172)


def _islow_1d(d):
    """d[..., 8] int64 -> un-descaled outputs (jidctint.c even / odd parts)"""
    c = _C
    z1 = (d[..., 2] + d[..., 6]) * c["F_0_541"]
    t2 = z1 - d[..., 6] * c["F_1_847"]
    t3 = z1 + d[..., 2] * c["F_0_765"]
    t0 = (d[..., 0] + d[..., 4]) << 13
    t1 = (d[..., 0] - d[..., 4]) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    a0, a1, a2, a3 = d[..., 7], d[..., 5], d[..., 3], d[..., 1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * c["F_1_175"]
    a0, a1, a2, a3 = a0 * c["F_0_298"], a1 * c["F_2_053"], a2 * c["F_3_072"], a3 * c["F_1_501"]
    z1, z2 = z1 * -c["F_0_899"], z2 * -c["F_2_562"]
    z3, z4 = z3 * -c["F_1_961"] + z5, z4 * -c["F_0_390"] + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    return np.stack([t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3], -1)


def idct_islow(coef, q):
    """coef [n][64] natural order, q [n][64] -> uint8 [n][8][8]"""
    d = (coef * q.astype(np.int16).astype(np.int64)).reshape(-1, 8, 8)
    ws = (_islow_1d(np.swapaxes(d, 1, 2)) + (1 << 10)) >> 11          # columns: ws[n][col][row]
    o = _islow_1d(np.swapaxes(ws, 1, 2))                              # rows:    o[n][row][col]
    m = ((o + (1 << 17)) >> 18) & 1023
    t = np.where(m < 512, m, m - 1024) + 128
    return np.clip(t, 0, 255).astype(np.uint8)


def planes(coef, layout, mcu, h):
    mcux, mcuy = mcu
    bpm = len(layout)
    out = []
    for c in range(h.ncomp):
        hc, vc = (1, 1) if h.ncomp == 1 else h.comps[c][1:3]
        sel = [j for j in range(bpm) if layout[j][0] == c]
        q = np.broadcast_to(h.qtables[h.comps[c][3]], (1, 64))
        idx = (np.arange(mcux * mcuy)[:, None] * bpm + np.array(sel)[None, :]).reshape(-1)
        px = idct_islow(coef[idx], q).reshape(mcuy, mcux, vc, hc, 8, 8)
        out.append(px.transpose(0, 2, 4, 1, 3, 5).reshape(mcuy * vc * 8, mcux * hc * 8))
    return out


def _fancy_h2(p, dw, bias_even, bias_odd, shift, w_edge):
    """one axis of fancy upsampling over the first dw columns of p (values already column sums for h2v2)"""
    a = p[:, :dw].astype(np.int64)
    left = np.concatenate([a[:, :1], a[:, :-1]], 1)
    right = np.concatenate([a[:, 1:], a[:, -1:]], 1)
    even = (a * 3 + left + bias_even) >> shift
    odd = (a * 3 + right + bias_odd) >> shift
    return np.stack([even, odd], -1).reshape(a.shape[0], 2 * dw)


def upsample(p, dw, dh, hup, vup):
    if not hup:
        return p.astype(np.int64)
    if dw <= 2:   # jinit_upsampler: no fancy filter below 3 samples -> h2v1_upsample / h2v2_upsample (replication)
        a = p[:dh, :dw].astype(np.int64)
        return np.repeat(np.repeat(a, 2, 1), 2 if vup else 1, 0)
    if not vup:   # h2v1: 3/4 nearer + 1/4 further, biases +1 / +2; edge columns replicated
        return _fancy_h2(p[:dh], dw, 1, 2, 2, None)
    a = p[:dh, :].astype(np.int64)
    above = np.concatenate([a[:1], a[:-1]], 0)
    below = np.concatenate([a[1:], a[-1:]], 0)
    cs = np.stack([a * 3 + above, a * 3 + below], 1).reshape(2 * dh, a.shape[1])      # column sums per output row
    return _fancy_h2(cs, dw, 8, 7, 4, None)


def decode(data):
    coef, layout, mcu, h, stats = entropy_decode(data)
    pl = planes(coef, layout, mcu, h)
    W, H = h.width, h.height
    Y = pl[0][:H, :W].astype(np.int64)
    if h.ncomp == 1:
        g = Y.astype(np.uint8)
        return np.stack([g, g, g], -1), stats
    hup, vup = h.comps[0][1] == 2, h.comps[0][2] == 2
    dw, dh = -(-W // 2) if hup else W, -(-H // 2) if vup else H
    cb = upsample(pl[1], dw, dh, hup, vup)[:H, :W] - 128
    cr = upsample(pl[2], dw, dh, hup, vup)[:H, :W] - 128
    r = Y + ((91881 * cr + 32768) >> 16)
    g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = Y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8), stats
