"""JPEG decode of the loader's frames on the GPU (csrc/jpeg.cu): what Image.open(f).convert('RGB') does per image in the
reference's loader (BP/Dataloader/Load_Data_new.py:118-119), bit-identical to Pillow, for a batch of same-size frames.

    dec = JpegDecoder("cuda")
    frames = dec([open(p, "rb").read() for p in paths])      # uint8 [N,H,W,3] on the device; never synchronises
    x = FramePreprocessor(256)(frames)                        # crop / resize / flip / ToTensor (input_pipeline.py)
    dec.check()                                               # one sync: raises if any entropy-coded data was corrupt

Supported: baseline sequential DCT (SOF0, or SOF1 with 8-bit samples), Huffman coding, one scan, YCbCr 4:4:4 / 4:2:2 /
4:2:0 or one grayscale component (replicated into R, G, B as convert('RGB') does), with or without restart markers,
8- or 16-bit quantisation tables; APPn and COM segments are skipped.  Everything else raises ValueError on the host,
naming the feature.  There is no CPU fallback.

Host work per image is a walk over the markers (no per-byte Python loop: finding the end of the entropy-coded segment is
one regular-expression search, unstuffing and restart markers are handled on the device).  The frames belong to the
stream current at the call; a consumer on another stream waits for that stream and calls frames.record_stream(...).

JpegEncoder is the other direction (csrc/jpeg_enc.cu): frames -> files byte-identical to Pillow's baseline encoder."""
import functools
import re

import numpy as np

from . import _capi

_ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                    21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                    60, 61, 54, 47, 55, 62, 63], dtype=np.int64)   # zig-zag index -> natural index
_ECS_END = re.compile(rb"\xff[^\x00\xd0-\xd7\xff]")
_SAMPLINGS = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0"}
_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical (differential sequential)",
              0xC6: "hierarchical (differential progressive)", 0xC7: "hierarchical (differential lossless)",
              0xC9: "arithmetic-coded", 0xCA: "progressive arithmetic-coded", 0xCB: "lossless arithmetic-coded",
              0xCD: "hierarchical arithmetic-coded", 0xCE: "hierarchical arithmetic-coded", 0xCF: "hierarchical arithmetic-coded"}


class JpegHeader:
    """What the decoder needs from one file: size, components, sampling, tables, restart interval, and where the
    entropy-coded segment (ECS) lies."""
    __slots__ = ("width", "height", "ncomp", "comps", "qtables", "dc_tables", "ac_tables", "restart", "scan", "ecs_off",
                 "ecs_len", "sof")

    @property
    def sampling(self):
        """(h, v) of the first component relative to the others, as Pillow's get_sampling reports: -1 grayscale, 0 4:4:4,
        1 4:2:2, 2 4:2:0."""
        if self.ncomp == 1:
            return -1
        return {(1, 1): 0, (2, 1): 1, (2, 2): 2}[self.comps[0][1:3]]


def _u16(b, i):
    return (b[i] << 8) | b[i + 1]


def parse(data):
    """Walk the markers of one JPEG file.  Raises ValueError for anything outside the supported subset."""
    b = memoryview(data)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise ValueError("not a JPEG file (no SOI marker)")
    h = JpegHeader()
    h.qtables, h.dc_tables, h.ac_tables, h.restart, h.sof, h.scan = {}, {}, {}, 0, None, None
    jfif, adobe = False, None
    i = 2
    while True:
        while i < n and b[i] == 0xFF and i + 1 < n and b[i + 1] == 0xFF:   # fill bytes
            i += 1
        if i + 1 >= n or b[i] != 0xFF:
            raise ValueError("corrupt marker structure at byte %d" % i)
        m = b[i + 1]
        if m == 0xD9:
            raise ValueError("no scan (EOI before SOS)")
        if m in (0x01,) or 0xD0 <= m <= 0xD7:
            i += 2
            continue
        if i + 4 > n:
            raise ValueError("truncated marker segment")
        ln = _u16(b, i + 2)
        seg = b[i + 4:i + 2 + ln]
        if len(seg) != ln - 2:
            raise ValueError("truncated marker segment")
        if m in _SOF_NAMES:
            raise ValueError("unsupported JPEG: %s frames (SOF%d)" % (_SOF_NAMES[m], m - 0xC0))
        if m == 0xCC:
            raise ValueError("unsupported JPEG: arithmetic coding (DAC)")
        if m in (0xDE, 0xDF):
            raise ValueError("unsupported JPEG: hierarchical frames")
        if m == 0xDC:
            raise ValueError("unsupported JPEG: DNL marker")
        if m in (0xC0, 0xC1):
            if h.sof is not None:
                raise ValueError("corrupt JPEG: two frame headers")
            if seg[0] != 8:
                raise ValueError("unsupported JPEG: %d-bit samples (only 8-bit)" % seg[0])
            h.sof = m - 0xC0
            h.height, h.width, h.ncomp = _u16(seg, 1), _u16(seg, 3), seg[5]
            if h.height == 0:
                raise ValueError("unsupported JPEG: height defined by a DNL marker")
            if h.width == 0:
                raise ValueError("corrupt JPEG: zero width")
            if h.ncomp == 4:
                raise ValueError("unsupported JPEG: 4 components (CMYK / YCCK)")
            if h.ncomp not in (1, 3):
                raise ValueError("unsupported JPEG: %d components" % h.ncomp)
            h.comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(h.ncomp)]
        elif m == 0xC4:
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                bits = np.frombuffer(seg[j + 1:j + 17], dtype=np.uint8).astype(np.int64)
                nv = int(bits.sum())
                vals = bytes(seg[j + 17:j + 17 + nv])
                if tc > 1 or th > 3 or len(bits) != 16 or len(vals) != nv:
                    raise ValueError("corrupt JPEG: bad DHT segment")
                (h.ac_tables if tc else h.dc_tables)[th] = (bytes(seg[j + 1:j + 17]), vals)
                j += 17 + nv
        elif m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                if tq > 3 or pq > 1:
                    raise ValueError("corrupt JPEG: bad DQT segment")
                raw = bytes(seg[j + 1:j + 1 + 64 * (pq + 1)])
                if len(raw) != 64 * (pq + 1):
                    raise ValueError("corrupt JPEG: bad DQT segment")
                zz = np.frombuffer(raw, dtype=">u2" if pq else np.uint8).astype(np.uint16)
                nat = np.empty(64, np.uint16)
                nat[_ZIGZAG] = zz
                h.qtables[tq] = nat
                j += 1 + 64 * (pq + 1)
        elif m == 0xDD:
            h.restart = _u16(seg, 0)
        elif m == 0xE0:
            jfif = jfif or bytes(seg[:5]) == b"JFIF\x00"
        elif m == 0xEE:
            if bytes(seg[:5]) == b"Adobe" and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDA:
            if h.scan is not None:
                raise ValueError("unsupported JPEG: more than one scan")
            if h.sof is None:
                raise ValueError("corrupt JPEG: SOS before the frame header")
            ns = seg[0]
            scan = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            ss, se, ahl = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ns != h.ncomp:
                raise ValueError("unsupported JPEG: more than one scan (this scan codes %d of %d components)" % (ns, h.ncomp))
            if ss != 0 or se != 63 or ahl != 0:
                raise ValueError("unsupported JPEG: spectral selection / successive approximation in a sequential scan")
            ids = [c[0] for c in h.comps]
            order = []
            for cid, td, ta in scan:
                if cid not in ids:
                    raise ValueError("corrupt JPEG: scan names an unknown component")
                order.append((ids.index(cid), td, ta))
            if [o[0] for o in order] != list(range(h.ncomp)):
                raise ValueError("unsupported JPEG: scan components out of frame order")
            h.scan = order
            h.ecs_off = i + 2 + ln
            mm = _ECS_END.search(data, h.ecs_off)
            end = mm.start() if mm else n
            h.ecs_len = end - h.ecs_off
            i = end
            # after the scan: EOI, or markers before another scan / a DNL
            while mm is not None:
                m2 = data[mm.start() + 1]
                if m2 == 0xD9:
                    break
                if m2 == 0xDA:
                    raise ValueError("unsupported JPEG: more than one scan")
                if m2 == 0xDC:
                    raise ValueError("unsupported JPEG: DNL marker")
                if mm.start() + 4 > n:
                    break
                nxt = mm.start() + 2 + _u16(b, mm.start() + 2)
                mm = _ECS_END.search(data, nxt) if nxt < n else None
                if mm is not None and mm.start() != nxt:
                    raise ValueError("corrupt JPEG: data between markers after the scan")
            break
        i += 2 + ln
    _check_frame(h, jfif, adobe)
    return h


def _check_frame(h, jfif, adobe):
    if h.ncomp == 3:
        ids = tuple(c[0] for c in h.comps)
        # libjpeg's choice of colour space (jdapimin.c default_decompress_parms)
        if not jfif and ((adobe is not None and adobe == 0) or (adobe is None and ids == (82, 71, 66))):
            raise ValueError("unsupported JPEG: stored RGB (Adobe transform 0 or component IDs 'R','G','B')")
        if adobe is not None and adobe == 2:
            raise ValueError("unsupported JPEG: YCCK")
        if tuple(c[1:3] for c in h.comps[1:]) != ((1, 1), (1, 1)) or h.comps[0][1:3] not in _SAMPLINGS:
            raise ValueError("unsupported JPEG: sampling factors %s" % [c[1:3] for c in h.comps])
    for c in h.comps:
        if c[3] not in h.qtables:
            raise ValueError("corrupt JPEG: missing quantisation table %d" % c[3])
    for _, td, ta in h.scan:
        if td not in h.dc_tables or ta not in h.ac_tables:
            raise ValueError("corrupt JPEG: missing Huffman table")


def huffman_table(bits, vals, is_dc):
    """Decode tables of one DHT entry (libjpeg jdhuff.c jpeg_make_d_derived_tbl): a 9-bit lookahead of (length << 8) |
    symbol, and maxcode / valoff per code length for longer codes.  Returns an LfJpegHuff as a numpy record, shared
    between calls with the same table (read it, do not modify it).  Files usually share their tables (the standard ones),
    but optimised tables differ per file, so the cache keeps only the most recently used ones."""
    return _huffman_table(bytes(bits), bytes(vals), bool(is_dc))


@functools.lru_cache(maxsize=64)
def _huffman_table(bits, vals, is_dc):
    cnt = np.frombuffer(bits, dtype=np.uint8).astype(np.int64)
    nv = int(cnt.sum())
    if nv > 256:
        raise ValueError("corrupt JPEG: bad Huffman table")
    lens = np.repeat(np.arange(1, 17), cnt)
    first = np.zeros(18, np.int64)       # first code of each length (canonical Huffman)
    code = 0
    for l in range(1, 17):
        first[l] = code
        code += int(cnt[l - 1])
        if code >= (1 << l):             # as libjpeg: no code may be all ones
            raise ValueError("corrupt JPEG: bad Huffman table")
        code <<= 1
    start = np.concatenate([[0], np.cumsum(cnt)])[:16]       # index of the first symbol of each length
    codes = first[lens] + (np.arange(nv) - start[lens - 1])
    v = np.frombuffer(vals, dtype=np.uint8)
    if is_dc and nv and int(v.max()) > 15:
        raise ValueError("corrupt JPEG: bad Huffman table")
    rec = np.zeros(1, dtype=np.dtype(_capi.LfJpegHuff))[0]
    look = np.zeros(512, np.uint16)
    short = lens <= 9
    if short.any():
        sl, sc, sv = lens[short], codes[short], v[short].astype(np.int64)
        span = 1 << (9 - sl)
        idx = np.repeat(sc << (9 - sl), span) + (np.arange(int(span.sum())) - np.repeat(np.cumsum(span) - span, span))
        look[idx] = np.repeat((sl << 8) | sv, span)
    rec["look"] = look
    maxcode = np.full(18, -1, np.int64)
    valoff = np.zeros(18, np.int64)
    for l in range(1, 17):
        if cnt[l - 1]:
            maxcode[l] = first[l] + cnt[l - 1] - 1
            valoff[l] = start[l - 1] - first[l]
    maxcode[17] = 0x7fffffff
    rec["maxcode"] = maxcode.astype(np.int32)
    rec["valoff"] = valoff.astype(np.int32)
    vv = np.zeros(256, np.uint8)
    vv[:nv] = v
    rec["val"] = vv
    return rec


_IMG_DTYPE = np.dtype(_capi.LfJpegImage)


def descriptor(h, ecs_off):
    """LfJpegImage of one parsed header (layout fields are filled by lf_jpeg_workspace_bytes)."""
    d = np.zeros(1, dtype=_IMG_DTYPE)[0]
    W, H = h.width, h.height
    d["ecs_off"], d["ecs_len"], d["W"], d["H"], d["ncomp"] = ecs_off, h.ecs_len, W, H, h.ncomp
    if h.ncomp == 1:                      # non-interleaved scan: the block grid is ceil(W/8) x ceil(H/8)
        hmax = vmax = 1
        mcux, mcuy, layout = -(-W // 8), -(-H // 8), [(0, 0, 0)]
        hs = vs = [1]
    else:
        hs = [c[1] for c in h.comps]
        vs = [c[2] for c in h.comps]
        hmax, vmax = max(hs), max(vs)
        mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
        layout = [(c, dx, dy) for c in range(3) for dy in range(vs[c]) for dx in range(hs[c])]
    nmcu = mcux * mcuy
    d["mcux"], d["mcuy"], d["bpm"], d["restart"] = mcux, mcuy, len(layout), h.restart
    d["nint"] = -(-nmcu // h.restart) if h.restart else 1
    for c in range(h.ncomp):
        d["hs"][c], d["vs"][c] = hs[c], vs[c]
        d["comp_w"][c], d["comp_h"][c] = -(-W * hs[c] // hmax), -(-H * vs[c] // vmax)
        d["qtab"][c] = h.comps[c][3]
    for k, (c, dx, dy) in enumerate(layout):
        d["blk_comp"][k], d["blk_dx"][k], d["blk_dy"][k] = c, dx, dy
        d["blk_dc"][k], d["blk_ac"][k] = h.scan[c][1], h.scan[c][2]
    for t, q in h.qtables.items():
        d["qt"][t] = q
    for t, (bits, vals) in h.dc_tables.items():
        d["dc"][t] = huffman_table(bits, vals, True)
    for t, (bits, vals) in h.ac_tables.items():
        d["ac"][t] = huffman_table(bits, vals, False)
    return d


class JpegDecoder:
    """Batch JPEG decoder on one device.  Calls are ordered among themselves (they share the decoder's buffers); the
    status word collects LF_STATUS_JPEG_CORRUPT over calls until check() reads and clears it."""

    def __init__(self, device="cuda"):
        import torch
        self.device = torch.device(device)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._coef = None
        self._ws = None
        self._last = torch.cuda.Event()   # event of the previous call: the next one waits for it (shared buffers);
        self._last.record(torch.cuda.current_stream(self.device))   # first: the zeroing of the status word

    def prepare(self, datas):
        """Host half of a call: parse every file, build the descriptors and the blob (descriptors + ECS bytes).
        Returns (blob uint8 numpy, N, W, H, workspace bytes, coefficient bytes)."""
        import ctypes
        hs = [parse(d) for d in datas]
        W, H = hs[0].width, hs[0].height
        for h in hs[1:]:
            if (h.width, h.height) != (W, H):
                raise ValueError("images of different sizes in one batch: %dx%d and %dx%d" % (W, H, h.width, h.height))
        N = len(hs)
        desc = np.zeros(N, dtype=_IMG_DTYPE)
        off = N * _IMG_DTYPE.itemsize
        for k, h in enumerate(hs):
            desc[k] = descriptor(h, off)
            off += (h.ecs_len + 15) & ~15
        cb = ctypes.c_size_t(0)
        wsb = _capi.lib().lf_jpeg_workspace_bytes(desc.ctypes.data, N, ctypes.byref(cb))
        if wsb == 0:
            raise ValueError("lf_jpeg_workspace_bytes rejected the descriptors")
        blob = np.zeros(off, np.uint8)
        blob[:desc.nbytes] = desc.view(np.uint8)
        for h, d, data in zip(hs, desc, datas):
            o = int(d["ecs_off"])
            blob[o:o + h.ecs_len] = np.frombuffer(data, np.uint8, h.ecs_len, h.ecs_off)
        return blob, N, W, H, wsb, cb.value

    def __call__(self, datas):
        import torch
        if len(datas) == 0:
            raise ValueError("empty batch")
        blob, N, W, H, wsb, cbytes = self.prepare(datas)
        stream = torch.cuda.current_stream(self.device)
        if self._last is not None:
            stream.wait_event(self._last)
        if self._coef is None or self._coef.numel() < cbytes:
            self._coef = torch.zeros(cbytes, dtype=torch.uint8, device=self.device)    # zero once; every launch leaves it zero
        if self._ws is None or self._ws.numel() < wsb:
            self._ws = torch.empty(wsb, dtype=torch.uint8, device=self.device)
        for t in (self._coef, self._ws, self.status):
            t.record_stream(stream)
        pinned = torch.empty(blob.size, dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = blob
        dblob = pinned.to(self.device, non_blocking=True)                              # one pinned copy
        out = torch.empty(N, H, W, 3, dtype=torch.uint8, device=self.device)
        _capi.call("lf_jpeg_decode", _capi.ptr(dblob), N, W, H, _capi.ptr(out), _capi.ptr(self.status), _capi.ptr(self._coef),
                   self._coef.numel(), _capi.ptr(self._ws), self._ws.numel(), _capi.stream_ptr(), nbytes=blob.size + out.numel())
        self._last = torch.cuda.Event()
        self._last.record(stream)
        return out

    def check(self):
        """Read the status word (one synchronisation) and raise if a decoded file had corrupt entropy-coded data.  Waits for
        the last decode whatever stream it ran on; the next decode waits for the word to be cleared."""
        import torch
        stream = torch.cuda.current_stream(self.device)
        if self._last is not None:
            stream.wait_event(self._last)
        s = int(self.status.item())
        if s:
            self.status.zero_()
            self._last = torch.cuda.Event()
            self._last.record(stream)
            raise ValueError("corrupt JPEG data: entropy-coded segment truncated or invalid (status 0x%x)" % s)


_SAMPLING_IDS = {"4:2:0": 2, "4:4:4": 0}


class JpegEncoder:
    """Batch baseline JPEG encoder on one device (csrc/jpeg_enc.cu): uint8 [N,H,W,3] RGB or [N,H,W] grayscale frames ->
    one file per frame, byte-identical to Image.fromarray(frame).save(buf, "JPEG", quality=quality,
    subsampling=subsampling) of Pillow.  quality 1..100 (libjpeg's scaling of the Annex K tables, forced baseline);
    subsampling "4:2:0" (Pillow's default) or "4:4:4".  Standard Huffman tables, no restart markers.

        enc = JpegEncoder("cuda", quality=75)
        files = enc(frames)                               # list of bytes; one synchronisation to read the lengths
        buf, offsets, lengths = enc.encode_async(frames)  # device tensors: file n is buf[offsets[n]:offsets[n] + lengths[n]]

    Calls are ordered among themselves (they share the workspace); the outputs belong to the stream current at the call.
    encode_async can be captured into a CUDA graph once the workspace for its shape exists (one eager call first)."""

    def __init__(self, device="cuda", quality=75, subsampling="4:2:0"):
        import torch
        if subsampling not in _SAMPLING_IDS:
            raise ValueError("subsampling must be one of %s, got %r" % (sorted(_SAMPLING_IDS), subsampling))
        if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
            raise ValueError("quality must be an integer in 1..100, got %r" % (quality,))
        self.device = torch.device(device)
        self.quality, self.subsampling = int(quality), subsampling
        self._qt = {}
        for ncomp in (1, 3):
            qt = np.zeros((2, 64), np.uint16)
            _capi.check(_capi.lib().lf_jpeg_quality_tables(self.quality, ncomp, qt.ctypes.data), "lf_jpeg_quality_tables")
            self._qt[ncomp] = qt
        self._ws = None
        self._last = None

    def encode_async(self, frames):
        """frames: uint8 CUDA tensor [N,H,W,3] or [N,H,W] -> (buffer uint8, offsets int64 [N], lengths int64 [N]), all on
        the device; no synchronisation."""
        import torch
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() not in (3, 4) or \
                (frames.dim() == 4 and frames.shape[3] != 3) or frames.shape[0] < 1:
            raise ValueError("frames must be a uint8 tensor [N,H,W,3] or [N,H,W], got %s %s"
                             % (getattr(frames, "dtype", type(frames)), tuple(getattr(frames, "shape", ()))))
        _capi.require_cuda(frames)
        N, H, W = (int(v) for v in frames.shape[:3])
        ncomp = 3 if frames.dim() == 4 else 1
        sampling = _SAMPLING_IDS[self.subsampling]
        lib = _capi.lib()
        cap = lib.lf_jpeg_encode_bound(W, H, ncomp, sampling)
        wsb = lib.lf_jpeg_encode_workspace_bytes(N, W, H, ncomp, sampling)
        if cap <= 0 or wsb == 0:
            raise ValueError("cannot encode %dx%d frames (JPEG sizes are 1..65535)" % (W, H))
        frames = frames.contiguous()
        stream = torch.cuda.current_stream(self.device)
        capturing = torch.cuda.is_current_stream_capturing()      # a graph orders its own replays
        if self._last is not None and not capturing:
            stream.wait_event(self._last)
        if self._ws is None or self._ws.numel() < wsb:
            self._ws = torch.empty(wsb, dtype=torch.uint8, device=self.device)
        if not capturing:
            self._ws.record_stream(stream)
        buf = torch.empty(N * cap, dtype=torch.uint8, device=self.device)
        lengths = torch.empty(N, dtype=torch.int64, device=self.device)
        _capi.call("lf_jpeg_encode", _capi.ptr(frames), N, W, H, ncomp, sampling, self._qt[ncomp].ctypes.data, _capi.ptr(buf), cap,
                   _capi.ptr(lengths), _capi.ptr(self._ws), _capi.stream_ptr(), nbytes=frames.numel())
        if not capturing:
            self._last = torch.cuda.Event()
            self._last.record(stream)
        offsets = torch.arange(N, dtype=torch.int64, device=self.device) * cap
        return buf, offsets, lengths

    def __call__(self, frames):
        """frames -> list of N JPEG files (bytes)."""
        import torch
        buf, offsets, lengths = self.encode_async(frames)
        lens = lengths.cpu().tolist()                     # the one synchronisation
        cap = int(buf.numel()) // len(lens)
        packed = torch.cat([buf[n * cap:n * cap + l] for n, l in enumerate(lens)]).cpu().numpy()
        out, o = [], 0
        for l in lens:
            out.append(packed[o:o + l].tobytes())
            o += l
        return out
