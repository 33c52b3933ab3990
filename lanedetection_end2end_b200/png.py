"""PNG decode of the loader's ground-truth label maps on the GPU (csrc/png.cu): what Image.open(f).convert('P') does per
image in the reference's loader (BP/Dataloader/Load_Data_new.py:120-121), bit-identical to Pillow, for a batch of
same-size maps.

    dec = PngDecoder("cuda")
    maps = dec([open(p, "rb").read() for p in paths])        # uint8 [N,H,W] on the device; never synchronises
    gt = LabelPreprocessor(256, nclasses=4)(maps, flip=mask)  # crop / NEAREST resize / class rules (input_pipeline.py)
    dec.check()                                               # one sync: raises if any compressed stream was corrupt

Supported: non-interlaced PNGs of colour type 0 (grayscale) at 8 bits or colour type 3 (palette) at 1, 2, 4 or 8 bits --
what Pillow and OpenCV write for a uint8 label map.  The frame holds the gray values or the palette indices, which is
what convert('P') returns for these files (PLTE, tRNS and the other ancillary chunks do not change it, so they are
skipped).  Everything else raises ValueError on the host, naming the feature: Adam7 interlace, colour types 2 / 4 / 6
(their convert('P') quantises to the web palette with dithering), 16-bit samples, grayscale below 8 bits, a zlib preset
dictionary, a compression or filter method other than 0, a bad signature or IHDR, no IDAT.  There is no CPU fallback.

Host work per image is a walk over the chunks and one copy of the IDAT payloads into the batch's pinned blob; inflate,
unfiltering and unpacking run on the device.  The frames belong to the stream current at the call; a consumer on another
stream waits for that stream and calls maps.record_stream(...)."""
import struct

import numpy as np

from . import _capi

SIGNATURE = b"\x89PNG\r\n\x1a\n"
_COLOUR_NAMES = {2: "RGB", 4: "grayscale + alpha", 6: "RGBA"}
_DEPTHS = {0: (1, 2, 4, 8, 16), 3: (1, 2, 4, 8), 2: (8, 16), 4: (8, 16), 6: (8, 16)}


class PngHeader:
    """What the decoder needs from one file: size, colour type, bit depth and its IDAT payloads (joined)."""
    __slots__ = ("width", "height", "depth", "colour", "zdata")


def parse(data):
    """Walk the chunks of one PNG file.  Raises ValueError for anything outside the supported subset."""
    b = memoryview(data)
    n = len(b)
    if n < 8 or bytes(b[:8]) != SIGNATURE:
        raise ValueError("not a PNG file (bad signature)")
    h = PngHeader()
    idat = []
    i = 8
    first = True
    while True:
        if i + 8 > n:
            raise ValueError("corrupt PNG: truncated chunk" if idat or not first else "corrupt PNG: no IHDR")
        ln, ctype = struct.unpack_from(">I4s", b, i)
        if i + 12 + ln > n:
            raise ValueError("corrupt PNG: truncated %s chunk" % ctype.decode("latin-1"))
        body = b[i + 8:i + 8 + ln]
        if first:
            if ctype != b"IHDR" or ln != 13:
                raise ValueError("corrupt PNG: bad IHDR")
            _ihdr(h, body)
            first = False
        elif ctype == b"IDAT":
            idat.append(body)
        elif ctype == b"IEND":
            break
        elif ctype == b"IHDR":
            raise ValueError("corrupt PNG: bad IHDR (a second one)")
        i += 12 + ln
    if not idat:
        raise ValueError("corrupt PNG: no IDAT chunk")
    h.zdata = b"".join(idat)
    _check_zlib_header(h.zdata)
    return h


def _ihdr(h, body):
    w, hh, depth, colour, comp, filt, interlace = struct.unpack(">IIBBBBB", body)
    if w == 0 or hh == 0 or w >= 1 << 31 or hh >= 1 << 31 or colour not in _DEPTHS or depth not in _DEPTHS[colour]:
        raise ValueError("corrupt PNG: bad IHDR (%dx%d, colour type %d, bit depth %d)" % (w, hh, colour, depth))
    if comp != 0:
        raise ValueError("unsupported PNG: compression method %d" % comp)
    if filt != 0:
        raise ValueError("unsupported PNG: filter method %d" % filt)
    if interlace == 1:
        raise ValueError("unsupported PNG: Adam7 interlace")
    if interlace != 0:
        raise ValueError("corrupt PNG: bad IHDR (interlace method %d)" % interlace)
    if colour in _COLOUR_NAMES:
        raise ValueError("unsupported PNG: colour type %d (%s); label maps are grayscale or palette images"
                         % (colour, _COLOUR_NAMES[colour]))
    if depth == 16:
        raise ValueError("unsupported PNG: 16-bit samples")
    if colour == 0 and depth < 8:
        raise ValueError("unsupported PNG: %d-bit grayscale (only 8-bit)" % depth)
    h.width, h.height, h.depth, h.colour = w, hh, depth, colour


def _check_zlib_header(z):
    if len(z) < 2:
        raise ValueError("corrupt PNG: zlib stream too short")
    cmf, flg = z[0], z[1]
    if cmf & 15 != 8:
        raise ValueError("unsupported PNG: zlib compression method %d" % (cmf & 15))
    if cmf >> 4 > 7 or (cmf * 256 + flg) % 31:
        raise ValueError("corrupt PNG: bad zlib header")
    if flg & 0x20:
        raise ValueError("unsupported PNG: zlib preset dictionary")


_IMG_DTYPE = np.dtype(_capi.LfPngImage)


class PngDecoder:
    """Batch PNG decoder on one device.  Calls are ordered among themselves (they share the decoder's workspace); the
    status word collects LF_STATUS_PNG_CORRUPT over calls until check() reads and clears it."""

    def __init__(self, device="cuda"):
        import torch
        self.device = torch.device(device)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._ws = None
        self._last = torch.cuda.Event()   # event of the previous call: the next one waits for it (shared workspace);
        self._last.record(torch.cuda.current_stream(self.device))   # first: the zeroing of the status word

    def prepare(self, datas):
        """Host half of a call: parse every file, build the descriptors and the blob (descriptors + zlib streams).
        Returns (blob uint8 numpy, N, W, H, workspace bytes)."""
        hs = [parse(d) for d in datas]
        W, H = hs[0].width, hs[0].height
        for h in hs[1:]:
            if (h.width, h.height) != (W, H):
                raise ValueError("images of different sizes in one batch: %dx%d and %dx%d" % (W, H, h.width, h.height))
        N = len(hs)
        desc = np.zeros(N, dtype=_IMG_DTYPE)
        off = N * _IMG_DTYPE.itemsize
        for k, h in enumerate(hs):
            d = desc[k]
            d["zoff"], d["zlen"], d["W"], d["H"], d["depth"] = off, len(h.zdata), W, H, h.depth
            off += (len(h.zdata) + 15) & ~15
        wsb = _capi.lib().lf_png_workspace_bytes(desc.ctypes.data, N)
        if wsb == 0:
            raise ValueError("lf_png_workspace_bytes rejected the descriptors (image too large?)")
        blob = np.zeros(off, np.uint8)
        blob[:desc.nbytes] = desc.view(np.uint8)
        for h, d in zip(hs, desc):
            o = int(d["zoff"])
            blob[o:o + len(h.zdata)] = np.frombuffer(h.zdata, np.uint8)
        return blob, N, W, H, wsb

    def __call__(self, datas):
        import torch
        if len(datas) == 0:
            raise ValueError("empty batch")
        blob, N, W, H, wsb = self.prepare(datas)
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(self._last)
        if self._ws is None or self._ws.numel() < wsb:
            self._ws = torch.empty(wsb, dtype=torch.uint8, device=self.device)
        for t in (self._ws, self.status):
            t.record_stream(stream)
        pinned = torch.empty(blob.size, dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = blob
        dblob = pinned.to(self.device, non_blocking=True)                              # one pinned copy
        out = torch.empty(N, H, W, dtype=torch.uint8, device=self.device)
        _capi.call("lf_png_decode", _capi.ptr(dblob), N, W, H, _capi.ptr(out), _capi.ptr(self.status), _capi.ptr(self._ws),
                   self._ws.numel(), _capi.stream_ptr(), nbytes=blob.size + out.numel())
        self._last = torch.cuda.Event()
        self._last.record(stream)
        return out

    def check(self):
        """Read the status word (one synchronisation) and raise if a decoded file had a corrupt compressed stream.  Waits
        for the last decode whatever stream it ran on; the next decode waits for the word to be cleared."""
        import torch
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(self._last)
        s = int(self.status.item())
        if s:
            self.status.zero_()
            self._last = torch.cuda.Event()
            self._last.record(stream)
            raise ValueError("corrupt PNG data: invalid or truncated zlib stream, bad Adler-32 or filter type (status 0x%x)" % s)
