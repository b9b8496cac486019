"""numpy restatement of the GPU PNG decode (csrc/png_plan.cpp, csrc/png_dec.cu): which files the GPU takes, and the
page it gives for them, equal to cv2.imdecode(buf, IMREAD_COLOR) with cv2 4.13's libpng 1.6.53 and zlib 1.2.11.

The chunk walk restates png_plan.cpp rule for rule.  The zlib stream is inflated with Python's zlib at the window the
header declares; a valid stream inflates to the same bytes on every zlib version.  Then the rows are unfiltered and
converted as libpng does under OpenCV's settings: png_set_strip_16 (a 16-bit sample keeps its high byte),
png_set_expand_gray_1_2_4_to_8 (1/2/4-bit grey times 255/85/17), png_set_palette_to_rgb (an index past the PLTE
entries reads (0, 0, 0)), png_set_gray_to_rgb, png_set_bgr and png_set_strip_alpha (no compositing); tRNS and gAMA
change nothing.  The eXIf orientation is applied as OpenCV's ExifTransform applies a JPEG's.

`decode(buf)` -> (status name, page or None): the status the GPU path must give, and the page for status "ok".  A file
with any other status is decoded by cv2, so for those only "result == cv2's" is judged, not the reason.
"""
import struct
import zlib

import numpy as np

from oracle import jpeg_ref

STATUS = ["ok", "not_png", "truncated", "header", "interlaced", "apng", "chunks", "exif", "zlib", "size", "crc", "data"]
SIGNATURE = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}


class Decline(Exception):
    def __init__(self, reason):
        super().__init__(reason)
        self.reason = reason


def _letters(t):
    return all(65 <= c <= 90 or 97 <= c <= 122 for c in t)


def parse(d, check_crc=True):
    """png_plan.cpp's walk -> dict of the IHDR fields, palette, orientation, zlib stream and window; raises Decline"""
    d = bytes(d)
    n = len(d)
    if n < 8 or d[:8] != SIGNATURE:
        raise Decline("not_png")
    if n < 16 or struct.unpack(">I", d[8:12])[0] != 13 or d[12:16] != b"IHDR":
        raise Decline("not_png")
    if n < 33:
        raise Decline("truncated")
    w, h, depth, ctype, cm, fm, il = struct.unpack(">IIBBBBB", d[16:29])
    if w == 0 or h == 0 or w > 0x7FFFFFFF or h > 0x7FFFFFFF or cm or fm or depth not in DEPTHS.get(ctype, ()):
        raise Decline("header")
    if il == 1:
        raise Decline("interlaced")
    if il:
        raise Decline("header")
    rowbytes = (w * CHANNELS[ctype] * depth + 7) // 8
    filtered = h * (1 + rowbytes)
    size_ok = w <= 1000000 and h <= 1000000 and w * h <= 1 << 30 and filtered < 1 << 31
    ihdr_crc_ok = not check_crc or zlib.crc32(d[12:29]) == struct.unpack(">I", d[29:33])[0]
    plte, orient, exif, idat, idat_done = None, 1, False, [], False
    p = 33
    while True:
        if p + 12 > n:
            raise Decline("truncated")
        L = struct.unpack(">I", d[p:p + 4])[0]
        t = d[p + 4:p + 8]
        if L > 0x7FFFFFFF or p + 12 + L > n:
            raise Decline("truncated")
        if not _letters(t):
            raise Decline("chunks")
        s = d[p + 8:p + 8 + L]
        if check_crc and zlib.crc32(t + s) != struct.unpack(">I", d[p + 8 + L:p + 12 + L])[0]:
            raise Decline("crc")
        if t != b"IDAT" and idat:
            idat_done = True
        if t == b"IDAT":
            if idat_done or (ctype == 3 and plte is None):
                raise Decline("chunks")
            idat.append(s)
        elif t == b"IEND":
            if L:
                raise Decline("chunks")
            break
        elif t == b"PLTE":
            if ctype != 3 or plte is not None or idat or L == 0 or L % 3 or L > 768:
                raise Decline("chunks")
            plte = s
        elif t in (b"acTL", b"fcTL", b"fdAT"):
            raise Decline("apng")
        elif t == b"eXIf":
            if exif:
                raise Decline("exif")
            exif = True
            try:
                orient = jpeg_ref._parse_exif(s)
            except jpeg_ref.Reject:
                raise Decline("exif")
        elif not t[0] & 0x20:
            raise Decline("chunks")
        p += 12 + L
    if not idat:
        raise Decline("truncated")
    if not ihdr_crc_ok:
        raise Decline("crc")
    z = b"".join(idat)
    if not size_ok or len(z) >= 1 << 30:
        raise Decline("size")
    if len(z) < 6 or z[0] & 15 != 8 or z[0] >> 4 > 7 or ((z[0] << 8) | z[1]) % 31 or z[1] & 0x20:
        raise Decline("zlib")
    pal = np.zeros((256, 3), np.uint8)
    if plte is not None:
        pal[:len(plte) // 3] = np.frombuffer(plte, np.uint8).reshape(-1, 3)
    return dict(w=w, h=h, depth=depth, ctype=ctype, rowbytes=rowbytes, filtered=filtered, zlib=z,
                wbits=(z[0] >> 4) + 8, palette=pal, plte_n=0 if plte is None else len(plte) // 3, orient=orient)


def inflate(info):
    """the filtered stream; Decline("data") unless the zlib stream is exactly one complete stream of `filtered` bytes"""
    try:
        dz = zlib.decompressobj(info["wbits"])
        if info["wbits"] < 15:
            # a distance past the header's window: zlib (without INFLATE_STRICT) takes one that stays inside the output
            # of the current call, so it is fed one output byte per call, as the decoder checks every distance against
            # the window (a 32 KiB window bounds every deflate distance, so wbits 15 needs no such care)
            parts, data = [], info["zlib"]
            while not dz.eof and len(parts) <= info["filtered"]:
                parts.append(dz.decompress(data, 1))
                data = dz.unconsumed_tail
                if not parts[-1] and not data:
                    break
            raw = b"".join(parts)
        else:
            raw = dz.decompress(info["zlib"])
    except zlib.error:
        raise Decline("data")
    if not dz.eof or dz.unused_data or len(raw) != info["filtered"]:
        raise Decline("data")
    return raw


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def unfilter(raw, h, rowbytes, bpp):
    """[h][rowbytes] u8 rows; Decline("data") for a filter type above 4"""
    a = np.frombuffer(raw, np.uint8).reshape(h, rowbytes + 1)
    if (a[:, 0] > 4).any():
        raise Decline("data")
    out = np.zeros((h, rowbytes), np.uint8)
    prev = np.zeros(rowbytes, np.int64)
    for y in range(h):
        ft, x = int(a[y, 0]), a[y, 1:].astype(np.int64)
        if ft == 0:
            r = x
        elif ft == 1:   # per byte lane, a prefix sum mod 256
            pad = -rowbytes % bpp
            r = np.cumsum(np.r_[x, np.zeros(pad, np.int64)].reshape(-1, bpp), axis=0).reshape(-1)[:rowbytes]
        elif ft == 2:
            r = x + prev
        else:
            xs, up, r = x.tolist(), prev.tolist(), [0] * rowbytes
            for i in range(rowbytes):
                left = r[i - bpp] if i >= bpp else 0
                ul = up[i - bpp] if i >= bpp else 0
                pr = (left + up[i]) >> 1 if ft == 3 else _paeth(left, up[i], ul)
                r[i] = (xs[i] + pr) & 255
            r = np.array(r, np.int64)
        prev = r & 255
        out[y] = prev
    return out


def convert(rows, info):
    """libpng's transforms under OpenCV's settings -> u8 BGR [h][w][3]"""
    w, d, ct = info["w"], info["depth"], info["ctype"]
    if d < 8:
        bits = np.unpackbits(rows, axis=1)[:, :w * d].reshape(rows.shape[0], w, d)
        v = (bits * (1 << np.arange(d - 1, -1, -1, dtype=np.uint8))).sum(-1).astype(np.int64)
        if ct == 3:
            rgb = info["palette"][v]
        else:
            g = (v * {1: 255, 2: 85, 4: 17}[d]).astype(np.uint8)
            rgb = np.stack([g, g, g], -1)
    else:
        s = rows[:, ::d // 8].reshape(rows.shape[0], w, -1) if d == 16 else rows.reshape(rows.shape[0], w, -1)
        if ct == 3:
            rgb = info["palette"][s[..., 0]]
        elif ct in (0, 4):
            rgb = np.repeat(s[..., :1], 3, -1)
        else:
            rgb = s[..., :3]
    return np.ascontiguousarray(rgb[..., ::-1]).astype(np.uint8)


def decode(buf):
    """(status name, page or None) as the GPU path must give them"""
    try:
        info = parse(buf)
        raw = inflate(info)
        bpp = max(1, CHANNELS[info["ctype"]] * info["depth"] // 8)
        rows = unfilter(raw, info["h"], info["rowbytes"], bpp)
    except Decline as e:
        return e.reason, None
    return "ok", jpeg_ref.orient(convert(rows, info), info["orient"])


def probe(buf):
    """the status `ctd_png_probe` gives: the walk without the CRCs and the image data"""
    try:
        parse(buf, check_crc=False)
    except Decline as e:
        return e.reason
    return "ok"
