"""Seeded PNG files for the GPU PNG decoder's tests: every colour type and bit depth it takes, every filter, zlib
levels / strategies / windows / memLevel 1, hand-made deflate blocks, split IDAT chunks, ancillary chunks, eXIf
orientations, odd and large sizes, PIL's adaptive filtering, cv2's and PngEncoder's own files, and every decline.

`corpus(large=...)` -> list of (name, file bytes, expected status name).  The expected status is what the GPU path
gives: "ok", a probe reason, or "crc" / "data" for what only the decode finds.
"""
import io
import struct
import zlib

import cv2
import numpy as np

from oracle.png_ref import BitWriter
from oracle.png_decode_ref import CHANNELS

SIGNATURE = b"\x89PNG\r\n\x1a\n"


def chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows, bpp, filters):
    """[h][rowbytes] u8 rows, one filter type per row -> the filtered stream"""
    h, rb = rows.shape
    out, prev = [], np.zeros(rb, np.int64)
    for y in range(h):
        x = rows[y].astype(np.int64)
        a = np.r_[np.zeros(bpp, np.int64), x[:-bpp]][:rb]
        c = np.r_[np.zeros(bpp, np.int64), prev[:-bpp]][:rb]
        ft = int(filters[y])
        pred = [0, a, prev, (a + prev) >> 1, _paeth(a, prev, c)][ft]
        out.append(bytes([ft]) + ((x - pred) & 255).astype(np.uint8).tobytes())
        prev = x
    return b"".join(out)


def ihdr(w, h, depth, ctype, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace))


def assemble(w, h, depth, ctype, z, pre=b"", post=b"", split=None, interlace=0):
    """a PNG file around zlib stream z; split: IDAT payload sizes (the rest in a last chunk)"""
    idats, p = [], 0
    for s in split or []:
        idats.append(chunk(b"IDAT", z[p:p + s]))
        p += s
    idats.append(chunk(b"IDAT", z[p:]))
    return SIGNATURE + ihdr(w, h, depth, ctype, interlace) + pre + b"".join(idats) + post + chunk(b"IEND", b"")


def rows_for(rng, w, h, depth, ctype):
    rb = (w * CHANNELS[ctype] * depth + 7) // 8
    return rng.integers(0, 256, (h, rb), dtype=np.uint8)


def make(rng, w, h, depth, ctype, filters=None, level=6, pre=b"", post=b"", plte=None, **zkw):
    rows = rows_for(rng, w, h, depth, ctype)
    bpp = max(1, CHANNELS[ctype] * depth // 8)
    if filters is None:
        filters = rng.integers(0, 5, h)
    elif np.isscalar(filters):
        filters = np.full(h, filters)
    if ctype == 3:
        pre = chunk(b"PLTE", plte if plte is not None else rng.integers(0, 256, 3 << depth, dtype=np.uint8).tobytes()) + pre
    co = zlib.compressobj(level, zlib.DEFLATED, zkw.get("wbits", 15), zkw.get("mem", 8), zkw.get("strategy", 0))
    z = co.compress(filter_rows(rows, bpp, filters)) + co.flush()
    return assemble(w, h, depth, ctype, z, pre, post)


def exif(orient, le=True):
    e = "<" if le else ">"
    return (b"II" if le else b"MM") + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHI", 0x0112, 3, 1) + struct.pack(e + "H", orient) + b"\0\0" + struct.pack(e + "I", 0)


def structured(seed, h, w):
    rng = np.random.default_rng(seed)
    page = np.full((h, w, 3), 255, np.uint8)
    for _ in range(max(1, h * w // 4000)):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        cv2.putText(page, "TEXT", (x, y), cv2.FONT_HERSHEY_SIMPLEX, 0.6, tuple(int(v) for v in rng.integers(0, 200, 3)), 1)
    page[: h // 3, : w // 3] = rng.integers(0, 256, (h // 3, w // 3, 3), dtype=np.uint8) // 64 * 64
    return page


def pil_png(img, mode, **kw):
    from PIL import Image
    if mode in ("RGB", "RGBA"):
        im = Image.fromarray(np.ascontiguousarray(img[..., ::-1]), "RGB").convert(mode)
    elif mode in ("L", "LA", "1"):
        im = Image.fromarray(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), "L").convert(mode)
    elif mode == "I;16":
        g = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY).astype(np.uint16) * 257 + 3
        im = Image.fromarray(g, "I;16")
    else:   # palette
        im = Image.fromarray(np.ascontiguousarray(img[..., ::-1]), "RGB").quantize(kw.pop("colors", 256))
    b = io.BytesIO()
    im.save(b, "PNG", **kw)
    return b.getvalue()


def _dynamic_literals(data):
    """one final dynamic block of literals with a single one-bit distance code: litlen lengths 8 for 0..254 and 9 for
    255 and 256 (a complete code), code-length code lengths 1 (for 8) and 2 (for 1 and 9)"""
    bw = BitWriter()

    def huff(code, n):   # a Huffman code, first bit first
        bw.put(int(format(code, "0%db" % n)[::-1], 2), n)
    bw.put(1, 1)
    bw.put(2, 2)
    bw.put(0, 5)   # HLIT 257
    bw.put(0, 5)   # HDIST 1
    bw.put(15, 4)  # HCLEN 19
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    cl = {8: 1, 1: 2, 9: 2}
    for s in order:
        bw.put(cl.get(s, 0), 3)
    clcode = {8: (0, 1), 1: (2, 2), 9: (3, 2)}
    for L in [8] * 255 + [9, 9] + [1]:
        huff(*clcode[L])
    for v in data:
        huff(v, 8) if v < 255 else huff(510, 9)
    huff(511, 9)
    return bw.tobytes()


def zwrap(deflate, raw, cmf=0x78):
    flg = 31 - ((cmf << 8) % 31)
    return bytes([cmf, flg % 256 if flg != 31 else 0]) + deflate + struct.pack(">I", zlib.adler32(raw))


def stored(raw, sizes):
    bw = BitWriter()
    p = 0
    for i, s in enumerate(sizes):
        bw.put(1 if i == len(sizes) - 1 else 0, 1)
        bw.put(0, 2)
        bw.align()
        bw.put(s, 16)
        bw.put(s ^ 0xFFFF, 16)
        bw.put(int.from_bytes(raw[p:p + s], "little"), 8 * s)
        p += s
    return bw.tobytes()


def eob_then(raw):
    """a fixed block with only EOB, an empty stored block to reach a byte, then zlib's raw deflate of raw"""
    bw = BitWriter()
    bw.put(0, 1)
    bw.put(1, 2)
    bw.put(0, 7)
    bw.put(0, 1)
    bw.put(0, 2)
    bw.align()
    bw.put(0, 16)
    bw.put(0xFFFF, 16)
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    return bw.tobytes() + co.compress(raw) + co.flush()


def recrc(data, kind=b"IDAT", mutate=None):
    """the file with the first `kind` chunk's payload passed through mutate and its CRC recomputed"""
    p = 8
    while True:
        L = struct.unpack(">I", data[p:p + 4])[0]
        if data[p + 4:p + 8] == kind:
            body = mutate(bytearray(data[p + 8:p + 8 + L]))
            return data[:p] + chunk(kind, bytes(body)) + data[p + 12 + L:]
        p += 12 + L


def corpus(large=True):
    rng = np.random.default_rng(2026)
    out = []
    add = lambda name, data, expect="ok": out.append((name, bytes(data), expect))
    # every colour type x bit depth, odd widths, a random filter per row
    for ct, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for d in depths:
            for w, h in ((7, 5), (13, 9), (1, 3)):
                add("ct%d_d%d_%dx%d" % (ct, d, w, h), make(rng, w, h, d, ct))
    # a short palette: indices past it read (0, 0, 0)
    add("plte_short", make(rng, 9, 4, 8, 3, plte=bytes(range(12))))
    add("plte_short_2bit", make(rng, 9, 4, 2, 3, plte=bytes([10, 20, 30])))
    # each filter on every row
    for ft in range(5):
        for ct, d in ((2, 8), (0, 2), (6, 16), (4, 8)):
            add("filter%d_ct%d_d%d" % (ft, ct, d), make(rng, 11, 6, d, ct, filters=ft))
    # zlib levels x strategies, windows, memLevel 1
    for lv in range(10):
        for strat in range(5):
            add("z_l%d_s%d" % (lv, strat), make(rng, 40, 30, 8, 2, level=lv, strategy=strat))
    for wb in range(9, 16):
        add("z_wbits%d" % wb, make(rng, 64, 48, 8, 0, level=9, wbits=wb, filters=2))
    add("z_mem1", make(rng, 120, 90, 8, 2, level=6, mem=1))
    # hand-made blocks
    raw = filter_rows(rows_for(rng, 65534, 1, 8, 0), 1, [1])
    add("stored_65535", assemble(65534, 1, 8, 0, zwrap(stored(raw, [0, 65535]), raw)))
    raw = filter_rows(rows_for(rng, 20, 7, 8, 2), 3, rng.integers(0, 5, 7))
    add("dynamic_one_distance_code", assemble(20, 7, 8, 2, zwrap(_dynamic_literals(raw), raw)))
    add("eob_only_block", assemble(20, 7, 8, 2, zwrap(eob_then(raw), raw)))
    # IDAT split into 1-byte and empty chunks
    z = zlib.compress(raw, 6)
    add("idat_split", assemble(20, 7, 8, 2, z, split=[1, 0, 1, 3, 0, 1] + [1] * 20))
    # ancillary chunks before and after the image data
    anc = chunk(b"gAMA", struct.pack(">I", 100000)) + chunk(b"tEXt", b"Comment\0hi") + chunk(b"pHYs", bytes(9))
    add("ancillary", assemble(20, 7, 8, 2, z, pre=anc + chunk(b"tRNS", bytes(6)), post=chunk(b"tEXt", b"After\0x")))
    add("trns_grey", make(rng, 9, 5, 8, 0, pre=chunk(b"tRNS", b"\0\x40")))
    add("trns_palette", make(rng, 9, 5, 4, 3, pre=chunk(b"tRNS", bytes([0, 7, 255]))))
    # eXIf orientations, before and after IDAT, both byte orders
    for o in range(1, 9):
        add("exif%d_before" % o, make(rng, 13, 6, 8, 2, pre=chunk(b"eXIf", exif(o, o % 2 == 0))))
        add("exif%d_after" % o, make(rng, 13, 6, 8, 0, post=chunk(b"eXIf", exif(o, o % 2 == 1))))
    # odd sizes
    for w, h in ((1, 1), (8193, 1), (1, 8193)):
        add("size_%dx%d" % (w, h), make(rng, w, h, 8, 2))
    # PIL: adaptive filters (Paeth and friends), every mode it writes
    img = structured(5, 61, 83)
    for mode, kw in (("RGB", {}), ("RGBA", {}), ("L", {}), ("LA", {}), ("1", {}), ("I;16", {}), ("P", {}),
                     ("P", {"colors": 16, "bits": 4}), ("P", {"colors": 4, "bits": 2}), ("P", {"colors": 2, "bits": 1}),
                     ("RGB", {"compress_level": 9}), ("RGB", {"compress_level": 1})):
        add("pil_%s_%s" % (mode.replace(";", ""), "_".join("%s%s" % kv for kv in kw.items())), pil_png(img, mode, **kw))
    # cv2's own files: pages and masks
    add("cv2_page", cv2.imencode(".png", img)[1])
    add("cv2_mask", cv2.imencode(".png", (cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) > 128).astype(np.uint8) * 255)[1])
    add("cv2_level9", cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 9])[1])
    if large:
        for ct, name in ((0, "grey"), (2, "rgb")):
            big = structured(9, 7016, 4960)
            page = cv2.cvtColor(big, cv2.COLOR_BGR2GRAY) if ct == 0 else big
            add("a4_300dpi_%s" % name, cv2.imencode(".png", page)[1])
    # declines the probe finds
    good = make(rng, 13, 6, 8, 2)
    add("interlaced", SIGNATURE + ihdr(4, 4, 8, 0, 1) + chunk(b"IDAT", zlib.compress(bytes(40))) + chunk(b"IEND", b""),
        "interlaced")
    add("apng", good[:33] + chunk(b"acTL", bytes(8)) + good[33:], "apng")
    add("bad_depth", SIGNATURE + ihdr(4, 4, 4, 2) + good[33:], "header")
    add("two_exif", make(rng, 5, 5, 8, 2, pre=chunk(b"eXIf", exif(6)) + chunk(b"eXIf", exif(3))), "exif")
    add("bad_exif", make(rng, 5, 5, 8, 2, pre=chunk(b"eXIf", b"II*\0junk")), "exif")
    split = good[:-12] + chunk(b"tEXt", b"a\0b") + chunk(b"IDAT", b"") + chunk(b"IEND", b"")
    add("idat_not_consecutive", split, "chunks")
    add("palette_without_plte", SIGNATURE + ihdr(4, 4, 8, 3) + good[33:], "chunks")
    add("no_iend", good[:-12], "truncated")
    add("truncated", good[:len(good) // 2], "truncated")
    add("bad_zlib_header", recrc(good, mutate=lambda b: bytes([0x79]) + b[1:]), "zlib")
    add("not_png", b"junk" * 10, "not_png")
    # declines only the decode finds
    add("bad_idat_crc", good[:-16] + bytes([good[-16] ^ 1]) + good[-15:], "crc")
    add("bad_ancillary_crc", (lambda d: d[:-1] + bytes([d[-1] ^ 1]))(good[:33] + chunk(b"tEXt", b"a\0b")) + good[33:],
        "crc")

    def flip(k):
        def m(b):
            b[k] ^= 0x5A
            return b
        return m
    add("bad_adler", recrc(good, mutate=lambda b: b[:-1] + bytes([b[-1] ^ 1])), "data")
    for k in (2, 5, 9, 20):
        add("corrupt_idat_%d" % k, recrc(good, mutate=flip(k)), None)   # cv2 decides; the status is not fixed
    raw = filter_rows(rows_for(rng, 13, 6, 8, 2), 3, [0] * 6)
    add("not_enough_data", assemble(13, 6, 8, 2, zlib.compress(raw[:-5])), "data")
    add("too_much_data", assemble(13, 6, 8, 2, zlib.compress(raw + b"\0" * 7)), "data")
    add("data_after_final_block", assemble(13, 6, 8, 2, zlib.compress(raw)[:-4] + b"\0\0" +
                                           struct.pack(">I", zlib.adler32(raw))), "data")
    add("filter_type_5", assemble(13, 6, 8, 2, zlib.compress(b"\5" + raw[1:])), "data")
    half = rng.integers(0, 256, 999, dtype=np.uint8).tobytes()
    far = b"\0" + half + half   # one row whose second half repeats its first at distance 999
    z = bytearray(zlib.compress(far, 9))
    z[0], z[1] = 0x18, 31 - ((0x18 << 8) % 31)   # the header declares a 512-byte window
    add("distance_past_window", assemble(1998, 1, 8, 0, bytes(z)), "data")
    add("block_type_3", assemble(13, 6, 8, 2, zwrap(bytes([0x07, 0, 0]), raw)), "data")
    return out
