"""TEST INFRASTRUCTURE (oracle side): a numpy restatement of the baseline JPEG decode that `cv2.imdecode(buf,
IMREAD_COLOR)` performs with its bundled libjpeg-turbo, for the files the GPU decoder takes (csrc/jpeg_plan.cpp
decides which; `parse` here applies the same rules).

Stage by stage, after libjpeg-turbo's defaults (JDCT_ISLOW, do_fancy_upsampling):
  - Huffman decode of one interleaved scan, restart intervals reset the DC predictors (jdhuff.c); DC values are summed
    in 32-bit ints and stored as int16 (JCOEF);
  - dequantise + `jpeg_idct_islow` (jidctint.c): 13-bit constants, PASS1_BITS = 2, output through the post-IDCT
    range-limit table indexed with `x & 1023` (jdmaster.c prepare_range_limit_table);
  - "fancy" h2v1 / h2v2 chroma upsampling (jdsample.c): triangle filter, rounding +1/+2 (h2v1) and +8/+7 (h2v2)
    alternating between the two output columns, edge samples replicated (context rows at the image's top and bottom
    edge repeat the first / last chroma row); a chroma plane at most 2 samples wide is box-upsampled instead
    (jinit_upsampler takes the fancy filters only above that width);
  - YCbCr -> BGR through `build_ycc_rgb_table` (jdcolor.c, 16-bit fixed point) and the sample range limit; one
    component gives B = G = R = Y;
  - EXIF orientation as OpenCV's `ExifTransform` applies it (flips and a transpose).

`decode` returns (page, exact): `exact` is False for a block whose IDCT leaves the range on which libjpeg-turbo's C
and SIMD IDCTs agree (a dequantised coefficient or a pass-1 value beyond +-16383, an output beyond [-512, 511]); the
GPU decoder hands such a page to cv2, so the oracle does not claim it.  Slow (pure Python bit reader): small images.
Nothing in the package imports this module.
"""
import struct

import numpy as np

# reason codes of ctd_jpeg_probe (include/ctd_b200.h CTD_JPEG_*)
OK, NOT_JPEG, TRUNCATED, PROGRESSIVE, ARITHMETIC, PRECISION, LOSSLESS, SAMPLING, COLOR, SCANS, EXIF, TABLES, \
    ENTROPY, RANGE_CODE, SIZE = range(15)
MAX_SCAN_BYTES = 1 << 28   # an interval's bit length stays inside int32

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


class Reject(Exception):
    def __init__(self, code, why):
        super().__init__(why)
        self.code = code


def _u16(d, o):
    return (d[o] << 8) | d[o + 1]


def _parse_exif(seg):
    """IFD0 orientation of an APP1 'Exif\\0\\0' payload (after the 6-byte header): 1 when absent; Reject(EXIF) when the
    TIFF structure does not parse cleanly or the orientation is not 1..8"""
    t = bytes(seg)
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        raise Reject(EXIF, "bad TIFF header")
    e = "<" if t[:2] == b"II" else ">"
    if struct.unpack(e + "H", t[2:4])[0] != 42:
        raise Reject(EXIF, "bad TIFF magic")
    ifd = struct.unpack(e + "I", t[4:8])[0]
    if ifd < 8 or ifd + 2 > len(t):
        raise Reject(EXIF, "IFD0 outside the block")
    n = struct.unpack(e + "H", t[ifd:ifd + 2])[0]
    if ifd + 2 + 12 * n > len(t):
        raise Reject(EXIF, "IFD0 entries outside the block")
    sizes = {1: 1, 2: 1, 3: 2, 4: 4, 5: 8, 6: 1, 7: 1, 8: 2, 9: 4, 10: 8, 11: 4, 12: 8}
    orient, seen = 1, False
    for i in range(n):
        o = ifd + 2 + 12 * i
        tag, typ, cnt = struct.unpack(e + "HHI", t[o:o + 8])
        if typ not in sizes:
            raise Reject(EXIF, "unknown entry type")
        nb = sizes[typ] * cnt
        if nb > 4:
            off = struct.unpack(e + "I", t[o + 8:o + 12])[0]
            if off + nb > len(t):
                raise Reject(EXIF, "entry data outside the block")
        if tag == 0x0112:
            if seen:
                raise Reject(EXIF, "two orientation entries")
            seen = True
            if typ != 3 or cnt != 1:
                raise Reject(EXIF, "orientation is not one SHORT")
            orient = struct.unpack(e + "H", t[o + 8:o + 10])[0]
            if not 1 <= orient <= 8:
                raise Reject(EXIF, "orientation %d" % orient)
    return orient


def parse(buf):
    """the marker walk of ctd_jpeg_probe -> dict (frame, components, tables, scan, restart interval, entropy-coded
    segments, orientation); raises Reject(code, why) for every file the GPU decoder does not take"""
    d = np.frombuffer(bytes(buf), np.uint8).tolist() if not isinstance(buf, list) else buf
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Reject(NOT_JPEG, "no SOI")
    qt, ht = {}, {}
    frame, restart, orient, exif_seen, adobe = None, 0, 1, False, None
    p = 2
    while True:
        # markers may be preceded by fill bytes 0xFF
        if p >= n or d[p] != 0xFF:
            raise Reject(TRUNCATED if p >= n else NOT_JPEG, "marker expected at %d" % p)
        while p < n and d[p] == 0xFF:
            p += 1
        if p >= n:
            raise Reject(TRUNCATED, "file ends in a marker")
        m = d[p]
        p += 1
        if m == 0xD9:
            raise Reject(TRUNCATED, "EOI before any scan")
        if 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if p + 2 > n:
            raise Reject(TRUNCATED, "segment length")
        L = _u16(d, p)
        if L < 2 or p + L > n:
            raise Reject(TRUNCATED, "segment of %d bytes" % L)
        seg = d[p + 2:p + L]
        p += L
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise Reject(SCANS, "second frame")
            if len(seg) < 6:
                raise Reject(TRUNCATED, "SOF")
            prec, h, w, nc = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if prec != 8:
                raise Reject(PRECISION, "%d-bit samples" % prec)
            if h == 0:
                raise Reject(SCANS, "height 0 (DNL)")
            if w == 0:
                raise Reject(TRUNCATED, "width 0")
            if len(seg) != 6 + 3 * nc or nc not in (1, 3):
                raise Reject(COLOR if len(seg) == 6 + 3 * nc else TRUNCATED, "%d components" % nc)
            comps = [dict(id=seg[6 + 3 * i], h=seg[7 + 3 * i] >> 4, v=seg[7 + 3 * i] & 15, tq=seg[8 + 3 * i])
                     for i in range(nc)]
            frame = dict(h=h, w=w, comps=comps)
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise Reject(PROGRESSIVE, "progressive")
        elif m in (0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF, 0xCC):
            raise Reject(ARITHMETIC, "arithmetic coding")
        elif m in (0xC3, 0xC5, 0xC7):
            raise Reject(LOSSLESS, "lossless / hierarchical")
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    raise Reject(TABLES, "DHT")
                tc, th = seg[q] >> 4, seg[q] & 15
                counts = seg[q + 1:q + 17]
                tot = sum(counts)
                if tc > 1 or th > 3 or tot > 256 or q + 17 + tot > len(seg):
                    raise Reject(TABLES, "DHT")
                ht[(tc, th)] = (counts, seg[q + 17:q + 17 + tot])
                q += 17 + tot
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                sz = 64 * (2 if pq else 1)
                if pq > 1 or tq > 3 or q + 1 + sz > len(seg):
                    raise Reject(TABLES, "DQT")
                vals = seg[q + 1:q + 1 + sz]
                zz = [(_u16(vals, 2 * i) if pq else vals[i]) for i in range(64)]
                if max(zz) > 32767:
                    raise Reject(TABLES, "quantiser above 32767")
                tab = np.zeros(64, np.int64)
                tab[ZIGZAG] = zz
                qt[tq] = tab
                q += 1 + sz
        elif m == 0xDD:
            if len(seg) != 2:
                raise Reject(TRUNCATED, "DRI")
            restart = _u16(seg, 0)
        elif m == 0xE1 and len(seg) >= 6 and bytes(seg[:6]) == b"Exif\0\0":
            if exif_seen:
                raise Reject(EXIF, "two Exif blocks")
            exif_seen = True
            orient = _parse_exif(seg[6:])
        elif m == 0xEE and len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
            adobe = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise Reject(TRUNCATED, "SOS before SOF")
            ns = seg[0] if seg else 0
            if len(seg) != 4 + 2 * ns or ns != len(frame["comps"]):
                raise Reject(SCANS, "scan of %d components" % ns)
            for i, c in enumerate(frame["comps"]):
                if seg[1 + 2 * i] != c["id"]:
                    raise Reject(SCANS, "scan component order")
                c["td"], c["ta"] = seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15
            if seg[1 + 2 * ns:4 + 2 * ns] != [0, 63, 0]:
                raise Reject(PROGRESSIVE, "spectral selection")
            return _finish(d, p, frame, qt, ht, restart, orient, adobe)
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            pass
        else:
            raise Reject(NOT_JPEG if m in (0x00, 0xFF) else SCANS, "marker 0x%02X" % m)


def _finish(d, p, frame, qt, ht, restart, orient, adobe):
    comps = frame["comps"]
    if len(comps) == 3:
        ids = [c["id"] for c in comps]
        if ids == [82, 71, 66] or (adobe is not None and adobe != 1):
            raise Reject(COLOR, "RGB components")
        hv = [(c["h"], c["v"]) for c in comps]
        if hv[1] != (1, 1) or hv[2] != (1, 1) or hv[0] not in ((1, 1), (2, 1), (2, 2)):
            raise Reject(SAMPLING, "sampling %s" % hv)
        hmax, vmax = hv[0]
    else:
        hmax = vmax = 1
        comps[0]["h"] = comps[0]["v"] = 1
    tabs = {}
    for c in comps:
        if c["tq"] not in qt or (0, c["td"]) not in ht or (1, c["ta"]) not in ht:
            raise Reject(TABLES, "missing table")
        c["qt"] = qt[c["tq"]]
        c["dc"] = _derive(*ht[(0, c["td"])], True)
        c["ac"] = _derive(*ht[(1, c["ta"])], False)
    h, w = frame["h"], frame["w"]
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    nmcu = mcux * mcuy
    nint = -(-nmcu // restart) if restart else 1
    # entropy-coded segments: FF00 unstuffed, split at RSTn (in order), EOI right after the last one
    segs, cur, q, n, rst = [], [], p, len(d), 0
    while True:
        if q >= n:
            raise Reject(TRUNCATED, "scan without EOI")
        b = d[q]
        if b != 0xFF:
            cur.append(b)
            q += 1
            continue
        if q + 1 >= n:
            raise Reject(TRUNCATED, "scan without EOI")
        m = d[q + 1]
        q += 2
        if m == 0x00:
            cur.append(0xFF)
        elif 0xD0 <= m <= 0xD7:
            if not restart or m != 0xD0 + (rst & 7):
                raise Reject(ENTROPY, "restart marker out of order")
            rst += 1
            segs.append(cur)
            cur = []
        elif m == 0xD9:
            segs.append(cur)
            break
        else:
            raise Reject(SCANS if m in (0xDA, 0xDC) else ENTROPY, "marker 0x%02X in the scan" % m)
    if q - 2 - p >= MAX_SCAN_BYTES:
        raise Reject(SIZE, "scan of %d bytes" % (q - 2 - p))
    if len(segs) != nint:
        raise Reject(ENTROPY, "%d intervals, %d expected" % (len(segs), nint))
    return dict(h=h, w=w, comps=comps, hmax=hmax, vmax=vmax, mcux=mcux, mcuy=mcuy, restart=restart, segs=segs,
                orient=orient, ecs_bytes=q - 2 - p, scan_begin=p)


def _derive(counts, vals, is_dc):
    """jdhuff.c jpeg_make_d_derived_tbl: canonical codes; the all-ones code of any length is not allowed"""
    look, code, k = {}, 0, 0
    for L in range(1, 17):
        for _ in range(counts[L - 1]):
            look[(L, code)] = vals[k]
            code += 1
            k += 1
        if code >= (1 << L):
            raise Reject(TABLES, "bad Huffman table")
        code <<= 1
    if is_dc and any(v > 15 for v in vals):
        raise Reject(TABLES, "DC symbol above 15")
    return look


class _Bits:
    def __init__(self, data):
        self.d, self.p = data, 0   # p: bit position

    def bit(self):
        i = self.p >> 3
        if i >= len(self.d):
            raise Reject(ENTROPY, "past the end of an interval")
        b = (self.d[i] >> (7 - (self.p & 7))) & 1
        self.p += 1
        return b

    def bits(self, s):
        v = 0
        for _ in range(s):
            v = (v << 1) | self.bit()
        return v

    def huff(self, look):
        code = 0
        for L in range(1, 17):
            code = (code << 1) | self.bit()
            s = look.get((L, code))
            if s is not None:
                return s
        raise Reject(ENTROPY, "invalid code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(info):
    """per component int16 [rows][cols][64] (natural order) of every block of the scan"""
    comps, mcux, mcuy = info["comps"], info["mcux"], info["mcuy"]
    single = len(comps) == 1
    if single:
        mcux, mcuy = -(-info["w"] // 8), -(-info["h"] // 8)
    out = [np.zeros((mcuy * c["v"], mcux * c["h"], 64), np.int64) for c in comps]
    R = info["restart"] or mcux * mcuy
    for iv, seg in enumerate(info["segs"]):
        br = _Bits(seg)
        pred = [0] * len(comps)
        for m in range(iv * R, min((iv + 1) * R, mcux * mcuy)):
            my, mx = divmod(m, mcux)
            for ci, c in enumerate(comps):
                for by in range(c["v"]):
                    for bx in range(c["h"]):
                        blk = out[ci][my * c["v"] + by, mx * c["h"] + bx]
                        s = br.huff(c["dc"])
                        pred[ci] = (pred[ci] + _extend(br.bits(s), s) + 2 ** 31) % 2 ** 32 - 2 ** 31
                        blk[0] = (pred[ci] + 2 ** 15) % 2 ** 16 - 2 ** 15
                        k = 1
                        while k < 64:
                            rs = br.huff(c["ac"])
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                if k > 63:
                                    raise Reject(ENTROPY, "run past coefficient 63")
                                blk[ZIGZAG[k]] = _extend(br.bits(s), s)
                                k += 1
                            elif r == 15:
                                k += 16
                                if k > 64:
                                    raise Reject(ENTROPY, "run past coefficient 63")
                            else:
                                break
        info.setdefault("ends", []).append(br.p)
        if len(seg) * 8 - br.p >= 8:
            raise Reject(ENTROPY, "bytes left in an interval")
    return out


def _range_limit():
    """prepare_range_limit_table's post-IDCT part: value at x & 1023"""
    t = np.empty(1024, np.int64)
    x = np.arange(1024)
    t[:] = np.where(x < 128, x + 128, np.where(x < 512, 255, np.where(x < 896, 0, x - 896)))
    return t


RANGE = _range_limit()
F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
         f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(v, shift):
    """one jpeg_idct_islow pass over axis 0 of v (int64 [8][...]); returns the 8 outputs before descaling"""
    c = F
    z2, z3 = v[2], v[6]
    z1 = (z2 + z3) * c["f0541"]
    tmp2 = z1 + z3 * -c["f1847"]
    tmp3 = z1 + z2 * c["f0765"]
    tmp0 = (v[0] + v[4]) << 13
    tmp1 = (v[0] - v[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = v[7], v[5], v[3], v[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * c["f1175"]
    t0, t1, t2, t3 = t0 * c["f0298"], t1 * c["f2053"], t2 * c["f3072"], t3 * c["f1501"]
    z1, z2, z3, z4 = z1 * -c["f0899"], z2 * -c["f2562"], z3 * -c["f1961"] + z5, z4 * -c["f0390"] + z5
    t0 += z1 + z3
    t1 += z2 + z4
    t2 += z2 + z3
    t3 += z1 + z4
    o = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return np.stack([(x + (1 << (shift - 1))) >> shift for x in o])


def idct_islow(coef, q):
    """coef int [..][64] natural order, q int [64] -> (u8 [..][8][8], exact per block)"""
    deq = coef.astype(np.int64) * q
    b = deq.reshape(-1, 8, 8)                                  # [blk][row v][col u]
    ws = _idct_1d(np.moveaxis(b, 1, 0), 11)                    # columns: [y][blk][u]
    ws = np.moveaxis(ws, 0, 1)                                 # [blk][y][u]
    out = _idct_1d(np.moveaxis(ws, 2, 0), 18)                  # rows: [x][blk][y]
    out = np.moveaxis(out, 0, 2)                               # [blk][y][x]
    exact = (np.abs(b).max(axis=(1, 2)) <= 16383) & (np.abs(ws).max(axis=(1, 2)) <= 16383) & \
        (out.min(axis=(1, 2)) >= -512) & (out.max(axis=(1, 2)) <= 511)
    return RANGE[out & 1023].reshape(coef.shape[:-1] + (8, 8)).astype(np.uint8), exact.reshape(coef.shape[:-1])


def _plane(coef, q):
    """component plane u8 [rows*8][cols*8] of one component's blocks"""
    px, exact = idct_islow(coef, q)
    r, c = coef.shape[:2]
    return px.transpose(0, 2, 1, 3).reshape(r * 8, c * 8), bool(exact.all())


def upsample(plane, h_fac, v_fac, ch, cw, oh, ow):
    """jdsample.c fancy upsampling of a chroma plane (its first ch x cw samples are real) to oh x ow"""
    x = plane[:ch, :cw].astype(np.int64)
    if cw <= 2:
        # jinit_upsampler: fancy only when the downsampled width is above 2, else the box filter
        out = np.repeat(np.repeat(x, v_fac, 0), h_fac, 1)
    elif v_fac == 2:
        up = np.vstack([x[:1], x[:-1]])
        dn = np.vstack([x[1:], x[-1:]])
        rows = np.empty((2 * ch, cw), np.int64)
        rows[0::2] = 3 * x + up
        rows[1::2] = 3 * x + dn
        lf = np.hstack([rows[:, :1], rows[:, :-1]])
        rt = np.hstack([rows[:, 1:], rows[:, -1:]])
        out = np.empty((2 * ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * rows + lf + 8) >> 4
        out[:, 1::2] = (3 * rows + rt + 7) >> 4
    elif h_fac == 2:
        lf = np.hstack([x[:, :1], x[:, :-1]])
        rt = np.hstack([x[:, 1:], x[:, -1:]])
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * x + lf + 1) >> 2
        out[:, 1::2] = (3 * x + rt + 2) >> 2
    else:
        out = x
    return out[:oh, :ow]


def ycc_tables():
    """jdcolor.c build_ycc_rgb_table"""
    x = np.arange(256, dtype=np.int64) - 128
    fix = lambda v: int(v * 65536 + 0.5)
    half = 1 << 15
    cr_r = (fix(1.40200) * x + half) >> 16
    cb_b = (fix(1.77200) * x + half) >> 16
    cr_g = -fix(0.71414) * x
    cb_g = -fix(0.34414) * x + half
    return cr_r, cb_b, cr_g, cb_g


def orient(img, o):
    """OpenCV ExifTransform"""
    if o >= 5:
        img = img.transpose(1, 0, 2)
    flip = {2: 1, 3: -1, 4: 0, 6: 1, 7: -1, 8: 0}.get(o)
    if flip in (1, -1):
        img = img[:, ::-1]
    if flip in (0, -1):
        img = img[::-1]
    return np.ascontiguousarray(img)


def decode(buf):
    """-> (u8 BGR [h][w][3] as cv2.imdecode(buf, IMREAD_COLOR) returns it, exact); raises Reject"""
    info = parse(buf)
    h, w = info["h"], info["w"]
    planes, exact = [], True
    for c, co in zip(info["comps"], coefficients(info)):
        p, e = _plane(co, c["qt"])
        planes.append(p)
        exact &= e
    y = planes[0][:h, :w].astype(np.int64)
    if len(planes) == 1:
        bgr = np.stack([y, y, y], -1)
    else:
        hm, vm = info["hmax"], info["vmax"]
        ch, cw = -(-h // vm), -(-w // hm)
        cb = upsample(planes[1], hm, vm, ch, cw, h, w)
        cr = upsample(planes[2], hm, vm, ch, cw, h, w)
        cr_r, cb_b, cr_g, cb_g = ycc_tables()
        r = np.clip(y + cr_r[cr], 0, 255)
        g = np.clip(y + ((cb_g[cb] + cr_g[cr]) >> 16), 0, 255)
        b = np.clip(y + cb_b[cb], 0, 255)
        bgr = np.stack([b, g, r], -1)
    return orient(bgr.astype(np.uint8), info["orient"]), exact


def probe(buf):
    """(status, shape as cv2 returns it or None, orientation) by this module's rules"""
    try:
        info = parse(buf)
    except Reject as e:
        return e.code, None, 0
    h, w = info["h"], info["w"]
    return OK, ((w, h) if info["orient"] >= 5 else (h, w)), info["orient"]
