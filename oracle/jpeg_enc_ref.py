"""TEST INFRASTRUCTURE (oracle side): a numpy restatement of the baseline JPEG file `cv2.imencode('.jpg', img, params)`
writes with OpenCV 4.13's bundled libjpeg-turbo 3.1, for u8 grey [h][w] and BGR [h][w][3] images.

Stage by stage, after what OpenCV sets (JCS_EXT_BGR or JCS_GRAYSCALE input, jpeg_set_defaults, jpeg_set_quality with
force_baseline, optimize_coding, restart_interval, the luma sampling factors; JDCT_ISLOW, no smoothing):
  - parameters (`parse_params`): quality clamped to [0, 100] and quality 0 scaled as 1 (jpeg_quality_scaling); the
    restart interval clamped to [0, 65535]; OPTIMIZE clamped to [0, 1]; a sampling value that is not one of the
    five IMWRITE_JPEG_SAMPLING_FACTOR_* constants falls back to 4:2:0; a grey image is one component with factors 1x1
    whatever the sampling parameter says;
  - BGR -> YCbCr with jccolor.c's 16-bit fixed-point tables (rounding 1/2 on Y, 1/2 - epsilon on Cb / Cr);
  - edges: the bottom input row is repeated to a whole row group (max_v rows), each component is downsampled, its
    last downsampled row is repeated to whole iMCU rows, and the right edge is repeated to whole blocks of the
    component (jcprepct.c, jcsample.c expand_right_edge);
  - downsampling (jcsample.c): h2v1 with bias 0, 1, 0, 1, ..., h2v2 with bias 1, 2, 1, 2, ... (both restarting each
    row), `int_downsample` (rounded mean) for 4:1:1 and 4:4:0;
  - dummy blocks of an interleaved MCU past a component's width or height: zero AC and the DC of the MCU's previous
    block (jccoefct.c): the last real block of the row for a right-edge dummy, the MCU's last block of the row above
    for a bottom dummy row;
  - `jpeg_fdct_islow` (jfdctint.c: CONST_BITS 13, PASS1_BITS 2) on samples - 128, output scaled by 8;
  - quantisation by libjpeg-turbo's reciprocals (jcdctmgr.c compute_reciprocal / quantize) of divisor 8 * q;
  - quantisation tables: Annex K.1 scaled by jpeg_quality_scaling, (t * scale + 50) / 100 clamped to [1, 255];
  - Huffman tables: Annex K.3, or with OPTIMIZE jchuff.c's jpeg_gen_optimal_table on the image's counts (Cb and Cr
    share table 1);
  - entropy coding (jchuff.c): DC differences with the predictor reset to 0 at each restart, AC runs with ZRL and
    EOB, bits MSB first, FF 00 stuffing, each interval padded with 1-bits, RSTn markers modulo 8 between intervals;
  - markers: SOI, APP0 JFIF 1.01 (units 0, density 1x1), one DQT per table, SOF0, DHT DC0 AC0 (DC1 AC1), DRI when the
    interval is nonzero, SOS, the entropy-coded data, EOI.

`encode(img, params)` returns the file as a 1-D np.uint8 array; `coefficients` and `scan_blocks` expose the stages.
Nothing in the package imports this module.
"""
import numpy as np

QUALITY, PROGRESSIVE, OPTIMIZE, RST_INTERVAL, LUMA_QUALITY, CHROMA_QUALITY, SAMPLING_FACTOR = 1, 2, 3, 4, 5, 6, 7
# IMWRITE_JPEG_SAMPLING_FACTOR_*: 0xHV1111 with the luma factors H, V
SAMPLING = {0x411111: (4, 1), 0x221111: (2, 2), 0x211111: (2, 1), 0x121111: (1, 2), 0x111111: (1, 1)}

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# Annex K.1, natural order
STD_LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113,
                       92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
STD_CHROMA_Q = np.full(64, 99)
STD_CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# Annex K.3: (bits[1..16], values) of DC0, AC0, DC1, AC1
_AC_LUMA_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5"
    "a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHROMA_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4"
    "a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STD_HUFF = [
    ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], list(_AC_LUMA_VALS)),
    ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119], list(_AC_CHROMA_VALS)),
]


def parse_params(params):
    """cv2's reading of a flat [key, value, ...] list: (quality, (h, v) luma factors, optimize, restart_interval).
    Keys this encoder does not implement raise ValueError."""
    params = list(params or [])
    if len(params) % 2:
        raise ValueError("params must be [key, value, ...] pairs")
    quality, hv, optimize, rst = 95, (2, 2), False, 0
    for k, v in zip(params[0::2], params[1::2]):
        k, v = int(k), int(v)
        if k == QUALITY:
            quality = min(max(v, 0), 100)
        elif k == SAMPLING_FACTOR:
            hv = SAMPLING.get(v, (2, 2))
        elif k == OPTIMIZE:
            optimize = v > 0
        elif k == RST_INTERVAL:
            rst = min(max(v, 0), 65535)
        else:
            raise ValueError("unsupported JPEG parameter %d" % k)
    return quality, hv, optimize, rst


def quant_tables(quality):
    """jpeg_set_quality(quality, force_baseline=TRUE): the luma and chroma tables, natural order"""
    q = min(max(quality, 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((t * scale + 50) // 100, 1, 255) for t in (STD_LUMA_Q, STD_CHROMA_Q)]


def reciprocal(divisor):
    """compute_reciprocal: (reciprocal, correction, shift) with q = ((|x| + correction) * reciprocal) >> shift"""
    d = np.asarray(divisor, np.int64)
    b = np.floor(np.log2(d)).astype(np.int64)
    r = 16 + b
    fq = (np.int64(1) << r) // d
    fr = (np.int64(1) << r) % d
    c = d // 2
    pow2 = fr == 0
    fq = np.where(pow2, fq >> 1, fq)
    r = np.where(pow2, r - 1, r)
    low = ~pow2 & (fr <= d // 2)
    c = np.where(low, c + 1, c)
    fq = np.where(~pow2 & ~low, fq + 1, fq)
    return fq, c, r


def ycc(img):
    """jccolor.c rgb_ycc_convert on a BGR image: three int64 planes"""
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))
    half = 1 << 15
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + half - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + half - 1) >> 16
    return [y, cb, cr]


class Geometry:
    """the frame and scan geometry of jcmaster.c for an image of h x w with nc components and luma factors hv"""

    def __init__(self, h, w, nc, hv):
        self.h, self.w, self.nc = h, w, nc
        self.samp = [hv] + [(1, 1)] * (nc - 1) if nc == 3 else [(1, 1)]
        self.maxh = max(s[0] for s in self.samp)
        self.maxv = max(s[1] for s in self.samp)
        cdiv = lambda a, b: -(-a // b)
        self.wib = [cdiv(w * s[0], self.maxh * 8) for s in self.samp]
        self.hib = [cdiv(h * s[1], self.maxv * 8) for s in self.samp]
        if nc == 1:     # one component: a non-interleaved scan, one block per MCU
            self.mcux, self.mcuy = self.wib[0], self.hib[0]
        else:
            self.mcux, self.mcuy = cdiv(w, self.maxh * 8), cdiv(h, self.maxv * 8)


def component_planes(img, g):
    """each component's downsampled plane, hib * 8 rows by wib * 8 columns, edges as jcprepct / jcsample make them"""
    planes = ycc(img) if g.nc == 3 else [img.astype(np.int64)]
    out = []
    ngroups = -(-g.h // g.maxv)
    for c, (hs, vs) in enumerate(g.samp):
        he, ve = g.maxh // hs, g.maxv // vs
        rows = np.minimum(np.arange(ngroups * g.maxv), g.h - 1)
        cols = np.minimum(np.arange(g.wib[c] * 8 * he), g.w - 1)
        p = planes[c][rows][:, cols]
        R, C = p.shape[0] // ve, p.shape[1] // he
        s = p.reshape(R, ve, C, he).sum(axis=(1, 3))
        x = np.arange(C)
        if he == 1 and ve == 1:
            d = s
        elif he == 2 and ve == 1:
            d = (s + (x & 1)) >> 1
        elif he == 2 and ve == 2:
            d = (s + 1 + (x & 1)) >> 2
        else:
            n = he * ve
            d = (s + n // 2) // n
        d = d[np.minimum(np.arange(g.hib[c] * 8), R - 1)]
        out.append(d)
    return out


def fdct_islow(blk):
    """jpeg_fdct_islow on [n, 8, 8] int64 samples already shifted by -128"""
    d = blk.astype(np.int64).copy()

    def one_pass(v, first):
        # v: [..., 8] along the transformed axis
        s = [v[..., k] for k in range(8)]
        t0, t7 = s[0] + s[7], s[0] - s[7]
        t1, t6 = s[1] + s[6], s[1] - s[6]
        t2, t5 = s[2] + s[5], s[2] - s[5]
        t3, t4 = s[3] + s[4], s[3] - s[4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        sh = 13 - 2 if first else 13 + 2
        ds = lambda x, n: (x + (1 << (n - 1))) >> n
        o = [None] * 8
        if first:
            o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
        else:
            o[0], o[4] = ds(t10 + t11, 2), ds(t10 - t11, 2)
        z1 = (t12 + t13) * 4433
        o[2] = ds(z1 + t13 * 6270, sh)
        o[6] = ds(z1 - t12 * 15137, sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * 9633
        t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069, z4 * -3196
        z3 += z5
        z4 += z5
        o[7] = ds(t4 + z1 + z3, sh)
        o[5] = ds(t5 + z2 + z4, sh)
        o[3] = ds(t6 + z2 + z3, sh)
        o[1] = ds(t7 + z1 + z4, sh)
        return np.stack(o, axis=-1)

    d = one_pass(d, True)                                        # rows
    d = one_pass(d.transpose(0, 2, 1), False).transpose(0, 2, 1)  # columns
    return d


def scan_blocks(g):
    """every block of the scan in coding order: (component, bx, by, dummy, ref_bx, ref_by, mcu index)"""
    if g.nc == 1:
        by, bx = np.mgrid[0:g.hib[0], 0:g.wib[0]]
        bx, by = bx.ravel(), by.ravel()
        z = np.zeros_like(bx)
        return np.stack([z, bx, by, z, bx, by, np.arange(bx.size)], axis=1)
    rows = []
    for c, (hs, vs) in enumerate(g.samp):
        my, mx, dy, dx = np.meshgrid(np.arange(g.mcuy), np.arange(g.mcux), np.arange(vs), np.arange(hs), indexing="ij")
        bx, by = mx * hs + dx, my * vs + dy
        real_x, real_y = bx < g.wib[c], by < g.hib[c]
        # right-edge dummies take the row's last real block; a bottom dummy row takes the MCU's last block of the row
        # above, itself the row's last real block when the MCU runs past the right edge
        rx = np.where(real_y, np.minimum(bx, g.wib[c] - 1), np.minimum(mx * hs + hs - 1, g.wib[c] - 1))
        ry = np.minimum(by, g.hib[c] - 1)
        rows.append(np.stack([np.full(bx.shape, c), bx, by, ~(real_x & real_y), rx, ry, my * g.mcux + mx,
                              dy * hs + dx], axis=-1).reshape(g.mcuy * g.mcux, vs * hs, 8))
    allb = np.concatenate(rows, axis=1)          # [mcu, blocks per MCU, 8], components in order inside an MCU
    return allb.reshape(-1, 8)[:, :7]


def coefficients(img, quality=95, hv=(2, 2)):
    """(geometry, blocks in scan order, quantised coefficients [n, 64] in zig-zag order, luma / chroma tables)"""
    nc = 1 if img.ndim == 2 else 3
    g = Geometry(img.shape[0], img.shape[1], nc, hv)
    planes = component_planes(img, g)
    blocks = scan_blocks(g)
    qt = quant_tables(quality)
    out = np.zeros((len(blocks), 64), np.int64)
    for c in range(nc):
        sel = blocks[:, 0] == c
        rx, ry = blocks[sel, 4], blocks[sel, 5]
        p = planes[c]
        Hb, Wb = g.hib[c], g.wib[c]
        tiles = p.reshape(Hb, 8, Wb, 8).transpose(0, 2, 1, 3)[ry, rx] - 128
        d = fdct_islow(tiles).reshape(-1, 64)
        fq, corr, sh = reciprocal(qt[min(c, 1)] * 8)
        a = np.abs(d)
        q = ((a + corr) * fq) >> sh
        q = np.where(d < 0, -q, q)
        q = q[:, ZIGZAG]
        q[blocks[sel, 3].astype(bool), 1:] = 0
        out[sel] = q
    return g, blocks, out, qt


def nbits(v):
    a = np.abs(np.asarray(v, np.int64))
    n = np.zeros(a.shape, np.int64)
    while (a > 0).any():
        n += a > 0
        a >>= 1
    return n


def gen_optimal_table(freq):
    """jchuff.c jpeg_gen_optimal_table: (bits[1..16], values) for counts of symbols 0..255"""
    freq = [int(f) for f in freq] + [1]
    codesize = [0] * 257
    others = [-1] * 257
    while True:
        c1 = c2 = -1
        v = v2 = 1000000000
        for i in range(257):
            f = freq[i]
            if f and f <= v2:
                if f <= v:
                    c2, v2, c1, v = c1, v, i, f
                else:
                    c2, v2 = i, f
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    vals = [j for L in range(1, 33) for j in range(256) if codesize[j] == L]
    return bits[1:17], vals


def derive(bits, vals):
    """jpeg_make_c_derived_tbl: per symbol (code, size) arrays"""
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            code[vals[k]], size[vals[k]] = c, L
            c += 1
            k += 1
        c <<= 1
    return code, size


def _symbols(blocks, coef, g, rst, tbl_of):
    """every entropy-coded event in stream order: (block, table, symbol, extra value, extra bits); table 0..3 =
    DC0 AC0 DC1 AC1, symbol -1 for pure extra bits"""
    n = len(blocks)
    comp = blocks[:, 0]
    mcu = blocks[:, 6]
    # DC predictor: previous block of the component in the interval
    dc = coef[:, 0]
    diff = np.empty(n, np.int64)
    for c in range(g.nc):
        idx = np.nonzero(comp == c)[0]
        v = dc[idx]
        prev = np.r_[0, v[:-1]]
        m = mcu[idx]
        first = np.r_[True, m[1:] != m[:-1]] & ((m % rst == 0) if rst else (m == 0))
        prev[first] = 0
        diff[idx] = v - prev
    t = tbl_of[comp]
    ev_b, ev_k, ev_s, ev_t, ev_sym, ev_val, ev_nb = [], [], [], [], [], [], []

    def add(b, k, s, tab, sym, val, nb):
        ev_b.append(b); ev_k.append(k); ev_s.append(s); ev_t.append(tab); ev_sym.append(sym)
        ev_val.append(val); ev_nb.append(nb)

    nb_dc = nbits(diff)
    ar = np.arange(n)
    add(ar, np.zeros(n, np.int64), np.zeros(n, np.int64), 2 * t, nb_dc, np.where(diff < 0, diff - 1, diff), nb_dc)
    ac = coef[:, 1:]
    bi, ki = np.nonzero(ac)
    ki = ki + 1
    prevk = np.r_[0, ki[:-1]]
    newb = np.r_[True, bi[1:] != bi[:-1]]
    prevk[newb] = 0
    run = ki - prevk - 1
    nz = run // 16
    if nz.sum():
        zb = np.repeat(bi, nz)
        zk = np.repeat(ki, nz)
        zs = np.arange(nz.sum()) - np.repeat(np.cumsum(nz) - nz, nz)
        add(zb, zk, zs, 2 * t[zb] + 1, np.full(zb.size, 0xF0), np.zeros(zb.size, np.int64), np.zeros(zb.size, np.int64))
    v = ac[bi, ki - 1]
    nbv = nbits(v)
    add(bi, ki, np.full(bi.size, 100), 2 * t[bi] + 1, ((run % 16) << 4) + nbv, np.where(v < 0, v - 1, v), nbv)
    last = np.zeros(n, np.int64)
    if bi.size:
        np.maximum.at(last, bi, ki)
    eob = np.nonzero(last < 63)[0]
    add(eob, np.full(eob.size, 64), np.zeros(eob.size, np.int64), 2 * t[eob] + 1, np.zeros(eob.size, np.int64),
        np.zeros(eob.size, np.int64), np.zeros(eob.size, np.int64))
    cat = lambda L: np.concatenate([np.asarray(x, np.int64) for x in L])
    b, k, s = cat(ev_b), cat(ev_k), cat(ev_s)
    order = np.lexsort((s, k, b))
    return b[order], cat(ev_t)[order], cat(ev_sym)[order], cat(ev_val)[order], cat(ev_nb)[order]


def _marker(m, payload):
    return bytes([0xFF, m]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def encode(img, params=None):
    """the file cv2.imencode('.jpg', img, params) writes, as a 1-D np.uint8 array"""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] != 3) or 0 in img.shape:
        raise ValueError("need a non-empty u8 [h][w] or [h][w][3] image, got %s %s" % (img.dtype, img.shape))
    quality, hv, optimize, rst = parse_params(params)
    g, blocks, coef, qt = coefficients(img, quality, hv)
    tbl_of = np.array([0, 1, 1])
    b, tab, sym, val, nb = _symbols(blocks, coef, g, rst, tbl_of)
    ntab = 2 if g.nc == 1 else 4
    if optimize:
        huff = []
        for k in range(ntab):
            sel = tab == k
            huff.append(gen_optimal_table(np.bincount(sym[sel], minlength=256)))
    else:
        huff = STD_HUFF[:ntab]
    der = [derive(*h) for h in huff]
    codes = np.zeros(len(b), np.int64)
    sizes = np.zeros(len(b), np.int64)
    for k in range(ntab):
        sel = tab == k
        codes[sel] = der[k][0][sym[sel]]
        sizes[sel] = der[k][1][sym[sel]]
    # event list: code then extra bits
    v2 = np.stack([codes, val & ((np.int64(1) << nb) - 1)], 1).ravel()
    n2 = np.stack([sizes, nb], 1).ravel()
    b2 = np.repeat(b, 2)
    # intervals: MCUs [j * rst, (j + 1) * rst), each padded to a byte with 1-bits
    interval = blocks[:, 6] // rst if rst else np.zeros(len(blocks), np.int64)
    nint = int(interval[-1]) + 1
    blk_bits = np.bincount(b2, weights=n2, minlength=len(blocks)).astype(np.int64)
    int_bits = np.bincount(interval, weights=blk_bits, minlength=nint).astype(np.int64)
    int_bytes = (int_bits + 7) // 8
    int_start = np.r_[0, np.cumsum(int_bytes)[:-1]]
    int_first_bit = np.r_[0, np.cumsum(int_bits)[:-1]]
    ev_pos = np.cumsum(n2) - n2
    iv = interval[b2]
    ev_pos = int_start[iv] * 8 + ev_pos - int_first_bit[iv]
    total = int(int_bytes.sum())
    bits = np.ones(total * 8, np.uint8)
    keep = n2 > 0
    v2, n2, ev_pos = v2[keep], n2[keep], ev_pos[keep]
    rep_n = np.repeat(n2, n2)
    j = np.arange(rep_n.size) - np.repeat(np.cumsum(n2) - n2, n2)
    bits[np.repeat(ev_pos, n2) + j] = (np.repeat(v2, n2) >> (rep_n - 1 - j)) & 1
    data = np.packbits(bits)
    # stuffing and restart markers
    pieces = []
    for q in range(nint):
        seg = data[int_start[q]:int_start[q] + int_bytes[q]]
        ff = np.nonzero(seg == 0xFF)[0]
        pieces.append(np.insert(seg, ff + 1, 0))
        if q + 1 < nint:
            pieces.append(np.array([0xFF, 0xD0 + (q & 7)], np.uint8))
    # headers
    hdr = bytearray(b"\xff\xd8")
    hdr += _marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for k in range(1 if g.nc == 1 else 2):
        hdr += _marker(0xDB, [k] + [int(x) for x in qt[k][ZIGZAG]])
    sof = [8, g.h >> 8, g.h & 255, g.w >> 8, g.w & 255, g.nc]
    for c in range(g.nc):
        sof += [c + 1, (g.samp[c][0] << 4) | g.samp[c][1], min(c, 1)]
    hdr += _marker(0xC0, sof)
    for k in range(ntab):
        bits_k, vals_k = huff[k]
        hdr += _marker(0xC4, [(k & 1) << 4 | (k >> 1)] + list(bits_k) + list(vals_k))
    if rst:
        hdr += _marker(0xDD, [rst >> 8, rst & 255])
    sos = [g.nc]
    for c in range(g.nc):
        sos += [c + 1, 0 if c == 0 else 0x11]
    hdr += _marker(0xDA, sos + [0, 63, 0])
    return np.concatenate([np.frombuffer(bytes(hdr), np.uint8)] + pieces + [np.array([0xFF, 0xD9], np.uint8)])
