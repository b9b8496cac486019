"""JPEG test files, generated from seeds with cv2.imencode and PIL (no file of them is committed except the golden
page): qualities, optimised tables, restart intervals, samplings, grayscale, odd sizes, strips and the eight EXIF
orientations; plus files the GPU path must decline."""
import io
import os

import cv2
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "AisazuNihaIrarenai-003.jpg")

S444, S422, S420 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422, \
    cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420
SAMPLINGS = {"444": S444, "422": S422, "420": S420}


def image(h, w, seed):
    """a BGR page with smooth gradients, edges and noise: every coefficient band gets used"""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.sin(xx / 5.0 + seed) * 80 + np.cos(yy / 7.0) * 60 + 128 + g.normal(0, 25, (h, w))
    b = np.stack([a, 255 - a, (xx * 3 + yy * 5 + seed) % 256], -1)
    return np.clip(b, 0, 255).astype(np.uint8)


def encode(img, quality=90, sampling=S420, optimize=False, rst=0):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    ok, e = cv2.imencode(".jpg", img, params)
    assert ok
    return e.tobytes()


def pil_encode(img_bgr, mode="RGB", **kw):
    from PIL import Image
    im = Image.fromarray(np.ascontiguousarray(img_bgr[:, :, ::-1]))
    if mode != "RGB":
        im = im.convert(mode)
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def exif_jpeg(orientation, h=13, w=21, seed=3):
    """written by PIL with an Exif IFD0 orientation tag"""
    from PIL import Image
    ex = Image.Exif()
    ex[0x0112] = orientation
    return pil_encode(image(h, w, seed + orientation), quality=90, exif=ex.tobytes())


def corpus(small=False):
    """[(name, bytes)] of files the GPU path takes.  small: the subset the pure-Python oracle decodes quickly."""
    out = []
    sizes = [(1, 1), (3, 17), (15, 16), (33, 65), (2, 3), (5, 2)]
    for h, w in sizes:
        for q in (10, 50, 90, 100):
            for sn, s in SAMPLINGS.items():
                out.append(("%dx%d_q%d_%s" % (h, w, q, sn), encode(image(h, w, h * w + q), q, s)))
    for sn, s in SAMPLINGS.items():
        img = image(33, 65, 7)
        out.append(("opt_%s" % sn, encode(img, 75, s, optimize=True)))
        for rst in (1, 7):
            out.append(("rst%d_%s" % (rst, sn), encode(img, 75, s, rst=rst)))
    for h, w in ((33, 65), (3, 17), (1, 1)):
        out.append(("gray_%dx%d" % (h, w), encode(image(h, w, 11)[:, :, 0], 90)))
    out.append(("gray_rst3", encode(image(33, 65, 12)[:, :, 0], 90, rst=3)))
    for o in range(1, 9):
        out.append(("exif%d" % o, exif_jpeg(o)))
    for sub in (0, 1, 2):
        out.append(("pil_sub%d" % sub, pil_encode(image(20, 30, 5), quality=80, subsampling=sub)))
    if not small:
        for h, w in ((1, 8193), (8193, 1)):
            for sn in ("420", "444"):
                out.append(("strip%dx%d_%s" % (h, w, sn), encode(image(h, w, 2), 90, SAMPLINGS[sn])))
        out.append(("gray_pil_exif6", pil_encode(image(40, 24, 9), mode="L", quality=85,
                                                 exif=_exif_bytes(6))))
    return out


def _exif_bytes(o):
    from PIL import Image
    ex = Image.Exif()
    ex[0x0112] = o
    return ex.tobytes()


def truncated(data, keep=0.5):
    return data[:int(len(data) * keep)]


def corrupt_scan(data, seed=0):
    """flips bytes inside the entropy-coded data (never creating a 0xFF), markers left intact"""
    b = bytearray(data)
    sos = b.find(b"\xff\xda")
    g = np.random.default_rng(seed)
    start = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    for i in g.integers(start, len(b) - 2, 12):
        if b[i] != 0xFF and b[i - 1] != 0xFF and b[i] ^ 0x5A != 0xFF:
            b[i] ^= 0x5A
    return bytes(b)


def broken_exif(data):
    """the Exif block's IFD0 offset pointed past the block's end"""
    b = bytearray(data)
    i = b.find(b"Exif\0\0")
    assert i > 0
    t = i + 6
    le = b[t:t + 2] == b"II"
    b[t + 4:t + 8] = (0x7FFFFF00).to_bytes(4, "little" if le else "big")
    return bytes(b)


def png(img):
    ok, e = cv2.imencode(".png", img)
    assert ok
    return e.tobytes()


def exif_orientations(data, orientations):
    """data with an APP1 Exif block right after SOI whose IFD0 holds one orientation entry per value (little endian)"""
    n = len(orientations)
    tiff = b"II*\0" + (8).to_bytes(4, "little") + n.to_bytes(2, "little")
    for o in orientations:
        tiff += (0x0112).to_bytes(2, "little") + (3).to_bytes(2, "little") + (1).to_bytes(4, "little") + \
            int(o).to_bytes(2, "little") + b"\0\0"
    tiff += b"\0\0\0\0"
    payload = b"Exif\0\0" + tiff
    seg = b"\xff\xe1" + (len(payload) + 2).to_bytes(2, "big") + payload
    return data[:2] + seg + data[2:]


def zero_padded(data):
    """data with the padding bits after each restart interval's last MCU set to 0 instead of 1 (what some encoders
    write): every MCU decodes as before, but the zero bits left in an interval can start a block of their own"""
    from oracle import jpeg_ref
    info = jpeg_ref.parse(data)
    jpeg_ref.coefficients(info)
    segs = []
    for seg, end in zip(info["segs"], info["ends"]):
        seg = list(seg)
        if end % 8:
            seg[-1] &= 0xFF << (8 - end % 8) & 0xFF
        segs.append(bytes(seg).replace(b"\xff", b"\xff\x00"))
    scan = b"".join(s + (bytes([0xFF, 0xD0 + (i & 7)]) if i + 1 < len(segs) else b"") for i, s in enumerate(segs))
    return bytes(data[:info["scan_begin"]]) + scan + b"\xff\xd9"


def raised_dc_quantiser(q):
    """a white 8x8 page at quality 100 with its luma DC quantiser set to q: from q = 5 on, the IDCT output leaves the
    range on which libjpeg-turbo's C and SIMD IDCTs agree"""
    data = bytearray(encode(np.full((8, 8, 3), 255, np.uint8), 100, S444))
    i = data.find(b"\xff\xdb")
    data[i + 5] = q
    return bytes(data)
