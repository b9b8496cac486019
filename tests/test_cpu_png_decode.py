"""The PNG decode oracle (oracle/png_decode_ref.py) equals cv2.imdecode(buf, IMREAD_COLOR) byte for byte on every file
of the generated corpus the GPU takes, and `png_probe` gives each file the status the chunk walk must give.  The
conversion facts the decoder restates are pinned one by one against cv2."""
import struct
import zlib

import cv2
import numpy as np
import pytest

import ctd_b200
import png_decode_corpus as pc
from oracle import png_decode_ref as ref


def _cv2(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    return pc.corpus(large=False)


def test_oracle_equals_cv2(files):
    for name, data, expect in files:
        status, page = ref.decode(data)
        if expect is not None:
            assert status == expect, name
        got = _cv2(data)
        if status == "ok":
            assert got is not None and got.shape == page.shape and np.array_equal(got, page), name


def test_probe_status(files):
    for name, data, expect in files:
        want = ref.probe(data)
        assert ctd_b200.png_probe(data)["reason"] == want, name
        if expect is not None and expect not in ("crc", "data"):
            assert want == expect, name


def test_large_pages():
    for ct in (0, 2):
        page = pc.structured(3, 2339, 1654)
        page = cv2.cvtColor(page, cv2.COLOR_BGR2GRAY) if ct == 0 else page
        data = cv2.imencode(".png", page)[1].tobytes()
        status, got = ref.decode(data)
        assert status == "ok" and np.array_equal(got, _cv2(data))
        info = ctd_b200.png_probe(data)
        assert info["reason"] == "ok" and (info["height"], info["width"]) == (2339, 1654)


def _one(w, h, depth, ctype, rows, pre=b""):
    return pc.assemble(w, h, depth, ctype, zlib.compress(b"".join(b"\0" + r for r in rows)), pre=pre)


def test_conversion_facts():
    # 16 bits: the high byte (0x12ff -> 0x12, not 0x13)
    v = np.array([0x12FF, 0x1280, 0x127F, 0xFE80], ">u2")
    im = _cv2(_one(4, 1, 16, 0, [v.tobytes()]))
    assert im[0, :, 0].tolist() == [0x12, 0x12, 0x12, 0xFE]
    # 1/2/4-bit grey scaled: 0/255, x85, x17
    assert _cv2(_one(3, 1, 1, 0, [bytes([0b10100000])]))[0, :, 0].tolist() == [255, 0, 255]
    assert _cv2(_one(4, 1, 2, 0, [bytes([0b00011011])]))[0, :, 0].tolist() == [0, 85, 170, 255]
    assert _cv2(_one(2, 1, 4, 0, [bytes([0x1F])]))[0, :, 0].tolist() == [17, 255]
    # grey replicated, RGB stored as BGR, alpha dropped without compositing
    assert _cv2(_one(1, 1, 8, 0, [bytes([77])]))[0, 0].tolist() == [77, 77, 77]
    assert _cv2(_one(1, 1, 8, 2, [bytes([1, 2, 3])]))[0, 0].tolist() == [3, 2, 1]
    assert _cv2(_one(1, 1, 8, 4, [bytes([100, 0])]))[0, 0].tolist() == [100, 100, 100]
    assert _cv2(_one(1, 1, 8, 6, [bytes([100, 150, 200, 0])]))[0, 0].tolist() == [200, 150, 100]
    # tRNS and gAMA change nothing
    assert _cv2(_one(2, 1, 8, 0, [bytes([64, 65])], pc.chunk(b"tRNS", b"\0\x40")))[0, :, 0].tolist() == [64, 65]
    assert _cv2(_one(2, 1, 8, 0, [bytes([64, 200])], pc.chunk(b"gAMA", struct.pack(">I", 100000))))[0, :, 0].tolist() \
        == [64, 200]
    # palette: an index past PLTE reads (0, 0, 0), tRNS ignored
    pal = pc.chunk(b"PLTE", bytes([10, 20, 30])) + pc.chunk(b"tRNS", b"\0")
    assert _cv2(_one(2, 1, 8, 3, [bytes([0, 1])], pal))[0].tolist() == [[30, 20, 10], [0, 0, 0]]
    # eXIf orientation 6, before or after IDAT: transposed then columns flipped
    for where in ("pre", "post"):
        d = pc.assemble(3, 2, 8, 0, zlib.compress(b"\0\0\1\2\0\x0a\x0b\x0c"),
                        **{where: pc.chunk(b"eXIf", pc.exif(6, False))})
        assert _cv2(d)[..., 0].tolist() == [[10, 0], [11, 1], [12, 2]]
        assert ref.decode(d)[1][..., 0].tolist() == [[10, 0], [11, 1], [12, 2]]
    # errors: None; too much data: the image
    good = b"\0\1\2\3\4"
    assert _cv2(pc.assemble(4, 2, 8, 0, zlib.compress(good))) is None
    assert _cv2(pc.assemble(4, 1, 8, 0, zlib.compress(good + b"\0\1\2\3\4"))) is not None
    assert _cv2(pc.assemble(4, 1, 8, 0, zlib.compress(b"\5" + good[1:]))) is None
