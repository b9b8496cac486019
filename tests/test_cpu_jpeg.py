"""not-gpu: the JPEG decode's integer rules and its file selection.

The numpy restatement (oracle/jpeg_ref.py) equals cv2.imdecode byte for byte on the generated corpus; the host probe
(ctd_jpeg_probe) reports shapes, orientation and sampling as the oracle and cv2 see them, and the right reason code
for each kind of file the GPU path declines."""
import cv2
import numpy as np
import pytest

import ctd_b200
from oracle import jpeg_ref
import jpeg_corpus as jc

SMALL = jc.corpus(small=True)
FULL = jc.corpus()


def _cv2(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


@pytest.mark.parametrize("name,data", SMALL, ids=[n for n, _ in SMALL])
def test_oracle_equals_cv2(name, data):
    page, exact = jpeg_ref.decode(data)
    ref = _cv2(data)
    assert exact
    assert page.shape == ref.shape and np.array_equal(page, ref)


def test_oracle_equals_cv2_strips():
    for name, data in FULL:
        if name.startswith("strip"):
            page, exact = jpeg_ref.decode(data)
            assert exact and np.array_equal(page, _cv2(data)), name


def test_oracle_range_guard_marks_where_cv2_saturates():
    # a white q100 block with its DC quantiser raised: the IDCT output leaves [-512, 511]; libjpeg-turbo's C table
    # would wrap it, cv2's SIMD IDCT saturates, and the oracle (as the GPU decoder) declines to claim the page
    data = bytearray(jc.encode(np.full((8, 8, 3), 255, np.uint8), 100, jc.S444))
    i = data.find(b"\xff\xdb")
    for q, exact in ((1, True), (2, True), (5, False), (9, False)):
        data[i + 5] = q
        page, ok = jpeg_ref.decode(bytes(data))
        assert ok == exact, q
        if ok:
            assert np.array_equal(page, _cv2(bytes(data)))


@pytest.mark.parametrize("name,data", FULL, ids=[n for n, _ in FULL])
def test_probe_shape_orientation_sampling(name, data):
    info = ctd_b200.jpeg_probe(data)
    ref = _cv2(data)
    assert info["status"] == 0, info
    assert (info["height"], info["width"]) == ref.shape[:2]
    st, shape, orient = jpeg_ref.probe(data)
    assert st == 0 and shape == ref.shape[:2] and info["orientation"] == orient
    rotated = orient >= 5
    assert (info["frame_height"], info["frame_width"]) == (ref.shape[1], ref.shape[0]) if rotated else ref.shape[:2]
    if name.startswith("gray"):
        assert info["components"] == 1 and (info["h_samp"], info["v_samp"]) == (1, 1)
    else:
        assert info["components"] == 3
    for sn, hv in (("444", (1, 1)), ("422", (2, 1)), ("420", (2, 2))):
        if name.endswith("_" + sn):
            assert (info["h_samp"], info["v_samp"]) == hv
    if name.startswith("rst"):
        assert info["restart_interval"] == int(name[3])
    assert 0 < info["ecs_bytes"] < len(data)


def test_probe_exif_orientations():
    for o in range(1, 9):
        info = ctd_b200.jpeg_probe(jc.exif_jpeg(o, 13, 21))
        assert info["status"] == 0 and info["orientation"] == o
        assert (info["height"], info["width"]) == ((21, 13) if o >= 5 else (13, 21))


def _declined():
    img = jc.image(40, 48, 1)
    base = jc.encode(img, 80, jc.S420)
    return [
        ("progressive", jc.pil_encode(img, quality=80, progressive=True), "progressive"),
        ("411", jc.encode(img, 80, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411), "sampling"),
        ("440", jc.encode(img, 80, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440), "sampling"),
        ("cmyk", jc.pil_encode(img, mode="CMYK", quality=80), "color"),
        ("truncated", jc.truncated(base), "truncated"),
        ("no_eoi", base[:-2], "truncated"),
        ("png", jc.png(img), "not_jpeg"),
        ("text", b"not a jpeg at all", "not_jpeg"),
        ("empty", b"", "not_jpeg"),
        ("broken_exif", jc.broken_exif(jc.exif_jpeg(6)), "exif"),
        # OpenCV takes the first of two orientation entries, other readers the last: left to cv2
        ("two_orientations_3_6", jc.exif_orientations(base, [3, 6]), "exif"),
        ("two_orientations_6_3", jc.exif_orientations(base, [6, 3]), "exif"),
    ]


@pytest.mark.parametrize("name,data,reason", _declined(), ids=[d[0] for d in _declined()])
def test_probe_reason_codes(name, data, reason):
    info = ctd_b200.jpeg_probe(data)
    assert info["reason"] == reason, info
    assert jpeg_ref.probe(data)[0] == info["status"]


def test_probe_takes_numpy_and_memoryview():
    data = jc.encode(jc.image(9, 9, 0))
    a = ctd_b200.jpeg_probe(np.frombuffer(data, np.uint8))
    b = ctd_b200.jpeg_probe(memoryview(data))
    c = ctd_b200.jpeg_probe(bytearray(data))
    assert a == b == c and a["status"] == 0
    with pytest.raises(ValueError):
        ctd_b200.jpeg_probe(np.zeros((3, 3), np.uint8))


def test_golden_page_probe():
    data = open(jc.GOLDEN, "rb").read()
    info = ctd_b200.jpeg_probe(data)
    assert info["status"] == 0
    assert (info["height"], info["width"]) == (1170, 1654)
    assert (info["components"], info["h_samp"], info["v_samp"]) == (3, 2, 2)


def test_exif_builder_single_orientation_is_taken():
    data = jc.exif_orientations(jc.encode(jc.image(13, 21, 1)), [6])
    info = ctd_b200.jpeg_probe(data)
    assert info["status"] == 0 and info["orientation"] == 6 and (info["height"], info["width"]) == (21, 13)
    assert _cv2(data).shape == (21, 13, 3)


@pytest.mark.parametrize("rst", [1, 3])
def test_zero_padded_intervals_are_taken_by_the_probe(rst):
    # zero padding bits before each RSTn: the probe takes the file (its structure is fine); the MCUs decode as cv2
    # decodes them, and the GPU decode must notice the partial block the zeros start (tests/test_gpu_jpeg.py)
    orig = jc.encode(jc.image(64, 80, 1), 90, jc.S420, rst=rst)
    data = jc.zero_padded(orig)
    assert data != orig and len(data) == len(orig)
    assert ctd_b200.jpeg_probe(data)["status"] == 0
    page, exact = jpeg_ref.decode(data)
    assert exact and np.array_equal(page, _cv2(data)) and np.array_equal(page, _cv2(orig))


def test_size_status_is_last():
    # the Python names follow ctd_jpeg_status
    assert ctd_b200.jpeg.JPEG_STATUS[jpeg_ref.RANGE_CODE] == "range"
    assert ctd_b200.jpeg.JPEG_STATUS[jpeg_ref.SIZE] == "size"
