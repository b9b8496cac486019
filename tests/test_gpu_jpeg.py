"""-m gpu: JPEG pages decoded on the GPU (`ctd_b200.JpegDecoder`, csrc/jpeg.cu) equal cv2.imdecode byte for byte, on
every file of the generated corpus, the golden scan and large synthetic pages, at subsequence lengths that force many
self-synchronisation rounds, the default and one longer than any stream; files the GPU declines come back as cv2's
own result.  `detect_stream` / `detect_batch` on encoded pages equal the stream on the cv2.imdecode pages."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from oracle import synth
from util import get_checkpoint
import jpeg_corpus as jc

pytestmark = pytest.mark.gpu

SUB_BITS = [5, 0, 1 << 30]   # tiny and not byte-aligned, the default, longer than any stream
SIZES_73 = [(1654, 1170), (1170, 1654), (2048, 1446), (1200, 800), (1024, 1024)]


def _cv2(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def _same(got, ref):
    if ref is None:
        return got is None
    if isinstance(got, torch.Tensor):
        got = got.cpu().numpy()
    return isinstance(got, np.ndarray) and got.shape == ref.shape and np.array_equal(got, ref)


@pytest.fixture(scope="module", params=SUB_BITS, ids=["sub5", "default", "serial"])
def dec(request):
    d = ctd_b200.JpegDecoder(0, subsequence_bits=request.param)
    yield d
    d.close()


def test_corpus(dec):
    files = jc.corpus()
    out = dec.decode([d for _, d in files])
    for (name, data), got, st in zip(files, out, dec.last_status):
        assert st == 0 and isinstance(got, torch.Tensor) and got.is_cuda, (name, st)
        assert _same(got, _cv2(data)), name


def test_golden_page(dec):
    data = open(jc.GOLDEN, "rb").read()
    got = dec.decode([data])[0]
    assert dec.last_status == [0]
    assert _same(got, _cv2(data))


def _pages_73():
    out = []
    for i, (h, w) in enumerate(SIZES_73):
        page = synth.structured_page(20_000 + i, h, w)
        for q in (75, 95):
            for s in (jc.S420, jc.S444):
                out.append(("%dx%d_q%d_%d" % (h, w, q, s), jc.encode(page, q, s)))
    return out


def test_large_pages(dec):
    files = _pages_73()
    out = dec.decode([d for _, d in files])
    assert dec.last_status == [0] * len(files)
    for (name, data), got in zip(files, out):
        assert _same(got, _cv2(data)), name


def test_subsequence_lengths_agree():
    files = [d for _, d in _pages_73()[:4]] + [open(jc.GOLDEN, "rb").read()] + [d for _, d in jc.corpus(True)[:40]]
    results = []
    for sb in SUB_BITS + [8, 77]:
        d = ctd_b200.JpegDecoder(0, subsequence_bits=sb)
        try:
            results.append([t.cpu().numpy() for t in d.decode(files)])
        finally:
            d.close()
    for r in results[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(results[0], r))


def test_mixed_list_is_cv2(dec):
    img = jc.image(40, 48, 1)
    good = jc.encode(img, 80, jc.S420)
    golden = open(jc.GOLDEN, "rb").read()
    files = [good, jc.pil_encode(img, quality=80, progressive=True), jc.png(img), jc.corrupt_scan(golden),
             jc.truncated(golden), jc.encode(img, 90, jc.S444, rst=2), b"junk", np.frombuffer(good, np.uint8)]
    out = dec.decode(files)
    for i, (data, got) in enumerate(zip(files, out)):
        assert _same(got, _cv2(bytes(data))), i
    assert isinstance(out[0], torch.Tensor) and isinstance(out[5], torch.Tensor)
    assert isinstance(out[1], np.ndarray) and isinstance(out[2], np.ndarray)
    assert out[4] is None or isinstance(out[4], np.ndarray)
    assert dec.last_status[1:3] == [3, 1] and dec.last_status[6] == 1


def test_declined_after_decode_is_cv2(dec):
    # pages the probe takes but the GPU decode declines, between pages it keeps: zero-padded restart intervals (the
    # zeros start a block that never ends: CTD_JPEG_ENTROPY) and blocks whose IDCT leaves the range on which cv2's SIMD
    # IDCT and libjpeg's C table agree (CTD_JPEG_RANGE); and a file with two EXIF orientation entries (probe: EXIF)
    img = jc.image(64, 80, 1)
    good = jc.encode(img, 90, jc.S420, rst=2)
    files = [jc.zero_padded(jc.encode(img, 90, jc.S420, rst=1)), good, jc.zero_padded(jc.encode(img, 90, jc.S420, rst=3)),
             jc.raised_dc_quantiser(5), good, jc.raised_dc_quantiser(9), jc.raised_dc_quantiser(2),
             jc.exif_orientations(jc.encode(jc.image(13, 21, 1)), [3, 6]),
             jc.exif_orientations(jc.encode(jc.image(13, 21, 1)), [6, 3])]
    out = dec.decode(files)
    assert dec.last_status == [12, 0, 12, 13, 0, 13, 0, 10, 10]
    for i, (data, got) in enumerate(zip(files, out)):
        assert _same(got, _cv2(data)), i
    assert _cv2(files[7]).shape == (13, 21, 3) and _cv2(files[8]).shape == (21, 13, 3)


def test_corrupt_scans_fall_back():
    golden = open(jc.GOLDEN, "rb").read()
    files = [jc.corrupt_scan(golden, s) for s in range(6)] + \
        [jc.corrupt_scan(jc.encode(jc.image(64, 80, s), 90, jc.S420, rst=3), s) for s in range(6)]
    d = ctd_b200.JpegDecoder(0)
    try:
        out = d.decode(files)
    finally:
        d.close()
    for i, (data, got) in enumerate(zip(files, out)):
        assert _same(got, _cv2(data)), (i, d.last_status[i])


# ---- the detector on encoded pages -------------------------------------------------------------------------------
NET = 256
DET_SIZES = [(NET, NET), (361, 251), (414, 292), (512, 512), (200, 150), (96, 700)]


@pytest.fixture(scope="module")
def det():
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=4)
    yield d
    d.close()


@pytest.fixture(scope="module")
def files():
    out = []
    for i, (h, w) in enumerate(DET_SIZES):
        page = synth.structured_page(700 + i, h, w)
        out.append(jc.encode(page, 90, jc.S420 if i % 2 == 0 else jc.S444))
    return out


def _same_item(got, ref):
    assert len(got) == len(ref)
    for k in (0, 1):
        g = got[k].cpu().numpy() if isinstance(got[k], torch.Tensor) else got[k]
        assert np.array_equal(g, ref[k]), k
    assert [vars(b).keys() for b in got[2]] == [vars(b).keys() for b in ref[2]]
    for g, r in zip(got[2], ref[2]):
        for k, v in vars(r).items():
            gv = vars(g)[k]
            assert (np.array_equal(gv, v) if isinstance(v, np.ndarray) else gv == v), k
    if len(ref) == 4:
        for gb, rb in zip(got[3], ref[3]):
            assert len(gb) == len(rb)
            for g, r in zip(gb, rb):
                assert (g is None) == (r is None)
                if r is not None:
                    g = g.cpu().numpy() if isinstance(g, torch.Tensor) else g
                    assert np.array_equal(g, r)


@pytest.mark.parametrize("kw", [{}, {"textheight": 48}, {"device_results": True},
                                {"textheight": 48, "device_results": True}],
                         ids=["plain", "textheight", "device", "textheight_device"])
def test_stream_bytes(det, files, kw):
    ref = list(det.detect_stream([_cv2(f) for f in files], textheight=kw.get("textheight")))
    got = list(det.detect_stream(files, **kw))
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        _same_item(g, r)


def test_stream_paths_and_mix(det, files, tmp_path):
    paths = []
    for i, f in enumerate(files):
        p = tmp_path / ("page%d.jpg" % i)
        p.write_bytes(f)
        paths.append(p if i % 2 else str(p))
    pages = [_cv2(f) for f in files]
    ref = list(det.detect_stream(pages, textheight=48))
    mix = [paths[0], pages[1], torch.from_numpy(pages[2]).cuda(), np.frombuffer(files[3], np.uint8),
           bytearray(files[4]), memoryview(files[5])]
    for imgs in (paths, mix):
        got = list(det.detect_stream(imgs, textheight=48))
        for g, r in zip(got, ref):
            _same_item(g, r)
    got = det.detect_batch(mix)
    ref = det.detect_batch(pages)
    for g, r in zip(got, ref):
        _same_item(g, r)


def test_stream_fallback_pages_and_errors(det, files, tmp_path):
    img = _cv2(files[1])
    prog = jc.pil_encode(img, quality=90, progressive=True)
    pngf = jc.png(img)
    ref = list(det.detect_stream([_cv2(prog), img]))
    got = list(det.detect_stream([prog, pngf]))
    for g, r in zip(got, ref):
        _same_item(g, r)
    bad = tmp_path / "bad.jpg"
    bad.write_bytes(b"junk")
    with pytest.raises(ValueError, match=r"page 5 \(.*bad\.jpg\)"):
        list(det.detect_stream(files[:5] + [str(bad)]))
    with pytest.raises(ValueError, match="page 1"):
        det.detect_batch([files[0], jc.truncated(files[0], 0.1)])
