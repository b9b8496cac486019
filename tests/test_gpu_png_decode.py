"""-m gpu: PNG pages decoded on the GPU (`ctd_b200.PngDecoder`, csrc/png_dec.cu) equal cv2.imdecode byte for byte on
every file of the generated corpus, in one mixed call with the declined files between the kept ones, at several
subsequence_bits values, across calls whose buffers grow and shrink.  `detect_stream` / `detect_batch` on PNG files
equal the stream on the cv2.imdecode pages, and `model2annotations` on a directory of PNG pages writes the same files
as on the same pages read by cv2."""
import os

import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200.png import PNG_STATUS
from ctd_b200 import annotations
from util import get_checkpoint
import jpeg_corpus as jc
import png_decode_corpus as pc

pytestmark = pytest.mark.gpu


def _cv2(data):
    return cv2.imdecode(np.frombuffer(bytes(data), np.uint8), cv2.IMREAD_COLOR)


def _same(got, ref):
    if ref is None:
        return got is None
    if isinstance(got, torch.Tensor):
        got = got.cpu().numpy()
    return isinstance(got, np.ndarray) and got.shape == ref.shape and np.array_equal(got, ref)


@pytest.fixture(scope="module")
def files():
    return pc.corpus(large=True)


@pytest.mark.parametrize("sub_bits", [32, 0, 1 << 30])
def test_corpus(files, sub_bits):
    d = ctd_b200.PngDecoder(0, subsequence_bits=sub_bits)
    try:
        out = d.decode([data for _, data, _ in files])
        status = d.last_status
    finally:
        d.close()
    for (name, data, expect), got, st in zip(files, out, status):
        if expect is not None:
            assert PNG_STATUS[st] == expect, (name, PNG_STATUS[st])
        if st == 0:
            assert isinstance(got, torch.Tensor) and got.is_cuda, name
        assert _same(got, _cv2(data)), name


def test_encoder_files_and_buffers_grow_and_shrink():
    enc = ctd_b200.PngEncoder(0)
    d = ctd_b200.PngDecoder(0)
    try:
        imgs = [pc.structured(40 + i, h, w) for i, (h, w) in enumerate([(1654, 1170), (64, 48), (2339, 1654), (9, 7)])]
        imgs += [cv2.cvtColor(imgs[0], cv2.COLOR_BGR2GRAY), (cv2.cvtColor(imgs[2], cv2.COLOR_BGR2GRAY) > 100) * np.uint8(255)]
        encoded = enc.encode(imgs)
        for img, f in zip(imgs, encoded):
            assert np.array_equal(f, cv2.imencode(".png", img)[1])
        batches = [encoded[:1], encoded, encoded[1:2], encoded[2:], encoded[3:4], encoded]
        for b in batches:
            out = d.decode(b)
            assert d.last_status == [0] * len(b)
            for f, got in zip(b, out):
                assert _same(got, _cv2(f))
    finally:
        enc.close()
        d.close()


# ---- the detector on PNG pages -----------------------------------------------------------------------------------
NET = 256
DET_SIZES = [(NET, NET), (361, 251), (414, 292), (512, 512), (200, 150), (96, 700)]


@pytest.fixture(scope="module")
def det():
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=4)
    yield d
    d.close()


@pytest.fixture(scope="module")
def pngs():
    from oracle import synth
    out = []
    for i, (h, w) in enumerate(DET_SIZES):
        page = synth.structured_page(700 + i, h, w)
        out.append(cv2.imencode(".png", page)[1].tobytes() if i % 2 else pc.pil_png(page, "RGB"))
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
def test_stream_bytes(det, pngs, kw):
    ref = list(det.detect_stream([_cv2(f) for f in pngs], textheight=kw.get("textheight")))
    got = list(det.detect_stream(pngs, **kw))
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        _same_item(g, r)


def test_stream_paths_mixed_with_jpeg_and_pages(det, pngs, tmp_path):
    paths = []
    for i, f in enumerate(pngs):
        p = tmp_path / ("page%d.png" % i)
        p.write_bytes(f)
        paths.append(p if i % 2 else str(p))
    pages = [_cv2(f) for f in pngs]
    jpg = jc.encode(pages[1], 90, jc.S420)
    ref_pages = [pages[0], _cv2(jpg), pages[2], pages[3], pages[4], pages[5]]
    ref = list(det.detect_stream(ref_pages, textheight=48))
    mix = [paths[0], jpg, torch.from_numpy(pages[2]).cuda(), np.frombuffer(pngs[3], np.uint8), pages[4],
           memoryview(pngs[5])]
    got = list(det.detect_stream(mix, textheight=48))
    for g, r in zip(got, ref):
        _same_item(g, r)
    for g, r in zip(det.detect_batch(mix), det.detect_batch(ref_pages)):
        _same_item(g, r)


def test_stream_undecodable_png_raises(det, pngs, tmp_path):
    bad = tmp_path / "bad.png"
    bad.write_bytes(pngs[0][:len(pngs[0]) // 3])
    with pytest.raises(ValueError, match=r"page 5 \(.*bad\.png\)"):
        list(det.detect_stream(pngs[:5] + [str(bad)]))


def test_model2annotations_on_png_pages(det, pngs, tmp_path):
    src, out_gpu, out_ref = tmp_path / "src", tmp_path / "gpu", tmp_path / "ref"
    src.mkdir()
    for i, f in enumerate(pngs):
        (src / ("p%d.png" % i)).write_bytes(f)
    annotations.model2annotations(None, str(src), str(out_gpu), save_json=True, detector=det)
    # the same pages read by cv2, page by page
    os.makedirs(out_ref)
    for p in annotations.find_all_imgs(str(src), abs_path=True):
        img = annotations.imread(p)
        _m, mask_refined, blks = det(img, refine_mode=ctd_b200.REFINEMASK_ANNOTATION, keep_undetected_mask=True)
        annotations.write_annotations(str(out_ref), os.path.basename(p), img, mask_refined, blks, save_json=True)
    names = sorted(os.listdir(out_ref))
    assert names == sorted(os.listdir(out_gpu)) and len(names) >= 2 * len(pngs)
    for n in names:
        assert (out_gpu / n).read_bytes() == (out_ref / n).read_bytes(), n
