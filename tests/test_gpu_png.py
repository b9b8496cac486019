"""gpu: PNG files encoded on the GPU (ctd_b200.PngEncoder, csrc/png.cu) equal cv2.imencode('.png') byte for byte.

Covers one call mixing numpy images and CUDA tensors (crops, permuted channels-first tensors, a tensor written by a
kernel still queued on the caller's stream), the seeded corpus of tests/png_corpus.py, the masks of a device-results
stream, large pages, buffers growing and shrinking, refused inputs, and model2annotations on a directory of baseline
JPEGs, a progressive JPEG, a PNG and an unreadable file."""
import os

import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import annotations
from oracle import png_ref, synth
import png_corpus as pc
from util import get_checkpoint

pytestmark = pytest.mark.gpu

# the sizes of the benchmark pages (scripts/pages_bench.py)
PAGE_SIZES = [(1654, 1170), (1170, 1654), (2048, 1446), (1200, 800), (1024, 1024)]


def _cv2(img):
    if isinstance(img, torch.Tensor):
        img = img.cpu().numpy()
    return cv2.imencode(".png", img)[1]


@pytest.fixture(scope="module")
def enc():
    e = ctd_b200.PngEncoder(0)
    yield e
    e.close()


def test_mixed_call(enc):
    rng = np.random.default_rng(7)
    dev = torch.device("cuda", 0)
    page = synth.structured_page(3, 600, 500)
    big = torch.from_numpy(page).to(dev)
    chw = torch.from_numpy(np.ascontiguousarray(page.transpose(2, 0, 1))).to(dev)
    grey = torch.from_numpy(rng.integers(0, 4, (333, 517), dtype=np.uint8) * 80).to(dev)
    # written by kernels still queued on the current stream when encode is called
    queued = torch.empty((700, 900, 3), dtype=torch.uint8, device=dev)
    torch.cuda._sleep(50_000_000)
    queued.copy_(torch.from_numpy(synth.structured_page(4, 700, 900)).to(dev))
    imgs = [page, big[17:411, 33:377], chw.permute(1, 2, 0), grey, grey[::2, 1::3], big[:, :, 1], queued,
            rng.integers(0, 256, (1, 1), dtype=np.uint8), np.ascontiguousarray(page[::-1]), big[5:6, :1]]
    got = enc.encode(imgs)
    assert len(got) == len(imgs)
    for i, (img, g) in enumerate(zip(imgs, got)):
        ref = _cv2(img)
        assert g.dtype == np.uint8 and g.ndim == 1
        assert np.array_equal(g, ref), i
        if i in (1, 4, 7, 9):
            host = img.cpu().numpy() if isinstance(img, torch.Tensor) else img
            assert np.array_equal(g, png_ref.encode(host)), i


def test_corpus(enc):
    cases = pc.corpus() + pc.golden_page()
    got = enc.encode([img for _n, img in cases])
    for (name, img), g in zip(cases, got):
        assert np.array_equal(g, _cv2(img)), name
    # the same images one by one, and as CUDA tensors
    for name, img in cases[:40]:
        assert np.array_equal(enc.encode([img])[0], _cv2(img)), name
    dev = [torch.from_numpy(img).cuda() for _n, img in cases]
    for (name, img), g in zip(cases, enc.encode(dev)):
        assert np.array_equal(g, _cv2(img)), name


def test_device_result_masks(enc):
    pages = [synth.structured_page(40 + i, h, w) for i, (h, w) in enumerate(PAGE_SIZES)]
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=1024, act="leaky", max_batch=4)
    try:
        res = list(det.detect_stream(pages, refine_mode=ctd_b200.REFINEMASK_ANNOTATION, keep_undetected_mask=True,
                                     device_results=True))
    finally:
        det.close()
    masks = [m for r in res for m in (r[0], r[1])]
    assert all(m.is_cuda for m in masks)
    got = enc.encode(masks)
    for m, g in zip(masks, got):
        assert np.array_equal(g, _cv2(m))


def test_large_pages(enc):
    rng = np.random.default_rng(11)
    a4 = synth.structured_page(9, 7016, 4960)
    wide = rng.integers(0, 3, (300, 8193, 3), dtype=np.uint8) * 100
    got = enc.encode([a4, torch.from_numpy(wide).cuda()])
    assert np.array_equal(got[0], _cv2(a4))
    assert np.array_equal(got[1], _cv2(wide))


def test_buffers_grow_and_shrink():
    e = ctd_b200.PngEncoder(0)
    try:
        rng = np.random.default_rng(5)
        for shape in [(8, 8), (300, 200, 3), (2000, 1500, 3), (50, 60), (1, 1), (1500, 2000, 3), (17, 3, 3)]:
            imgs = [rng.integers(0, 256, shape, dtype=np.uint8), np.full(shape, 9, np.uint8),
                    (rng.integers(0, 3, shape) * 90).astype(np.uint8)]
            for img, g in zip(imgs, e.encode(imgs)):
                assert np.array_equal(g, _cv2(img)), shape
    finally:
        e.close()


def test_refused_inputs(enc):
    ok = np.zeros((4, 4, 3), np.uint8)
    bad = [np.zeros((0, 4), np.uint8), np.zeros((4, 0, 3), np.uint8), np.zeros((4, 4, 4), np.uint8),
           np.zeros((4, 4, 1), np.uint8), np.zeros((4, 4), np.uint16), np.zeros(16, np.uint8),
           torch.zeros((4, 4, 3), dtype=torch.uint8), torch.zeros((4, 4), dtype=torch.int16, device="cuda"),
           torch.zeros((4, 4, 2), dtype=torch.uint8, device="cuda"), [[1, 2], [3, 4]], None]
    for b in bad:
        with pytest.raises(ValueError, match="image 1"):
            enc.encode([ok, b])
    assert np.array_equal(enc.encode([ok])[0], _cv2(ok))


def _same_tree(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    assert fa == fb
    for f in fa:
        with open(os.path.join(a, f), "rb") as x, open(os.path.join(b, f), "rb") as y:
            assert x.read() == y.read(), f


def test_model2annotations(tmp_path):
    src, out, ref = tmp_path / "src", tmp_path / "out", tmp_path / "ref"
    src.mkdir()
    ref.mkdir()
    pages = [synth.structured_page(70 + i, h, w) for i, (h, w) in enumerate(PAGE_SIZES)]
    for i, p in enumerate(pages):
        cv2.imwrite(str(src / ("p%d.jpg" % i)), p, [cv2.IMWRITE_JPEG_QUALITY, 90])
    cv2.imwrite(str(src / "prog.jpg"), pages[0][:900, :700], [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    cv2.imwrite(str(src / "flat.png"), pages[1][:500, :640])
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=1024, act="leaky", max_batch=3)
    try:
        annotations.model2annotations(None, str(src), str(out), save_json=True, detector=det)
        for fp in annotations.find_all_imgs(str(src), abs_path=True):
            img = annotations.imread(fp)
            _m, refined, blks = det(img, refine_mode=ctd_b200.REFINEMASK_ANNOTATION, keep_undetected_mask=True)
            annotations.write_annotations(str(ref), os.path.basename(fp), img, refined, blks, save_json=True)
        _same_tree(str(out), str(ref))
        # an unreadable file last: every page before it is written, then the error is raised
        (src / "zz_broken.png").write_bytes(b"not an image")
        out2 = tmp_path / "out2"
        with pytest.raises(ValueError, match="zz_broken"):
            annotations.model2annotations(None, str(src), str(out2), save_json=True, detector=det)
        names = [os.path.basename(f) for f in annotations.find_all_imgs(str(src))]
        before = names[:names.index("zz_broken.png")]
        written = sorted(os.listdir(out2))
        assert {annotations.png_path(n) for n in before} <= set(written)
        assert {"mask-" + os.path.splitext(n)[0] + ".png" for n in before} <= set(written)
        for f in written:
            with open(os.path.join(out2, f), "rb") as x, open(os.path.join(ref, f), "rb") as y:
                assert x.read() == y.read(), f
    finally:
        det.close()
