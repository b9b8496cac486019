"""-m gpu: text-line crops of caller block lists (`RegionCropper.crop_stream` / `crop_batch`, ctd_submit_regions).
Every crop is compared byte for byte with the cv2 restatement of the reference method (tests/region_ref.py), with None
exactly where that method raises: on the detector's own blocks (where the stream must also equal
`detect_stream(textheight=)`), on the reference's own crops (tests/golden/regions_ref.npz), on edited block lists, and
on batches mixing numpy pages, strided CUDA pages and encoded files."""
import json

import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding
from ctd_b200.annotations import NumpyEncoder
from ctd_b200.textblock import TextBlock
from oracle import synth
import region_cases as rc
import region_ref
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
SIZES = [(NET, NET), (361, 251), (414, 292), (2 * NET, 2 * NET), (200, 150), (96, 1500)]


def _pages(sizes, seed=900):
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _host(c):
    return c.cpu().numpy() if isinstance(c, torch.Tensor) else c


def _check(page, blk_list, crops, th):
    """crops against region_ref, None exactly where it raises; -> (crops compared, None lines)"""
    assert len(crops) == len(blk_list)
    n = raising = 0
    for b, blk in enumerate(blk_list):
        assert len(crops[b]) == len(blk.lines), b
        for i, c in enumerate(crops[b]):
            try:
                ref = region_ref.transformed_region(blk, page, i, th)
            except Exception:
                assert c is None, (b, i)
                raising += 1
                continue
            c = _host(c)
            assert c is not None and c.dtype == np.uint8 and c.shape == ref.shape, (b, i)
            assert np.array_equal(c, ref), (b, i, int((c != ref).any(-1).sum()))
            n += 1
    return n, raising


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for p, q in zip(x, y):
            assert (p is None) == (q is None)
            if p is not None:
                p, q = _host(p), _host(q)
                assert p.shape == q.shape and np.array_equal(p, q)


def _one_base(crops):
    bases = {id(c.base) for blk in crops for c in blk if c is not None}
    assert len(bases) <= 1


@pytest.fixture(scope="module")
def det():
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=4)
    yield d
    d.close()


@pytest.fixture(scope="module")
def cropper():
    r = ctd_b200.RegionCropper(max_batch=3)
    yield r
    r.close()


@pytest.mark.parametrize("th", [32, 48])
def test_detector_blocks_equal_detect_stream(det, cropper, th):
    pages = _pages(SIZES)
    res = det.detect_batch([p.copy() for p in pages], textheight=th)
    got = cropper.crop_batch([(p, r[2]) for p, r in zip(pages, res)], th)
    n = 0
    for p, r, g in zip(pages, res, got):
        _same(g, r[3])
        _one_base(g)
        n += _check(p, r[2], g, th)[0]
    assert n > 20


def test_reference_crops_through_the_stream(cropper):
    z = np.load(rc.GOLD)
    items = [rc.page_case(i) for i in range(len(rc.PAGE_CASES))]
    n = 0
    for th in (32, 48):
        idx = [i for i, (_p, _b, t) in enumerate(items) if t == th]
        for i, got in zip(idx, cropper.crop_stream([items[i][:2] for i in idx], th)):
            for b, crops in enumerate(got):
                for l, c in enumerate(crops):
                    assert np.array_equal(c, z["p%d_%d_%d" % (i, b, l)]), (i, b, l)
                    n += 1
    page = rc.hand_page()
    for th in (32, 48):
        hand, raising = cropper.crop_batch([(page, rc.hand_blocks()), (page, rc.raising_blocks())], th)
        for b, crops in enumerate(hand):
            for l, c in enumerate(crops):
                assert np.array_equal(c, z["h%d_%d_%d" % (th, b, l)]), (th, b, l)
                n += 1
        assert [b for b, crops in enumerate(raising) if crops[0] is None] == z["raises%d" % th].tolist()
    assert n == len([k for k in z.files if not k.startswith("raises")])


def _edited(blks, shape):
    """the detector's blocks edited as a caller would: every other block dropped, hand-made blocks added (eng, ja,
    unknown, vertical, past the page edge, no lines, the default font_size), a 1-px crop and a degenerate quad"""
    h, w = shape
    kept = blks[::2]
    added = [
        TextBlock([5, 5, 60, 20], lines=[rc.rect(5, 5, 60, 20)], language="eng", font_size=9),
        TextBlock([10, 30, 90, 44], lines=[rc.rect(10, 30, 90, 44)], language="ja"),   # font_size -1
        TextBlock([20, 50, 100, 70], lines=[rc.rect(20, 50, 100, 70), rc.rect(22, 72, 80, 88)], language="unknown",
                  font_size=11.5),
        TextBlock([30, 10, 46, 100], lines=[rc.rect(30, 10, 46, 100)], language="ja", vertical=True, font_size=14),
        TextBlock([w - 40, h - 20, w + 30, h + 15], lines=[rc.rect(w - 40, h - 20, w + 30, h + 15)], language="eng",
                  font_size=12),
        TextBlock([0, 0, 10, 10]),                                                     # no lines
        TextBlock([40, 40, 42, 100], lines=[rc.rect(40, 40, 42, 100), rc.rect(40, 40, 100, 40)], language="ja",
                  font_size=10),                                                     # 1-px crop, degenerate quad
    ]
    return kept + added


def test_edited_and_json_round_tripped_lists(det, cropper):
    pages = _pages(SIZES[:5], seed=950)
    res = det.detect_batch([p.copy() for p in pages])
    lists = [_edited(r[2], p.shape[:2]) for p, r in zip(pages, res)]
    # through the json writer of model2annotations and back with TextBlock(**d)
    back = [[TextBlock(**d) for d in json.loads(json.dumps([b.to_dict() for b in bl], cls=NumpyEncoder))]
            for bl in lists]
    for th in (32, 48):
        got = cropper.crop_batch(list(zip(pages, lists)), th)
        got_json = list(cropper.crop_stream(zip(pages, back), th))
        for p, bl, g, gj in zip(pages, lists, got, got_json):
            _same(g, gj)
            n, raising = _check(p, bl, g, th)
            assert n >= 6 and raising >= 1          # the other lines of a page with a raising line are still cut
            assert g[-2] == [] and g[-1][1] is None   # no lines; the degenerate quad
            assert (g[-1][0] is None) == (th == 32)   # a 1-px wide crop at textheight 32 only


def _encode(page, ext):
    return cv2.imencode(ext, page, [cv2.IMWRITE_JPEG_QUALITY, 93] if ext == ".jpg" else [])[1]


@pytest.mark.parametrize("max_batch", [1, 3, 16])
def test_mixed_batches(tmp_path, max_batch):
    pages = _pages(SIZES + [(300, 420)], seed=970)
    blocks = [rc.hand_blocks() + rc.raising_blocks() for _ in pages]
    dev = torch.device("cuda", 0)
    items, refs = [], []
    for k, p in enumerate(pages):
        kind = k % 6
        if kind == 0:
            items.append(p)
        elif kind == 1:   # a crop of a larger tensor
            big = torch.zeros((p.shape[0] + 7, p.shape[1] + 9, 3), dtype=torch.uint8, device=dev)
            big[3:3 + p.shape[0], 5:5 + p.shape[1]] = torch.from_numpy(p).to(dev)
            items.append(big[3:3 + p.shape[0], 5:5 + p.shape[1]])
        elif kind == 2:   # channels-first storage
            items.append(torch.from_numpy(np.ascontiguousarray(p.transpose(2, 0, 1))).to(dev).permute(1, 2, 0))
        elif kind == 3:
            items.append(_encode(p, ".jpg").tobytes())
        elif kind == 4:
            items.append(_encode(p, ".png"))
        else:
            fn = tmp_path / ("page%d.%s" % (k, "png" if k % 2 else "jpg"))
            cv2.imwrite(str(fn), p)
            items.append(str(fn))
        refs.append(p if kind < 3 else cv2.imdecode(np.fromfile(str(items[-1]), np.uint8) if kind == 5 else
                                                    np.frombuffer(bytes(items[-1]), np.uint8), cv2.IMREAD_COLOR))
    r = ctd_b200.RegionCropper(max_batch=max_batch)
    try:
        for th in (32, 48):
            got = list(r.crop_stream(zip(items, blocks), th))
            assert len(got) == len(items)
            for ref, bl, g in zip(refs, blocks, got):
                _one_base(g)
                _check(ref, bl, g, th)
            dres = r.crop_batch(list(zip(items, blocks)), th, device_results=True)
            for g, d in zip(got, dres):
                _same(g, d)
                assert all(c.is_cuda for blk in d for c in blk if c is not None)
    finally:
        r.close()


def test_cuda_page_written_by_queued_kernel(cropper):
    page = _pages([(414, 292)], seed=990)[0]
    src = torch.from_numpy(page).cuda()
    dst = torch.zeros_like(src)
    torch.cuda._sleep(200_000_000)   # the copy below stays queued behind this on the current stream
    dst.copy_(src)
    (got,) = list(cropper.crop_stream([(dst, rc.hand_blocks())], 48))
    _check(page, rc.hand_blocks(), got, 48)


def test_items_without_lines(cropper):
    page = _pages([(200, 150)])[0]
    got = cropper.crop_batch([(page, []), (page, [TextBlock([0, 0, 5, 5])]), (page, rc.raising_blocks()[2:])], 32)
    assert got[0] == [] and got[1] == [[]] and got[2] == [[None]]
    dres = cropper.crop_batch([(page, []), (torch.from_numpy(page).cuda(), [TextBlock([0, 0, 5, 5])])], 32,
                              device_results=True)
    assert dres == [[], [[]]]


def test_errors_before_gpu_work_and_reuse(cropper):
    page = _pages([(200, 150)])[0]
    good = (page, rc.hand_blocks())
    for th in (1, 0, 2.5, "32", None):
        with pytest.raises(ValueError, match="textheight"):
            cropper.crop_stream([good], th)
    bad_line = [TextBlock([0, 0, 5, 5], lines=[rc.rect(1, 1, 30, 9), [[1, 2], [3, 4]]])]
    cases = [(np.zeros((10, 10), np.uint8), rc.hand_blocks()), (page, bad_line),
             (np.zeros((1, 32767, 3), np.uint8), rc.hand_blocks())]
    for bad, match in zip(cases, ["item 1: a page must be", "item 1: block 0, line 1", "item 1: the page is 1x32767"]):
        with pytest.raises(ValueError, match=match):
            cropper.crop_batch([good, bad], 32)
        gen = cropper.crop_stream([good, bad, good], 32)   # max_batch 3: nothing reaches the GPU
        with pytest.raises(ValueError, match=match):
            next(gen)
    # the engine refuses the same page itself, naming it
    with pytest.raises(binding.CtdError, match="page 0"):
        cropper.net.submit_regions(0, [np.zeros((1, 32767, 3), np.uint8)], np.zeros((0,), binding.REGION_LINE_DTYPE),
                                   [0], 32)
    with pytest.raises(binding.CtdError, match="textheight"):
        cropper.net.submit_regions(0, [page], np.zeros((0,), binding.REGION_LINE_DTYPE), [0], 1)
    (got,) = cropper.crop_batch([good], 32)
    _check(page, rc.hand_blocks(), got, 32)


def test_abandoned_generator_leaves_engine_reusable():
    pages = _pages(SIZES, seed=1000)
    items = [(p, rc.hand_blocks()) for p in pages]
    r = ctd_b200.RegionCropper(max_batch=1)
    try:
        gen = r.crop_stream(items, 48)
        first = next(gen)
        gen.close()
        again = r.crop_batch(items, 48)
        _same(first, again[0])
        for p, g in zip(pages, again):
            _check(p, rc.hand_blocks(), g, 48)
    finally:
        r.close()
