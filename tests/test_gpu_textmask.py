"""-m gpu: refine_mask on caller block lists (ctd_submit_refine): the module-level `refine_mask` /
`refine_undetected_mask`, `MaskRefiner` and `annotations.traverse_by_dict`, byte for byte against the oracle
(tie_order="stable") in both refine modes, and against the detector's own masks on its own blocks."""
import json
import os

import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import annotations, binding
from ctd_b200.textblock import TextBlock
from oracle import pipeline_ref, postproc_ref, synth
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
SIZES = [(NET, NET), (361, 251), (414, 292), (200, 150), (96, 700)]
MODES = [ctd_b200.REFINEMASK_INPAINT, ctd_b200.REFINEMASK_ANNOTATION]


def _pages(sizes, seed=700):
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _blocks(boxes):
    return [TextBlock(b) for b in boxes]


def _oracle(img, mask, boxes, mode):
    return postproc_ref.refine_mask(img, mask, [list(b) for b in boxes], mode, "stable")


@pytest.fixture(scope="module")
def det():
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=4)
    yield d
    d.close()


@pytest.fixture(scope="module")
def detected(det):
    pages = _pages(SIZES)
    return pages, det.detect_batch([p.copy() for p in pages], keep_undetected_mask=False)


@pytest.fixture(scope="module")
def refiner():
    r = ctd_b200.MaskRefiner(max_batch=3)
    yield r
    r.close()


def _status(shape, boxes):
    return binding.refine_plan([shape], np.asarray(boxes, np.int32).reshape(-1, 4), [len(boxes)])[2]


def _refinable(blks, shape):
    """the blocks refine_mask takes: the detector can make a block whose window is empty (a block past the page's right
    or bottom edge); the reference raises on it, while the detector drops its window, so dropping the block leaves the
    detector's mask_refined as it is"""
    st = _status(shape, [b.xyxy for b in blks])
    return [b for b, s in zip(blks, st) if s == 0]


def _odd_boxes(ih, iw):
    return [[-5, -5, 20, 20], [iw - 10, ih - 10, iw + 30, ih + 30], [-40, 3, -33, 9], [3, -40, 9, -33],
            [30, 30, 10, 50], [0, 0, 0, 0], [iw - 1, ih - 1, iw - 1, ih - 1], [0, 0, iw, ih], [iw // 2, 0, iw // 2 + 1, ih],
            [0, ih // 2, iw, ih // 2], [-100, -100, 100, 100], [iw + 5, 0, iw + 9, 4], [5, 5, 6, 6]]


@pytest.mark.parametrize("mode", MODES)
def test_refine_mask_against_oracle(detected, mode):
    pages, res = detected
    for img, (mask, _mr, blks) in zip(pages, res):
        ih, iw = img.shape[:2]
        odd = _odd_boxes(ih, iw)
        st = _status((ih, iw), odd)
        ok = [b for b, s in zip(odd, st) if s == 0]
        assert len(ok) >= 6 and (st != 0).any()
        boxes = [b.xyxy for b in _refinable(blks, (ih, iw))] + ok
        got = ctd_b200.refine_mask(img, mask, _blocks(boxes), mode)
        assert np.array_equal(got, _oracle(img, mask, boxes, mode)), (img.shape, int((got != _oracle(img, mask, boxes, mode)).sum()))
        for b, s in zip(odd, st):
            if s != 0:
                with pytest.raises(ValueError, match="block 1 "):
                    ctd_b200.refine_mask(img, mask, _blocks([ok[0], b]), mode)


def test_refine_mask_rejects_bad_masks(detected):
    pages, res = detected
    img, mask = pages[1], res[1][0]
    for bad in (mask[:-1], mask.astype(np.int16), np.dstack([mask, mask]), mask[None]):
        with pytest.raises(ValueError, match="mask"):
            ctd_b200.refine_mask(img, bad, _blocks([[5, 5, 40, 40]]))
    with pytest.raises(ValueError, match="int32"):
        ctd_b200.refine_mask(img, mask, _blocks([[5, 5, 2 ** 31, 40]]))


@pytest.mark.parametrize("mode", MODES)
def test_refine_undetected_mask_against_oracle(detected, mode):
    pages, res = detected
    for img, (mask, mr, blks) in zip(pages, res):
        boxes = [b.xyxy for b in blks]
        # a caller mask_refined that is not refine_mask's output: every other block's part of it, plus a stripe
        other = ctd_b200.refine_mask(img, mask, _refinable(blks, img.shape[:2])[::2], mode)
        other[::7] |= 40
        keep = [b for i, b in enumerate(boxes) if i % 3]
        mp, mp_ref = mask.copy(), mask.copy()
        got = ctd_b200.refine_undetected_mask(img, mp, other.copy(), _blocks(keep), mode)
        want = pipeline_ref.refine_undetected_mask(img, mp_ref, other.copy(), keep, None, mode)
        assert np.array_equal(mp, mp_ref)
        assert np.array_equal(got, want), int((got != want).sum())


@pytest.mark.parametrize("mode", MODES)
def test_refine_batch_equals_the_detector(det, refiner, mode):
    pages = _pages(SIZES, seed=900)
    plain = det.detect_batch([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=False)
    kept = det.detect_batch([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=True)
    items = [(p, m, _refinable(blks, p.shape[:2])) for p, (m, _mr, blks) in zip(pages, plain)]
    for (m, mr), (m0, mr0, _b) in zip(refiner.refine_batch(items, refine_mode=mode), plain):
        assert m is m0 and np.array_equal(mr, mr0)
    masks = [m.copy() for _p, m, _b in items]
    whole = [len(b) == len(d[2]) for (_p, _m, b), d in zip(items, plain)]
    assert any(whole)
    for (m, mr), (mk, mrk, _b), src, (_p, m0, _b0), w in zip(refiner.refine_batch(items, mode, True), kept, masks, items,
                                                              whole):
        assert m is not m0 and np.array_equal(m0, src)   # the caller's mask is not modified
        if w:   # refine_undetected_mask compares the components with every block
            assert np.array_equal(m, mk) and np.array_equal(mr, mrk)
    # the reference's chain on the detector's whole block list: refine_mask, then refine_undetected_mask
    for p, (m0, mr0, blks), (mk, mrk, _b) in zip(pages, plain, kept):
        m = m0.copy()
        mr = ctd_b200.refine_undetected_mask(p, m, ctd_b200.refine_mask(p, m0, _refinable(blks, p.shape[:2]), mode),
                                             blks, mode)
        assert np.array_equal(m, mk) and np.array_equal(mr, mrk)


@pytest.mark.parametrize("mode", MODES)
def test_edited_block_lists(detected, refiner, mode):
    pages, res = detected
    rng = np.random.default_rng(5)
    items, want = [], []
    for img, (mask, _mr, blks) in zip(pages, res):
        ih, iw = img.shape[:2]
        boxes = [list(b.xyxy) for b in blks]
        added = [[int(rng.integers(0, iw - 20)), int(rng.integers(0, ih - 20))] for _ in range(3)]
        added = [[x, y, x + int(rng.integers(8, 60)), y + int(rng.integers(8, 40))] for x, y in added]
        moved = [[b[0] + 7, b[1] - 5, b[2] + 7, b[3] - 5] for b in boxes]
        for edit in (boxes[1:], boxes + added, moved, boxes + boxes[:2], [], added[:1]):
            edit = [b for b, s in zip(edit, _status((ih, iw), edit)) if s == 0]
            items.append((img, mask, _blocks(edit)))
            want.append(_oracle(img, mask, edit, mode))
    got = refiner.refine_batch(items, refine_mode=mode)
    for (m, mr), w, (_i, m0, blks) in zip(got, want, items):
        assert m is m0 and np.array_equal(mr, w)
        if not blks:
            assert not mr.any()


def _encoded(img, k):
    return cv2.imencode(".png" if k % 2 else ".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 95] if k % 2 == 0 else [])[1]


def test_stream_mixed_inputs(detected, refiner):
    pages, res = detected
    dev = torch.device("cuda", 0)
    items, want = [], []
    for k in range(10):
        img, (mask, _mr, blks) = pages[k % len(pages)], res[k % len(res)]
        boxes = [b.xyxy for b in _refinable(blks, img.shape[:2])]
        ih, iw = img.shape[:2]
        kind = k % 5
        if kind == 0:
            page, m = img, mask
        elif kind == 1:   # CUDA page, mask channel 0 of a CUDA page (a strided view)
            page = torch.from_numpy(img).to(dev)
            m = torch.from_numpy(np.dstack([mask, mask // 2, mask])).to(dev)[..., 0]
        elif kind == 2:   # crops of larger CUDA images
            big = torch.zeros((ih + 9, iw + 13, 3), dtype=torch.uint8, device=dev)
            big[4:4 + ih, 6:6 + iw] = torch.from_numpy(img).to(dev)
            bigm = torch.zeros((ih + 3, iw + 31), dtype=torch.uint8, device=dev)
            bigm[1:1 + ih, 5:5 + iw] = torch.from_numpy(mask).to(dev)
            page, m = big[4:4 + ih, 6:6 + iw], bigm[1:1 + ih, 5:5 + iw]
        elif kind == 3:   # encoded page, numpy mask with strides
            page, m = _encoded(img, k), np.dstack([mask, mask])[..., 0]
        else:             # channels-first CUDA page permuted, encoded PNG page with a CUDA mask
            page = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).to(dev).permute(1, 2, 0)
            m = torch.from_numpy(mask).to(dev).t().contiguous().t()
        src = img if kind != 3 else cv2.imdecode(page, cv2.IMREAD_COLOR)
        items.append((page, m, _blocks(boxes)))
        want.append(_oracle(src, mask, boxes, 0))
    host = list(refiner.refine_stream(items))
    devr = list(refiner.refine_stream(items, device_results=True))
    assert len(host) == len(devr) == 10
    for (m, mr), (dm, dmr), w, it in zip(host, devr, want, items):
        assert m is it[1] and dm is it[1]
        assert np.array_equal(mr, w)
        assert dmr.is_cuda and np.array_equal(dmr.cpu().numpy(), mr)
    kept = list(refiner.refine_stream(items, keep_undetected_mask=True))
    kept_dev = list(refiner.refine_stream(items, keep_undetected_mask=True, device_results=True))
    for (m, mr), (dm, dmr), it in zip(kept, kept_dev, items):
        assert isinstance(m, np.ndarray) and m is not it[1]
        assert np.array_equal(dm.cpu().numpy(), m) and np.array_equal(dmr.cpu().numpy(), mr)


def test_stream_waits_for_a_mask_written_on_the_callers_stream(detected, refiner):
    pages, res = detected
    img, (mask, mr, blks) = pages[2], res[2]
    blks = _refinable(blks, img.shape[:2])
    side = torch.cuda.Stream()
    src = torch.from_numpy(mask).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        m = torch.zeros_like(src)
        torch.cuda._sleep(50_000_000)
        m.copy_(src)
        out = list(refiner.refine_stream([(img, m, blks)]))
    assert np.array_equal(out[0][1], mr)


def test_stream_errors_before_gpu_work(detected, refiner):
    pages, res = detected
    img, (mask, _mr, blks) = pages[1], res[1]
    blks = _refinable(blks, img.shape[:2])
    bad_items = [
        [(img, mask[:, :-1], blks)],
        [(img[..., :2], mask, blks)],
        [(img, mask, _blocks([[10, 10, 30, 30], [30, 30, 10, 10]]))],
        [(img, torch.from_numpy(mask).cuda().to(torch.int16), blks)],
    ]
    for items in bad_items:
        with pytest.raises(ValueError, match="item 0"):
            refiner.refine_batch(items)
        with pytest.raises(ValueError, match="item 0"):
            list(refiner.refine_stream(items))
    # an encoded page: checked once decoded, with its batch
    with pytest.raises(ValueError, match="item 1"):
        list(refiner.refine_stream([(img, mask, blks), (_encoded(img, 1), mask[:-2], blks)]))
    # the refiner is still usable
    assert np.array_equal(refiner.refine_batch([(img, mask, blks)])[0][1], res[1][1])


def test_abandoned_stream_leaves_nothing_in_flight(detected, refiner):
    pages, res = detected
    items = [(p, m, _refinable(b, p.shape[:2])) for p, (m, _mr, b) in zip(pages, res)] * 3
    g = refiner.refine_stream(items)
    next(g)
    g.close()
    assert refiner.net._pg_inflight == [None, None]
    got = refiner.refine_batch(items[:4])
    for (m, mr), (_p, m0, _b), (_m, mr0, _bb) in zip(got, items[:4], res + res):
        assert np.array_equal(mr, mr0)


def test_traverse_by_dict_after_model2annotations(det, tmp_path):
    pages = _pages([(300, 220), (256, 256), (180, 340), (250, 190), (333, 111)], seed=1200)
    src, out = tmp_path / "src", tmp_path / "out"
    src.mkdir()
    for i, p in enumerate(pages):
        cv2.imwrite(str(src / ("page%d.%s" % (i, "jpg" if i % 2 else "png"))), p)
    annotations.model2annotations(None, str(src), str(out), save_json=True, detector=det)
    # the blocks refine_mask takes (_refinable), written back as a caller that edits the json would
    for i, p in enumerate(pages):
        fn = out / ("page%d.json" % i)
        dicts = json.loads(fn.read_text())
        st = _status(p.shape[:2], [d["xyxy"] for d in dicts])
        fn.write_text(json.dumps([d for d, s in zip(dicts, st) if s == 0]))
    r = ctd_b200.MaskRefiner(max_batch=2)
    try:
        got = list(annotations.traverse_by_dict(str(src), str(out), refiner=r))
    finally:
        r.close()
    paths = annotations.find_all_imgs(str(src), abs_path=True)
    assert [g[0] for g in got] == paths and len(got) == 5
    n_blocks = 0
    for img_path, img, mask_refined, blk_list in got:
        name = os.path.splitext(os.path.basename(img_path))[0]
        im = cv2.imread(img_path)
        mask = cv2.imread(str(out / ("mask-%s.png" % name)), cv2.IMREAD_GRAYSCALE)
        page = img.cpu().numpy() if getattr(img, "is_cuda", False) else img
        assert np.array_equal(page, im)
        assert all(isinstance(b, TextBlock) for b in blk_list)
        n_blocks += len(blk_list)
        boxes = [b.xyxy for b in blk_list]
        assert np.array_equal(mask_refined, _oracle(im, mask, boxes, 0))
    assert n_blocks > 0
    os.remove(str(out / "page0.json"))
    with pytest.raises(FileNotFoundError):
        list(annotations.traverse_by_dict(str(src), str(out)))
