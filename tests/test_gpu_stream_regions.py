"""-m gpu: text-line crops in the batched stream (`TextDetector.detect_stream` / `detect_batch` with a textheight,
ctd_submit_pages + ctd_collect_regions).  Every crop is compared byte for byte with the cv2 restatement of the
reference method (tests/region_ref.py), None exactly where that method raises, and with the blocking per-page
`get_transformed_regions` on pages where no line raises; the first three fields of every item must equal the stream
without a textheight."""
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import binding
from oracle import synth
import region_ref
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
# net-sized (identity letterbox), odd, the reference's example page scaled to the net, exactly 2x the net, smaller than
# the net (upscale), a thin strip
SIZES = [(NET, NET), (361, 251), (414, 292), (2 * NET, 2 * NET), (200, 150), (96, 1500)]


def _pages(sizes, seed=500):
    # the synthetic page generator needs at least ~128 px per side: smaller pages are crops of a larger one
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _detector(max_batch, net=NET):
    return ctd_b200.TextDetector(get_checkpoint(0, True), input_size=net, act="leaky", max_batch=max_batch)


def _same_value(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)
    return type(a) is type(b) and a == b


def _same_result(got, ref):
    assert np.array_equal(got[0], ref[0]), int((got[0] != ref[0]).sum())
    assert np.array_equal(got[1], ref[1]), int((got[1] != ref[1]).sum())
    assert len(got[2]) == len(ref[2])
    for g, r in zip(got[2], ref[2]):
        dg, dr = vars(g), vars(r)
        assert list(dg) == list(dr)
        for k in dr:
            assert _same_value(dg[k], dr[k]), (k, dg[k], dr[k])


def _check_crops(det, page, blk_list, crops, th):
    """crops against region_ref line by line (None exactly where it raises) and, on a page where no line raises,
    against get_transformed_regions; all crops of the page are views of one array.  Returns
    (crops compared, lines without a crop)."""
    assert len(crops) == len(blk_list)
    n = raising = 0
    bases = set()
    for b, blk in enumerate(blk_list):
        assert len(crops[b]) == len(blk.lines)
        for i, c in enumerate(crops[b]):
            try:
                ref = region_ref.transformed_region(blk, page, i, th)
            except Exception:
                assert c is None, (b, i)
                raising += 1
                continue
            assert c is not None and c.dtype == np.uint8 and c.shape == ref.shape, (b, i, None if c is None else c.shape)
            assert np.array_equal(c, ref), (b, i, int((c != ref).any(-1).sum()))
            assert c.base is not None
            bases.add(id(c.base))
            n += 1
    assert len(bases) <= 1
    if not raising:
        for g, r in zip(det.get_transformed_regions(page, blk_list, th), crops):
            assert len(g) == len(r) and all(np.array_equal(x, y) and x.shape == y.shape for x, y in zip(g, r))
    return n, raising


@pytest.fixture(scope="module")
def det():
    d = _detector(4)
    yield d
    d.close()


@pytest.mark.parametrize("th", [32, 48])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("keep", [False, True])
def test_stream_crops_mixed_sizes(det, th, mode, keep):
    pages = _pages(SIZES)                       # 6 pages at max_batch 4: a full batch, then a partial one
    plain = list(det.detect_stream([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=keep))
    got = list(det.detect_stream([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=keep, textheight=th))
    assert len(got) == len(pages) and all(len(g) == 4 for g in got)
    n = 0
    page_bufs = set()
    for p, g, r in zip(pages, got, plain):
        _same_result(g[:3], r)
        n += _check_crops(det, p, g[2], g[3], th)[0]
        page_bufs.update(id(c.base) for blk in g[3] for c in blk if c is not None)
    assert n > 20
    assert len(page_bufs) == sum(1 for g in got if any(c is not None for blk in g[3] for c in blk))
    # detect_batch gives the same items
    bat = det.detect_batch([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=keep, textheight=th)
    for g, b in zip(got, bat):
        _same_result(b[:3], g[:3])
        assert all(len(x) == len(y) and all((u is None and v is None) or np.array_equal(u, v) for u, v in zip(x, y))
                   for x, y in zip(g[3], b[3]))


def test_stream_crops_realistic_pages():
    # an input_size-1024 detector on pages of the reference's example size: hundreds of lines per page, vertical lines,
    # crops thousands of pixels long
    d = _detector(2, net=1024)
    try:
        pages = [synth.structured_page(1000 + 1654 + 48, 1170, 1654), synth.structured_page(7001, 1654, 1170),
                 synth.structured_page(7002, 1170, 1654)]
        plain = list(d.detect_stream([p.copy() for p in pages]))
        got = list(d.detect_stream([p.copy() for p in pages], textheight=48))
        n = vert = longest = 0
        for p, g, r in zip(pages, got, plain):
            _same_result(g[:3], r)
            n += _check_crops(d, p, g[2], g[3], 48)[0]
            vert += sum(len(b.lines) for b in g[2] if b.vertical)
            longest = max([longest] + [max(c.shape[:2]) for blk in g[3] for c in blk if c is not None])
        print("realistic pages: %d crops, %d vertical lines, longest crop side %d px" % (n, vert, longest))
        assert n > 300, n
    finally:
        d.close()


def test_blank_pages_and_batches_without_crops(det):
    # uniform pages whose letterbox needs no padding (padding would draw an edge the network may see as text)
    blanks = [np.full((NET, NET, 3), 128, np.uint8), np.full((NET, NET, 3), 112, np.uint8),
              np.full((2 * NET, 2 * NET, 3), 128, np.uint8), np.full((NET // 2, NET // 2, 3), 144, np.uint8),
              np.zeros((300, 200, 3), np.uint8)]
    plain = list(det.detect_stream([p.copy() for p in blanks]))
    empty = [p for p, r in zip(blanks, plain) if sum(len(b.lines) for b in r[2]) == 0]
    assert len(empty) >= 2
    # a batch without a single crop: nothing launched or allocated, every page gets its blocks and no crops
    for batch in (empty[:1], empty, empty * 3):
        got = det.detect_batch([p.copy() for p in batch], textheight=32)
        for p, g in zip(batch, got):
            _same_result(g[:3], det(p.copy()))
            assert g[3] == [[] for _ in g[2]]
    # blank pages mixed with real ones in one batch
    real = _pages(SIZES[1:3], seed=800)
    mixed = [empty[0], real[0], empty[-1], real[1]]
    got = det.detect_batch([p.copy() for p in mixed], textheight=48)
    assert got[0][3] == [[] for _ in got[0][2]] and got[2][3] == [[] for _ in got[2][2]]
    assert _check_crops(det, real[0], got[1][2], got[1][3], 48)[0] > 0
    _check_crops(det, real[1], got[3][2], got[3][3], 48)
    # a page without blocks gives []
    assert [g[3] for g, p in zip(got, mixed) if not g[2]] == [[] for g in got if not g[2]]


def test_crop_buffers_grow_and_stay_correct():
    d = _detector(3)
    try:
        small = _pages([(120, 90), (200, 150), (NET, NET), (150, 150)], seed=3000)
        large = _pages([(2000, 3000), (1654, 1170), (3000, 2000)], seed=3100)
        for pages in (small, large + small[:2], small):
            got = list(d.detect_stream([p.copy() for p in pages], refine_mode=0, keep_undetected_mask=True,
                                       textheight=48))
            n = 0
            for p, g in zip(pages, got):
                _same_result(g[:3], d(p.copy(), refine_mode=0, keep_undetected_mask=True))
                n += _check_crops(d, p, g[2], g[3], 48)[0]
            assert n > 0
    finally:
        d.close()


def test_call_and_crops_between_stream_yields():
    # __call__ and get_transformed_regions (engine stream, io scratch) while the other batch of a crop stream is still
    # in flight (post stream, the slot's crop buffers): both sides give their stand-alone results
    d = _detector(2)
    try:
        pages = _pages([(700, 500), (520, 760), (NET, NET), (900, 640), (361, 251), (640, 900), (500, 700), (300, 420)],
                       seed=6100)
        others = _pages([(620, 410), (NET, NET), (1000, 700)], seed=6200)
        ref = [d(p.copy(), refine_mode=1, keep_undetected_mask=True) for p in pages]
        ref_o, ref_oc = [], []
        for p in others:
            r = d(p.copy(), refine_mode=1, keep_undetected_mask=True)
            ref_o.append(r)
            try:
                ref_oc.append(d.get_transformed_regions(p, r[2], 32))
            except binding.CtdError as e:
                ref_oc.append(str(e))
        k = 0
        for i, got in enumerate(d.detect_stream([p.copy() for p in pages], refine_mode=1, keep_undetected_mask=True,
                                                textheight=32)):
            _same_result(got[:3], ref[i])
            _check_crops(d, pages[i], got[2], got[3], 32)
            o = k % len(others)
            r = d(others[o].copy(), refine_mode=1, keep_undetected_mask=True)
            _same_result(r, ref_o[o])
            if isinstance(ref_oc[o], str):
                with pytest.raises(binding.CtdError):
                    d.get_transformed_regions(others[o], r[2], 32)
            else:
                c = d.get_transformed_regions(others[o], r[2], 32)
                assert all(len(x) == len(y) and all(np.array_equal(u, v) for u, v in zip(x, y))
                           for x, y in zip(c, ref_oc[o]))
            k += 1
        assert k == len(pages)
    finally:
        d.close()


def test_stream_region_errors(det):
    pages = _pages(SIZES[:5], seed=900)
    # an abandoned crop stream leaves the engine usable
    g = det.detect_stream([p.copy() for p in pages], textheight=48)
    first = next(g)
    g.close()
    again = det.detect_batch([p.copy() for p in pages], textheight=48)
    _same_result(again[0][:3], first[:3])
    for p, a in zip(pages, again):
        _check_crops(det, p, a[2], a[3], 48)
    # a bad textheight raises before any page is read or submitted
    seen = []

    def feed():
        for p in pages:
            seen.append(1)
            yield p.copy()

    for bad in (1, 2.5, True, 0, -4, "48"):
        with pytest.raises(ValueError):
            det.detect_stream(feed(), textheight=bad)
        with pytest.raises(ValueError):
            det.detect_batch(pages, textheight=bad)
    assert not seen
    # the C ABI refuses textheight < 2 (0 means no crops) and crops of a batch that did not ask for them
    eng = det.net
    ent, ib, rb = binding.pages_plan([p.shape[:2] for p in pages[:2]], NET, NET)
    buf = np.zeros((ib,), np.uint8)
    out = np.zeros((rb,), np.uint8)
    for th in (1, -1):
        rc = eng.lib.ctd_submit_pages(eng.h, 1, binding._ptr(ent), 2, NET, NET, binding._ptr(buf), None, 0, 0, th, 0,
                                      binding._ptr(out))
        assert rc == -1   # CTD_E_INVALID
    eng.submit_pages(1, pages[:2], NET, NET)
    eng.collect_pages(1)
    with pytest.raises(ctd_b200.CtdError):
        eng.collect_regions(1, [[], []])
    # the engine still works after every refusal
    res = det.detect_batch([pages[1]], textheight=32)[0]
    _same_result(res[:3], det(pages[1]))
    _check_crops(det, pages[1], res[2], res[3], 32)
