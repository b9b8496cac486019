"""-m gpu: batches of pages of any size (ctd_submit_pages, TextDetector.detect_batch / detect_stream) against the
page-by-page call (ctd_detect_page) byte for byte, the letterbox kernel against the host letterbox, one page against
the oracle chain at the page's own scale, model2annotations through the stream, and the error paths."""
import filecmp
import os

import numpy as np
import pytest

import ctd_b200
from ctd_b200 import annotations, binding
from ctd_b200.inference import letterbox, letterbox_geometry
from oracle import synth, textblock_ref
from pages_ref import postprocess_page_any_size
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
# net-sized (identity letterbox), odd, the reference's example page scaled to the net, exactly 2x the net (INTER_AREA),
# smaller than the net (upscale), a thin strip
SIZES = [(NET, NET), (361, 251), (414, 292), (2 * NET, 2 * NET), (200, 150), (96, 1500)]


def _pages(sizes, seed=500):
    # the synthetic page generator needs at least ~128 px per side: smaller pages are crops of a larger one
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _detector(max_batch):
    return ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=max_batch)


def _same_value(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)
    return type(a) is type(b) and a == b


def _same_blocks(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        dg, dr = vars(g), vars(r)
        assert list(dg) == list(dr)
        for k in dr:
            assert _same_value(dg[k], dr[k]), (k, dg[k], dr[k])


def _same_result(got, ref):
    assert np.array_equal(got[0], ref[0]), int((got[0] != ref[0]).sum())
    assert np.array_equal(got[1], ref[1]), int((got[1] != ref[1]).sum())
    _same_blocks(got[2], ref[2])


@pytest.fixture(scope="module")
def det():
    d = _detector(4)
    yield d
    d.close()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("keep", [False, True])
def test_detect_batch_equals_call(det, mode, keep):
    pages = _pages(SIZES)                       # 6 pages at max_batch 4: a full batch, then a partial one
    got = det.detect_batch([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=keep)
    n_blocks = 0
    for p, g in zip(pages, got):
        ref = det(p.copy(), refine_mode=mode, keep_undetected_mask=keep)
        _same_result(g, ref)
        n_blocks += len(ref[2])
    assert n_blocks > 5


def test_letterbox_kernel_equals_host_letterbox(det):
    # the forward of a batch sees exactly the host letterbox of every page: a net-sized page is copied unchanged
    pages = _pages(SIZES[:4], seed=900)
    eng = det.net
    eng.submit_pages(0, pages, NET, NET)
    eng.collect_pages(0)
    blks, mask, lines = eng.net_outputs()
    boxed = np.stack([letterbox(p, (NET, NET))[0] for p in pages])
    assert np.array_equal(boxed[0], pages[0])
    eng.forward(boxed)
    rb, rm, rl = eng.net_outputs()
    assert np.array_equal(blks, rb) and np.array_equal(mask, rm) and np.array_equal(lines, rl)


def test_batched_page_matches_oracle_at_page_scale(det):
    # oracle chain for a non-net-sized page that never goes through ctd_detect_page: host letterbox -> engine forward ->
    # oracle post-processing at the page's scale, against the batched result for that page, with refine_undetected_mask
    keep = True
    pages = _pages([(1654 * NET // 1024, 1170 * NET // 1024), (NET, NET)], seed=42)
    page = pages[0]
    got = det.detect_batch([p.copy() for p in pages], refine_mode=1, keep_undetected_mask=keep)[0]
    _r, (uw, uh), _dw, _dh = letterbox_geometry(page.shape[:2], (NET, NET))
    eng = det.net
    eng.forward(letterbox(page, (NET, NET))[0][None])
    blks, mask, lines = eng.net_outputs()
    rmask, rref, rblk = postprocess_page_any_size(page.copy(), (NET, NET), (uh, uw), blks[0], mask[0, 0], lines[0],
                                                  textblock_ref.group_output, refine_mode=1, keep_undetected_mask=keep)
    key = lambda b: (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
                     float(b.font_size), int(b.angle))
    assert len(rblk) > 0
    assert [key(a) for a in got[2]] == [key(b) for b in rblk]
    assert np.array_equal(got[0], rmask)
    assert np.array_equal(got[1], rref), int((got[1] != rref).sum())


def test_stream_in_order_and_growing():
    d = _detector(3)
    try:
        # small pages first, then a page several times larger than anything before it: the packed buffers grow while
        # the other slot is still in flight
        sizes = [(120, 90), (NET, NET), (300, 200), (64, 700), (150, 150), (200, 330), (2000, 3000), (361, 251),
                 (NET, NET), (96, 1500), (700, 500)]
        pages = _pages(sizes, seed=3000)
        seen = []

        def feed():
            for p in pages:
                seen.append(p.shape)
                yield p.copy()

        got = list(d.detect_stream(feed(), refine_mode=0, keep_undetected_mask=True))
        assert seen == [p.shape for p in pages]
        assert [g[0].shape for g in got] == [p.shape[:2] for p in pages]
        ref = d.detect_batch([p.copy() for p in pages], refine_mode=0, keep_undetected_mask=True)
        for g, r in zip(got, ref):
            _same_result(g, r)
        for i in (0, 6, 10):
            _same_result(got[i], d(pages[i].copy(), refine_mode=0, keep_undetected_mask=True))
    finally:
        d.close()


def test_model2annotations_through_stream(det, tmp_path):
    import cv2
    src = tmp_path / "src"
    src.mkdir()
    for i, p in enumerate(_pages([(361, 251), (NET, NET), (414, 292), (96, 1500), (300, 420)], seed=77)):
        cv2.imwrite(str(src / ("page%d.png" % i)), p)
    a, b = tmp_path / "stream", tmp_path / "call"
    annotations.model2annotations(None, str(src), str(a), save_json=True, detector=det)
    os.makedirs(b)
    for fp in annotations.find_all_imgs(str(src), abs_path=True):
        img = annotations.imread(fp)
        _m, refined, blks = det(img, refine_mode=ctd_b200.REFINEMASK_ANNOTATION, keep_undetected_mask=True)
        annotations.write_annotations(str(b), os.path.basename(fp), img, refined, blks, True)
    names = sorted(os.listdir(b))
    assert sorted(os.listdir(a)) == names and len(names) >= 15
    match, mismatch, errors = filecmp.cmpfiles(str(a), str(b), names, shallow=False)
    assert not mismatch and not errors


def test_pages_batch_errors(det):
    eng = det.net
    pages = _pages([(300, 200), (200, 300)])
    eng.submit_pages(0, pages, NET, NET)
    with pytest.raises(ctd_b200.CtdError):
        eng.submit_pages(0, pages, NET, NET)            # busy slot
    eng.collect_pages(0)
    with pytest.raises(ctd_b200.CtdError):
        eng.submit_pages(1, _pages([(100, 100)] * 5), NET, NET)     # n > max_batch
    with pytest.raises(ctd_b200.CtdError) as e:
        eng.submit_pages(1, pages, NET, NET - 32)       # net shape not a multiple of 64
    assert "(-4)" in str(e.value)
    with pytest.raises(ctd_b200.CtdError):
        eng.submit_pages(1, pages, 2 * NET, 2 * NET)    # larger than the engine's max shape
    for bad in (np.zeros((50, 60, 3), np.float32), np.zeros((50, 60), np.uint8), np.zeros((50, 60, 4), np.uint8),
                np.zeros((0, 60, 3), np.uint8)):
        with pytest.raises(ValueError):
            det.detect_batch([pages[0], bad])
        with pytest.raises(ValueError):
            list(det.detect_stream([pages[0], bad]))
    # a pre-planned entry with tampered offsets is refused by the library
    ent, ib, rb = binding.pages_plan([p.shape[:2] for p in pages], NET, NET)
    ent[1]["mask_off"] += 256
    buf = np.zeros((ib,), np.uint8)
    out = np.zeros((rb,), np.uint8)
    rc = eng.lib.ctd_submit_pages(eng.h, 1, binding._ptr(ent), 2, NET, NET, binding._ptr(buf), None, 0, 0, 0, 0,
                                  binding._ptr(out))
    assert rc == -1   # CTD_E_INVALID
    # the engine still works after every refusal
    _same_result(det.detect_batch([pages[0]])[0], det(pages[0]))


def test_skip_postproc_engine_refused():
    prog = ctd_b200.compiler.compile_checkpoint(get_checkpoint(0, True))
    eng = ctd_b200.Engine(prog, max_batch=1, max_h=NET, max_w=NET, skip_postproc=True)
    try:
        with pytest.raises(ctd_b200.CtdError):
            eng.submit_pages(0, _pages([(100, 100)]), NET, NET)
    finally:
        eng.close()


def test_results_layout_block_section(det):
    # the block-section offsets the engine reports are the layout the plan and the decoder assume, for any engine shape
    from test_cpu_pages_plan import _section_layout
    sec = _section_layout()
    for lay in (det.net.results_layout(), ctd_b200.Engine(det.program, max_batch=2, max_h=128, max_w=192).results_layout()):
        assert {k: lay[k] for k in sec} == sec
    ent, _ib, _rb = binding.pages_plan([(100, 100), (50, 70)], NET, NET)
    assert int(ent[1]["blocks_off"]) - int(ent[0]["blocks_off"]) == (sec["blocks_stride"] + 255) // 256 * 256


def test_call_between_stream_yields():
    # TextDetector.__call__ (engine stream) while the stream's other batch is still in its refine phase (post stream):
    # each path has its own refine scratch, so both give the page-by-page results
    d = _detector(2)
    try:
        pages = _pages([(700, 500), (520, 760), (NET, NET), (900, 640), (361, 251), (640, 900), (500, 700), (300, 420)],
                       seed=6100)
        others = _pages([(620, 410), (NET, NET), (1000, 700)], seed=6200)
        ref = [d(p.copy(), refine_mode=1, keep_undetected_mask=True) for p in pages]
        ref_o = [d(p.copy(), refine_mode=1, keep_undetected_mask=True) for p in others]
        k = 0
        for i, got in enumerate(d.detect_stream([p.copy() for p in pages], refine_mode=1, keep_undetected_mask=True)):
            _same_result(got, ref[i])
            o = k % len(others)
            _same_result(d(others[o].copy(), refine_mode=1, keep_undetected_mask=True), ref_o[o])
            k += 1
        assert k == len(pages)
    finally:
        d.close()


def test_model2annotations_unreadable_page(tmp_path):
    # the pages read before an unreadable one are written, then the error is raised (as page by page)
    import cv2
    d = _detector(4)
    try:
        src, out = tmp_path / "src", tmp_path / "out"
        src.mkdir()
        for i, p in enumerate(_pages([(361, 251), (NET, NET), (414, 292), (300, 420), (200, 330), (96, 1500)], seed=88)):
            cv2.imwrite(str(src / ("page%d.png" % i)), p)
        (src / "broken.png").write_bytes(b"not an image")
        imglist = annotations.find_all_imgs(str(src), abs_path=True)
        k = [os.path.basename(f) for f in imglist].index("broken.png")
        with pytest.raises(ValueError):
            annotations.model2annotations(None, str(src), str(out), detector=d)
        written = set(os.listdir(out))
        for fp in imglist[:k]:
            name = os.path.basename(fp)
            assert name in written and "mask-" + name in written
            img = annotations.imread(fp)
            _m, refined, _b = d(img, refine_mode=ctd_b200.REFINEMASK_ANNOTATION, keep_undetected_mask=True)
            assert np.array_equal(annotations.imread(str(out / ("mask-" + name)), cv2.IMREAD_GRAYSCALE), refined)
        for fp in imglist[k + 1:]:
            assert os.path.basename(fp) not in written
    finally:
        d.close()
