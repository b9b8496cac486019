"""-m gpu: error behaviour and edge inputs of the C ABI / drop-in class (the reference raises Python exceptions at the
same places: bad shapes, oversize batches), plus size-independent properties at the full 1024x1024 page size."""
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import multigpu
from oracle import synth
from util import get_checkpoint

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def prog():
    return ctd_b200.compiler.compile_checkpoint(get_checkpoint(0, True))


def test_shape_and_capacity_errors(prog):
    eng = ctd_b200.Engine(prog, max_batch=2, max_h=256, max_w=256)
    try:
        with pytest.raises(ctd_b200.binding.CtdError, match="multiple of 64"):
            eng.forward(np.zeros((1, 100, 128, 3), np.uint8))
        with pytest.raises(ctd_b200.binding.CtdError, match="multiple of 64"):
            eng.forward(np.zeros((1, 320, 256, 3), np.uint8))       # larger than the reserved workspace
        with pytest.raises(ctd_b200.binding.CtdError, match="max_batch"):
            eng.forward(np.zeros((3, 256, 256, 3), np.uint8))
        with pytest.raises(ctd_b200.binding.CtdError):
            eng.collect(0)                                            # nothing in flight
        eng.forward(np.zeros((2, 128, 192, 3), np.uint8))           # smaller, non-square shapes are fine
        assert eng.mask_u8().shape == (2, 128, 192)
    finally:
        eng.close()


@pytest.mark.parametrize("ph", [0, 32])
def test_profile_forward_rejects_bad_shapes(prog, ph):
    """the per-op profiler checks the page size like the forward does (at least 64, a multiple of 64)"""
    eng = ctd_b200.Engine(prog, max_batch=1, max_h=256, max_w=256)
    try:
        with pytest.raises(ctd_b200.binding.CtdError, match="multiple of 64"):
            eng.profile_forward(np.zeros((1, ph, 256, 3), np.uint8))
    finally:
        eng.close()


@pytest.mark.parametrize("fill", [0, 255])
def test_blank_pages_through_the_detector(fill):
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=256, act="leaky")
    try:
        img = np.full((256, 256, 3), fill, np.uint8)
        mask, mask_refined, blk_list = det(img, keep_undetected_mask=True)
        assert mask.shape == (256, 256) and mask_refined.shape == (256, 256)
        assert mask.dtype == np.uint8 and mask_refined.dtype == np.uint8
        if len(blk_list) == 0:
            assert not mask_refined.any() or mask.max() > 30      # only the undetected-mask pass can add pixels
        for b in blk_list:
            x1, y1, x2, y2 = b.xyxy
            assert 0 <= x1 <= x2 <= 256 and 0 <= y1 <= y2 <= 256
    finally:
        det.close()


def test_letterboxed_page_keeps_reference_shapes():
    """page != net size: aspect-preserving resize + bottom/right padding (imgproc_utils.py:86-117); mask comes back at
    the page size, boxes inside the page (inference.py:164-172)."""
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=256, act="leaky")
    try:
        page = synth.structured_page(5, 360, 250)          # portrait, not a multiple of anything
        mask, mask_refined, blk_list = det(page.copy())
        assert mask.shape == (360, 250) and mask_refined.shape == (360, 250)
        assert len(blk_list) > 0
        for b in blk_list:
            x1, y1, x2, y2 = b.xyxy
            assert x1 <= x2 and y1 <= y2        # (the reference does not clip detector boxes to the page)
            for ln in b.lines:
                a = np.array(ln)
                assert a.shape == (4, 2)
    finally:
        det.close()


def test_full_size_forward_deterministic_batch_invariant_and_arena_layout(prog):
    """1024x1024, batch 3 vs batch 1: bit-identical result arenas run to run, and page k of a batch equals the same page
    processed alone (pages are independent, inference.py:141-178)."""
    h = w = 1024
    pages = np.stack([synth.structured_page(1000 + i, h, w) for i in range(3)])
    eng = ctd_b200.Engine(prog, max_batch=3, max_h=h, max_w=w)
    try:
        def snapshot(pg):
            eng.forward(pg)
            boxes, scores = eng.text_lines()
            return eng.mask_u8().copy(), eng.detections(), boxes, scores, eng.db_components(want_labels=False)[0].copy()
        a = snapshot(pages)
        b = snapshot(pages)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[4], b[4])
        for i in range(3):
            assert np.array_equal(a[1][i], b[1][i]) and np.array_equal(a[2][i], b[2][i]) and np.array_equal(a[3][i], b[3][i])
        one = snapshot(pages[1:2])
        assert np.array_equal(one[0][0], a[0][1]) and np.array_equal(one[4][0], a[4][1])
        assert np.array_equal(one[1][0], a[1][1]) and np.array_equal(one[2][0], a[2][1]) and np.array_equal(one[3][0], a[3][1])
        # structure of the result: counts within the reference's caps, scores in [0,1], boxes inside the page
        for i in range(3):
            assert len(a[1][i]) <= 300 and len(a[2][i]) <= 1000
            assert np.all((a[3][i] >= 0) & (a[3][i] <= 1))
            assert a[2][i].min(initial=0) >= 0 and a[2][i].max(initial=0) <= 1024
        assert multigpu.arena_layout(3, h, w)["phase_a_bytes"] == eng.results_layout()["phase_a_bytes"]
    finally:
        eng.close()


RESIZE_CASES = [((360, 250), (178, 256)), ((1654, 1170), (724, 1024)), ((724, 1024), (1170, 1654)), ((100, 100), (50, 50)),
                ((100, 100), (200, 200)), ((77, 33), (100, 211)), ((512, 512), (511, 513)), ((17, 5), (3, 9)),
                ((2, 2), (7, 5)), ((1, 9), (4, 4)), ((9, 1), (1, 30)), ((640, 480), (320, 480)), ((64, 64), (64, 64))]


@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda c: "%dx%d_to_%dx%d" % (c[0][0], c[0][1], c[1][1], c[1][0]))
@pytest.mark.parametrize("channels", [1, 3])
def test_gpu_resize_is_cv2_exact(prog, case, channels):
    """ctd_resize_linear_u8 against the oracle (itself pinned against cv2 in tests/test_cpu_resize.py) and, where the
    box has OpenCV, against cv2.resize directly: bit-exact."""
    from oracle.resize_ref import resize_linear_u8
    (sh, sw), (dw, dh) = case
    rng = np.random.default_rng(sh * 131 + sw * 7 + dw)
    src = rng.integers(0, 256, (sh, sw, channels), dtype=np.uint8)
    if channels == 1:
        src = src[:, :, 0]
    eng = ctd_b200.Engine(prog, max_batch=1, max_h=64, max_w=64)
    try:
        got = eng.resize_linear_u8(src, (dw, dh))
    finally:
        eng.close()
    assert np.array_equal(got, resize_linear_u8(src, (dw, dh)))
    try:
        import cv2
    except ImportError:
        return
    assert np.array_equal(got, cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR))


def test_gpu_letterbox_equals_host_letterbox():
    """TextDetector on a page that is not net-sized: the GPU letterbox + mask back-projection must reproduce the
    host path (reference `letterbox` + `cv2.resize` of the cropped mask) bit for bit."""
    import cv2
    from ctd_b200 import inference
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=256, act="leaky")
    try:
        for shape in [(361, 251), (200, 300), (512, 512)]:
            page = synth.structured_page(11, shape[0], shape[1])
            mask, mask_refined, blk_list = det(page.copy())
            im_in, _ratio, (dw, dh) = inference.letterbox(page, (256, 256))
            det.net.forward(im_in[None])
            m = det.net.mask_u8()[0][: 256 - dh, : 256 - dw]
            want = cv2.resize(m, (shape[1], shape[0]), interpolation=cv2.INTER_LINEAR)
            assert mask.shape == shape and np.array_equal(mask, want), shape
            assert mask_refined.shape == shape
    finally:
        det.close()


def test_model2annotations_writes_the_reference_files(tmp_path):
    """`model2annotations` (inference.py:19-70) end to end on the GPU detector: per page <name>.txt (YOLO), line-<name>.txt,
    <name>.json, <name>.png, mask-<name>.png; the file FORMATS are pinned byte-for-byte against the reference's writer
    in tests/test_cpu_annotations.py."""
    import json
    import cv2
    from ctd_b200 import annotations as ann
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    for i, shape in enumerate([(256, 256), (300, 212)]):
        cv2.imwrite(str(src / ("page%d.jpg" % i)), synth.structured_page(20 + i, shape[0], shape[1]))
    (src / "notes.txt").write_text("not an image")
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=256, act="leaky")
    try:
        ann.model2annotations(None, str(src), str(dst), save_json=True, detector=det)
    finally:
        det.close()
    names = sorted(p.name for p in dst.iterdir())
    for i in range(2):
        for f in ("page%d.txt", "page%d.json", "page%d.png", "mask-page%d.png"):
            assert f % i in names, (f % i, names)
        blks = json.loads((dst / ("page%d.json" % i)).read_text())
        labels = (dst / ("page%d.txt" % i)).read_text()
        assert len(blks) == (len(labels.split("\n")) if labels else 0)
        n_lines = sum(len(b["lines"]) for b in blks)
        if n_lines:
            rows = (dst / ("line-page%d.txt" % i)).read_text().strip().split("\n")
            assert len(rows) == n_lines and all(len(r.split()) == 8 for r in rows)
        m = cv2.imread(str(dst / ("mask-page%d.png" % i)), cv2.IMREAD_GRAYSCALE)
        assert m.shape == cv2.imread(str(dst / ("page%d.png" % i))).shape[:2]
    assert not any(n.startswith("notes") for n in names)


def test_gpu_resize_equals_committed_cv2_goldens(prog):
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_cv2.npz"))
    eng = ctd_b200.Engine(prog, max_batch=1, max_h=64, max_w=64)
    try:
        for k in g.files:
            if k.startswith("src_"):
                want = g["dst_" + k[4:]]
                assert np.array_equal(eng.resize_linear_u8(g[k], (want.shape[1], want.shape[0])), want), k
    finally:
        eng.close()
