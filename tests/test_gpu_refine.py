"""-m gpu: refine_mask (utils/textmask.py:159-169) on the GPU (csrc/refine_mk.cu), bit-exact against the oracle
restatement (which equals the unmodified reference except for the documented stable tie order of np.argsort)."""
import cv2
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref, synth

pytestmark = pytest.mark.gpu

CHUNK_PX = 8192   # kRefineChunkPx (csrc/kernels.h): windows wider than this are cut into row segments


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=1024, max_w=1024, skip_postproc=True)
    yield e
    e.close()


def draw_text(rng, img, m, h_page, w_page):
    """one text block the way the detector's windows see it: glyphs in the page and a stroke mask; returns its box"""
    x0, y0 = int(rng.integers(0, w_page - 112)), int(rng.integers(0, h_page - 92))
    w, h = int(rng.integers(30, 110)), int(rng.integers(20, 90))
    txt = "Ab%d" % rng.integers(0, 99)
    cv2.putText(m, txt, (x0 + 4, y0 + h - 6), cv2.FONT_HERSHEY_SIMPLEX, h / 40, 1.0, 3)
    cv2.putText(img, txt, (x0 + 4, y0 + h - 6), cv2.FONT_HERSHEY_SIMPLEX, h / 40, (10, 10, 10), 2)
    return [x0, y0, min(w_page - 1, x0 + w), min(h_page - 1, y0 + h)]


def blur_mask(m):
    return (cv2.GaussianBlur(m, (0, 0), 1.5) * 255).clip(0, 255).astype(np.uint8)


def make_case(seed, size=512, nblk=10):
    rng = np.random.default_rng(seed)
    img = synth.structured_page(2000 + seed, size, size)
    m = np.zeros((size, size), np.float32)
    wins = [draw_text(rng, img, m, size, size) for _ in range(nblk)]
    return img, blur_mask(m), wins


def oracle_refine_windows(img, mask, windows, mode):
    """postproc_ref.refine_mask on windows that are already expanded (the windows the engine is given)"""
    out = np.zeros_like(mask)
    for x1, y1, x2, y2 in windows:
        im = np.ascontiguousarray(img[y1:y2, x1:x2])
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        out[y1:y2, x1:x2] |= postproc_ref.merge_masks(postproc_ref.candidate_masks(im, msk), msk, mode)
    return out


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
@pytest.mark.parametrize("seed", range(12))
def test_refine_mask_matches_oracle(eng, seed, mode):
    img, mask, wins = make_case(seed)
    ref = postproc_ref.refine_mask(img, mask.copy(), wins, mode)
    ex = [postproc_ref.expand_textwindow(img.shape, w, expand_r=16) for w in wins]
    got = eng.refine_mask(img, mask, ex, mode)
    assert np.array_equal(got, ref), int((got != ref).sum())


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_mask_edge_cases(eng, mode):
    img, mask, _ = make_case(3, 256, 4)
    # window covering the whole page, an empty-mask window, a 1-pixel-high window, no windows at all
    wins = [[0, 0, 255, 255], [200, 200, 240, 240], [10, 10, 60, 11]]
    mask[190:256, 190:256] = 0
    ref = postproc_ref.refine_mask(img, mask.copy(), wins, mode)
    ex = [postproc_ref.expand_textwindow(img.shape, w, expand_r=16) for w in wins]
    assert np.array_equal(eng.refine_mask(img, mask, ex, mode), ref)
    assert not eng.refine_mask(img, mask, np.zeros((0, 4), np.int32), mode).any()


def test_refine_large_windows_match_oracle(eng):
    """a 1024x1024 page with overlapping page-sized windows (many chunks of whole rows per window), in both modes"""
    img, mask, wins = make_case(11, 1024, 30)
    wins += [[0, 0, 1023, 1023], [100, 50, 900, 1000], [0, 300, 1023, 700]]
    ex = [postproc_ref.expand_textwindow(img.shape, w, expand_r=16) for w in wins]
    for mode in (0, 1):
        ref = postproc_ref.refine_mask(img, mask.copy(), wins, mode)
        got = eng.refine_mask(img, mask, ex, mode)
        assert ref.any() and np.array_equal(got, ref), (mode, int((got != ref).sum()))


def make_wide_case():
    """a 160 x 20000 page whose windows are wider than one chunk, with strokes across the row-segment seams; returns
    the page, the mask and the (already expanded) windows"""
    h, w = 160, 20000
    rng = np.random.default_rng(7)
    img = synth.structured_page(2100, h, w)
    m = np.zeros((h, w), np.float32)
    narrow = [postproc_ref.expand_textwindow(img.shape, draw_text(rng, img, m, h, w), expand_r=16) for _ in range(120)]
    wide = [
        [0, 0, w, h],                              # full width: segments of 8192, 8192 and 3616 px
        [100, 10, 100 + CHUNK_PX, 150],            # exactly one chunk wide: whole rows, one row per chunk
        [3000, 5, 3000 + CHUNK_PX + 1, 155],       # a 1-px second segment per row
        [500, 80, 500 + 9000, 81],                 # 1 px high
        [700, 40, 700 + 12000, 42],                # 2 px high
    ]

    def stroke(x, y0, y1, col):
        # white band around the seam at page column x, then strokes that cross it
        img[y0:y1, x - 40:x + 40] = 255
        cv2.line(img, (x - 30, y0 + 5), (x + 30, y0 + 5), col, 3)                           # horizontal bar
        cv2.line(img, (x - 20, y0 + 10), (x - 20 + (y1 - y0 - 20), y1 - 10), col, 1, cv2.LINE_8)   # 1-px diagonal
        cv2.line(m, (x - 30, y0 + 5), (x + 30, y0 + 5), 1.0, 3)
        cv2.line(m, (x - 20, y0 + 10), (x - 20 + (y1 - y0 - 20), y1 - 10), 1.0, 1, cv2.LINE_8)

    for x1, y1, x2, y2 in wide[:3]:
        for s in range(x1 + CHUNK_PX, x2, CHUNK_PX):
            stroke(s, y1 + 2, y2 - 2, (20, 20, 20))
    # a closed ring across the first seam of the full-width window: a hole for the hole-filling round (and area0)
    img[60:140, 8150:8235] = 255
    cv2.circle(img, (CHUNK_PX, 100), 30, (15, 15, 15), 4)
    cv2.circle(m, (CHUNK_PX, 100), 30, 1.0, 4)
    # the 1-px-high window: a run across its seam; the 2-px-high one: a diagonal-only contact across its seam
    s1 = 500 + CHUNK_PX
    img[78:83, s1 - 40:s1 + 40] = 255
    img[80, s1 - 20:s1 + 20] = 20
    m[80, s1 - 20:s1 + 20] = 1.0
    s2 = 700 + CHUNK_PX
    img[38:44, s2 - 40:s2 + 40] = 255
    img[40, s2 - 10:s2] = 20
    img[41, s2:s2 + 10] = 20
    m[40, s2 - 10:s2] = 1.0
    m[41, s2:s2 + 10] = 1.0
    return img, blur_mask(m), wide + narrow


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_wide_windows_match_oracle(eng, mode):
    """windows wider than one chunk (row segments, and their seams) next to ordinary narrow windows in one call"""
    img, mask, wins = make_wide_case()
    ref = oracle_refine_windows(img, mask, wins, mode)
    got = eng.refine_mask(img, mask, wins, mode)
    assert ref.any() and np.array_equal(got, ref), int((got != ref).sum())
