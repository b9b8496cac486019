"""-m gpu: refine_mask (csrc/refine_mk.cu) against the oracle, byte for byte, on the cases its 1-bit planes make sharp:
chunks whose pixel count is not a multiple of 32 (tail bits of the last word), windows 31, 32 and 33 pixels wide (row
ends inside, at and past a word), windows of 3 and of 4 candidate rounds in one launch (each round's merge is applied
once, by the next kernel that reads `merged`), and rings whose inside the hole filling fills."""
import cv2
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref

pytestmark = pytest.mark.gpu

CHUNK_PX = 8192   # kRefineChunkPx (csrc/kernels.h)


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=1024, max_w=1024, skip_postproc=True)
    yield e
    e.close()


def oracle(img, mask, windows, mode):
    out = np.zeros_like(mask)
    for x1, y1, x2, y2 in windows:
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        cands = postproc_ref.candidate_masks(np.ascontiguousarray(img[y1:y2, x1:x2]), msk)
        out[y1:y2, x1:x2] |= postproc_ref.merge_masks(cands, msk, mode)
    return out


def blur(m):
    return (cv2.GaussianBlur(m, (0, 0), 1.2) * 255).clip(0, 255).astype(np.uint8)


def chunk_pixels(rw, rh):
    rows_per = max(1, CHUNK_PX // rw)
    if rows_per >= 8:
        rows_per &= ~3
    return [min(rows_per, rh - y0) * rw for y0 in range(0, rh, rows_per)]


def narrow_case(rw):
    """a 600 x 256 page with one window rw wide and 560 high (three chunks) of strokes, some along the window's edges"""
    rng = np.random.default_rng(rw)
    h, w = 600, 256
    img = np.full((h, w, 3), 235, np.uint8)
    img += rng.integers(0, 12, img.shape, dtype=np.uint8)
    m = np.zeros((h, w), np.float32)
    x1, y1 = 64, 20
    for x in (x1, x1 + rw - 1, x1 + rw // 2):
        for y in range(y1 + 4, y1 + 550, 37):
            ln = int(rng.integers(8, 30))
            cv2.line(img, (x, y), (x, y + ln), (12, 12, 12), 1)
            cv2.line(m, (x, y), (x, y + ln), 1.0, 1)
    for y in range(y1 + 10, y1 + 550, 23):
        cv2.line(img, (x1, y), (x1 + rw - 1, y + 5), (12, 12, 12), 2)
        cv2.line(m, (x1, y), (x1 + rw - 1, y + 5), 1.0, 2)
    return img, blur(m), [[x1, y1, x1 + rw, y1 + 560]]


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
@pytest.mark.parametrize("rw", [31, 32, 33])
def test_refine_window_width_around_a_word(eng, rw, mode):
    img, mask, wins = narrow_case(rw)
    px = chunk_pixels(rw, 560)
    assert len(px) == 3 and (rw == 32) == all(p % 32 == 0 for p in px), px
    ref = oracle(img, mask, wins, mode)
    got = eng.refine_mask(img, mask, wins, mode)
    assert ref.any() and np.array_equal(got, ref), int((got != ref).sum())


def ring_case():
    """Two windows in one launch.  Left: rings whose left half is dark and right half light grey on a lighter page, under
    a mask of filled discs (four candidate rounds).  Right: dark strokes of one grey (three rounds)."""
    h, w = 300, 640
    img = np.full((h, w, 3), 250, np.uint8)
    m = np.zeros((h, w), np.float32)
    for (cx, cy, r) in ((110, 150, 70), (260, 150, 30)):
        cv2.ellipse(img, (cx, cy), (r, r), 0, 90, 270, (20, 20, 20), 5)
        cv2.ellipse(img, (cx, cy), (r, r), 0, -90, 90, (190, 190, 190), 5)
        cv2.circle(m, (cx, cy), r + 2, 1.0, -1)
    rng = np.random.default_rng(11)
    for _ in range(10):
        p = (int(rng.integers(360, 600)), int(rng.integers(30, 270)))
        q = (int(rng.integers(360, 600)), int(rng.integers(30, 270)))
        cv2.line(img, p, q, (15, 15, 15), 2)
        cv2.line(m, p, q, 1.0, 2)
    return img, blur(m), [[20, 40, 320, 260], [350, 20, 610, 280]]


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_rings_next_to_a_window_of_fewer_rounds(eng, mode):
    img, mask, wins = ring_case()
    rounds = []
    for x1, y1, x2, y2 in wins:
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        rounds.append(len(postproc_ref.candidate_masks(np.ascontiguousarray(img[y1:y2, x1:x2]), msk)))
    assert rounds == [4, 3], rounds   # the right window skips round 3: its round 2 is merged by that round's kernel
    ref = oracle(img, mask, wins, mode)
    # the hole filling has filled the inside of the small ring (window 0 starts at (20, 40))
    assert ref[140:160, 250:270].all()
    got = eng.refine_mask(img, mask, wins, mode)
    assert np.array_equal(got, ref), int((got != ref).sum())
