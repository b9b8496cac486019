"""-m gpu: refine_mask (csrc/refine_mk.cu) against the oracle, byte for byte, on the cases that its front end (the
per-window histograms, xor sums and candidate order) and its run labelling make sharp.  Front end: windows at every
x1 mod 16 with widths off multiples of 4, a window of 40 chunks, overlapping windows, row segments, 1, 2 and 3 colours,
a winning negative polarity, exact ties (negative against positive, a colour against the Otsu candidate).  Labelling,
where a run that crosses word seams is one forest node: dense planes with runs over many words, runs that end at bit 31
and rows that start at bit 0 right after a foreground bit 31, and hole fillings over a mostly foreground inverse."""
import cv2
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref, synth

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


def candidates(img, mask, win):
    x1, y1, x2, y2 = win
    return postproc_ref.candidate_masks(np.ascontiguousarray(img[y1:y2, x1:x2]), np.ascontiguousarray(mask[y1:y2, x1:x2]))


def oracle(img, mask, windows, mode):
    out = np.zeros_like(mask)
    for x1, y1, x2, y2 in windows:
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        out[y1:y2, x1:x2] |= postproc_ref.merge_masks(candidates(img, mask, [x1, y1, x2, y2]), msk, mode)
    return out


def n_chunks(rw, rh):
    rows_per = max(1, CHUNK_PX // rw)
    if rows_per >= 8:
        rows_per &= ~3
    return -(-rh // rows_per) * -(-rw // CHUNK_PX)


def strokes(rng, img, m, x1, y1, x2, y2, n, col=(15, 15, 15)):
    for _ in range(n):
        p = (int(rng.integers(x1, x2)), int(rng.integers(y1, y2)))
        q = (int(rng.integers(x1, x2)), int(rng.integers(y1, y2)))
        t = int(rng.integers(1, 4))
        cv2.line(img, p, q, col, t)
        cv2.line(m, p, q, 1.0, t)


def blur(m):
    return (cv2.GaussianBlur(m, (0, 0), 1.2) * 255).clip(0, 255).astype(np.uint8)


def check(eng, img, mask, wins, mode):
    ref = oracle(img, mask, wins, mode)
    got = eng.refine_mask(img, mask, wins, mode)
    assert ref.any() and np.array_equal(got, ref), int((got != ref).sum())


def alignment_case():
    """a 1024^2 page: 16 windows with x1 = 0..15 mod 16 and widths that are not multiples of 4, with 1, 2 or 3 stroke
    colours; a 1000 x 320 window of 40 chunks; and a window overlapping it and two of the small ones"""
    rng = np.random.default_rng(7)
    h = w = 1024
    img = synth.structured_page(4000, h, w)
    m = np.zeros((h, w), np.float32)
    wins = []
    for j in range(16):
        x1, y1 = 64 * (j % 8) + j, 20 + 150 * (j // 8)
        rw, rh = 41 + 2 * j, 110 + 3 * j
        img[y1:y1 + rh, x1:x1 + rw] = 240 - 3 * j
        cols = ([20], [20, 110], [20, 80, 160])[j % 3]
        for k, cv in enumerate(cols):
            strokes(rng, img, m, x1, y1 + k * rh // len(cols), x1 + rw, y1 + (k + 1) * rh // len(cols), 4, (cv, cv, cv))
        wins.append([x1, y1, x1 + rw, y1 + rh])
        assert x1 % 16 == j and rw % 4 != 0
    x1, y1 = 11, 380
    strokes(rng, img, m, x1, y1, x1 + 1000, y1 + 320, 120)
    cv2.circle(img, (500, 540), 60, (20, 20, 20), 4)
    cv2.circle(m, (500, 540), 60, 1.0, 4)
    wins.append([x1, y1, x1 + 1000, y1 + 320])
    assert n_chunks(1000, 320) == 40
    wins.append([300, 200, 640, 460])   # overlaps the 40-chunk window and windows of the second row
    return img, blur(m), wins


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_frontend_alignment_and_many_chunks(eng, mode):
    img, mask, wins = alignment_case()
    rounds = {len(candidates(img, mask, wn)) for wn in wins}
    assert rounds == {2, 3, 4}, rounds
    check(eng, img, mask, wins, mode)


def otsu_sums(img, mask, win):
    """(positive, negative) xor sums of the three Otsu candidates of a window"""
    x1, y1, x2, y2 = win
    msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
    out = []
    for c in range(3):
        _, t = cv2.threshold(np.ascontiguousarray(img[y1:y2, x1:x2, c]), 1, 255, cv2.THRESH_OTSU + cv2.THRESH_BINARY)
        out.append((int(cv2.bitwise_xor(t, msk).sum()), int(cv2.bitwise_xor(255 - t, msk).sum())))
    return out


def tie_case():
    """Window 0: grey quadrants, the left half 200 and the right half 50, under a hard mask over the top half: every
    candidate disagrees with the mask on exactly half the pixels (negative == positive), and the colour candidate of 200
    is the Otsu plane (a colour and the Otsu candidate tie).  Window 1: dark strokes on a light page, whose Otsu
    candidates win with the negative polarity.  Window 2: light strokes on a dark page."""
    h, w = 200, 400
    img = np.full((h, w, 3), 235, np.uint8)
    mask = np.zeros((h, w), np.uint8)
    img[10:74, 10:42] = 200
    img[10:74, 42:74] = 50
    mask[10:42, 10:74] = 255
    rng = np.random.default_rng(3)
    m = np.zeros((h, w), np.float32)
    strokes(rng, img, m, 100, 10, 240, 180, 14)
    img[10:190, 260:390] = 25
    strokes(rng, img, m, 260, 10, 390, 180, 14, (225, 225, 225))
    mask = np.maximum(mask, blur(m))
    return img, mask, [[10, 10, 74, 74], [100, 10, 240, 180], [260, 10, 390, 190]]


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_frontend_polarity_and_ties(eng, mode):
    img, mask, wins = tie_case()
    assert all(p == n for p, n in otsu_sums(img, mask, wins[0]))               # negative == positive: positive wins
    sums = [s for _, s in candidates(img, mask, wins[0])]
    assert sums[-1] in sums[:-1], sums                                          # a colour ties with the Otsu candidate
    assert all(n < p for p, n in otsu_sums(img, mask, wins[1]))                # the negative wins
    check(eng, img, mask, wins, mode)


def dense_case():
    """Dense candidate planes: windows 64, 96 and 160 wide (rows of whole words, so a row ends at bit 31 and the next
    starts at bit 0) that are dark and under the mask almost everywhere, with small light holes; full-row bands and
    runs ending at columns 31 and 63.  And a window of sparse thin strokes and a ring: its hole filling labels a mostly
    foreground inverse."""
    rng = np.random.default_rng(9)
    h, w = 420, 700
    img = np.full((h, w, 3), 240, np.uint8)
    m = np.zeros((h, w), np.float32)
    wins = []
    for x1, rw in ((16, 64), (96, 96), (224, 160)):
        y1, rh = 10, 400
        img[y1:y1 + rh, x1:x1 + rw] = 30
        m[y1:y1 + rh, x1:x1 + rw] = 1.0
        for _ in range(40):
            hx, hy = int(rng.integers(x1, x1 + rw - 6)), int(rng.integers(y1, y1 + rh - 6))
            s = int(rng.integers(2, 6))
            img[hy:hy + s, hx:hx + s] = 235
            m[hy:hy + s, hx:hx + s] = 0.0
        for yb in range(y1 + 40, y1 + rh - 20, 60):   # light bands with dark runs ending at columns 31 and 63
            img[yb:yb + 8, x1:x1 + rw] = 235
            m[yb:yb + 8, x1:x1 + rw] = 0.0
            img[yb + 2:yb + 6, x1 + 5:x1 + 32] = 30
            m[yb + 2:yb + 6, x1 + 5:x1 + 32] = 1.0
            img[yb + 2:yb + 6, x1 + 40:x1 + 64] = 30
            m[yb + 2:yb + 6, x1 + 40:x1 + 64] = 1.0
        wins.append([x1, y1, x1 + rw, y1 + rh])
    x1, y1 = 420, 20
    strokes(rng, img, m, x1, y1, x1 + 260, y1 + 380, 6)
    cv2.circle(img, (550, 200), 50, (20, 20, 20), 2)
    cv2.circle(m, (550, 200), 50, 1.0, 2)
    wins.append([x1, y1, x1 + 260, y1 + 380])
    return img, blur(m), wins


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_frontend_dense_planes(eng, mode):
    img, mask, wins = dense_case()
    for wn in wins[:3]:
        t = candidates(img, mask, wn)[0][0]
        assert (t > 0).mean() > 0.7, (wn, float((t > 0).mean()))   # the first round's plane is dense
    check(eng, img, mask, wins, mode)


def segment_case():
    """a 40 x 9000 page: a window 8996 px wide (two row segments per row, x1 = 3) and a narrow window overlapping it;
    long dark bands whose runs cross the segment seam and hundreds of words"""
    h, w = 40, 9000
    rng = np.random.default_rng(13)
    img = np.full((h, w, 3), 230, np.uint8)
    img += rng.integers(0, 20, img.shape, dtype=np.uint8)
    m = np.zeros((h, w), np.float32)
    img[8:14, 100:8900] = 20
    m[8:14, 100:8900] = 1.0
    img[20:22, 3000:8999] = 20
    m[20:22, 3000:8999] = 1.0
    for _ in range(30):
        x = int(rng.integers(0, w - 60))
        strokes(rng, img, m, x, 0, x + 60, h, 2)
    return img, blur(m), [[3, 2, 8999, 38], [8150, 0, 8250, 40]]


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_frontend_row_segments(eng, mode):
    img, mask, wins = segment_case()
    assert wins[0][2] - wins[0][0] > CHUNK_PX
    check(eng, img, mask, wins, mode)
