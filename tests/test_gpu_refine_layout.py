"""-m gpu: refine_mask (csrc/refine_mk.cu) against the oracle, byte for byte, on windows that exercise the labelling's
layout: 16-bit chunk-local labels (a pixel's root is its chunk's start + its label), per-chunk root lists, chunks
that start off a 32-pixel boundary, row segments, components spread over several chunks, rounds that windows skip,
and windows too large for a 16-bit window-global index."""
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


def oracle_refine_windows(img, mask, windows, mode, rounds=None):
    """postproc_ref.refine_mask on windows that are already expanded (the windows the engine is given); `rounds`
    (a list) receives each window's number of candidate masks, i.e. the labelling rounds before the hole filling"""
    out = np.zeros_like(mask)
    for x1, y1, x2, y2 in windows:
        im = np.ascontiguousarray(img[y1:y2, x1:x2])
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        cands = postproc_ref.candidate_masks(im, msk)
        if rounds is not None:
            rounds.append(len(cands))
        out[y1:y2, x1:x2] |= postproc_ref.merge_masks(cands, msk, mode)
    return out


def chunks_of(rw, rh):
    """(chunk starts as window pixel indices) of the host's cut (RefineJob::add, csrc/pipeline.cu)"""
    rows_per = max(1, CHUNK_PX // rw)
    if rows_per >= 8:
        rows_per &= ~3
    return [y0 * rw + x0 for y0 in range(0, rh, rows_per) for x0 in range(0, rw, CHUNK_PX)]


def strokes(rng, img, m, x1, y1, x2, y2, n, col=(15, 15, 15)):
    for _ in range(n):
        p = (int(rng.integers(x1, x2)), int(rng.integers(y1, y2)))
        q = (int(rng.integers(x1, x2)), int(rng.integers(y1, y2)))
        t = int(rng.integers(1, 4))
        cv2.line(img, p, q, col, t)
        cv2.line(m, p, q, 1.0, t)


def blur(m):
    return (cv2.GaussianBlur(m, (0, 0), 1.2) * 255).clip(0, 255).astype(np.uint8)


def page_case(seed):
    """a 1024^2 page: narrow multi-chunk windows whose chunk starts are off 32-px boundaries, components across 3+
    chunks, single-chunk windows, overlapping windows, one window over 65 535 pixels, and windows of 1, 2 and 3
    dominant colours, so that windows have 2, 3 and 4 candidate masks and skip rounds"""
    rng = np.random.default_rng(seed)
    h = w = 1024
    img = synth.structured_page(3000 + seed, h, w)
    m = np.zeros((h, w), np.float32)
    wins = []
    # 101 px wide: 80-row chunks of 8080 px, whose starts are not multiples of 32; a vertical stroke spans 5 chunks
    x1, y1 = 20, 20
    img[y1:y1 + 420, x1:x1 + 101] = 240
    cv2.line(img, (x1 + 50, y1 + 5), (x1 + 50, y1 + 410), (10, 10, 10), 3)
    cv2.line(m, (x1 + 50, y1 + 5), (x1 + 50, y1 + 410), 1.0, 3)
    strokes(rng, img, m, x1, y1, x1 + 101, y1 + 420, 12)
    wins.append([x1, y1, x1 + 101, y1 + 420])
    assert any(s % 32 for s in chunks_of(101, 420)) and len(chunks_of(101, 420)) >= 3
    # 333 px wide (24 rows per chunk, 7992 px), a ring across several chunks: a hole for the hole-filling round
    x1, y1 = 150, 20
    img[y1:y1 + 300, x1:x1 + 333] = 230
    cv2.circle(img, (x1 + 160, y1 + 150), 100, (20, 20, 20), 5)
    cv2.circle(m, (x1 + 160, y1 + 150), 100, 1.0, 5)
    strokes(rng, img, m, x1, y1, x1 + 333, y1 + 300, 20)
    wins.append([x1, y1, x1 + 333, y1 + 300])
    # over 65 535 pixels (420 x 400 = 168 000), overlapping the previous window
    x1, y1 = 400, 100
    strokes(rng, img, m, x1, y1, x1 + 420, y1 + 400, 60)
    wins.append([x1, y1, x1 + 420, y1 + 400])
    wins.append([300, 250, 600, 450])
    # windows of 1, 2 and 3 grey levels under the mask: 1, 2 or 3 top colours -> 2, 3 or 4 rounds
    for k, cols in enumerate(([20], [20, 120], [20, 90, 170])):
        x1, y1 = 40 + 300 * k, 600
        img[y1:y1 + 120, x1:x1 + 200] = 250
        for j, cv in enumerate(cols):
            strokes(rng, img, m, x1 + 60 * j, y1, x1 + 60 * j + 60, y1 + 120, 6, (cv, cv, cv))
        wins.append([x1, y1, x1 + 200, y1 + 120])
    # small single-chunk windows
    for _ in range(12):
        x1, y1 = int(rng.integers(0, w - 80)), int(rng.integers(760, h - 60))
        strokes(rng, img, m, x1, y1, x1 + 70, y1 + 50, 3)
        wins.append([x1, y1, x1 + int(rng.integers(20, 80)), y1 + int(rng.integers(10, 60))])
    return img, blur(m), wins


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
@pytest.mark.parametrize("seed", range(3))
def test_refine_layout_page(eng, seed, mode):
    img, mask, wins = page_case(seed)
    rounds = []
    ref = oracle_refine_windows(img, mask, wins, mode, rounds)
    # the batch holds windows that run 2, 3 and 4 of the 4 candidate rounds, so rounds 2 and 3 are skipped by some
    # windows and not by others (a window always has the Otsu candidate and at least one top colour: never fewer than 2)
    assert set(rounds) == {2, 3, 4}, rounds
    got = eng.refine_mask(img, mask, wins, mode)
    assert ref.any() and np.array_equal(got, ref), int((got != ref).sum())


def wide_case():
    """a 48 x 17000 page: a window of exactly 8192 columns (one row per chunk), wider ones cut into row segments,
    with strokes and a ring across the segment seams"""
    h, w = 48, 17000
    rng = np.random.default_rng(5)
    img = synth.structured_page(3100, h, w)
    m = np.zeros((h, w), np.float32)
    wins = [[0, 0, w, h], [200, 4, 200 + CHUNK_PX, 44], [1000, 2, 1000 + CHUNK_PX + 33, 46]]
    for s in (CHUNK_PX, 2 * CHUNK_PX, 200 + CHUNK_PX // 2, 1000 + CHUNK_PX):
        img[4:44, s - 40:s + 40] = 245
        cv2.line(img, (s - 30, 10), (s + 30, 10), (15, 15, 15), 3)
        cv2.line(m, (s - 30, 10), (s + 30, 10), 1.0, 3)
        cv2.line(img, (s - 15, 15), (s + 15, 40), (15, 15, 15), 1)
        cv2.line(m, (s - 15, 15), (s + 15, 40), 1.0, 1)
        cv2.circle(img, (s, 28), 10, (20, 20, 20), 2)
        cv2.circle(m, (s, 28), 10, 1.0, 2)
    for _ in range(40):
        x = int(rng.integers(0, w - 60))
        strokes(rng, img, m, x, 0, x + 60, h, 2)
    return img, blur(m), wins


@pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])
def test_refine_layout_row_segments(eng, mode):
    img, mask, wins = wide_case()
    ref = oracle_refine_windows(img, mask, wins, mode)
    got = eng.refine_mask(img, mask, wins, mode)
    assert ref.any() and np.array_equal(got, ref), int((got != ref).sum())
