"""Seeded images for the PNG encoder's tests: every case names the rule of libpng / zlib 1.2.11 it reaches.

`corpus()` gives (name, image) pairs, grey and BGR, made from fixed seeds: the same bytes on every machine, so
tests/golden/png_cv2_sha256.json can pin cv2's files for them."""
import numpy as np

SEED = 20261017
WINDOW_SIZES = [1 << k for k in range(8, 15)]     # 256 .. 16384: where libpng's window and CINFO rules step


def _noise(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


def row_from_filtered(d):
    """a 1-row grey image whose SUB-filtered bytes (after the filter byte) are `d`"""
    return (np.cumsum(np.asarray(d, np.int64)) % 256).astype(np.uint8)[None, :]


def distinct_run(rng, n, first_not=1):
    """n bytes, no two neighbours equal and the first one != first_not: n literal tokens"""
    d = rng.integers(0, 255, n)
    prev = first_not
    for i in range(n):
        if d[i] >= prev:
            d[i] += 1
        prev = d[i]
    return d


def corpus(large=True):
    rng = np.random.default_rng(SEED)
    out = []
    # 1x1, 1xN, Nx1 (an image one pixel wide is written with filter NONE)
    for c in (None, 3):
        sh = (lambda h, w: (h, w) if c is None else (h, w, 3))
        tag = "g" if c is None else "c"
        out += [("one_%s" % tag, _noise(rng, sh(1, 1))),
                ("row8193_%s" % tag, _noise(rng, sh(1, 8193))),
                ("col8193_%s" % tag, _noise(rng, sh(8193, 1)))]
    # filtered sizes around each window / CINFO boundary: S = w + 1 for one grey row; both of libpng's tests
    # (data_size + 262 <= half window, data_size <= half window) step at these sizes
    for B in WINDOW_SIZES:
        for S in sorted({B - 1, B, B + 1, B - 262 - 1, B - 262, B - 262 + 1}):
            if S >= 2:
                out.append(("win%d" % S, _noise(rng, (1, S - 1))))
    out.append(("win16405", _noise(rng, (1, 16404))))
    # constant and all-zero images
    out += [("zeros_64c", np.zeros((64, 64, 3), np.uint8)),
            ("zeros_1000x999", np.zeros((1000, 999), np.uint8)),
            ("const_517x300c", np.full((517, 300, 3), 201, np.uint8))]
    if large:
        out += [("zeros_4096c", np.zeros((4096, 4096, 3), np.uint8)),
                ("const_4096g", np.full((4096, 4096), 77, np.uint8))]
    # runs of length 258 k + {0 .. 4}: a literal, then one run of equal filtered bytes
    for k in (0, 1, 2, 5):
        for e in range(5):
            R = 258 * k + e
            if R < 1:
                continue
            d = np.r_[distinct_run(rng, 7), np.full(R, 0), distinct_run(rng, 5, 0)]
            out.append(("run%d" % R, row_from_filtered(d)))
    # token counts 16383 k and +-1: a row of distinct filtered bytes is 1 + w literal tokens
    for k in (1, 2, 3):
        for e in (-1, 0, 1):
            out.append(("tok%d" % (16383 * k + e), row_from_filtered(distinct_run(rng, 16383 * k + e - 1))))
    # a block spanning more than the 32 KiB window (long zero runs) between literal blocks
    d = np.r_[distinct_run(rng, 16000), np.zeros(70000, np.int64), distinct_run(rng, 20000, 0)]
    out.append(("span_window", row_from_filtered(d)))
    # incompressible data: stored blocks
    out += [("noise_256c", _noise(rng, (256, 256, 3))), ("noise_300x77g", _noise(rng, (300, 77)))]
    if large:
        out.append(("noise_700x900c", _noise(rng, (700, 900, 3))))
    # 2-4 levels: static and dynamic blocks
    for lv in (2, 3, 4):
        out.append(("levels%d_g" % lv, (rng.integers(0, lv, (123, 457)) * (255 // (lv - 1))).astype(np.uint8)))
        out.append(("levels%d_c" % lv, (rng.integers(0, lv, (97, 311, 3)) * 60).astype(np.uint8)))
    out.append(("sparse_c", np.where(rng.random((400, 600, 1)) < 0.01, _noise(rng, (400, 600, 3)), 255)
                .astype(np.uint8)))
    return out


def golden_page():
    """the golden scan decoded as the reference reads it, and a binary mask of it"""
    import os
    import cv2
    here = os.path.dirname(os.path.abspath(__file__))
    page = cv2.imdecode(np.fromfile(os.path.join(here, "golden", "AisazuNihaIrarenai-003.jpg"), np.uint8),
                        cv2.IMREAD_COLOR)
    mask = np.where(cv2.cvtColor(page, cv2.COLOR_BGR2GRAY) < 128, 255, 0).astype(np.uint8)
    return [("golden_page", page), ("golden_mask", mask)]
