"""Window shapes for refine_mask (csrc/refine_mk.cu) and the content that makes them sharp, shared by
tests/test_gpu_refine_shapes.py (the engine against the oracle) and tests/test_cpu_refine_shapes.py (the oracle against
the unmodified reference).  Every case is (img u8 [H,W,3], mask u8 [H,W], windows): the windows are already expanded
(what the engine is given; each tiny window is also a block whose expand_textwindow padding rounds to 0).  Grey levels
are built directly: the candidates a window gets follow from them, not from glyph rendering."""
import cv2
import numpy as np

from oracle import postproc_ref

CHUNK_PX = 8192   # kRefineChunkPx (csrc/kernels.h)
LIGHT, DARK = 230, 20
# grey levels of the noise windows: no three of them are evenly spaced, so that no window with equal counts has two
# Otsu thresholds in different gaps at exactly the same between-class variance
LEVELS = (20, 75, 180, 235)


def rows_per_chunk(rw):
    """refine_rows_per_chunk (csrc/kernels.h)"""
    q = CHUNK_PX // rw
    return q & ~3 if q >= 8 else max(q, 1)


def oracle_refine_windows(img, mask, windows, mode):
    """postproc_ref.refine_mask on windows that are already expanded (the windows the engine is given)"""
    out = np.zeros_like(mask)
    for x1, y1, x2, y2 in windows:
        im = np.ascontiguousarray(img[y1:y2, x1:x2])
        msk = np.ascontiguousarray(mask[y1:y2, x1:x2])
        out[y1:y2, x1:x2] |= postproc_ref.merge_masks(postproc_ref.candidate_masks(im, msk), msk, mode)
    return out


def _dense(h, w):
    """a page of dark pixels under mask 255: any read outside a window changes its erosions, dilation or labels"""
    return np.full((h, w, 3), DARK, np.uint8), np.full((h, w), 255, np.uint8)


# ---- tiny windows -------------------------------------------------------------------------------------------------
TINY = (1, 2, 3, 4, 5, 7)
# offsets of the window's pixels from its first one: single pixel, 2-pixel components in the four orientations
# (horizontal, vertical, diagonal, anti-diagonal) and the four 3-pixel L shapes
SHAPES = {"px": (), "h": ((0, 1),), "v": ((1, 0),), "d": ((1, 1),), "a": ((1, -1),),
          "L0": ((0, 1), (1, 0)), "L1": ((0, 1), (1, 1)), "L2": ((1, 0), (1, 1)), "L3": ((1, 0), (1, -1))}
TINY_COLS = 8        # windows per row: x1 = 0, x1 = 0, 1, 30, 31 (mod 32), ... and x2 = W - 1
TINY_W = 64 * TINY_COLS


def tiny_contents(rw, rh):
    """(shape name, pixels) of every shape at every position where it fits a rw x rh window"""
    out = []
    for y in range(rh):
        for x in range(rw):
            for name, d in SHAPES.items():
                pts = [(y, x)] + [(y + dy, x + dx) for dy, dx in d]
                if all(0 <= py < rh and 0 <= px < rw for py, px in pts):
                    out.append((name, pts))
    return out


def tiny_case(rw, rh, seed=0):
    """One page of rw x rh windows, one per (shape, position) of tiny_contents, in rows of TINY_COLS: the first column
    at the page's left edge, the last against the clamped right edge (x2 = W - 1, as expand_textwindow makes it), the
    others at x1 = 0, 1, 30, 31, 0, 1 (mod 32); the first row at the top edge, the last against the clamped bottom edge.
    A window is light with the shape dark; its mask is 255 on the shape's 3 x 3 neighbourhood (the shape is the positive
    candidate and predicted, so the w*h < 3 rule decides whether it merges), on the shape only, or random 0 / 255, in
    turn.  Around the windows: dark pixels under mask 255."""
    rng = np.random.default_rng(1000 * rw + 10 * rh + seed)
    contents = tiny_contents(rw, rh)
    nrows = -(-len(contents) // TINY_COLS)
    h, w = 10 * nrows + 2, TINY_W
    img, mask = _dense(h, w)
    offs = (None, 0, 1, 30, 31, 0, 1, None)
    wins = []
    for i, (_name, pts) in enumerate(contents):
        r, c = divmod(i, TINY_COLS)
        x1 = 0 if c == 0 else (w - 1 - rw if c == TINY_COLS - 1 else 64 * c + offs[c])
        y1 = 0 if r == 0 else (h - 1 - rh if r == nrows - 1 else 10 * r)
        img[y1:y1 + rh, x1:x1 + rw] = LIGHT
        kind = i % 3
        mask[y1:y1 + rh, x1:x1 + rw] = 0 if kind < 2 else rng.integers(0, 2, (rh, rw)).astype(np.uint8) * 255
        for py, px in pts:
            img[y1 + py, x1 + px] = DARK
            if kind == 0:
                mask[y1 + max(py - 1, 0):y1 + min(py + 2, rh), x1 + max(px - 1, 0):x1 + min(px + 2, rw)] = 255
            mask[y1 + py, x1 + px] = 255
        wins.append([x1, y1, x1 + rw, y1 + rh])
    return img, mask, wins


def two_wide_case():
    """A 2 x 26 component (area 52 > 50, the smallest refine_undetected_mask keeps) has expand_textwindow padding
    round(8 / 16) = 0: its window is 2 px wide.  Light windows of 2 x 26 and 2 x 20 with anti-diagonal pairs
    (r, 1)-(r+1, 0) of dark pixels (2 x 2 boxes, which the w*h < 3 rule keeps) and, for contrast, horizontal and
    vertical pairs (1 x 2 and 2 x 1 boxes, which it skips), each under a band of mask 255 from the row above it to
    the third row below its first: the pair is the positive candidate and predicted, so it merges unless skipped."""
    h, w = 40, 64
    img, mask = _dense(h, w)
    wins = []
    for x1, rh, pairs in ((3, 26, (((2, 1), (3, 0)), ((9, 1), (10, 0)), ((20, 0), (20, 1)))),
                          (10, 20, (((0, 1), (1, 0)), ((18, 1), (19, 0)), ((8, 0), (9, 0)))),
                          (33, 26, (((5, 1), (6, 0)),)),
                          (61, 26, (((12, 1), (13, 0)),))):      # x2 = W - 1
        y1 = 4
        img[y1:y1 + rh, x1:x1 + 2] = LIGHT
        mask[y1:y1 + rh, x1:x1 + 2] = 0
        for pair in pairs:
            r = pair[0][0]
            mask[y1 + max(r - 1, 0):y1 + min(r + 4, rh), x1:x1 + 2] = 255
            for py, px in pair:
                img[y1 + py, x1 + px] = DARK
        wins.append([x1, y1, x1 + 2, y1 + rh])
    return img, mask, wins


# ---- rows per chunk -----------------------------------------------------------------------------------------------
# widths on both sides of every change of refine_rows_per_chunk from 8 rows down to 1, and the widest whole-row window
SEAM_ROWS = {1023: 8, 1024: 8, 1025: 7, 1170: 7, 1171: 6, 1365: 6, 1366: 5, 1638: 5, 1639: 4, 2048: 4, 2049: 3,
             2730: 3, 2731: 2, 4096: 2, 4097: 1, 8191: 1}


def _seam_window(img, m, x1, y1, rw, rh):
    """strokes at every chunk seam of a rw x rh window at (x1, y1): vertical strokes across it, diagonal-only contacts
    at both row ends and inside the row, runs across 32-pixel word boundaries in the rows on both sides, and a ring
    from the row above the first seam to the row below the second (a hole for the hole filling)"""
    rp = rows_per_chunk(rw)

    def put(y, x0, x1_, v=1.0):
        if 0 <= y < rh:
            img[y1 + y, x1 + x0:x1 + x1_] = DARK
            m[y1 + y, x1 + x0:x1 + x1_] = v

    for s in range(rp, rh, rp):
        for xs, t in ((33, 1), (64, 2), (95, 1), (rw // 2, 3), (rw // 2 + 31, 1), (rw - 40, 2)):
            for y in range(s - 2, s + 2):
                put(y, xs, xs + t)
        for (ya, xa), (yb, xb) in (((s - 1, 0), (s, 1)), ((s - 1, rw - 1), (s, rw - 2)), ((s - 1, 200), (s, 201)),
                                   ((s - 1, 301), (s, 300))):
            put(ya, xa, xa + 1)
            put(yb, xb, xb + 1)
        for k in range(20, 25):
            put(s - 1, 32 * k - 4, 32 * k + 4)
            put(s, 32 * k + 2, 32 * k + 9)
        put(s, 700, 800)
    s1, s2 = rp, 2 * rp
    for y in range(s1 - 1, min(s2 + 1, rh - 1) + 1):
        if y in (s1 - 1, min(s2 + 1, rh - 1)):
            put(y, 400, 441)
        else:
            put(y, 400, 401)
            put(y, 440, 441)


def seam_case():
    """one window of every SEAM_ROWS width, 3 chunks and a partial one high, stacked on one 8231-px-wide page (one
    launch), light with the strokes of _seam_window under a blurred stroke mask, and one window overlapping two"""
    rng = np.random.default_rng(5)
    w = 8191 + 40
    rhs = {rw: 3 * rp + 2 for rw, rp in SEAM_ROWS.items()}
    h = sum(rh + 6 for rh in rhs.values()) + 4
    img = np.full((h, w, 3), LIGHT, np.uint8)
    img += rng.integers(0, 8, img.shape, dtype=np.uint8)
    m = np.zeros((h, w), np.float32)
    wins = []
    y1 = 3
    for i, (rw, rh) in enumerate(rhs.items()):
        x1 = (7 * i) % (w - rw + 1)
        _seam_window(img, m, x1, y1, rw, rh)
        wins.append([x1, y1, x1 + rw, y1 + rh])
        y1 += rh + 6
    wins.append([500, wins[1][1] + 3, 2600, wins[2][3] - 2])
    mask = (cv2.GaussianBlur(m, (0, 0), 1.0) * 255).clip(0, 255).astype(np.uint8)
    return img, mask, wins


# ---- dense noise --------------------------------------------------------------------------------------------------
def noise_fill(rng, img, mask, x1, y1, rw, rh):
    """per-pixel grey from 2 - 4 of LEVELS, mask of random blobs plus salt and pepper: thousands of 1 - 3 pixel
    components in every candidate and in the hole filling"""
    lv = rng.choice(LEVELS, int(rng.integers(2, 5)), replace=False)
    img[y1:y1 + rh, x1:x1 + rw] = lv[rng.integers(0, len(lv), (rh, rw))][..., None]
    mk = np.zeros((rh, rw), np.uint8)
    for _ in range(int(rng.integers(1, 2 + rw * rh // 200))):
        c = (int(rng.integers(0, rw)), int(rng.integers(0, rh)))
        cv2.ellipse(mk, c, (int(rng.integers(1, 8)), int(rng.integers(1, 6))), float(rng.uniform(0, 180)), 0, 360,
                    int(rng.integers(100, 256)), -1)
    salt = rng.random((rh, rw))
    mk[salt < 0.08] = 255
    mk[salt > 0.95] = 0
    mask[y1:y1 + rh, x1:x1 + rw] = mk


def _tie_window(img, mask, x1, y1):
    """31 x 20: a dark wall down the middle column under a 3-column mask band splits the window into two mirror-image
    halves, each with a ring; the hole filling sees the two largest areas tied (sorted_area[-2] == sorted_area[-1])"""
    rw, rh = 31, 20
    img[y1:y1 + rh, x1:x1 + rw] = LIGHT
    mask[y1:y1 + rh, x1:x1 + rw] = 0
    img[y1:y1 + rh, x1 + 15] = DARK
    mask[y1:y1 + rh, x1 + 14:x1 + 17] = 255
    for xa in (3, 21):                                # mirror images: columns 3..9 and 21..27
        img[y1 + 4, x1 + xa:x1 + xa + 7] = DARK
        img[y1 + 10, x1 + xa:x1 + xa + 7] = DARK
        img[y1 + 4:y1 + 11, x1 + xa] = DARK
        img[y1 + 4:y1 + 11, x1 + xa + 6] = DARK
        mask[y1 + 3:y1 + 12, x1 + xa - 1:x1 + xa + 8] = 255
    return [x1, y1, x1 + rw, y1 + rh]


def noise_case(seed=0):
    """noise windows of several shapes (two overlapping), and the hole filling's edge cases: two holes tied for the
    largest area, one component in the inverse besides label 0, a window that merges entirely (dark under mask 255),
    and one where nothing merges (light under mask 0: area0 = 0)"""
    rng = np.random.default_rng(seed)
    h, w = 120, 260
    img, mask = _dense(h, w)
    wins = []
    for x1, y1, rw, rh in ((2, 2, 40, 30), (50, 2, 33, 17), (90, 2, 64, 9), (160, 2, 7, 50), (170, 5, 31, 21),
                           (185, 15, 40, 30), (2, 40, 1, 30), (10, 40, 60, 2), (80, 60, 17, 33)):
        noise_fill(rng, img, mask, x1, y1, rw, rh)
        wins.append([x1, y1, x1 + rw, y1 + rh])
    wins.append(_tie_window(img, mask, 100, 80))
    # one hole: a light window whose left column is a dark wall under mask 255
    img[80:100, 140:160] = LIGHT
    mask[80:100, 140:160] = 0
    img[80:100, 140] = DARK
    mask[80:100, 140:142] = 255
    wins.append([140, 80, 160, 100])
    wins.append([165, 80, 185, 100])                  # dark under mask 255: merges entirely
    img[80:100, 190:215] = LIGHT                       # light under mask 0: nothing merges
    mask[80:100, 190:215] = 0
    wins.append([190, 80, 215, 100])
    return img, mask, wins


# ---- seeded random sweep ------------------------------------------------------------------------------------------
SWEEP_W, SWEEP_H = 9100, 320


def sweep_case(seed, n=8):
    """n windows of log-uniform width 1 - 9000 and height 1 - 300 at random positions of one page (one launch):
    windows under 4000 px get noise content, larger ones dark strokes and rings under a blurred mask on a light page
    with mild noise; the page around them is dark under mask 255"""
    rng = np.random.default_rng(seed)
    img, mask = _dense(SWEEP_H, SWEEP_W)
    m = np.zeros((SWEEP_H, SWEEP_W), np.float32)
    wins, big = [], []
    for _ in range(n):
        rw = int(np.exp(rng.uniform(0, np.log(9000))))
        rh = int(np.exp(rng.uniform(0, np.log(300))))
        x1 = int(rng.integers(0, SWEEP_W - rw))
        y1 = int(rng.integers(0, SWEEP_H - rh))
        if rng.random() < 0.2:                        # against the clamped right / bottom edge
            x1 = SWEEP_W - 1 - rw
        if rng.random() < 0.2:
            y1 = SWEEP_H - 1 - rh
        wins.append([x1, y1, x1 + rw, y1 + rh])
        if rw * rh < 4000:
            noise_fill(rng, img, mask, x1, y1, rw, rh)
        else:
            big.append((x1, y1, rw, rh))
    for x1, y1, rw, rh in big:
        img[y1:y1 + rh, x1:x1 + rw] = LIGHT + rng.integers(0, 8, (rh, rw, 1), dtype=np.uint8)
        for _ in range(int(rng.integers(2, 6 + rw * rh // 20000))):
            p = (x1 + int(rng.integers(0, rw)), y1 + int(rng.integers(0, rh)))
            q = (x1 + int(rng.integers(0, rw)), y1 + int(rng.integers(0, rh)))
            t = int(rng.integers(1, 4))
            cv2.line(img, p, q, (DARK, DARK, DARK), t)
            cv2.line(m, p, q, 1.0, t)
            if rng.random() < 0.3:
                r = int(rng.integers(3, 20))
                cv2.circle(img, p, r, (DARK, DARK, DARK), 1)
                cv2.circle(m, p, r, 1.0, 1)
    sm = (cv2.GaussianBlur(m, (0, 0), 1.2) * 255).clip(0, 255).astype(np.uint8)
    for x1, y1, rw, rh in big:
        mask[y1:y1 + rh, x1:x1 + rw] = sm[y1:y1 + rh, x1:x1 + rw]
    return img, mask, wins
