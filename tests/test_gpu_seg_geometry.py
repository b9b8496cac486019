"""-m gpu: the text-line boxes and scores of `SegDetectorRepresenter.boxes_from_bitmap` (`csrc/segrep.cu`, the per-contour
geometry of `csrc/geom.h`) contour by contour, on maps aimed at the geometry's float arithmetic and at the score's fill.

Every box the device gives equals the host build of the same geometry on cv2's contours bit for bit, skipped rows
included; the host equals the oracle (cv2's `minAreaRect`) on every contour but exact area ties, which are counted and
pinned.  Scores equal cv2's mean bit for bit on maps quantised to multiples of 2^-24, and are within one float32 ulp
elsewhere (`tests/seg_geometry.py`).  Each map asserts on the CPU the property it exists for; the not-gpu test pins the
host-vs-oracle residuals of every map, so that a GPU run that passes also speaks for the oracle."""
import math
import os

import cv2
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import geom_ref, postproc_ref
import seg_geometry as sg
import stress_maps
from util import get_checkpoint

T = sg.T


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return sg.build_host_geom(tmp_path_factory.mktemp("geom"))


def texture(mask, rng, quantised=True):
    """pred that differs from pixel to pixel: (0.31, 1) on the mask, [0, 0.29) off it, so that one pixel more or less in a
    contour's fill moves its score by many ulps"""
    m = np.where(mask, rng.uniform(0.31, 1.0, mask.shape), rng.uniform(0.0, 0.29, mask.shape))
    return sg.quantise(m) if quantised else m.astype(np.float32)


def first_sides(cs):
    """min(cv2.minAreaRect(c)[1]) of every contour: the short side the reference skips below 2"""
    return np.array([min(cv2.minAreaRect(c)[1]) for c in cs], np.float64)


def grid(h, w, pitch):
    return [(x + pitch // 2, y + pitch // 2) for y in range(0, h - pitch + 1, pitch) for x in range(0, w - pitch + 1, pitch)]


# ---- maps: (h, w, rng) -> pred f32 [h][w] -----------------------------------------------------------------------------
ANGLES = np.arange(0.0, 90.0 + 1e-9, 0.25)   # 361 angles, 0 and 90 included


def rects(sizes, min_angles):
    """filled cv2.boxPoints rectangles at every angle of ANGLES, for each (long, short) side pair: the caliper angle, and
    the atan2 / cos / sin of the angle and of boxPoints.  A map too small for all of them takes every k-th one.
    min_angles: the fraction of them whose cv2.minAreaRect angles must be distinct after rasterisation"""
    def make(h, w, rng):
        diag = max(math.hypot(a, b) for a, b in sizes)
        cells = grid(h, w, int(diag) + 4)
        jobs = [(a, s) for s in sizes for a in ANGLES]
        jobs = jobs[::-(-len(jobs) // len(cells))]
        assert len(jobs) <= sg.MAX_CANDIDATES
        mask = np.zeros((h, w), np.uint8)
        for (a, (L, S)), (cx, cy) in zip(jobs, cells):
            cx += float(rng.uniform(-0.5, 0.5))
            cy += float(rng.uniform(-0.5, 0.5))
            pts = cv2.boxPoints(((cx, cy), (L, S), float(a)))
            cv2.fillPoly(mask, [np.round(pts * 16).astype(np.int32)], 1, cv2.LINE_8, 4)
        m = texture(mask > 0, rng)
        cs = sg.contours(m)
        assert len(cs) == len(jobs)                          # one contour per rectangle
        ang = {round(float(cv2.minAreaRect(c)[2]), 3) for c in cs}
        assert len(ang) >= min_angles * len(jobs), len(ang)   # the rasterised rectangles keep many distinct angles
        assert (first_sides(cs) >= 2).all()
        return m
    return make


def shelf(h, w, sizes):
    """pack squares of the given sides left to right in rows, largest first -> [(side, (x0, y0))]; what does not fit is
    left out"""
    out, x, y, row = [], 0, 0, 0
    for s in sorted(sizes, reverse=True):
        if x + s > w:
            x, y, row = 0, y + row, 0
        if y + s > h or s > w:
            continue
        out.append((s, (x, y)))
        x += s
        row = max(row, s)
    return out


def clipper_steps(cs):
    """round(pi / acos(1 - 0.25 / delta)) of every contour that is not skipped: Clipper's round-join steps per turn"""
    steps = []
    for c in cs:
        p4, ss = postproc_ref._get_mini_boxes(c.squeeze(1))
        if ss >= 2:
            p4 = np.array(p4)
            d = geom_ref.geos_ring_area(p4) * 1.5 / geom_ref.geos_ring_length(p4)
            steps.append(int(round(math.pi / math.acos(1 - min(0.25, d * 0.25) / d))))
    return steps


def discs(h, w, rng):
    """discs and ellipses of radii 1 .. 160 at random angles, as many as fit: the first boxes' distance covers a wide
    range of Clipper round-join steps (acos, sin, cos of the step angle)"""
    mask = np.zeros((h, w), np.uint8)
    radii = [int(r) for r in np.unique(np.round(np.geomspace(1, 160, 70)))]
    placed = shelf(h, w, [2 * r + 4 + kind for r in radii for kind in (0, 1)])
    for s, (x0, y0) in placed:
        r, kind = (s - 4) // 2, (s - 4) % 2
        c = (x0 + s // 2, y0 + s // 2)
        if kind == 0:
            cv2.circle(mask, c, r, 1, -1)
        else:
            cv2.ellipse(mask, c, (r, max(1, int(rng.integers(1, r + 1)))), float(rng.uniform(0, 180)), 0, 360, 1, -1)
    m = texture(mask > 0, rng)
    cs = sg.contours(m)
    assert len(cs) == len(placed)
    steps = set(clipper_steps(cs))
    assert len(steps) >= min(25, len(placed) // 4), sorted(steps)   # many distinct Clipper steps per turn
    return m


def thin(h, w, rng):
    """1-3 px lines at every 3 degrees and specks of 1-4 px sides: first minAreaRect short sides on both sides of the
    reference's `sside < 2` skip"""
    mask = np.zeros((h, w), np.uint8)
    cells = grid(h, w, 40)
    k = 0
    for t in (1, 2, 3):
        for a in range(0, 180, 3):
            cx, cy = cells[k]
            k += 1
            d = np.array([math.cos(math.radians(a)), math.sin(math.radians(a))]) * float(rng.uniform(6, 16))
            p0 = np.round((np.array([cx, cy]) - d) * 16).astype(int)
            p1 = np.round((np.array([cx, cy]) + d) * 16).astype(int)
            cv2.line(mask, tuple(int(v) for v in p0), tuple(int(v) for v in p1), 1, t, cv2.LINE_8, 4)
    for sy in range(1, 5):
        for sx in range(1, 5):
            for _ in range(3):
                cx, cy = cells[k]
                k += 1
                mask[cy:cy + sy, cx:cx + sx] = 1
    for _ in range(20):                                       # diagonal pairs and anti-diagonal triples
        cx, cy = cells[k]
        k += 1
        mask[cy, cx] = mask[cy + 1, cx + 1] = 1
        cx, cy = cells[k]
        k += 1
        mask[cy + 2, cx] = mask[cy + 1, cx + 1] = mask[cy, cx + 2] = 1
    m = texture(mask > 0, rng)
    ss = first_sides(sg.contours(m))
    assert (ss < 2).sum() > 50 and (ss == 2).sum() >= 10 and ((ss > 2) & (ss < 3)).sum() > 10, np.unique(np.round(ss, 2))
    return m


def off_frame(h, w, rng):
    """ellipses and rotated rectangles across every side and corner: unclipped boxes leave [0, w] x [0, h]"""
    mask = np.zeros((h, w), np.uint8)
    for _ in range(40):
        side = int(rng.integers(4))
        t = float(rng.uniform(0, 1))
        c = [(t * w, 0), (t * w, h - 1), (0, t * h), (w - 1, t * h)][side]
        c = (int(c[0] + rng.uniform(-3, 3)), int(c[1] + rng.uniform(-3, 3)))
        ax = (int(rng.integers(4, max(5, min(h, w) // 6))), int(rng.integers(2, max(3, min(h, w) // 12))))
        cv2.ellipse(mask, c, ax, float(rng.uniform(0, 180)), 0, 360, 1, -1)
    for c in ((0, 0), (w - 1, 0), (0, h - 1), (w - 1, h - 1)):
        pts = cv2.boxPoints((c, (min(h, w) / 5, min(h, w) / 9), float(rng.uniform(0, 90))))
        cv2.fillPoly(mask, [np.round(pts).astype(np.int32)], 1)
    m = texture(mask > 0, rng)
    rb, _ = postproc_ref.seg_represent(m, 0.3)
    kept = rb.reshape(len(rb), -1).any(1)
    assert rb[kept, :, 0].min() == 0 and rb[kept, :, 0].max() == w      # clipped on the left and the right
    assert rb[kept, :, 1].min() == 0 and rb[kept, :, 1].max() == h      # and at the top and the bottom
    return m


def ties(h, w, rng):
    """exact area ties between minAreaRect candidates: axis-aligned squares, right isosceles triangles in all four
    orientations, diamonds and regular octagons, over a range of sizes"""
    mask = np.zeros((h, w), np.uint8)
    cells = grid(h, w, 48)
    k = 0
    for s in range(3, 40, 2):
        for kind in range(8):
            cx, cy = cells[k]
            k += 1
            x0, y0 = cx - s // 2, cy - s // 2
            if kind == 0:
                mask[y0:y0 + s, x0:x0 + s] = 1
            elif kind <= 4:
                tri = [[(0, 0), (s, 0), (0, s)], [(0, 0), (s, 0), (s, s)], [(s, 0), (s, s), (0, s)], [(0, 0), (s, s), (0, s)]]
                cv2.fillPoly(mask, [np.array(tri[kind - 1], np.int32) + (x0, y0)], 1)
            elif kind == 5:
                cv2.fillPoly(mask, [np.array([(s // 2, 0), (s, s // 2), (s // 2, s), (0, s // 2)], np.int32) + (x0, y0)], 1)
            else:
                a, b = s // 3, s - s // 3
                oct_ = [(a, 0), (b, 0), (s, a), (s, b), (b, s), (a, s), (0, b), (0, a)]
                cv2.fillPoly(mask, [np.array(oct_, np.int32) + (x0, y0)], 1)
    m = texture(mask > 0, rng)
    cs = sg.contours(m)
    assert len(cs) == k
    sq = [c for c in cs if cv2.boundingRect(c)[2] == cv2.boundingRect(c)[3] and cv2.contourArea(c) > 0]
    assert len(sq) > k // 2                                    # symmetric: equal width and height
    return m


def graded(h, w, rng):
    """a smooth field crossing the threshold, as a network's output does, plus sub-ulp texture: pred differs between
    every two neighbouring pixels inside and around each component; not quantised (the one-ulp rule)"""
    yy, xx = np.indices((h, w), dtype=np.float64)
    f = 0.3 + 0.22 * np.sin(xx / 17.0 + 0.3 * np.sin(yy / 23.0)) * np.cos(yy / 13.0 + 0.2 * np.cos(xx / 29.0))
    f += 0.05 * np.sin((xx + 2 * yy) / 7.0) + rng.uniform(-1e-3, 1e-3, (h, w))
    m = np.clip(f, 0, 1).astype(np.float32)
    assert (np.diff(m, axis=0) != 0).mean() > 0.999 and (np.diff(m, axis=1) != 0).mean() > 0.999
    assert not sg.is_quantised(m) and len(sg.contours(m)) > 20
    return m


def blobs_q(h, w, rng):
    """the blurred blob map of stress_maps, quantised: holes, nested rings and scores summed over hole borders"""
    m = sg.quantise(stress_maps.blobs(int(rng.integers(1 << 30)), h, w, max(4, h * w // 6000)))
    assert sg.is_quantised(m) and len(sg.contours(m)) > 10
    return m


MAP_KINDS = {
    "rects_small": rects([(7.0, 3.0), (11.5, 4.5)], 0.025),
    "rects_mid": rects([(30.0, 9.0), (41.0, 21.5)], 0.15),
    "rects_large": rects([(90.0, 24.0)], 0.3),
    "discs": discs,
    "thin": thin,
    "off_frame": off_frame,
    "ties": ties,
    "graded": graded,
    "blobs_q": blobs_q,
}

# (kind, h, w): the stage-isolated maps; non-square shapes up to the 2048 limit so that a swapped w / h shows
MAPS = [
    ("rects_small", 1024, 1024), ("rects_mid", 1024, 2048), ("rects_mid", 2048, 1024), ("rects_large", 2048, 2048),
    ("discs", 2048, 2048),
    ("thin", 768, 1024), ("off_frame", 512, 1536), ("off_frame", 1536, 512), ("off_frame", 64, 2048),
    ("off_frame", 2048, 40), ("ties", 1024, 1024), ("graded", 1000, 700), ("blobs_q", 700, 1000),
    ("blobs_q", 2048, 96), ("blobs_q", 40, 2048), ("blobs_q", 2048, 2048),
]


def make_map(kind, h, w):
    return MAP_KINDS[kind](h, w, np.random.default_rng(sum(map(ord, kind)) * 7919 + h * 31 + w))


def map_id(m):
    return "%s_%dx%d" % m


# host-vs-oracle residuals per map: axis-aligned rectangles whose cv2.minAreaRect comes out 1 ulp off the integers when
# cv2's hull starts at another vertex (its result depends on the order of the contour points); pyclipper then truncates
# the corners of the first box to the next integer down and the final box moves by one unit
RESIDUALS = {"rects_mid_1024x2048": 1, "blobs_q_700x1000": 2, "blobs_q_2048x2048": 3}


def test_host_geometry_matches_oracle_but_ties(geom):
    """not-gpu: the host build of the geometry equals the oracle on every contour of every map but the pinned ties"""
    got = {}
    for m in MAPS:
        ref = sg.Reference(geom, make_map(*m))
        got[map_id(m)] = (len(ref.cs), int(ref.resid.sum()))
    print({k: v for k, v in got.items()})
    assert {k: v[1] for k, v in got.items() if v[1]} == RESIDUALS


# the smallest contour on which dividing the exact double sum by the pixel count gives another float32 score than cv2's
# mean, which multiplies by the reciprocal: 210 px of a right isosceles triangle on a quantised map (26 x 26)
GOLDEN_RECIPROCAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seg_score_reciprocal.npz")


def test_score_reciprocal_fixture():
    """not-gpu: the fixture's oracle score is cv2's mean, float32(sum * (1 / n)), one ulp above float32(sum / n)"""
    g = np.load(GOLDEN_RECIPROCAL)
    pred = g["pred"]
    assert sg.is_quantised(pred)
    rb, rs = postproc_ref.seg_represent(pred, 0.3)
    assert np.array_equal(rb, g["boxes"]) and np.array_equal(rs, g["score"]) and len(rs) == 1
    cs = sg.contours(pred)
    mask = np.zeros(pred.shape, np.uint8)
    cv2.fillPoly(mask, [cs[0]], 1)
    v = pred[mask > 0].astype(np.float64)
    s, n = v.sum(), len(v)
    assert n == 210 and rs[0] == np.float32(s * (1.0 / n)) and rs[0] != np.float32(s / n)


@pytest.mark.gpu
def test_score_reciprocal_golden(eng, geom):
    g = np.load(GOLDEN_RECIPROCAL)
    gb, gs = eng.seg_represent(g["pred"], 0.3)
    assert np.array_equal(gb, g["boxes"]) and gs.tobytes() == g["score"].tobytes(), (gb, gs, g["boxes"], g["score"])


# ---- the stage-isolated kernels ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=2048, max_w=2048, skip_postproc=True)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m", MAPS, ids=map_id)
def test_seg_represent_geometry(eng, geom, m):
    pred = make_map(*m)
    ref = sg.Reference(geom, pred)
    gb, gs = eng.seg_represent(pred, 0.3)
    n = sg.assert_text_lines(ref, gb, gs, map_id(m))
    print(map_id(m), "contours", len(ref.cs), "host-vs-oracle residuals", n)
    assert n == RESIDUALS.get(map_id(m), 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(stress_maps.CASES))
def test_seg_represent_stress_maps(eng, geom, name):
    pred = stress_maps.CASES[name]()
    ref = sg.Reference(geom, pred)
    gb, gs = eng.seg_represent(pred, 0.3)
    n = sg.assert_text_lines(ref, gb, gs, name)
    print(name, "contours", len(ref.cs), "host-vs-oracle residuals", n)
    assert n == 0


# ---- the forward's batched post-processing ------------------------------------------------------------------------------
def rows_per_image(s):
    return 3 * ((s // 8) ** 2 + (s // 16) ** 2 + (s // 32) ** 2)


@pytest.fixture(scope="module")
def prog():
    return cc.compile_checkpoint(get_checkpoint(0, True))


@pytest.mark.gpu
@pytest.mark.parametrize("n,s", [(16, 1024), (8, 1536)])
def test_batched_text_lines(prog, geom, n, s):
    """every map kind at the benchmarked batch shapes through `debug_postprocess` (the forward's own DB post-processing);
    each page equals the host geometry and cv2's scores, and itself run alone: boxes bit for bit, scores within 1 ulp"""
    kinds = (list(MAP_KINDS) * (n // len(MAP_KINDS) + 1))[:n]
    np.random.default_rng(s).shuffle(kinds)
    lines = np.zeros((n, 2, s, s), np.float32)
    for i, k in enumerate(kinds):
        lines[i, 0] = MAP_KINDS[k](s, s, np.random.default_rng(1000 * i + s))
    blks = np.zeros((n, rows_per_image(s), 7), np.float32)      # no Detect candidates: this test is about the lines
    e = ctd_b200.Engine(prog, max_batch=n, max_h=s, max_w=s, use_graph=True)
    try:
        e.debug_postprocess(blks, lines)
        boxes, scores = e.text_lines()
        for i, k in enumerate(kinds):
            ref = sg.Reference(geom, lines[i, 0])
            nres = sg.assert_text_lines(ref, boxes[i], scores[i], (i, k, s))
            print(i, k, s, "contours", len(ref.cs), "host-vs-oracle residuals", nres)
        for i, k in enumerate(kinds):
            e.debug_postprocess(blks[i:i + 1], lines[i:i + 1])
            b1, s1 = e.text_lines()
            assert np.array_equal(b1[0], boxes[i]), (i, k, "alone")
            sg.assert_scores_within_ulp(s1[0], scores[i], (i, k, "alone"))
    finally:
        e.close()
