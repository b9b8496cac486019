"""Crafted Detect rows that put the NMS at its decision boundaries, and the property each one exists for.

Every builder asserts its property with numpy float32 (and float16) arithmetic in the order the kernels and
torchvision use: xywh2xyxy in the rows' dtype (yolov5_utils.py:172,220-227), widened to float32, the class offset
`cls * 4096` added to the corners (yolov5_utils.py:198), then `inter / ((area_i + area_j) - inter)`.  Rows are
[k][5 + nc] arrays of float32 or float16; the cases hold no GPU and no oracle, so tests/test_cpu_nms_boundaries.py
checks them on the CPU and tests/test_gpu_nms_boundaries.py feeds them to the kernels.

  * IoU ties: pairs and greedy chains whose IoU after the offset is exactly float32(t), one ulp below and one ulp
    above, in class 0 and in class 1 (fractional corners that the +4096 offset rounds), and the chain where A
    suppresses B (IoU the smallest float32 over t), B would have suppressed C, and C survives;
  * degenerate boxes: zero width or height (IoU 0 / 0 = NaN, never over t), negative sides, identical boxes;
  * score boundaries, float32 and float16: obj and the class score exactly at, and one ulp around, the threshold as
    the rows' dtype compares it; class scores tied for the maximum (the first class wins); half corners that round;
  * order and caps: more than 300 survivors with a score tie across the max_det cut, and more than 4096 candidates
    with the cut inside a tie."""
import functools

import numpy as np

THRESHOLDS = (0.35, 0.3, 0.4, 0.45, 0.5, 0.6, 0.8)   # IoU thresholds: rounding down, up, and exact in float32
CONFS = (0.4, 0.3, 0.55)                             # conf thresholds of the score cases
MAX_WH = np.float32(4096)
MAX_DET = 300
CAP = 4096   # the engine's NMS candidate workspace per page (include/ctd_b200.h, ctd_get_nms_status)


# ---- float32 / float16 arithmetic of the reference ------------------------------------------------------------------
def rd_f32(t):
    """t rounded toward -inf to float32: for a float32 x, `x > t` (t a double) exactly when `x > rd_f32(t)`"""
    f = np.float32(t)
    return np.nextafter(f, np.float32(-np.inf)) if float(f) > t else f


def above_f32(t):
    """the smallest float32 > t"""
    return np.nextafter(rd_f32(t), np.float32(np.inf))


def rounds_up(t):
    return float(np.float32(t)) > t


def corners(rows):
    """xywh2xyxy in the rows' dtype, widened to float32: [k][4]"""
    x = np.asarray(rows)
    two = x.dtype.type(2)
    hw, hh = x[:, 2] / two, x[:, 3] / two
    return np.stack([x[:, 0] - hw, x[:, 1] - hh, x[:, 0] + hw, x[:, 1] + hh], 1).astype(np.float32)


def scores(rows, conf):
    """(candidate mask, best class score, best class) as non_max_suppression computes them in the rows' dtype: obj >
    conf, cls * obj, the first maximal class, score > conf; conf is conf_thres as that dtype compares it"""
    x = np.asarray(rows)
    c = x.dtype.type(np.float32(conf))
    prod = x[:, 5:] * x[:, 4:5]
    best = prod.max(1)
    return (x[:, 4] > c) & (best > c), best.astype(np.float32), prod.argmax(1)


def offset_boxes(rows):
    """the class-offset boxes torchvision's NMS sees for rows whose best class is the class column"""
    _, _, cls = scores(rows, 0.0)
    return corners(rows) + cls.astype(np.float32)[:, None] * MAX_WH


def iou(a, b):
    """float32 IoU of float32 xyxy boxes a [..][4] and b [..][4], in torchvision's (and nms_mask_kernel's) order"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    zero = np.float32(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.maximum(zero, np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]))
        h = np.maximum(zero, np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]))
        inter = w * h
        area_a = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
        area_b = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
        return inter / ((area_a + area_b) - inter)


def greedy(rows, conf, suppress):
    """the kept row indices of the greedy NMS with the decision `suppress(iou)` (no max_det, no cap): stable by
    score descending, then row order"""
    cand, best, _ = scores(rows, conf)
    idx = np.nonzero(cand)[0]
    order = idx[np.lexsort((idx, -best[idx]))]
    boxes = offset_boxes(rows)
    keep, gone = [], set()
    for k, i in enumerate(order):
        if i in gone:
            continue
        keep.append(int(i))
        for j in order[k + 1:]:
            if j not in gone and suppress(iou(boxes[i], boxes[j])):
                gone.add(j)
    return keep


def kept_double(rows, conf, t):
    """torchvision's CPU rule: float32 IoU > t, compared in double"""
    return greedy(rows, conf, lambda v: float(v) > t)


def kept_float(rows, conf, t):
    """the float rule with t rounded to nearest: float32 IoU > float32(t)"""
    return greedy(rows, conf, lambda v: v > np.float32(t))


def row(cx, cy, w, h, obj, cls=0, nc=2, dtype=np.float32):
    r = np.zeros(5 + nc, dtype)
    r[:5] = (cx, cy, w, h, obj)
    r[5 + cls] = 1
    return r


# ---- IoU ties ---------------------------------------------------------------------------------------------------------
def _link(a, target, rng, dtype, t, others=()):
    """a row of a's class right of a, whose IoU with a after the class offset is exactly the float32 target and whose
    IoU with each of `others` is under 0.95 t: a seeded search around the analytic shift w (1 - t) / (1 + t), in the
    rows' dtype"""
    cls = int(np.argmax(a[5:]))
    box_a = offset_boxes(a[None])[0]
    cx, cy, w, h = (float(v) for v in a[:4])
    d0 = w * (1 - t) / (1 + t)
    if dtype == np.float16:
        # half rows are too coarse for a shift: integer corners instead, the next box of any integer size overlapping
        # a's bottom-right corner by ox x oy px, so that the IoU ox oy / (area_a + w h - ox oy) has a large denominator
        # (sides and overlaps in steps of 0.25 px, exact in half below 512).  t is a fraction of small denominator
        # d, and p / q != t is at least 1 / (d q) away from it: an IoU one float32 ulp from t needs unions of
        # some 10^5 px^2
        x2, y2 = cx + w / 2, cy + h / 2
        tries = []
        for _ in range(16):
            wb, hb = rng.integers(480, 1000, 1 << 17) / 4, rng.integers(480, 1000, 1 << 17) / 4
            oy = rng.integers(4 * np.minimum(h, hb) // 2, 4 * np.minimum(h, hb) + 1) / 4
            ox0 = t * (w * h + wb * hb) / ((1 + t) * oy)
            for r in (np.floor(4 * ox0) / 4, np.ceil(4 * ox0) / 4):
                ok = (r >= 1) & (r <= np.minimum(w, wb))
                b = np.repeat(a[None], int(ok.sum()), 0).astype(dtype)
                b[:, 2], b[:, 3] = wb[ok], hb[ok]
                b[:, 0] = x2 - r[ok] + wb[ok] / 2
                b[:, 1] = y2 - oy[ok] + hb[ok] / 2
                tries.append(b)
    else:
        # random sizes and vertical overlaps, the horizontal overlap solved for the target; the corners' rounding
        # (in class 1 to the 2^-11 grid of the offset boxes) scatters the IoU over a few hundred ulps around it
        x2, y2 = cx + w / 2, cy + h / 2
        tries = []
        for _ in range(16):
            n = 1 << 15
            wb, hb = w * rng.uniform(0.8, 1.2, n), h * rng.uniform(0.8, 1.2, n)
            oy = np.minimum(h, hb) * rng.uniform(0.8, 1.0, n)
            ox = t * (w * h + wb * hb) / ((1 + t) * oy)
            b = np.repeat(a[None], n, 0).astype(dtype)
            b[:, 0], b[:, 1] = x2 - ox + wb / 2, y2 - oy + hb / 2
            b[:, 2], b[:, 3] = wb, hb
            tries.append(b)
    for b in tries:
        boxes = corners(b) + np.float32(cls) * MAX_WH
        ok = iou(box_a, boxes) == np.float32(target)
        if cls:   # the offset must change the IoU
            ok &= iou(corners(a[None])[0], corners(b)) != np.float32(target)
        for o in others:
            ok &= iou(offset_boxes(o[None])[0], boxes) < np.float32(0.95 * t)
        hit = np.nonzero(ok)[0]
        if hit.size:
            return b[hit[rng.integers(hit.size)]].copy()
    raise AssertionError("no row at IoU %r" % float(target))


def tie_targets(t):
    """{name: float32 IoU}: exactly float32(t), one ulp below, one ulp above"""
    f = np.float32(t)
    return {"at": f, "below": np.nextafter(f, np.float32(0)), "above": np.nextafter(f, np.float32(1))}


def tie_chain(t, target, cls, length, seed, dtype=np.float32):
    """`length` rows of class cls, scores descending along the chain, each adjacent pair at IoU exactly `target`
    after the offset and every other pair far below t.  Class 1 sits at fractional corners that the +4096 offset
    rounds, so that the IoU with the offset differs from the IoU without it."""
    rng = np.random.default_rng(seed)
    if dtype == np.float16:
        first = row(130, 120, 240, 200, 0.9, cls, dtype=dtype)
    else:
        x0 = 20.0 + (0.37 if cls else 0.0)
        first = row(x0 + rng.uniform(0, 0.01) * cls, 30.0 + 0.123 * cls, 7.0 + 0.0517 * cls, 10.0 + 0.0313 * cls, 0.9,
                    cls, dtype=dtype)
        if cls == 0:
            first[:4] = np.round(first[:4].astype(np.float64) * 8) / 8
    rows = [first]
    for k in range(1, length):
        nxt = _link(rows[-1], target, rng, dtype, t, rows[:-1])
        nxt[4] = dtype(0.9 - 0.05 * k)
        rows.append(nxt)
    rows = np.stack(rows).astype(dtype)
    boxes = offset_boxes(rows)
    for i in range(length):
        for j in range(i + 1, length):
            v = iou(boxes[i], boxes[j])
            assert (v == np.float32(target)) if j == i + 1 else (v < np.float32(t) * np.float32(0.95)), (i, j, v)
    if cls == 1 and dtype == np.float32:
        plain = corners(rows)
        assert iou(plain[0], plain[1]) != iou(boxes[0], boxes[1])   # the offset rounds the corners
    return rows


@functools.lru_cache(maxsize=None)
def tie_rows(t, seed=0):
    """{name: rows} of the IoU-tie cases at threshold t, float32 and float16"""
    out = {}
    for dtype, tag in ((np.float32, "f32"), (np.float16, "f16")):
        for name, target in tie_targets(t).items():
            for cls in (0, 1):
                if dtype == np.float16 and (cls == 1 or name != "at"):
                    # half corners are coarse: the +4096 offset rounds none of them, and an IoU one float32 ulp from a
                    # t of small denominator is out of reach of boxes on a half grid below 512 px
                    continue
                out["%s_pair_%s_c%d" % (tag, name, cls)] = tie_chain(t, target, cls, 2, seed + 7 * cls, dtype)
                if dtype == np.float32:   # a half chain would leave the 0.25 px grid of half below 512
                    out["%s_chain_%s_c%d" % (tag, name, cls)] = tie_chain(t, target, cls, 5, seed + 1 + 7 * cls,
                                                                          dtype)
        if dtype == np.float32 or rounds_up(t):   # in half, only where the smallest float32 over t is float32(t)
            out["%s_survivor" % tag] = survivor_chain(t, seed + 3, dtype)
    if t == 0.4:
        # the integer pair of the float rule's failure: overlap 40 px^2, union 100 px^2
        out["f32_integer_pair"] = np.stack([row(3.5, 5, 7, 10, 0.9), row(6.5, 5, 7, 10, 0.8)])
        assert iou(*offset_boxes(out["f32_integer_pair"])) == np.float32(0.4)
    return out


def survivor_chain(t, seed, dtype=np.float32):
    """A, B, C with scores descending: IoU(A, B) is the smallest float32 over t, so A suppresses B; IoU(B, C) is well
    over t, so B would have suppressed C; IoU(A, C) is below t, so C survives.  Where float32(t) rounds up, IoU(A, B)
    is float32(t) itself and the float rule keeps B instead (and drops C)."""
    rng = np.random.default_rng(seed)
    a = row(40.0, 30.0, 12.0, 9.0, 0.9, dtype=dtype) if dtype == np.float32 else row(130, 120, 240, 200, 0.9, dtype=dtype)
    b = _link(a, above_f32(t), rng, dtype, t)
    b[4] = dtype(0.8)
    c = b.copy()
    c[0] = b[0] + b[2] * dtype(0.25) * dtype(1 - t)
    c[4] = dtype(0.7)
    rows = np.stack([a, b, c]).astype(dtype)
    boxes = offset_boxes(rows)
    assert iou(boxes[0], boxes[1]) == above_f32(t) and float(iou(boxes[1], boxes[2])) > t + 0.02
    assert float(iou(boxes[0], boxes[2])) < t
    assert kept_double(rows, 0.4, t) == [0, 2]
    return rows


# ---- degenerate boxes -------------------------------------------------------------------------------------------------
def degenerate_rows(dtype=np.float32):
    """rows of zero width or height, negative sides and identical boxes, each group far from the others:
    * two zero-width boxes at one place and two zero-height ones: union 0, IoU 0 / 0 = NaN, never over t: both kept;
    * a box and one of the same centre with its width negated: inter 0, areas 100 and -100, NaN: both kept;
    * a box and one with both sides negated (a positive area, corners swapped): inter 0, IoU 0: both kept;
    * identical boxes and identical scores: the lower row is kept, the other suppressed (IoU 1);
    * a zero-width box inside a normal one: inter 0, IoU 0: both kept"""
    r = [row(10, 10, 0, 8, 0.9), row(10, 10, 0, 8, 0.8),
         row(40, 10, 8, 0, 0.9), row(40, 10, 8, 0, 0.85),
         row(70, 10, 10, 10, 0.9), row(70, 10, -10, 10, 0.8),
         row(100, 10, 10, 10, 0.9), row(100, 10, -10, -10, 0.8),
         row(130, 10, 10, 6, 0.7), row(130, 10, 10, 6, 0.7),
         row(160, 10, 10, 10, 0.9), row(160, 10, 0, 4, 0.8)]
    rows = np.stack(r).astype(dtype)
    b = offset_boxes(rows)
    v = [iou(b[i], b[i + 1]) for i in range(0, len(r), 2)]
    assert np.isnan(v[0]) and np.isnan(v[1]) and np.isnan(v[2]) and v[3] == 0 and v[4] == 1 and v[5] == 0, v
    for t in THRESHOLDS:
        assert kept_double(rows, 0.4, t) == [0, 2, 4, 6, 10, 3, 1, 5, 7, 11, 8], kept_double(rows, 0.4, t)
    return rows


# ---- score boundaries -------------------------------------------------------------------------------------------------
def _spaced(k, nc, dtype, pitch=16.0):
    """k rows of class 0 on a grid of disjoint 6 x 6 boxes (every candidate survives the NMS)"""
    g = np.arange(k)
    rows = np.zeros((k, 5 + nc), dtype)
    rows[:, 0] = 8 + (g % 60) * pitch
    rows[:, 1] = 8 + (g // 60) * pitch
    rows[:, 2:4] = 6
    return rows


def score_rows_f32(conf, nc, seed=0):
    """float32 rows around conf (compared as float32(conf), the scalar cast to the tensor's dtype):
    obj at, one ulp below and above; the best class score cls * obj rounding onto, below and above float32(conf);
    class scores that tie for the maximum (the first class must win).  -> rows, {row: expected best class or -1}"""
    rng = np.random.default_rng(seed)
    c = np.float32(conf)
    up, dn = np.nextafter(c, np.float32(1)), np.nextafter(c, np.float32(0))
    specs = []   # (obj, class scores)
    for obj in (c, up, dn):
        specs.append((obj, [1.0] + [0.5] * (nc - 1)))
    for target in (c, up, dn):
        # an obj over conf and a class score whose float32 product rounds to the target (searched)
        for _ in range(100):
            obj = np.float32(rng.uniform(0.7, 0.99))
            base = np.float32(target / obj)
            hit = [s for s in (np.float32(base + np.float32(k) * np.spacing(base)) for k in range(-8, 9))
                   if s * obj == target and float(s) * float(obj) != float(target)]
            if hit:
                s = hit[0]
                break
        assert s * obj == target and float(s) * float(obj) != float(target)   # rounds onto the target
        specs.append((obj, [s] + [0.0] * (nc - 1)))
    for k in range(4):
        obj = np.float32(rng.uniform(0.6, 1.0))
        tie = np.float32(rng.uniform(0.7, 1.0))
        cs = list(rng.uniform(0, 0.5, nc).astype(np.float32))
        for j in range(nc):
            if j >= k % nc:
                cs[j] = tie
        specs.append((obj, cs))
    rows = _spaced(len(specs), nc, np.float32)
    for i, (obj, cs) in enumerate(specs):
        rows[i, 4] = obj
        rows[i, 5:] = cs
    cand, best, cls = scores(rows, conf)
    expect = {i: (int(cls[i]) if cand[i] else -1) for i in range(len(rows))}
    assert [expect[i] >= 0 for i in range(3)] == [False, True, False]
    assert [expect[i] >= 0 for i in range(3, 6)] == [False, True, False]
    for i in range(6, len(rows)):
        prod = rows[i, 5:] * rows[i, 4]
        assert expect[i] == int(np.nonzero(prod == prod.max())[0][0])
    assert any(expect[i] > 0 for i in range(6, len(rows))) or nc == 1
    return rows, expect


HALF_ULP = lambda v: np.spacing(np.float16(v))   # noqa: E731


def score_rows_f16(conf, seed=0):
    """float16 rows (nc = 2) around conf as a half tensor compares it, half(float32(conf)): obj at, one half-ulp below
    and above; products cls * obj that round in half onto, below and above it (and whose float32 product lies on the
    other side where one exists); class scores that tie only once rounded to half."""
    c = np.float16(np.float32(conf))
    up, dn = np.nextafter(c, np.float16(1)), np.nextafter(c, np.float16(0))
    all_h = np.arange(0x3c01, dtype=np.uint16).view(np.float16)   # 0 .. 1
    all_h = all_h[all_h > np.float16(0.5)]
    specs = [(c, (1, 0)), (up, (1, 0)), (dn, (1, 0))]
    for target in (c, up, dn):
        objs = all_h[all_h > up][::37]
        found = 0
        for obj in objs:
            s = np.float16(np.float32(target) / np.float32(obj))
            for cand in (np.nextafter(s, np.float16(0)), s, np.nextafter(s, np.float16(1))):
                if cand * obj == target and float(cand) * float(obj) != float(target) and cand <= 1:
                    specs.append((obj, (cand, 0)))
                    found += 1
                    break
            if found == 3:
                break
        assert found == 3, float(target)
    # class scores equal in half once multiplied, different in float32: the first class wins
    c0 = np.float16(0.9)
    c1 = np.nextafter(c0, np.float16(1))
    obj = next(o for o in all_h[all_h > np.float16(0.6)] if o * c0 == o * c1)
    specs += [(obj, (c0, c1)), (obj, (c1, c0))]
    rows = _spaced(len(specs), 2, np.float16)
    for i, (obj, cs) in enumerate(specs):
        rows[i, 4] = obj
        rows[i, 5:] = cs
    cand, _, cls = scores(rows, conf)
    # obj at, over and under half(conf); then three products each rounding onto, over and under it
    assert list(cand[:12]) == [False, True, False] + [False] * 3 + [True] * 3 + [False] * 3
    p32 = rows[-2:, 5:].astype(np.float32) * rows[-2:, 4:5].astype(np.float32)
    assert (p32[:, 0] != p32[:, 1]).all() and (cls[-2:] == 0).all()
    return rows


def half_corner_rows():
    """float16 rows whose corners round in half: w subnormal (RN_half(w / 2) rounds, ties to even), and a large cx
    where RN_half(cx -/+ RN_half(w / 2)) rounds.  Every box is apart from the others, so every row survives."""
    sub = np.arange(1, 64, dtype=np.uint16).view(np.float16)            # subnormal widths
    rows = _spaced(len(sub) + 120, 2, np.float16, pitch=32.0)
    rows[:, 4] = np.float16(0.9)
    rows[:, 5] = 1
    rows[:len(sub), 2] = sub
    rows[:len(sub), 3] = sub[::-1]
    rng = np.random.default_rng(5)
    k = slice(len(sub), None)
    rows[k, 0] = (np.arange(120) * 40 + 1030 + rng.integers(0, 8, 120) / 8).astype(np.float16)   # ulp 1 above 1024
    rows[k, 1] = rng.uniform(300, 900, 120).astype(np.float16)                                  # ulp 0.25 .. 0.5
    rows[k, 2] = rng.uniform(1, 20, 120).astype(np.float16)
    rows[k, 3] = rng.uniform(1, 20, 120).astype(np.float16)
    x = rows.astype(np.float32)
    exact = np.stack([x[:, 0] - x[:, 2] / 2, x[:, 1] - x[:, 3] / 2, x[:, 0] + x[:, 2] / 2, x[:, 1] + x[:, 3] / 2], 1)
    c = corners(rows)
    assert (c[:len(sub)] != exact[:len(sub)]).any(1).mean() > 0.4    # half of a subnormal rounds
    assert (c[k] != exact[k]).any(1).mean() > 0.5                   # the large-cx sums round
    return rows


# ---- order and caps ---------------------------------------------------------------------------------------------------
def max_det_rows(seed=0):
    """420 disjoint boxes, so that every candidate survives: 200 of distinct scores over 0.9, then 220 tied at 0.75
    in scattered rows.  The 300-detection cut falls inside the tie, and row order decides which 100 of it are kept."""
    rng = np.random.default_rng(seed)
    rows = _spaced(420, 2, np.float32)
    rows[:, 5] = 1
    perm = rng.permutation(420)
    rows[perm[:200], 4] = np.sort(rng.uniform(0.9, 1.0, 200)).astype(np.float32)[::-1]
    rows[perm[200:], 4] = np.float32(0.75)
    _, best, _ = scores(rows, 0.4)
    order = np.lexsort((np.arange(420), -best))
    assert best[order[MAX_DET - 1]] == best[order[MAX_DET]] == np.float32(0.75)
    return rows


def overflow_rows(seed=0, total=6000):
    """more than CAP candidates, all disjoint boxes, with the cut at CAP inside a score tie: the engine keeps the CAP
    best by (score descending, row ascending)"""
    rng = np.random.default_rng(seed)
    rows = _spaced(total, 2, np.float32, pitch=8.0)
    rows[:, 2:4] = 3
    rows[:, 5] = 1
    rows[:, 4] = np.round(rng.uniform(0.5, 1.0, total), 2).astype(np.float32)
    cand, best, _ = scores(rows, 0.4)
    idx = np.nonzero(cand)[0]
    order = idx[np.lexsort((idx, -best[idx]))]
    assert len(idx) > CAP and best[order[CAP - 1]] == best[order[CAP]]
    return rows


def capped(rows, conf):
    """the rows the engine runs the NMS on: past CAP candidates, the CAP best by (score descending, row ascending)"""
    cand, best, _ = scores(rows, conf)
    idx = np.nonzero(cand)[0]
    if len(idx) <= CAP:
        return rows
    return rows[np.sort(idx[np.lexsort((idx, -best[idx]))][:CAP])]


def oracle_nms(rows, conf, t):
    """the reference's non_max_suppression on rows as the engine runs them (past CAP candidates, the CAP best): float32
    rows through oracle/postproc_ref, float16 rows through oracle/postproc_half_ref -> float32 [k][6]"""
    import torch
    from oracle import postproc_half_ref, postproc_ref
    rows = capped(rows, conf)
    if rows.dtype == np.float16:
        return postproc_half_ref.non_max_suppression_half(rows[None], conf, t)[0].numpy()
    return postproc_ref.non_max_suppression(torch.from_numpy(np.ascontiguousarray(rows))[None], conf, t)[0].numpy()


def expected_rows(rows, conf, kept):
    """the NMS output rows (x1, y1, x2, y2, score, class) float32 of the kept row indices"""
    _, best, cls = scores(rows, conf)
    return np.concatenate([corners(rows), best[:, None], cls[:, None].astype(np.float32)], 1)[kept]
