"""Convex lattice polygons with as many vertices as a map of a given size allows, filled exactly.

A strictly convex polygon with integer vertices has edges of pairwise distinct directions, so the most vertices fit
when its edges are the shortest primitive integer vectors, chained in angle order.  `many_vertex_polygon()` takes every
primitive vector of L1 norm <= 20 and then norm-21 vectors in quadruples closed under quarter turns (so the chain
closes and the polygon keeps the symmetry of the square): 560 vertices inside 1998 x 1998.  `fill_exact` rasterises it
with integer half-plane tests, so every vertex is a pixel of the component and cv2.convexHull of the pixels gives the
polygon back.  (cv2.fillPoly's rasterisation loses vertices: it leaves 364.)"""
from math import atan2, gcd

import numpy as np


def _primitive(norm):
    """primitive integer vectors (a, b) with |a| + |b| == norm"""
    out = []
    for a in range(-norm, norm + 1):
        r = norm - abs(a)
        for b in {r, -r}:
            if gcd(abs(a), abs(b)) == 1:
                out.append((a, b))
    return out


def many_vertex_polygon(n_vertices=560, max_norm=20):
    """int64 [n_vertices, 2] (x, y) vertices, counter-clockwise in (x, y), min corner at (0, 0)"""
    vecs = [v for k in range(1, max_norm + 1) for v in _primitive(k)]
    # next norm, in quarter-turn orbits (a, b) -> (-b, a), taken in a fixed order until the count is reached
    orbits = sorted({tuple(sorted([(a, b), (-b, a), (-a, -b), (b, -a)])) for a, b in _primitive(max_norm + 1)})
    for orb in orbits:
        if len(vecs) + 4 > n_vertices:
            break
        vecs.extend(orb)
    assert len(vecs) == n_vertices, (len(vecs), n_vertices)
    vecs.sort(key=lambda v: atan2(v[1], v[0]))
    pts = np.cumsum(np.array(vecs, np.int64), axis=0)
    assert not pts[-1].any()          # the chain closes
    return pts - pts.min(0)


def fill_exact(pts, h, w, x0=0, y0=0, value=1.0, dtype=np.float32):
    """[h, w] map with `value` on every pixel inside or on the polygon `pts` (counter-clockwise, integer) shifted by
    (x0, y0), 0 elsewhere"""
    P = np.asarray(pts, np.int64) + np.array([x0, y0], np.int64)
    D = np.roll(P, -1, axis=0) - P
    out = np.zeros((h, w), dtype)
    ys = np.arange(h, dtype=np.int64)
    lo = np.zeros(h, np.int64)
    hi = np.full(h, w - 1, np.int64)
    ok = np.ones(h, bool)
    for (vx, vy), (dx, dy) in zip(P, D):
        # inside: cross(d, p - v) = dx * (py - vy) - dy * (px - vx) >= 0  <=>  px * dy <= vx * dy + dx * (py - vy)
        num = vx * dy + dx * (ys - vy)
        if dy > 0:
            hi = np.minimum(hi, num // dy)
        elif dy < 0:
            lo = np.maximum(lo, -((-num) // dy))
        else:
            ok &= dx * (ys - vy) >= 0
    for y in np.nonzero(ok & (lo <= hi))[0]:
        out[y, lo[y]:hi[y] + 1] = value
    return out
