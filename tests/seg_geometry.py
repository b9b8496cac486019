"""The text-line boxes and scores of `SegDetectorRepresenter.boxes_from_bitmap`, contour by contour.

Boxes: the per-contour geometry (`csrc/geom.h`) built for the host (`tests/geom_host.cpp`, as `test_cpu_geom.py` builds
it) and run on cv2's own contours is the reference the device must equal bit for bit, skipped rows included.  The host
build follows OpenCV's float32 rotating calipers and Clipper's offset step by step; it differs from the oracle (cv2's
`minAreaRect` itself) only where cv2's answer depends on the start vertex of its hull, which follows the order of the
contour points.  Those residuals are counted, and on every other contour host, device and oracle agree.

Scores: the mean of float32 `pred` over the filled contour (`box_score_fast`), summed in double.  On a map whose values
are multiples of 2^-24 in [0, 1] every such double sum of fewer than 2^29 pixels is exact in any order, so the device's
score must equal cv2's bit for bit (cv2.mean scales the sum by the reciprocal of the count, and so does the device); on
any map only the order of the double additions differs, so it must be within
one float32 ulp, and bit-exact on at least 99.9 % of the contours."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np

from oracle import postproc_ref

HERE = os.path.dirname(os.path.abspath(__file__))
T = np.float32(0.3)           # db_thresh
MAX_CANDIDATES = 1000
Q24 = 2.0 ** -24


def build_host_geom(dirpath):
    """g++ build of csrc/geom.h for the host, loaded with ctypes (the build of tests/test_cpu_geom.py)"""
    so = os.path.join(str(dirpath), "geom_host.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "geom_host.cpp")])
    lib = C.CDLL(so)
    lib.geom_contour_box.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p]
    return lib


def contours(pred):
    """cv2.findContours(RETR_LIST, CHAIN_APPROX_SIMPLE) on pred > float32(0.3): the first 1000, in OpenCV's order"""
    cs, _ = cv2.findContours((np.asarray(pred) > T).astype(np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_SIMPLE)
    return list(cs)[:MAX_CANDIDATES]


def host_boxes(lib, pred, cs=None):
    """-> (boxes int16 [k,4,2], kept bool [k]): geom_contour_box on every contour; a skipped row is all zeros"""
    h, w = pred.shape
    cs = contours(pred) if cs is None else cs
    boxes = np.zeros((len(cs), 4, 2), np.int16)
    kept = np.zeros(len(cs), bool)
    for i, c in enumerate(cs):
        pts = np.ascontiguousarray(c.reshape(-1, 2).astype(np.int32))
        box = np.zeros(8, np.int16)
        kept[i] = lib.geom_contour_box(pts.ctypes.data, len(pts), w, h, w, h, 1.5, box.ctypes.data) == 1
        boxes[i] = box.reshape(4, 2)
    return boxes, kept


def is_quantised(pred):
    """every value a multiple of 2^-24 in [0, 1]"""
    p = np.asarray(pred, np.float64)
    return bool(((p >= 0) & (p <= 1)).all() and (np.round(p / Q24) * Q24 == p).all())


def quantise(pred):
    return (np.round(np.clip(np.asarray(pred, np.float64), 0, 1) / Q24) * Q24).astype(np.float32)


def residuals(hb, hkept, rb, rs):
    """rows where the host geometry and the oracle (cv2) disagree: the box, or whether the row is skipped"""
    rkept = rb.reshape(len(rb), 8).any(1) | (rs != 0)
    return (hb.reshape(len(hb), 8) != rb.reshape(len(rb), 8)).any(1) | (hkept != rkept)


class Reference:
    """host boxes, oracle boxes and oracle scores of one map"""

    def __init__(self, lib, pred, oracle=None):
        self.pred = np.ascontiguousarray(pred, np.float32)
        self.cs = contours(self.pred)
        self.hb, self.hkept = host_boxes(lib, self.pred, self.cs)
        self.rb, self.rs = postproc_ref.seg_represent(self.pred, 0.3) if oracle is None else oracle
        assert len(self.rb) == len(self.cs) == len(self.rs)
        self.resid = residuals(self.hb, self.hkept, self.rb, self.rs)
        # the score of every row the host keeps: the oracle's where it kept the row too, box_score_fast where only the
        # host did (a start-vertex residual on the first minAreaRect's short side)
        self.scores = np.where(self.hkept, self.rs, np.float32(0)).astype(np.float32)
        for i in np.nonzero(self.hkept & (self.rs == 0))[0]:
            self.scores[i] = np.float32(postproc_ref._box_score_fast(self.pred, self.cs[i].squeeze(1)))


def assert_text_lines(ref, gb, gs, what):
    """the device's boxes equal the host geometry bit for bit (skipped rows included); its scores equal cv2's bit for bit
    on a quantised map, else within one float32 ulp and bit for bit on >= 99.9 % of the contours.
    -> the number of host-vs-oracle residuals"""
    k = len(ref.hb)
    assert gb.shape == (k, 4, 2) and gs.shape == (k,), (what, gb.shape, gs.shape, k)
    if k == 0:
        return 0
    bad = np.nonzero((gb.reshape(k, -1) != ref.hb.reshape(k, -1)).any(1))[0]
    assert len(bad) == 0, (what, "boxes differ from the host geometry", len(bad),
                           [(int(i), gb[i].tolist(), ref.hb[i].tolist(), ref.rb[i].tolist()) for i in bad[:5]])
    # where the host agrees with the oracle the device therefore does too; the residual rows are host-defined
    assert np.array_equal(gs[~ref.hkept], np.zeros(int((~ref.hkept).sum()), np.float32)), (what, "skipped-row scores")
    want = ref.scores
    exact = gs == want
    if is_quantised(ref.pred):
        bad = np.nonzero(~exact)[0]
        assert len(bad) == 0, (what, "scores on a quantised map", [(int(i), float(gs[i]), float(want[i])) for i in bad[:5]])
    else:
        ulp = np.spacing(np.maximum(np.abs(gs), np.abs(want)))
        bad = np.nonzero(np.abs(gs.astype(np.float64) - want) > ulp)[0]
        assert len(bad) == 0, (what, "scores beyond one ulp", [(int(i), float(gs[i]), float(want[i])) for i in bad[:5]])
        assert exact.sum() >= 0.999 * k, (what, "scores not bit-exact", int((~exact).sum()), k)
    return int(ref.resid.sum())


def assert_scores_within_ulp(a, b, what):
    """two runs of the same map: the double sums may only differ in their order"""
    assert a.shape == b.shape, what
    ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)))
    assert (np.abs(a.astype(np.float64) - b) <= ulp).all(), (what, float(np.abs(a - b).max()))
