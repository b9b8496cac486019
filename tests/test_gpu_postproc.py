"""-m gpu: integer / index post-processing kernels, bit-exact against the oracle."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=1024, max_w=1024, skip_postproc=True)
    yield e
    e.close()


def _blobs(rng, h, w, n=40):
    img = np.zeros((h, w), np.uint8)
    for _ in range(n):
        c = (int(rng.integers(0, w)), int(rng.integers(0, h)))
        ax = (int(rng.integers(2, 60)), int(rng.integers(2, 40)))
        cv2.ellipse(img, c, ax, float(rng.uniform(0, 180)), 0, 360, 255, -1 if rng.random() < 0.7 else 2)
    return img


CCL_IMAGES = {
    "noise30_1024": lambda r: (r.random((1024, 1024)) < 0.3).astype(np.uint8) * 255,
    "noise55_1024": lambda r: (r.random((1024, 1024)) < 0.55).astype(np.uint8),
    "blobs_1024": lambda r: _blobs(r, 1024, 1024, 120),
    "blobs_odd": lambda r: _blobs(r, 173, 95, 12),
    "tiny": lambda r: (r.random((3, 5)) < 0.5).astype(np.uint8),
    "empty": lambda r: np.zeros((64, 64), np.uint8),
    "full": lambda r: np.full((70, 33), 255, np.uint8),
    "checker": lambda r: ((np.indices((128, 128)).sum(0) % 2) * 255).astype(np.uint8),
    "stripes": lambda r: np.tile(np.array([[255, 0]], np.uint8), (64, 40)),
    "diag_pair": lambda r: np.array([[255, 0], [0, 255]], np.uint8),
    "spiral": lambda r: cv2.resize(_blobs(r, 64, 64, 10), (640, 384), interpolation=cv2.INTER_NEAREST),
}


@pytest.mark.parametrize("name", list(CCL_IMAGES))
def test_ccl_matches_cv2(eng, name):
    img = CCL_IMAGES[name](np.random.default_rng(abs(hash(name)) % 2**31 if False else sum(map(ord, name))))
    n_ref, lab_ref, stats_ref, _ = postproc_ref.connected_components_cv2(img)
    n, lab, stats = eng.connected_components(img, stats_cap=max(n_ref, 1) + 4)
    assert n == n_ref
    assert np.array_equal(lab, lab_ref)
    if img.any() and not img.all():
        assert np.array_equal(stats[:n_ref], stats_ref)
    else:
        assert np.array_equal(stats[:n_ref, 4], stats_ref[:, 4])


def _pred(rng, rows, n_obj, nc=2):
    p = np.zeros((rows, 5 + nc), np.float32)
    p[:, 0] = rng.uniform(0, 1024, rows)
    p[:, 1] = rng.uniform(0, 1024, rows)
    p[:, 2] = rng.uniform(4, 300, rows)
    p[:, 3] = rng.uniform(4, 300, rows)
    p[:, 4] = rng.uniform(0, 0.39, rows)
    p[:, 5:] = rng.uniform(0, 1, (rows, nc))
    hot = rng.choice(rows, n_obj, replace=False)
    p[hot, 4] = rng.uniform(0.3, 1.0, n_obj)
    # clusters of near-duplicates so that suppression really happens
    for k in hot[: n_obj // 2]:
        j = int(rng.integers(0, rows))
        p[j] = p[k]
        p[j, :4] += rng.normal(0, 3, 4).astype(np.float32)
        p[j, 4] = min(1.0, p[k, 4] * float(rng.uniform(0.8, 1.2)))
    return p.astype(np.float32)


@pytest.mark.parametrize("rows,n_obj,seed", [(64512, 200, 0), (64512, 1500, 1), (64512, 0, 2), (1000, 900, 3), (64512, 3500, 4)])
def test_nms_matches_reference(eng, rows, n_obj, seed):
    rng = np.random.default_rng(seed)
    pred = _pred(rng, rows, n_obj)
    if seed == 3:  # exact score ties: stable order must decide
        pred[:, 4] = np.round(pred[:, 4], 1)
        pred[:, 5:] = 1.0
    ref = postproc_ref.non_max_suppression(torch.from_numpy(pred)[None], 0.4, 0.35)[0].numpy()
    got = eng.nms(pred, 0.4, 0.35)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("seed,ties", [(10, False), (11, True)])
def test_nms_candidate_overflow_is_deterministic_top_by_score(eng, seed, ties):
    """More candidates than the 4096-slot workspace (ADVICE r1: the atomicAdd slot race made the survivors depend on
    thread scheduling): the engine must keep exactly the 4096 best rows by (score descending, row ascending), i.e.
    equal the reference NMS run on that subset, report the true count, and repeat bit-identically."""
    rng = np.random.default_rng(seed)
    rows = 64512
    pred = _pred(rng, rows, 9000)
    if ties:   # many exact ties straddling the cut: the lowest rows must win
        pred[:, 4] = np.round(pred[:, 4], 2)
        pred[:, 5:] = 1.0
    obj = pred[:, 4]
    score = (pred[:, 5:] * obj[:, None]).max(1)
    cand = np.where((obj > 0.4) & (score > 0.4))[0]
    assert len(cand) > 4096
    order = cand[np.lexsort((cand, -score[cand]))][:4096]
    sub = pred[np.sort(order)]
    ref = postproc_ref.non_max_suppression(torch.from_numpy(sub)[None], 0.4, 0.35)[0].numpy()
    got = eng.nms(pred, 0.4, 0.35)
    tot, cap = eng.nms_status()
    assert cap == 4096 and int(tot[0]) == len(cand)
    assert got.shape == ref.shape and np.array_equal(got, ref)
    for _ in range(3):
        assert np.array_equal(eng.nms(pred, 0.4, 0.35), got)


# ---------------------------------------------------------------------------------------------------
import seg_geometry as sg  # noqa: E402
import stress_maps  # noqa: E402


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return sg.build_host_geom(tmp_path_factory.mktemp("geom"))


@pytest.mark.parametrize("name", list(stress_maps.CASES))
def test_seg_represent_matches_oracle(eng, geom, name):
    """SegDetectorRepresenter on stage-isolated maps.  Contour count and order and skipped rows exact; every int16 box
    equals the host build of the same geometry (csrc/geom.h) on cv2's contours bit for bit, and on these maps the host
    equals the oracle on every contour; scores within one float32 ulp of cv2's mean (tests/seg_geometry.py)."""
    pred = stress_maps.CASES[name]()
    ref = sg.Reference(geom, pred)
    gb, gs = eng.seg_represent(pred, 0.3)
    assert sg.assert_text_lines(ref, gb, gs, name) == 0
