"""-m gpu: the DB post-processing's connected components and text lines at the places its labelling splits the page: the
32 x 32-pixel tile seams of the foreground (8-connected) and background (4-connected) passes, diagonal-only contacts
exactly on a seam, rings that straddle one, a component over every tile of a page, deep nesting, and widths that are not
multiples of 32.  Labels and counts against cv2, text lines against the host geometry and cv2's scores
(tests/seg_geometry.py).  The OpenCV-numbered label plane of a forward is built when `db_components` asks for it: it is
asked twice after one forward, and after a `submit_full` batch."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref, synth
import seg_geometry as sg
from util import get_checkpoint

pytestmark = pytest.mark.gpu


def rect(m, x0, y0, x1, y1, v=1):
    """inclusive corners"""
    m[y0:y1 + 1, x0:x1 + 1] = v


def seam_holes(h=256, w=256):
    """rings and holes whose edges sit on and across the seams at multiples of 32"""
    m = np.zeros((h, w), np.uint8)
    rect(m, 20, 20, 100, 76)
    rect(m, 31, 31, 64, 64, 0)            # a hole from the last pixel of one tile to the first of the next
    rect(m, 66, 24, 96, 72, 0)            # a hole that crosses a horizontal and a vertical seam
    rect(m, 40, 40, 56, 56)               # an island in the first hole
    rect(m, 128, 0, 160, 255)             # a bar over every tile row that touches the frame
    rect(m, 140, 31, 150, 32, 0)          # a 2-row hole split by a seam
    rect(m, 170, 95, 250, 97)             # a 3-row bar over the seam at y = 96
    return m


def diagonal_seams(h=128, w=128):
    """components that touch only diagonally, exactly at a seam (one foreground component, by 8-connectivity), and two
    holes that touch only diagonally at a seam corner (two holes, by 4-connectivity)"""
    m = np.zeros((h, w), np.uint8)
    rect(m, 10, 10, 31, 31)
    rect(m, 32, 32, 50, 50)               # diagonal at the corner of four tiles
    rect(m, 70, 20, 95, 40)
    rect(m, 96, 41, 120, 60)              # diagonal across the vertical seam x = 96 only
    rect(m, 4, 70, 60, 124)
    rect(m, 10, 76, 31, 95, 0)            # two holes, diagonal at the seam corner (31, 95) / (32, 96)
    rect(m, 32, 96, 54, 118, 0)
    return m


def thin_ring(h=96, w=96):
    """a one-pixel ring whose pixels lie on both sides of the seams x = 32, 64 and y = 32, 64"""
    m = np.zeros((h, w), np.uint8)
    rect(m, 31, 31, 64, 64)
    rect(m, 32, 32, 63, 63, 0)
    rect(m, 47, 47, 48, 48)
    return m


def mesh(h=512, w=512, pitch=24):
    """one component over every tile of the page: a lattice whose cells are holes"""
    m = np.zeros((h, w), np.uint8)
    m[::pitch, :] = 1
    m[:, ::pitch] = 1
    m[:, -1] = 1
    m[-1, :] = 1
    return m


def nested(h=300, w=300, levels=7):
    """square rings inside each other, alternating foreground and background, off the seams"""
    m = np.zeros((h, w), np.uint8)
    for k in range(levels * 2):
        rect(m, 7 + 9 * k, 5 + 9 * k, w - 1 - 11 - 9 * k, h - 1 - 13 - 9 * k, 1 - k % 2)
    return m


def blobs(h, w, seed, n=12):
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), np.uint8)
    for _ in range(n):
        c = (int(rng.integers(0, w)), int(rng.integers(0, h)))
        ax = (int(rng.integers(1, max(2, w // 4))), int(rng.integers(1, max(2, h // 4))))
        cv2.ellipse(m, c, ax, float(rng.uniform(0, 180)), 0, 360, 1, -1 if rng.random() < 0.6 else 1)
    return m


def noise(h, w, seed, p=0.45):
    return (np.random.default_rng(seed).random((h, w)) < p).astype(np.uint8)


MASKS = {
    "seam_holes": seam_holes,
    "diagonal_seams": diagonal_seams,
    "thin_ring": thin_ring,
    "mesh": mesh,
    "nested": nested,
    "blobs_37x41": lambda: blobs(37, 41, 1),
    "noise_37x41": lambda: noise(37, 41, 2),
    "blobs_3x2000": lambda: blobs(3, 2000, 3, 60),
    "blobs_2000x3": lambda: blobs(2000, 3, 4, 60),
    "noise_1x2000": lambda: noise(1, 2000, 5),
    "noise_2000x1": lambda: noise(2000, 1, 6),
}
# host-vs-oracle residuals (an exact minAreaRect area tie), pinned as in test_gpu_seg_geometry.py
RESIDUALS = {"blobs_3x2000": 1}
CC_ONLY = {
    "noise_1x5000": lambda: noise(1, 5000, 7),
    "noise_5000x1": lambda: noise(5000, 1, 8),
    "noise_33x4097": lambda: noise(33, 4097, 9, 0.6),
}


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=2048, max_w=2048, skip_postproc=True)
    yield e
    e.close()


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return sg.build_host_geom(tmp_path_factory.mktemp("geom"))


def test_crafted_masks_hold_their_property():
    """each map is what its name says: cv2 sees one foreground component over the diagonal seam contacts and two holes
    that touch only diagonally; the mesh is one component"""
    n, _, _, _ = postproc_ref.connected_components_cv2(diagonal_seams()[:64, :64])
    assert n == 2
    n, _, _, _ = postproc_ref.connected_components_cv2(diagonal_seams()[:64, 64:])
    assert n == 2
    bg = (diagonal_seams()[70:125, 4:61] == 0).astype(np.uint8)
    nb, _ = cv2.connectedComponents(bg, connectivity=4)
    assert nb - 1 == 2
    n, _, _, _ = postproc_ref.connected_components_cv2(mesh())
    assert n == 2


@pytest.mark.parametrize("name", list(MASKS) + list(CC_ONLY))
def test_components_match_cv2(eng, name):
    m = {**MASKS, **CC_ONLY}[name]() * 255
    n_ref, lab_ref, stats_ref, _ = postproc_ref.connected_components_cv2(m)
    n, lab, stats = eng.connected_components(m, stats_cap=n_ref + 4)
    assert n == n_ref
    assert np.array_equal(lab, lab_ref)
    assert np.array_equal(stats[1:n_ref], stats_ref[1:])


@pytest.mark.parametrize("name", list(MASKS))
def test_text_lines_match_oracle(eng, geom, name):
    m = MASKS[name]()
    rng = np.random.default_rng(len(name))
    pred = sg.quantise(np.where(m > 0, rng.uniform(0.31, 1.0, m.shape), rng.uniform(0.0, 0.29, m.shape)))
    ref = sg.Reference(geom, pred)
    gb, gs = eng.seg_represent(pred, 0.3)
    assert sg.assert_text_lines(ref, gb, gs, name) == RESIDUALS.get(name, 0)


@pytest.fixture(scope="module")
def prog():
    return cc.compile_checkpoint(get_checkpoint(0, True))


def _check_components(e, what):
    bm, lab, nl = e.db_components()
    for i in range(bm.shape[0]):
        n_ref, lab_ref, _, _ = postproc_ref.connected_components_cv2(bm[i])
        assert int(nl[i]) == n_ref and n_ref > 2, (what, i)
        assert np.array_equal(lab[i], lab_ref), (what, i)
    return lab


def test_db_components_on_demand(prog):
    """labels built on demand equal cv2's on the forward's own bitmap, asked twice after one forward, and after a
    submit_full batch of other pages (whose bitmap and labels they then are)"""
    n, s = 3, 512
    e = ctd_b200.Engine(prog, max_batch=n, max_h=s, max_w=s, use_graph=True)
    try:
        pages = np.stack([synth.structured_page(2000 + i, s, s) for i in range(n)])
        e.forward(pages)
        lab1 = _check_components(e, "first call")
        lab2 = _check_components(e, "second call")
        assert np.array_equal(lab1, lab2)
        lay = e.results_layout()
        out = torch.empty((lay["total_bytes"],), dtype=torch.uint8).pin_memory()
        other = torch.from_numpy(np.stack([synth.structured_page(2100 + i, s, s) for i in range(n)])).pin_memory()
        e.submit_full(0, other.data_ptr(), n, s, s, out.data_ptr())
        e.collect(0)
        lab3 = _check_components(e, "after submit_full")
        assert not np.array_equal(lab3, lab1)
    finally:
        e.close()
