"""-m gpu: refine_mask (csrc/refine_mk.cu) against the oracle, byte for byte and in both refine modes, over the window
shapes the engine can be given (tests/refine_shape_cases.py): windows 1 - 7 px wide and high at every alignment and
against every page edge, the 2-px-wide windows refine_undetected_mask produces, every width at which
refine_rows_per_chunk changes (chunks of 8 down to 1 rows, whose starts fall off 4- and 32-pixel boundaries), dense
noise with thousands of 1 - 3 pixel components and the hole filling's edge cases, and a seeded random sweep.  Also the
one window on which the engine once differed from the oracle in one pixel (tests/golden/refine_finding.npz)."""
import os

import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import postproc_ref
import refine_shape_cases as rc

pytestmark = pytest.mark.gpu

MODES = pytest.mark.parametrize("mode", [0, 1], ids=["inpaint", "annotation"])


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=1024, max_w=1024, skip_postproc=True)
    yield e
    e.close()


def mismatch(eng, img, mask, wins, mode):
    """(oracle result, '' or a description of the pixels in which the engine differs and the windows that hold them)"""
    ref = rc.oracle_refine_windows(img, mask, wins, mode)
    got = eng.refine_mask(img, mask, wins, mode)
    if np.array_equal(got, ref):
        return ref, ""
    bad = [w for w in wins if (got[w[1]:w[3], w[0]:w[2]] != ref[w[1]:w[3], w[0]:w[2]]).any()]
    return ref, "%d px differ in %d windows, e.g. %s" % (int((got != ref).sum()), len(bad), bad[:4])


def check(eng, img, mask, wins, mode, what):
    ref, msg = mismatch(eng, img, mask, wins, mode)
    assert not msg, "%s, mode %d: %s" % (what, mode, msg)
    return ref


@MODES
@pytest.mark.parametrize("rh", rc.TINY)
def test_tiny_windows(eng, rh, mode):
    merged, fails, x1_mod, edges = 0, [], set(), set()
    for rw in rc.TINY:
        img, mask, wins = rc.tiny_case(rw, rh)
        h, w = mask.shape
        x1_mod |= {wn[0] % 32 for wn in wins}
        edges |= {e for wn in wins for e, at in (("left", wn[0] == 0), ("top", wn[1] == 0), ("right", wn[2] == w - 1),
                                                   ("bottom", wn[3] == h - 1)) if at}
        ref, msg = mismatch(eng, img, mask, wins, mode)
        if msg:
            fails.append("%d x %d windows: %s" % (rw, rh, msg))
        merged += int(np.count_nonzero(ref))
    assert x1_mod >= {0, 1, 30, 31} and edges == {"left", "top", "right", "bottom"}
    assert not fails, fails
    assert merged > 0 or rh == 1     # in one row every shape is 1 x 1 or 1 x 2: the w*h < 3 rule skips them all


@MODES
def test_two_wide_windows(eng, mode):
    img, mask, wins = rc.two_wide_case()
    for x1, y1, x2, y2 in wins:
        # the block of a 2 x 26 component is its own window: padding round((26 * 0.25 + 2 * 0.75) / 16) = 0
        assert postproc_ref.expand_textwindow(img.shape, [x1, y1, x2, y2], expand_r=16) == [x1, y1, x2, y2]
    ref = check(eng, img, mask, wins, mode, "2-px-wide windows")
    # the anti-diagonal pairs (2 x 2 boxes) merge, the horizontal and vertical pairs (1 x 2, 2 x 1) do not
    x1, y1 = wins[0][:2]
    assert ref[y1 + 2, x1 + 1] and ref[y1 + 3, x1] and not ref[y1 + 20, x1] and not ref[y1 + 20, x1 + 1]


@MODES
def test_rows_per_chunk_regimes(eng, mode):
    img, mask, wins = rc.seam_case()
    for rw, rp in rc.SEAM_ROWS.items():
        assert rc.rows_per_chunk(rw) == rp
    for (x1, y1, x2, y2), (rw, rp) in zip(wins, rc.SEAM_ROWS.items()):
        assert x2 - x1 == rw and (y2 - y1) > 3 * rp           # at least three chunk seams... and a partial chunk
    check(eng, img, mask, wins, mode, "chunk seams")


@MODES
def test_dense_noise(eng, mode):
    for seed in range(4):
        img, mask, wins = rc.noise_case(seed)
        check(eng, img, mask, wins, mode, "noise seed %d" % seed)


@MODES
def test_seeded_sweep(eng, mode):
    fails = []
    for seed in range(25):
        img, mask, wins = rc.sweep_case(100 * mode + seed)
        ref = rc.oracle_refine_windows(img, mask, wins, mode)
        got = eng.refine_mask(img, mask, wins, mode)
        if not np.array_equal(got, ref):
            for w in wins:     # each window alone, to name the one that differs
                r1 = rc.oracle_refine_windows(img, mask, [w], mode)
                g1 = eng.refine_mask(img, mask, [w], mode)
                if not np.array_equal(g1, r1):
                    fails.append("seed %d window %s: %d px" % (100 * mode + seed, w, int((g1 != r1).sum())))
            if not fails:
                fails.append("seed %d: %d px differ in the launch of all its windows only" % (100 * mode + seed,
                                                                                              int((got != ref).sum())))
    assert not fails, fails


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_finding.npz")


def test_one_pixel_finding(eng):
    """The second refine_mask of refine_undetected_mask on structured_page(42, 413, 292) at input size 256,
    REFINEMASK_ANNOTATION (scripts/capture_refine_finding.py): the engine once set pixel (y 91, x 169) of the window
    (0, 0)-(291, 349), whose colour BGR (102, 59, 61) it turned into grey 65 with OpenCV's 14-bit coefficients where
    cv2 gives 64.  tests/test_cpu_refine_shapes.py holds the oracle to the reference's answer on the same inputs."""
    from oracle import synth
    d = np.load(GOLD)
    page, mask, blocks = synth.structured_page(42, 413, 292), d["mask"], d["blocks"].tolist()
    wins = [postproc_ref.expand_textwindow(page.shape, b, expand_r=16) for b in blocks]
    assert len(blocks) == 29 and [0, 0, 291, 349] in wins
    ref = postproc_ref.refine_mask(page, mask, blocks, 1)
    got = eng.refine_mask(page, mask, wins, 1)
    assert np.array_equal(got, ref), int((got != ref).sum())
