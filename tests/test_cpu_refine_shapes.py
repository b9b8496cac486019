"""not-gpu: the oracle's refine_mask (oracle/postproc_ref.py, numpy's own argsort tie order) on the window shapes of
tests/refine_shape_cases.py against the UNMODIFIED reference (`utils.textmask.refine_mask`): windows 1 - 7 px wide and
high including the 2-px-wide windows with anti-diagonal pairs, a window that merges entirely, two holes tied for the
largest area, and noise windows.  The reference expands every block it is given, so the tiny windows are blocks whose
expand_textwindow padding rounds to 0 (asserted).  Where the reference is absent the oracle is held to digests it
produced (tests/golden/refine_shapes_pins.json, written by `python tests/test_cpu_refine_shapes.py --regen` where the
reference exists, after checking every case against it)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import refine_shape_cases as rc  # noqa: E402
from oracle import postproc_ref, ref_shim  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_shapes_pins.json")
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="the reference tree is not present")


class _Blk:
    def __init__(self, xyxy):
        self.xyxy = xyxy


def _digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha1(a.tobytes()).hexdigest()[:16] + ":%d" % int(np.count_nonzero(a))


def cases():
    """name -> (img, mask, blocks, tiny): every rw x rh of tiny windows, the 2-px-wide windows, and the noise cases"""
    out = {}
    for rw in rc.TINY:
        for rh in rc.TINY:
            out["tiny_%dx%d" % (rw, rh)] = rc.tiny_case(rw, rh) + (True,)
    out["two_wide"] = rc.two_wide_case() + (True,)
    for seed in range(2):
        out["noise_%d" % seed] = rc.noise_case(seed) + (False,)
    return out


def oracle(img, mask, blocks, mode):
    return postproc_ref.refine_mask(img, mask.copy(), blocks, mode, tie_order="numpy")


def records():
    return {"%s/%d" % (name, mode): _digest(oracle(img, mask, blocks, mode))
            for name, (img, mask, blocks, _tiny) in cases().items() for mode in (0, 1)}


@needs_ref
@pytest.mark.parametrize("mode", [0, 1])
def test_oracle_equals_reference_on_window_shapes(mode):
    ns = ref_shim.load()
    for name, (img, mask, blocks, tiny) in cases().items():
        if tiny:
            for b in blocks:
                assert postproc_ref.expand_textwindow(img.shape, b, expand_r=16) == b, (name, b)
        ref = ns.textmask.refine_mask(img, mask.copy(), [_Blk(b) for b in blocks], refine_mode=mode)
        got = oracle(img, mask, blocks, mode)
        assert np.array_equal(ref, got), (name, int((ref != got).sum()))


def test_two_wide_anti_diagonal_pairs_merge():
    """the case the engine's w*h < 3 test once got wrong: in the reference's terms the anti-diagonal pair is a 2 x 2 box"""
    img, mask, wins = rc.two_wide_case()
    out = oracle(img, mask, wins, 1)
    x1, y1 = wins[0][:2]
    assert out[y1 + 2, x1 + 1] and out[y1 + 3, x1] and out[y1 + 9, x1 + 1] and out[y1 + 10, x1]
    assert not out[y1 + 20, x1] and not out[y1 + 20, x1 + 1]


def test_noise_edge_windows():
    """the hole filling's edge windows of noise_case: the tie window's halves stay open, the dark window merges
    entirely, the light one not at all"""
    img, mask, wins = rc.noise_case(0)
    for mode in (0, 1):
        tie, _one, full, empty = wins[-4:]
        out = np.zeros_like(mask)
        for w in (tie, full, empty):
            out |= rc.oracle_refine_windows(img, mask, [w], mode)
        x1, y1, x2, y2 = full
        assert out[y1:y2, x1:x2].all()
        x1, y1, x2, y2 = empty
        assert not out[y1:y2, x1:x2].any()
        x1, y1, x2, y2 = tie
        assert not out[y1 + 15, x1 + 1] and not out[y1 + 15, x1 + 29]


def test_one_pixel_finding_equals_reference_answer():
    """tests/golden/refine_finding.npz: refine_undetected_mask's second refine_mask on structured_page(42, 413, 292)
    (the page mask after the in-place edit, the blocks) and the reference's answer on them
    (oracle/make_refine_finding_ref.py); the stable histogram tie order changes 6 of its pixels"""
    from oracle import synth
    d = np.load(os.path.join(os.path.dirname(GOLD), "refine_finding.npz"))
    page, blocks = synth.structured_page(42, 413, 292), d["blocks"].tolist()
    assert np.array_equal(postproc_ref.refine_mask(page, d["mask"].copy(), blocks, 1, tie_order="numpy"), d["reference"])
    stable = postproc_ref.refine_mask(page, d["mask"].copy(), blocks, 1)
    assert int((stable != d["reference"]).sum()) == 6 and not stable[91, 169]


def test_oracle_matches_reference_digests():
    """runs everywhere: the digests were checked against the reference when written"""
    assert records() == json.load(open(GOLD))


if __name__ == "__main__":
    if "--regen" in sys.argv:
        assert ref_shim.available(), "regenerate where the reference tree exists"
        ns = ref_shim.load()
        for name, (img, mask, blocks, _tiny) in cases().items():
            for mode in (0, 1):
                ref = ns.textmask.refine_mask(img, mask.copy(), [_Blk(b) for b in blocks], refine_mode=mode)
                assert np.array_equal(ref, oracle(img, mask, blocks, mode)), (name, mode)
        json.dump(records(), open(GOLD, "w"), indent=1, sort_keys=True)
        print("wrote", GOLD)
