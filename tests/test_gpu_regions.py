"""-m gpu: the text-line crops (`ctd_transform_regions`, csrc/region.cu) on the GPU.  Every comparison is exact:
the warp kernel alone against cv2.warpPerspective (+ cv2.rotate) sampling with cv2's own inverse; the detector's
batched `get_transformed_regions` and the per-line `TextBlock.get_transformed_region` against the cv2 restatement of
the reference method (tests/region_ref.py); and the crops against the reference's own (tests/golden/regions_ref.npz)."""
import os
import sys

import cv2
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctd_b200  # noqa: E402
from ctd_b200 import binding, compiler as cc  # noqa: E402
from ctd_b200 import textblock as tb  # noqa: E402
from oracle import synth  # noqa: E402
import region_cases as rc  # noqa: E402
import region_ref  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=64, max_w=64, skip_postproc=True)
    yield e
    e.close()


def plan_with_cv2_inverse(blocks, page, th):
    """native plan with every `inverse` replaced by cv2.invert of cv2.findHomography's matrix"""
    rec, keys = tb.region_lines(blocks)
    plan, total = binding.region_plan(rec, page.shape[1], page.shape[0], th)
    for (b, i), p in zip(keys, plan):
        if p["status"] == 0:
            r = region_ref.plan_line(blocks[b].lines, i, blocks[b].language, blocks[b].vertical, blocks[b].font_size,
                                     page.shape[1], page.shape[0], th)
            p["inverse"] = r["inverse"].reshape(-1)
    return plan, total


def check_kernel(eng, page, blocks, th, device_page=None):
    plan, total = plan_with_cv2_inverse(blocks, page, th)
    if device_page is None:
        out = eng.transform_regions(page, plan)
    else:
        out = eng.transform_regions(device_page.data_ptr(), plan, page_shape=page.shape[:2])
    assert out.nbytes == total
    n = 0
    for p in plan:
        if p["status"] != 0:
            continue
        o, hh, ww = int(p["offset"]), int(p["out_h"]), int(p["out_w"])
        got = out[o:o + hh * ww * 3].reshape(hh, ww, 3)
        ref = region_ref.warp_with_inverse(page, p["inverse"].reshape(3, 3), hh, ww, int(p["rotate"]))
        assert np.array_equal(got, ref), (n, hh, ww, int((got != ref).any(-1).sum()))
        n += 1
    return n


@pytest.mark.parametrize("th", [32, 48])
def test_kernel_hand_made_blocks(eng, th):
    """every branch: clipped expansion, float font size, vertical (rotated) crops, both page-sized crops, quads that
    cross every page border"""
    assert check_kernel(eng, rc.hand_page(), rc.hand_blocks(), th) == 15


def test_kernel_crossing_borders_and_vertical_lines(eng):
    page = synth.structured_page(5, 512, 640)
    blocks = []
    for x0, y0 in ((-80, -30), (560, -25), (-90, 480), (580, 470), (300, -40), (300, 490), (-70, 250), (600, 250)):
        blocks.append(rc.blk([rc.rect(x0, y0, x0 + 150, y0 + 40)], "ja", False, 20))
        blocks.append(rc.blk([rc.rect(x0, y0, x0 + 36, y0 + 170)], "ja", True, 20))
    assert check_kernel(eng, page, blocks, 48) == 16


def test_kernel_long_crop_on_non_net_sized_page(eng):
    """a ~48 x 4000 crop and a random mix of lines on a 1654 x 1170 page (the size of the reference's example page)"""
    page = synth.structured_page(9, 1170, 1654)
    long_line = rc.blk([[[20, 600], [1620, 590], [1620, 609], [20, 619]]], "ja", False, 20)
    plan, _ = binding.region_plan(tb.region_lines([long_line])[0], 1654, 1170, 48)
    assert int(plan[0]["out_h"]) == 48 and 3900 < int(plan[0]["out_w"]) < 4100
    from test_cpu_regions import random_quads
    assert check_kernel(eng, page, [long_line] + random_quads(3, 200, 1654, 1170), 48) > 190


def test_kernel_page_on_device(eng):
    torch = pytest.importorskip("torch")
    page = synth.structured_page(12, 1170, 1654)
    dev = torch.from_numpy(page).cuda()
    from test_cpu_regions import random_quads
    blocks = random_quads(4, 80, 1654, 1170) + [rc.hand_blocks()[7]]
    assert check_kernel(eng, page, blocks, 32, device_page=dev) > 70


def test_capacity_and_empty_plan(eng):
    page = rc.hand_page()
    plan, total = binding.region_plan(tb.region_lines(rc.hand_blocks()[:3])[0], 800, 600, 32)
    with pytest.raises(binding.CtdError, match="-5"):
        eng.transform_regions(page, plan, out=np.empty((total - 1,), np.uint8))
    assert eng.transform_regions(page, np.zeros((0,), binding.REGION_DTYPE)).nbytes == 0
    # only raising lines: nothing to warp, nothing written
    bad, t = binding.region_plan(tb.region_lines(rc.raising_blocks())[0], 800, 600, 32)
    assert t == 0 and eng.transform_regions(page, bad).nbytes == 0


@pytest.fixture(scope="module")
def detector():
    det = ctd_b200.TextDetector(synth.make_checkpoint(0, smooth=True), input_size=1024, act="leaky")
    yield det
    det.close()


@pytest.mark.parametrize("th", [32, 48])
@pytest.mark.parametrize("shape", [(1024, 1024), (1170, 1654)])
def test_end_to_end_detector_crops(detector, shape, th):
    page = synth.structured_page(1000 + shape[1] + th, *shape)
    _, _, blk_list = detector(page.copy())
    assert len(blk_list) > 3
    ref, raising = [], []
    for b, blk in enumerate(blk_list):
        ref.append([])
        for i in range(len(blk.lines)):
            try:
                ref[-1].append(region_ref.transformed_region(blk, page, i, th))
            except Exception:
                raising.append((b, i))
    if raising:   # the batched call refuses the page; check the remaining lines without the raising ones
        with pytest.raises(binding.CtdError, match="block %d, line %d" % raising[0]):
            detector.get_transformed_regions(page, blk_list, th)
        keep = [b for b in range(len(blk_list)) if not any(r[0] == b for r in raising)]
        blk_list, ref = [blk_list[b] for b in keep], [ref[b] for b in keep]
    got = detector.get_transformed_regions(page, blk_list, th)
    n = 0
    for b, (g, r) in enumerate(zip(got, ref)):
        assert len(g) == len(r) == len(blk_list[b].lines)
        for i, (x, y) in enumerate(zip(g, r)):
            assert x.shape == y.shape and np.array_equal(x, y), (b, i, x.shape, y.shape)
            n += 1
    assert n > 5
    # the per-line method (its own engine, one upload per call) returns the same bytes
    for b in (0, len(blk_list) - 1):
        for i in range(len(blk_list[b].lines)):
            assert np.array_equal(blk_list[b].get_transformed_region(page, i, th), got[b][i])


def test_golden_reference_crops(eng):
    z = np.load(rc.GOLD)
    n = 0
    for i in range(len(rc.PAGE_CASES)):
        page, blks, th = rc.page_case(i)
        got = tb.transformed_regions(eng, page, blks, th)
        for b, crops in enumerate(got):
            for l, c in enumerate(crops):
                assert np.array_equal(c, z["p%d_%d_%d" % (i, b, l)]), (i, b, l)
                n += 1
    page = rc.hand_page()
    for th in (32, 48):
        got = tb.transformed_regions(eng, page, rc.hand_blocks(), th)
        for b, crops in enumerate(got):
            for l, c in enumerate(crops):
                assert np.array_equal(c, z["h%d_%d_%d" % (th, b, l)]), (th, b, l)
                n += 1
        raised = []
        for b, blk in enumerate(rc.raising_blocks()):
            try:
                tb.transformed_regions(eng, page, [blk], th)
            except binding.CtdError:
                raised.append(b)
        assert raised == z["raises%d" % th].tolist()
    assert n == len([k for k in z.files if not k.startswith("raises")])
