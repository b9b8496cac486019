"""not-gpu: the host side of the text-line crops (`TextBlock.get_transformed_region`, reference
utils/textblock.py:162-194).  `ctd_region_plan` (csrc/region_plan.cpp) must give the same shapes, rotation and
status as the reference and homographies / inverses BIT-IDENTICAL to cv2.findHomography(src, dst, RANSAC, 5.0) and
cv2.invert(M, DECOMP_LU); the cv2 restatement (tests/region_ref.py) must equal the reference's crops byte for byte;
and a numpy model of the warp kernel's arithmetic (csrc/region.cu) must equal cv2.warpPerspective, which pins the
order in which the kernel groups its double-precision sums."""
import os
import sys

import cv2
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ctd_b200 import binding  # noqa: E402
from ctd_b200 import textblock as tb  # noqa: E402
from oracle import ref_shim  # noqa: E402
import region_cases as rc  # noqa: E402
import region_ref  # noqa: E402
from test_cpu_textblock import make_case  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="/root/reference not present on this box")


def check_plan(blocks, im_w, im_h, th):
    """native plan of every line vs region_ref.plan_line; returns (lines checked, lines with status 0)"""
    rec, keys = tb.region_lines(blocks)
    plan, total = binding.region_plan(rec, im_w, im_h, th)
    off = 0
    n_ok = 0
    for (b, i), p in zip(keys, plan):
        blk = blocks[b]
        r = region_ref.plan_line(blk.lines, i, blk.language, blk.vertical, blk.font_size, im_w, im_h, th)
        assert int(p["status"]) == r["status"], (b, i, int(p["status"]), r)
        assert int(p["offset"]) == off
        if r["status"] != 0:
            continue
        n_ok += 1
        assert (int(p["out_h"]), int(p["out_w"]), int(p["rotate"])) == (r["out_h"], r["out_w"], r["rotate"]), (b, i)
        assert np.array_equal(p["homography"], r["homography"].reshape(-1)), (b, i, p["homography"], r["homography"])
        assert np.array_equal(p["inverse"], r["inverse"].reshape(-1)), (b, i)
        off += r["out_h"] * r["out_w"] * 3
    assert total == off
    return len(keys), n_ok


@pytest.mark.parametrize("th", [32, 48])
def test_plan_matches_cv2_on_group_output_lines(th):
    n = 0
    for seed in range(24):
        blks, lines, w, h, mask = make_case(seed)
        blocks = tb.group_output(blks, lines, w, h, mask)
        n += check_plan(blocks, w, h, th)[0]
    assert n > 300


def random_quads(seed, n, im_w, im_h):
    """n single-line blocks: integer axis-aligned rectangles, integer rotated quads and float rotated quads, all three
    languages, both directions, int and float font sizes"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        cx, cy = rng.uniform(0, im_w), rng.uniform(0, im_h)
        lw, lh = rng.uniform(10, 500), rng.uniform(8, 64)
        if rng.random() < 0.5:
            lw, lh = lh, lw
        if k % 3 == 0:
            x0, y0 = int(cx), int(cy)
            q = rc.rect(x0, y0, x0 + int(lw), y0 + int(lh))
        else:
            a = rng.normal(0, 0.3)
            u = np.array([np.cos(a), np.sin(a)]) * lw / 2
            v = np.array([-np.sin(a), np.cos(a)]) * lh / 2
            c = np.array([cx, cy])
            q = np.array([c - u - v, c + u - v, c + u + v, c - u + v])
            q = np.round(q).astype(int) if k % 3 == 1 else q
        fs = int(rng.integers(6, 64)) if rng.random() < 0.7 else float(rng.uniform(6, 64))
        out.append(rc.blk([q], region_ref.LANG_LIST[int(rng.integers(0, 3))], rng.random() < 0.4, fs))
    return out


@pytest.mark.parametrize("th", [32, 48])
@pytest.mark.parametrize("page", [(1024, 1024), (1654, 1170)])
def test_plan_matches_cv2_on_random_quads(th, page):
    """1500 quads per page and textheight: no exceptions (every matrix bit-identical)"""
    im_w, im_h = page
    n, n_ok = check_plan(random_quads(th + im_w, 1500, im_w, im_h), im_w, im_h, th)
    assert n == 1500 and n_ok > 1400


@pytest.mark.parametrize("th", [32, 48])
def test_plan_hand_made_and_raising_lines(th):
    check_plan(rc.hand_blocks() + rc.raising_blocks(), 800, 600, th)


def test_quirk_expansion_clipped_at_page_size():
    """the expanded corners are clipped to [0, im_w] x [0, im_h], not im_w - 1 / im_h - 1"""
    b = rc.hand_blocks()[1]
    src, _, _, _ = region_ref._geometry(b.lines, 0, b.language, b.vertical, b.font_size, 800, 600, 32)
    assert src[:, 0].max() == 800 and src[:, 1].max() == 600
    assert check_plan([b], 800, 600, 32) == (1, 1)


def test_quirk_float_font_size():
    b = rc.hand_blocks()[2]
    assert isinstance(b.font_size, float) and b.font_size / 3 != b.font_size // 3
    assert check_plan([b], 800, 600, 48) == (2, 2)


@pytest.mark.parametrize("vertical", [False, True])
def test_quirk_size_zero_gives_page_sized_crop(vertical):
    b = rc.hand_blocks()[8 if vertical else 7]
    plan, total = binding.region_plan(tb.region_lines([b])[0], 800, 600, 32)
    assert int(plan[0]["status"]) == 0 and int(plan[0]["rotate"]) == int(vertical)
    assert (int(plan[0]["out_h"]), int(plan[0]["out_w"])) == ((800, 600) if vertical else (600, 800))
    assert total == 800 * 600 * 3


def test_quirk_size_one_and_degenerate_quads_raise():
    plan, total = binding.region_plan(tb.region_lines(rc.raising_blocks())[0], 800, 600, 32)
    assert plan["status"].tolist() == [1, 1, 1] and total == 0
    for b in rc.raising_blocks():
        with pytest.raises(Exception):
            region_ref.transformed_region(b, rc.hand_page(), 0, 32)
    # the python surface refuses before it needs a GPU, naming the block and the line
    with pytest.raises(binding.CtdError, match="block 1, line 0"):
        tb.transformed_regions(None, rc.hand_page(), rc.hand_blocks()[:1] + rc.raising_blocks(), 32)


def test_textheight_below_two_and_non_integer_rejected():
    rec = tb.region_lines(rc.hand_blocks())[0]
    for th in (1, 0, -5):
        with pytest.raises(binding.CtdError):
            binding.region_plan(rec, 800, 600, th)
    with pytest.raises(ValueError):
        tb.transformed_regions(None, rc.hand_page(), rc.hand_blocks(), 32.5)
    assert tb._check_textheight(48.0) == 48 and tb._check_textheight(np.int64(32)) == 32


def test_plan_of_no_lines():
    plan, total = binding.region_plan(np.zeros((0,), binding.REGION_LINE_DTYPE), 800, 600, 32)
    assert len(plan) == 0 and total == 0


def kernel_model(img, Mi, ww, wh):
    """numpy restatement of k_warp_regions (csrc/region.cu) for one un-rotated crop: OpenCV's per-block grouping of
    the double sums, rint to 1/32 px, the 15-bit bilinear weights, BORDER_CONSTANT 0 per tap"""
    ih, iw = img.shape[:2]
    bh0 = min(16, wh)
    bw0 = min(1024 // bh0, ww)
    y, x = np.mgrid[0:wh, 0:ww].astype(np.int64)
    xb = (x // bw0) * bw0
    x1 = x - xb
    X0 = (Mi[0] * xb + Mi[1] * y) + Mi[2]
    Y0 = (Mi[3] * xb + Mi[4] * y) + Mi[5]
    W = ((Mi[6] * xb + Mi[7] * y) + Mi[8]) + Mi[6] * x1
    W = np.where(W != 0, 32.0 / np.where(W != 0, W, 1), 0)
    X = np.rint(np.clip((X0 + Mi[0] * x1) * W, -2 ** 31, 2 ** 31 - 1)).astype(np.int64)
    Y = np.rint(np.clip((Y0 + Mi[3] * x1) * W, -2 ** 31, 2 ** 31 - 1)).astype(np.int64)
    sx, sy, fx, fy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767), X & 31, Y & 31
    acc = np.zeros((wh, ww, 3), np.int64)
    for dy, dx, wgt in ((0, 0, (32 - fy) * (32 - fx)), (0, 1, (32 - fy) * fx), (1, 0, fy * (32 - fx)), (1, 1, fy * fx)):
        xx, yy = sx + dx, sy + dy
        inside = (xx >= 0) & (xx < iw) & (yy >= 0) & (yy < ih)
        v = img[np.clip(yy, 0, ih - 1), np.clip(xx, 0, iw - 1)].astype(np.int64) * inside[..., None]
        acc += v * (wgt * 32)[..., None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def test_kernel_arithmetic_model_matches_cv2_warp():
    """the kernel's sum grouping (per OpenCV pixel block) reproduces cv2.warpPerspective on crops of every width
    class, crossing the page borders; grouping by the absolute x instead does not (it differs on a few pixels)"""
    page = rc.hand_page()
    blocks = random_quads(7, 60, 800, 600) + rc.hand_blocks()
    rec, keys = tb.region_lines(blocks)
    plan, _ = binding.region_plan(rec, 800, 600, 48)
    n_px = 0
    for (b, i), p in zip(keys, plan):
        if p["status"] != 0 or p["out_h"] * p["out_w"] > 200000:
            continue
        blk = blocks[b]
        ref = region_ref.transformed_region(blk, page, i, 48)
        ww, wh = (int(p["out_h"]), int(p["out_w"])) if p["rotate"] else (int(p["out_w"]), int(p["out_h"]))
        got = kernel_model(page, p["inverse"], ww, wh)
        if p["rotate"]:
            got = cv2.rotate(got, cv2.ROTATE_90_COUNTERCLOCKWISE)
        assert np.array_equal(got, ref), (b, i, int((got != ref).any(-1).sum()))
        n_px += got.shape[0] * got.shape[1]
    assert n_px > 300000


def golden_items():
    z = np.load(rc.GOLD)
    for i in range(len(rc.PAGE_CASES)):
        page, blks, th = rc.page_case(i)
        for b, blk in enumerate(blks):
            for l in range(len(blk.lines)):
                yield "p%d_%d_%d" % (i, b, l), page, blk, l, th, z
    page = rc.hand_page()
    for th in (32, 48):
        for b, blk in enumerate(rc.hand_blocks()):
            for l in range(len(blk.lines)):
                yield "h%d_%d_%d" % (th, b, l), page, blk, l, th, z


def test_restatement_equals_golden():
    n = 0
    for key, page, blk, l, th, z in golden_items():
        got = region_ref.transformed_region(blk, page, l, th)
        assert got.dtype == np.uint8 and np.array_equal(got, z[key]), key
        n += 1
    z = np.load(rc.GOLD)
    assert n == len([k for k in z.files if not k.startswith("raises")]) and n > 90
    for th in (32, 48):
        raised = []
        for b, blk in enumerate(rc.raising_blocks()):
            try:
                region_ref.transformed_region(blk, rc.hand_page(), 0, th)
            except Exception:
                raised.append(b)
        assert raised == z["raises%d" % th].tolist()


@needs_ref
def test_restatement_equals_reference():
    ns = ref_shim.load()
    for key, page, blk, l, th, _z in golden_items():
        ref = ns.textblock.TextBlock([0, 0, 0, 0], lines=blk.lines, language=blk.language, vertical=blk.vertical,
                                     font_size=blk.font_size)
        assert np.array_equal(region_ref.transformed_region(blk, page, l, th), ref.get_transformed_region(page, l, th)), key
