"""not-gpu: `ctd_refine_plan`, the host layout and block check of a refine batch (ctd_submit_refine): each block's window
and status against the oracle's expand_textwindow plus Python slicing and against the unmodified reference's
refine_mask, which raises exactly on the status-1 blocks; the pixel layout against ctd_pages_plan's rule, also for
pages ctd_pages_plan refuses; and the greyscale read of masks that traverse_by_dict relies on."""
import cv2
import numpy as np
import pytest

import png_decode_corpus as pc
from ctd_b200 import binding
from oracle import postproc_ref, ref_shim, synth

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="/root/reference not present on this box")

I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1


def _odd_boxes(ih, iw, rng):
    """negative, off-page, reversed, zero-size and huge boxes, boxes whose x2 + pad wraps negative, and boxes on every
    edge of the page"""
    out = [[0, 0, iw, ih], [0, 0, 0, 0], [iw, ih, iw, ih], [-5, -5, -1, -1], [-50, -50, -2, -2], [-3, 0, 2, ih],
           [iw + 3, 0, iw + 40, ih], [0, ih + 1, iw, ih + 9], [iw - 1, ih - 1, 1, 1], [5, 5, 2, 9], [5, 5, 9, 2],
           [0, 0, iw - 1, 0], [0, 0, 0, ih - 1], [0, ih - 1, iw, ih - 1], [iw - 1, 0, iw - 1, ih], [-40, 0, -33, 1],
           [0, -40, 1, -33], [-100, -100, 100, 100], [1, 1, 2, 2], [0, 0, 1, 1], [iw - 1, ih - 1, iw, ih],
           [I32_MAX, I32_MAX, I32_MIN, I32_MIN], [I32_MIN, I32_MIN, I32_MAX, I32_MAX], [I32_MAX, 0, I32_MIN, ih],
           [0, 0, I32_MAX, I32_MAX], [I32_MIN, I32_MIN, -1, -1], [-2, -2, -1, -1]]
    for x in (0, iw // 2, iw - 1, iw):
        for y in (0, ih // 2, ih - 1, ih):
            out.append([x, y, x + 1, y + 1])
            out.append([x - 1, y - 1, x, y])
    for _ in range(60):
        a = rng.integers(-2 * max(ih, iw) - 20, 2 * max(ih, iw) + 20, 4)
        out.append([int(v) for v in a])
    return out


def _py_status(shape, xyxy):
    """the oracle's expand_textwindow on Python ints, then what img[by1:by2, bx1:bx2] gives"""
    win = postproc_ref.expand_textwindow(shape, xyxy, expand_r=16)
    if any(not I32_MIN <= v <= I32_MAX for v in win):
        return win, 2
    bx1, by1, bx2, by2 = win
    empty = np.zeros(shape[:2], np.uint8)[by1:by2, bx1:bx2].size == 0
    return win, 1 if empty else 0


SHAPES = [(1, 1), (1, 5000), (5000, 1), (1, 7), (9, 1), (2, 2), (37, 53), (300, 200)]


@pytest.mark.parametrize("shape", SHAPES)
def test_windows_and_status_match_python(shape):
    rng = np.random.default_rng(shape[0] * 7919 + shape[1])
    boxes = np.array(_odd_boxes(shape[0], shape[1], rng), np.int64)
    _e, win, status, _ib, _rb = binding.refine_plan([shape], boxes.astype(np.int32), [len(boxes)])
    seen = set()
    for b, xyxy in enumerate(boxes.tolist()):
        pw, ps = _py_status(shape, xyxy)
        assert int(status[b]) == ps, (b, xyxy, pw, win[b], status[b])
        if ps != 2:
            assert win[b].tolist() == pw, (b, xyxy, pw, win[b])
        seen.add(ps)
    # expand_textwindow clamps x2 to iw - 1 and the slice ends before it: on a page 1 px wide or high every window is
    # empty, and the reference raises on every block
    assert seen >= ({0, 1, 2} if shape[0] > 1 and shape[1] > 1 else {1})


@needs_ref
@pytest.mark.parametrize("shape", [(1, 40), (40, 1), (1, 1), (23, 31)])
def test_reference_raises_exactly_on_status_1(shape):
    """the unmodified reference's refine_mask, one block at a time: it raises where the plan gives status 1 or 2 and
    returns where it gives 0"""
    ns = ref_shim.load()
    rng = np.random.default_rng(11)
    page = np.ascontiguousarray(synth.structured_page(3, 128, 128)[:shape[0], :shape[1]])
    mask = (rng.random(shape) * 255).astype(np.uint8)
    boxes = np.array(_odd_boxes(shape[0], shape[1], rng)[:80], np.int64)
    _e, _win, status, _ib, _rb = binding.refine_plan([shape], boxes.astype(np.int32), [len(boxes)])
    for b, xyxy in enumerate(boxes.tolist()):
        blk = ns.textblock.TextBlock(xyxy)
        try:
            ns.textmask.refine_mask(page, mask, [blk])
            raised = False
        except Exception:
            raised = True
        assert raised == (int(status[b]) != 0), (b, xyxy, int(status[b]))


def _al(v):
    return (v + 255) // 256 * 256


def test_layout_rule_on_pages_the_letterbox_refuses():
    shapes = [(1, 5000), (5000, 1), (1, 1), (361, 251), (1, 3), (2, 70000)]
    counts = [1, 0, 2, 0, 0, 1]
    boxes = np.array([[0, 0, 10, 1], [0, 0, 1, 1], [0, 0, 0, 0], [5, 0, 60000, 2]], np.int32)
    entries, _win, _status, ib, rb = binding.refine_plan(shapes, boxes, counts)
    with pytest.raises(binding.CtdError):
        binding.pages_plan(shapes, 64, 64)
    p = 0
    offs = []
    for e, (ih, iw) in zip(entries, shapes):
        offs.append(p)
        assert (int(e["ih"]), int(e["iw"])) == (ih, iw)
        assert int(e["page_off"]) == 3 * p and int(e["mask_off"]) == p
        assert int(e["unpad_h"]) == int(e["unpad_w"]) == int(e["blocks_off"]) == 0
        p += _al(ih * iw)
    total = p
    for e, o in zip(entries, offs):
        assert int(e["refined_off"]) == total + o
    assert ib == 5 * total and rb == 2 * total
    # where ctd_pages_plan accepts the pages, the pixel offsets are its own
    ok = [(361, 251), (1024, 700), (64, 64)]
    pe, ib2, _rb2 = binding.pages_plan(ok, 1024, 1024)
    re, _w, _s, ib3, _rb3 = binding.refine_plan(ok, np.zeros((0, 4), np.int32), [0, 0, 0])
    assert ib2 * 5 == ib3 * 3
    m0 = int(pe[0]["mask_off"])
    for a, b in zip(pe, re):
        assert int(a["page_off"]) == int(b["page_off"])
        assert int(a["mask_off"]) - m0 == int(b["mask_off"])
        assert int(a["refined_off"]) - m0 == int(b["refined_off"])


def test_plan_refuses_empty_pages():
    with pytest.raises(binding.CtdError):
        binding.refine_plan([(0, 5)], np.zeros((0, 4), np.int32), [0])


def test_grey_png_reads_as_channel_0_of_the_colour_read():
    """cv2.imread(path, IMREAD_GRAYSCALE) of a greyscale PNG (colour type 0, any bit depth, eXIf included) is channel 0
    of cv2's colour read, the page PngDecoder returns, so traverse_by_dict reads such masks on the GPU"""
    n = 0
    for name, data, _expect in pc.corpus(large=False):
        b = np.frombuffer(data, np.uint8)
        if not (data[:8] == pc.SIGNATURE and len(data) > 25 and data[25] == 0):
            continue
        grey = cv2.imdecode(b, cv2.IMREAD_GRAYSCALE)
        colour = cv2.imdecode(b, cv2.IMREAD_COLOR)
        assert (grey is None) == (colour is None), name
        if grey is not None:
            assert grey.shape == colour.shape[:2] and np.array_equal(grey, colour[..., 0]), name
            n += 1
    assert n > 20
