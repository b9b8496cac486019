"""-m "not gpu": what `RegionCropper` checks and builds on the host before any GPU work: the column-wise line records
against `textblock.region_lines` on the same blocks, the argument checks, and the refusals of `ctd_submit_regions` that
need no device."""
import ctypes as C
import json

import numpy as np
import pytest

import ctd_b200
from ctd_b200 import binding, regions, textblock
from ctd_b200.annotations import NumpyEncoder
from ctd_b200.textblock import TextBlock
import region_cases as rc


def _lists():
    out = [rc.hand_blocks(), rc.raising_blocks(), [], [TextBlock([0, 0, 1, 1])]]
    for i in range(len(rc.PAGE_CASES)):
        out.append(rc.page_case(i)[1])
    # json round-tripped TextBlocks, hand-made blocks with the default font_size, float font sizes, numpy lines
    blks = rc.page_case(0)[1]
    out.append([TextBlock(**d) for d in json.loads(json.dumps([b.to_dict() for b in blks], cls=NumpyEncoder))])
    out.append([TextBlock([0, 0, 9, 9], lines=[rc.rect(1, 2, 40, 12)]),
                TextBlock([0, 0, 9, 9], lines=np.array([rc.rect(3, 4, 9, 60)], np.int32), vertical=True,
                          language="eng", font_size=np.float64(13.25)),
                TextBlock([0, 0, 9, 9], lines=[], language="unknown"),
                TextBlock([0, 0, 9, 9], lines=[rc.rect(0.5, 1.5, 20.25, 9)], language="fr", font_size=7)])
    return out


@pytest.mark.parametrize("k", range(len(_lists())))
def test_line_records_equal_region_lines(k):
    blks = _lists()[k]
    rec, counts = regions.line_records(blks)
    ref, keys = textblock.region_lines(blks)
    assert rec.dtype == binding.REGION_LINE_DTYPE and rec.tobytes() == ref.tobytes()
    assert counts == [len(b.lines) for b in blks]
    assert keys == [(b, i) for b, c in enumerate(counts) for i in range(c)]


@pytest.mark.parametrize("line", [[[1, 2], [3, 4]], [1, 2, 3, 4, 5, 6, 7, 8], [[1, 2], [3, 4], [5, 6], ["a", 8]],
                                  None, [[1, 2], [3, 4], [5, 6], [7, 8, 9]]])
def test_bad_line_named(line):
    blks = [TextBlock([0, 0, 1, 1], lines=[rc.rect(1, 1, 9, 9)]),
            TextBlock([0, 0, 1, 1], lines=[rc.rect(1, 1, 9, 9), line])]
    with pytest.raises(ValueError, match=r"item 4: block 1, line 1: a line must be 4 x 2 numbers"):
        regions.line_records(blks, "item 4: ")


@pytest.mark.parametrize("th,ok", [(2, 2), (48, 48), (np.int64(32), 32), (32.0, 32), (1, None), (0, None),
                                   (-3, None), (2.5, None), ("32", None), (None, None), (True, None)])
def test_textheight(th, ok):
    if ok is None:
        with pytest.raises(ValueError, match="textheight"):
            regions.check_textheight(th)
    else:
        assert regions.check_textheight(th) == ok


def test_page_side_limit():
    page = np.zeros((1, regions.MAX_SIDE - 1, 3), np.uint8)
    assert regions._check_side(page, "item 0: ") is page
    for shape in [(1, regions.MAX_SIDE, 3), (regions.MAX_SIDE, 1, 3)]:
        with pytest.raises(ValueError, match="item 7: the page is"):
            regions._check_side(np.zeros(shape, np.uint8), "item 7: ")


def test_submit_regions_refusals_without_a_device():
    lib = binding.load_library()
    entries, _w, _s, _ib, _rb = binding.refine_plan([(10, 10)], np.zeros((0, 4), np.int32), [0])
    counts = np.zeros((1,), np.int32)
    page = np.zeros((10, 10, 3), np.uint8)
    args = (binding._ptr(entries), 1, None, binding._ptr(counts), 32, binding._ptr(page), None, 0)
    assert lib.ctd_submit_regions(None, 0, *args) == -1             # CTD_E_INVALID: no handle
    assert lib.ctd_submit_regions(C.c_void_p(1), 2, *args) == -1    # a slot that is not 0 or 1
    assert lib.ctd_submit_regions(C.c_void_p(1), 0, args[0], 0, *args[2:]) == -1   # an empty batch
    assert "ctd_submit_regions" in binding.EXPORTS
    assert ctd_b200.RegionCropper.crop_stream.__doc__
