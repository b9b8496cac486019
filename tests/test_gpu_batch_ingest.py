"""-m gpu: the ingest every batch entry that takes caller pages shares (ctd_submit_pages, ctd_submit_outputs_dtype,
ctd_submit_refine, ctd_submit_regions, ctd_preprocess_pages), and the slot records of `Engine`.

* Kind mismatch: a batch of one kind (pages, refine, regions) refuses every collect of another kind with CtdError and
  stays in flight; its own collect then returns what a fresh engine returns for the same batch.
* Shared refusals: each entry refuses, with CTD_E_INVALID, a host pointer given as a device image, a stride past 2^31, a
  NULL image with no input_host, and entries whose page_off is not the plan's; a refusal about one image names its
  index.  A good call on the same slot (or into the same dst) then succeeds."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding
from oracle import synth
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
SIZES = [(200, 300), (150, 170)]
E_INVALID = -1


@pytest.fixture(scope="module")
def engines():
    dets = [ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=2) for _ in range(2)]
    yield [d.net for d in dets]
    for d in dets:
        d.close()


def _pages():
    return [np.ascontiguousarray(synth.structured_page(40 + i, 256, 320)[:h, :w]) for i, (h, w) in enumerate(SIZES)]


def _masks(pages):
    return [np.where(p[..., 0] > 128, 255, 0).astype(np.uint8) for p in pages]


def _lines():
    """two lines on page 0 (one block), one on page 1: records and the per-page block line counts"""
    def rec(x0, y0, x1, y1):
        r = np.zeros((), binding.REGION_LINE_DTYPE)
        r["quad"] = [x0, y0, x1, y0, x1, y1, x0, y1]
        r["font_size"] = y1 - y0
        return r
    lines = np.array([rec(10, 10, 150, 40), rec(20, 60, 180, 90), rec(5, 5, 100, 60)], binding.REGION_LINE_DTYPE)
    return lines, [2, 1], [[2], [1]]


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return a is None and b is None


BOXES = [np.array([[20, 20, 160, 90]], np.int32), np.array([[10, 10, 120, 100]], np.int32)]


def _submit(eng, kind):
    pages = _pages()
    if kind == "pages":
        eng.submit_pages(0, pages, NET, NET)
    elif kind == "refine":
        eng.submit_refine(0, pages, _masks(pages), BOXES)
    else:
        lines, n_lines, _counts = _lines()
        eng.submit_regions(0, pages, lines, n_lines, 32)


def _collect(eng, kind):
    if kind == "pages":
        return eng.collect_pages(0)
    if kind == "refine":
        return eng.collect_refine(0)
    return eng.collect_crops(0, _lines()[2])


@pytest.mark.parametrize("kind", ["pages", "refine", "regions"])
def test_kind_mismatch_leaves_batch_in_flight(engines, kind):
    eng, fresh = engines
    _submit(fresh, kind)
    want = _collect(fresh, kind)
    _submit(eng, kind)
    for other in ("pages", "refine", "regions"):
        if other != kind:
            with pytest.raises(binding.CtdError, match="submit_%s.*submit_%s" % (other, kind)):
                _collect(eng, other)
    got = _collect(eng, kind)
    assert _same(got, want), kind
    with pytest.raises(binding.CtdError, match="nothing"):
        _collect(eng, kind)


ENTRIES = ["pages", "outputs", "refine_pages", "refine_masks", "regions", "preprocess"]
CASES = ["host_pointer", "stride", "null_no_host", "page_off"]


def _raw_call(eng, entry, case, dst):
    """one ctd_* call of `entry` on two CUDA pages (and masks), with image 1 (page, or mask for refine_masks) or the
    entries broken as `case` says -> (rc, ctd_last_error)"""
    lib = eng.lib
    pages = [torch.from_numpy(p).cuda() for p in _pages()]
    masks = [torch.from_numpy(m).cuda() for m in _masks(_pages())]
    if entry in ("pages", "outputs", "preprocess"):
        ent, _in_bytes, res_bytes = binding.pages_plan(SIZES, NET, NET)
    else:
        boxes = np.concatenate(BOXES) if entry.startswith("refine") else np.zeros((0, 4), np.int32)
        counts = [1, 1] if entry.startswith("refine") else [0, 0]
        ent, _w, _s, _in_bytes, res_bytes = binding.refine_plan(SIZES, boxes, counts)
    results = torch.zeros((max(res_bytes, 1),), dtype=torch.uint8, pin_memory=True)
    host_img = np.zeros((1 << 20,), np.uint8)

    def dev_table(imgs, ch, broken):
        tab = (binding.CtdDevicePage * 2)()
        for i, t in enumerate(imgs):
            st = t.stride()
            tab[i] = binding.CtdDevicePage(t.data_ptr(), st[0], st[1], st[2] if ch == 3 else 0, None)
        if broken:
            if case == "host_pointer":
                tab[1].data = host_img.ctypes.data
            elif case == "stride":
                tab[1].stride_h = (1 << 31) + 1
            elif case == "null_no_host":
                tab[1].data = None
        return tab

    dev_p = dev_table(pages, 3, entry != "refine_masks")
    dev_m = dev_table(masks, 1, entry == "refine_masks")
    if case == "page_off":
        ent = ent.copy()
        ent[1]["page_off"] += 256
    ep, vp = binding._ptr(ent), C.c_void_p
    if entry == "pages":
        rc = lib.ctd_submit_pages(eng.h, 0, ep, 2, NET, NET, None, C.cast(dev_p, vp), 0, 0, 0, 0, vp(results.data_ptr()))
    elif entry == "outputs":
        outs = (binding.CtdNetOutput * 2)()
        dtypes = (C.c_int32 * 2)(binding.DTYPE_F32, binding.DTYPE_F32)
        rc = lib.ctd_submit_outputs_dtype(eng.h, 0, ep, 2, NET, NET, None, C.cast(dev_p, vp), C.cast(outs, vp),
                                          C.cast(dtypes, vp), 0, 0, 0, 0, vp(results.data_ptr()))
    elif entry.startswith("refine"):
        xyxy = np.ascontiguousarray(np.concatenate(BOXES))
        nb = np.array([1, 1], np.int32)
        rc = lib.ctd_submit_refine(eng.h, 0, ep, 2, binding._ptr(xyxy), binding._ptr(nb), None, C.cast(dev_p, vp),
                                   C.cast(dev_m, vp), 0, 0, 0, 0, vp(results.data_ptr()))
    elif entry == "regions":
        lines, n_lines, _counts = _lines()
        rc = lib.ctd_submit_regions(eng.h, 0, ep, 2, binding._ptr(lines), binding._ptr(np.array(n_lines, np.int32)),
                                    32, None, C.cast(dev_p, vp), 0)
    else:
        rc = lib.ctd_preprocess_pages(eng.h, ep, 2, NET, NET, None, C.cast(dev_p, vp), binding.PRE_F32_NCHW, 0,
                                      vp(dst.data_ptr()), vp(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, lib.ctd_last_error(eng.h).decode()


def _good_call(eng, entry, dst):
    pages = _pages()
    cuda_pages = [torch.from_numpy(p).cuda() for p in pages]
    if entry == "pages":
        eng.submit_pages(0, [pages[0], cuda_pages[1]], NET, NET)
        assert len(eng.collect_pages(0)) == 2
    elif entry == "outputs":
        outs = [(np.zeros((10, 7), np.float32), np.zeros((NET, NET), np.float32), np.zeros((NET, NET), np.float32))
                for _ in pages]
        eng.submit_outputs(0, [pages[0], cuda_pages[1]], outs, NET, NET)
        assert len(eng.collect_pages(0)) == 2
    elif entry.startswith("refine"):
        masks = _masks(pages)
        eng.submit_refine(0, cuda_pages, [masks[0], torch.from_numpy(masks[1]).cuda()], BOXES)
        assert len(eng.collect_refine(0)) == 2
    elif entry == "regions":
        lines, n_lines, counts = _lines()
        eng.submit_regions(0, [pages[0], cuda_pages[1]], lines, n_lines, 32)
        assert len(eng.collect_crops(0, counts)) == 2
    else:
        eng.preprocess_pages(cuda_pages, NET, NET, binding.PRE_F32_NCHW, False, dst.data_ptr(),
                             torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert not bool((dst == -7.0).all()), "the good call wrote nothing"


@pytest.mark.parametrize("entry", ENTRIES)
def test_shared_refusals(engines, entry):
    eng = engines[0]
    what = "mask" if entry == "refine_masks" else "page"
    dst = torch.full((2, 3, NET, NET), -7.0, device="cuda")
    want = {"host_pointer": "%s 1 .*is not device memory" % what, "stride": "%s 1: strides .*out of range" % what,
            "null_no_host": "%s 1 is in neither input_host nor device memory" % what, "page_off": "not the ones"}
    for case in CASES:
        rc, err = _raw_call(eng, entry, case, dst)
        assert rc == E_INVALID, (entry, case, rc, err)
        assert re.search(want[case], err), (entry, case, err)
        assert bool((dst == -7.0).all()), (entry, case, "a refused call wrote dst")
    _good_call(eng, entry, dst)
