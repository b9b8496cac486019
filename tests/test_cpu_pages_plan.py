"""not-gpu: `ctd_pages_plan`, the host layout of a batch of pages of any size (ctd_submit_pages), against the Python
letterbox arithmetic, the engine's block-section layout and the shape rules of ctd_detect_page."""
import ctypes as C

import numpy as np
import pytest

import ctd_b200
from ctd_b200 import binding, multigpu
from ctd_b200.inference import letterbox_geometry

CTD_E_SHAPE = -4


def _plan(shapes, net_h, net_w):
    lib = binding.load_library()
    pages = np.zeros((len(shapes),), binding.PAGE_ENTRY_DTYPE)
    for i, (ih, iw) in enumerate(shapes):
        pages[i]["ih"], pages[i]["iw"] = ih, iw
    ib, rb = C.c_size_t(), C.c_size_t()
    rc = lib.ctd_pages_plan(pages.ctypes.data_as(C.c_void_p), len(pages), net_h, net_w, C.byref(ib), C.byref(rb))
    return rc, pages, int(ib.value), int(rb.value)


def _al(v):
    return (v + 255) // 256 * 256


def _section_layout():
    # the block-section offsets ctd_create's arena uses (multigpu.arena_layout covers the phase-A part of the same
    # arena); blocks_stride etc. do not depend on the engine's shape
    rec_off = 64
    lines_off = rec_off + _al(binding.MAX_BLOCKS * binding.BLOCK_DTYPE.itemsize)
    dist_off = lines_off + _al(binding.MAX_BLOCKS * 32)
    return dict(blk_records_off=rec_off, blk_lines_off=lines_off, blk_dist_off=dist_off,
                blocks_stride=dist_off + _al(binding.MAX_BLOCK_DIST * 8))


def _sizes(rng, net_h, net_w):
    out = [(net_h, net_w), (net_h * 2, net_w * 2), (net_h // 2, net_w // 2), (40, 6000), (6000, 40), (1, 1),
           (1654, 1170), (361, 251), (96, 1500)]
    # size * r landing exactly on .5 (python's round: half to even): r = net / (2k), size = odd multiples of k
    for k in (1, 2, 3, 5):
        out.append((2 * k * 8, k * 7))
        out.append((k * 9, 2 * k * 8))
    while len(out) < 60:
        out.append((int(rng.integers(1, 4000)), int(rng.integers(1, 4000))))
    return out


@pytest.mark.parametrize("seed", range(40))
def test_plan_matches_python_letterbox(seed):
    rng = np.random.default_rng(seed)
    net_h, net_w = int(rng.integers(1, 33)) * 64, int(rng.integers(1, 33)) * 64
    shapes = _sizes(rng, net_h, net_w)
    rng.shuffle(shapes)
    keep = []
    for ih, iw in shapes:
        _r, (uw, uh), _dw, _dh = letterbox_geometry((ih, iw), (net_h, net_w))
        if uw >= 1 and uh >= 1:
            keep.append((ih, iw))
    rc, pages, ib, rb = _plan(keep, net_h, net_w)
    assert rc == 0
    for p, (ih, iw) in zip(pages, keep):
        _r, (uw, uh), _dw, _dh = letterbox_geometry((ih, iw), (net_h, net_w))
        assert (int(p["unpad_h"]), int(p["unpad_w"])) == (uh, uw), (ih, iw, net_h, net_w)
    _check_offsets(pages, ib, rb)


def test_half_to_even_ties():
    # 10 * 0.5 = 5 -> 5 (exact), 5 * 0.5 = 2.5 -> 2, 7 * 0.5 = 3.5 -> 4, 3 * 0.5 = 1.5 -> 2
    rc, pages, _ib, _rb = _plan([(128, 10), (128, 5), (128, 7), (128, 3)], 64, 64)
    assert rc == 0
    assert pages["unpad_w"].tolist() == [5, 2, 4, 2]
    assert pages["unpad_h"].tolist() == [64] * 4


def _check_offsets(pages, ib, rb):
    n = len(pages)
    sec = _section_layout()
    stride = _al(sec["blocks_stride"])
    px = [int(p["ih"]) * int(p["iw"]) for p in pages]
    for f in ("page_off", "mask_off", "refined_off", "blocks_off"):
        assert all(int(v) % 256 == 0 for v in pages[f]), f
    # input: pages back to back (each rounded up to 256 pixels), image offset = 3 x the page's pixel offset
    m0 = int(pages[0]["mask_off"])
    for i in range(n):
        assert int(pages[i]["page_off"]) == 3 * (int(pages[i]["mask_off"]) - m0)
        if i + 1 < n:
            assert int(pages[i + 1]["page_off"]) == int(pages[i]["page_off"]) + 3 * _al(px[i])
    assert ib == int(pages[-1]["page_off"]) + 3 * _al(px[-1])
    # results: masks, then mask_refined planes, then block sections, no overlaps, nothing past results_bytes
    spans = []
    for i in range(n):
        spans += [(int(pages[i]["mask_off"]), px[i]), (int(pages[i]["refined_off"]), px[i]),
                  (int(pages[i]["blocks_off"]), sec["blocks_stride"])]
    spans.sort()
    for (a, la), (b, _lb) in zip(spans, spans[1:]):
        assert a + la <= b
    assert rb == int(pages[-1]["blocks_off"]) + stride
    assert spans[-1][0] + spans[-1][1] <= rb
    for i in range(n - 1):
        assert int(pages[i + 1]["blocks_off"]) - int(pages[i]["blocks_off"]) == stride


def test_decode_block_section_shapes():
    # the decoder multigpu.unpack_arena and Engine.collect_pages share, on a section laid out as above (the engine's own
    # offsets, ctd_results_layout, are compared with this layout on the GPU: test_gpu_pages_batch.py)
    sec = _section_layout()
    lay = dict(multigpu.arena_layout(2, 128, 128), **sec)
    a = np.zeros((sec["blocks_stride"],), np.uint8)
    hdr, rec, lines, dist = binding.decode_block_section(a, lay)
    assert hdr.shape == (4,) and len(rec) == 0
    assert lines.shape == (binding.MAX_BLOCKS, 8) and dist.shape == (binding.MAX_BLOCK_DIST,)
    assert sec["blk_dist_off"] + binding.MAX_BLOCK_DIST * 8 <= sec["blocks_stride"]


def test_empty_batch():
    rc, _p, ib, rb = _plan([], 256, 256)
    assert rc == 0 and ib == 0 and rb == 0


@pytest.mark.parametrize("shape, net", [
    ((0, 100), (256, 256)), ((100, 0), (256, 256)), ((-5, 100), (256, 256)),
    ((1, 600), (64, 64)),            # 1 * 64/600 rounds to 0 rows
    ((700, 1), (64, 64)),            # 0 columns
    ((100, 100), (100, 128)), ((100, 100), (128, 100)), ((100, 100), (0, 64)), ((100, 100), (-64, 64)),
    ((100, 100), (32, 64)),
])
def test_shape_errors_as_detect_page(shape, net):
    rc, _p, _ib, _rb = _plan([(256, 256), shape], *net)
    assert rc == CTD_E_SHAPE
    with pytest.raises(ctd_b200.CtdError):
        binding.pages_plan([shape], *net)


def test_python_plan_wrapper():
    pages, ib, rb = binding.pages_plan([(1654, 1170), (512, 512)], 512, 512)
    assert pages["unpad_h"].tolist() == [512, 512] and pages["unpad_w"].tolist() == [362, 512]
    _check_offsets(pages, ib, rb)
