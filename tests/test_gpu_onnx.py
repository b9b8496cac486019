"""-m gpu: `TextDetector` on an `.onnx` model (the reference's OpenCV-DNN backend, comic-text-detector_b200/onnx_model.py).

* the accurate engines against the oracle forward of the SOURCE checkpoint on the channel-reversed page (the ONNX
  network sees RGB), the fp16 engine with the statistical bounds of the `.pt` engine;
* the drop-in call against the oracle chain on the engine's own maps, bit for bit;
* the unmodified reference's own results on the same model (oracle/make_onnx_ref.py): identical blocks wherever the
  engine's DB bitmap and boxes come out as cv2.dnn's, the mask within one level;
* the batched stream with CUDA pages, crops and device results against `__call__`;
* the same kernel launches as the `.pt` detector.

The model files come from oracle/make_onnx_ref.py; each test skips, naming the missing file, when they are absent."""
import json
import os

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200.inference import letterbox, letterbox_geometry
from oracle import pipeline_ref, postproc_ref, synth, textblock_ref
from oracle.net_ref import RefNet
from pages_ref import postprocess_page_any_size
from util import PREC_FP16_TC, PREC_FP32_SIMT, PREC_SPLIT_TC, page_to_net_input

pytestmark = pytest.mark.gpu

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
NET = 512


def _ref_file(name):
    p = os.path.join(REF, name)
    if not os.path.isfile(p):
        pytest.skip("%s is missing (made by oracle/make_onnx_ref.py where the reference tree exists)" % p)
    return p


def _detector(size=NET, **kw):
    return ctd_b200.TextDetector(_ref_file("ctd_%d.onnx" % size), input_size=size, **kw)


def _key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


@pytest.mark.parametrize("prec", [PREC_FP32_SIMT, PREC_SPLIT_TC, PREC_FP16_TC], ids=["fp32_simt", "split_tc", "fp16_tc"])
def test_net_maps_match_source_checkpoint_on_rgb(prec):
    det = _detector(precision=prec, max_batch=2)
    pages = np.stack([synth.structured_page(3100, NET, NET), synth.noise_page(3101, NET, NET)])
    try:
        det.net.forward(pages)
        blks, mask, lines = det.net.net_outputs()
    finally:
        det.close()
    with torch.no_grad():
        rb, rm, rl = (t.numpy() for t in RefNet(synth.make_checkpoint(0))(page_to_net_input(pages[..., ::-1])))
    e_mask, e_lines = float(np.abs(mask - rm).max()), float(np.abs(lines - rl).max())
    m_mask, m_lines = float(np.abs(mask - rm).mean()), float(np.abs(lines - rl).mean())
    e_blks = float((np.abs(blks - rb) / (np.abs(rb) + 1.0)).max())
    msg = "prec %d: max err mask %.3g lines %.3g blks(rel) %.3g; mean %.3g / %.3g" % (prec, e_mask, e_lines, e_blks,
                                                                                    m_mask, m_lines)
    print(msg)
    if prec == PREC_FP16_TC:   # test_gpu_net.py TOL[PREC_FP16_TC]
        assert e_mask <= 0.8 and e_lines <= 0.8 and m_mask <= 1.5e-2 and m_lines <= 1.5e-2 and e_blks <= 1.0, msg
    else:                      # test_gpu_net.py TOL[PREC_FP32_SIMT] / TOL[PREC_SPLIT_TC]
        assert e_mask <= 1e-3 and e_lines <= 1e-3 and m_mask <= 1e-4 and m_lines <= 1e-4 and e_blks <= 2e-3, msg


@pytest.mark.parametrize("keep", [False, True], ids=["", "keep_undetected"])
@pytest.mark.parametrize("mode", [0, 1])
def test_call_matches_oracle_chain(mode, keep):
    """`TextDetector(onnx)(page)` on a net-sized and an other-sized page: blocks, mask and mask_refined equal the
    oracle chain run on the engine's own maps of the letterboxed page"""
    det = _detector()
    try:
        n_blocks = 0
        for seed, (h, w) in ((3200, (NET, NET)), (3201, (640, 420))):
            page = synth.structured_page(seed, h, w)
            mask, mask_refined, blk_list = det(page.copy(), refine_mode=mode, keep_undetected_mask=keep)
            det.net.forward(letterbox(page, (NET, NET))[0][None])
            blks, mf, lf = det.net.net_outputs()
            if (h, w) == (NET, NET):
                rmask, rref, rblk = pipeline_ref.postprocess_page(page.copy(), blks[0], mf[0, 0], lf[0],
                                                                  textblock_ref.group_output, refine_mode=mode,
                                                                  keep_undetected_mask=keep)
            else:
                _r, (uw, uh), _dw, _dh = letterbox_geometry(page.shape[:2], (NET, NET))
                rmask, rref, rblk = postprocess_page_any_size(page.copy(), (NET, NET), (uh, uw), blks[0], mf[0, 0],
                                                              lf[0], textblock_ref.group_output, refine_mode=mode,
                                                              keep_undetected_mask=keep)
            assert [_key(a) for a in blk_list] == [_key(b) for b in rblk], (h, w)
            assert np.array_equal(mask, rmask), (h, w)
            assert np.array_equal(mask_refined, rref), ((h, w), int((mask_refined != rref).sum()))
            n_blocks += len(blk_list)
        assert n_blocks > 5
    finally:
        det.close()


def test_matches_reference_results():
    """Against the unmodified reference's `TextDetector(model_path=<onnx>)` on its OpenCV-DNN backend (oracle/_ref),
    at 512 and 1024 px.  The fp32 engine's maps differ from cv2.dnn's by ~1e-4, which moves ~0.5 % of the u8 mask
    (`(mask * 255).astype(uint8)`) by one level, so the u8 mask is held to one level everywhere; the blocks must be
    identical on every page whose DB bitmap (shrink > 0.3) and NMS boxes (after postprocess_yolo's casts) agree with
    cv2.dnn's, and at least one page must; mask and mask_refined must be identical where the u8 maps also agree.  The
    flipped pixels of every page are reported."""
    exact, report = 0, []
    for size in (512, 1024):
        meta = json.load(open(_ref_file("onnx_ref_%d.json" % size)))
        arrs = np.load(_ref_file("onnx_ref_%d.npz" % size))
        det = _detector(size, precision=PREC_FP32_SIMT)
        try:
            for k, p in enumerate(meta["pages"]):
                if "error" in p:
                    report.append("%d/%d: the reference raised" % (size, k))
                    continue
                page = synth.structured_page(p["seed"], p["h"], p["w"])
                _r, (uw, uh), _dw, _dh = letterbox_geometry(page.shape[:2], (size, size))
                det.net.forward(letterbox(page, (size, size))[0][None])
                blks, mf, lf = det.net.net_outputs()
                rs, rd = arrs["seg_%d" % k], arrs["det_%d" % k]
                flip_m = int(((mf[0, 0] * 255).astype(np.uint8) != (rs[0, 0] * 255).astype(np.uint8)).sum())
                flip_b = int(((lf[0, 0] > 0.3) != (rd[0, 0] > 0.3)).sum())
                same_boxes = _nms_ints(blks, p["w"] / uw, p["h"] / uh) == _nms_ints(arrs["blk_%d" % k], p["w"] / uw, p["h"] / uh)
                mask, mask_refined, blk_list = det(page.copy(), keep_undetected_mask=p["keep_undetected_mask"])
                rmask, rref = arrs["mask_%d" % k], arrs["mask_refined_%d" % k]
                same_blocks = [[list(kb[0])] + list(kb[1:]) for kb in map(_key, blk_list)] == [
                    [b["xyxy"], b["lines"], b["language"], b["vertical"], b["font_size"], b["angle"]] for b in p["blocks"]]
                # keep_undetected_mask zeroes the returned mask under mask_refined (textmask.py:135-156, in place)
                sel = (mask_refined <= 30) & (rref <= 30) if p["keep_undetected_mask"] else np.ones(mask.shape, bool)
                assert int(np.abs(mask.astype(int) - rmask)[sel].max()) <= 1, (size, k)
                if flip_b == 0 and same_boxes:
                    assert same_blocks, (size, k)
                    exact += 1
                    if flip_m == 0:
                        assert np.array_equal(mask, rmask) and np.array_equal(mask_refined, rref), (size, k)
                report.append("%d/%d %dx%d: u8 map %d px, bitmap %d px, boxes %s, blocks %s, mask %d px, mask_refined %d px"
                              % (size, k, p["h"], p["w"], flip_m, flip_b, "same" if same_boxes else "differ",
                                 "same" if same_blocks else "differ", int((mask != rmask).sum()),
                                 int((mask_refined != rref).sum())))
        finally:
            det.close()
    print("\n".join(report))
    assert exact >= 1, report


def _nms_ints(blks, rx, ry):
    """postprocess_yolo (inference.py:101-114): NMS, ratio scaling, int boxes, rounded confidences, classes"""
    d = postproc_ref.non_max_suppression(torch.as_tensor(blks[0])[None], 0.4, 0.35)[0].numpy()
    d[..., [0, 2]] *= rx
    d[..., [1, 3]] *= ry
    return d[..., 0:4].astype(np.int32).tolist(), np.round(d[..., 4], 3).tolist(), d[..., 5].astype(int).tolist()


def test_stream_with_device_pages_and_results_equals_call():
    det = _detector(max_batch=4)
    sizes = [(NET, NET), (640, 420), (300, 700), (NET, NET), (420, 420)]
    pages = [synth.structured_page(3300 + i, h, w) for i, (h, w) in enumerate(sizes)]
    try:
        cuda = [torch.from_numpy(p).cuda() for p in pages]
        got = list(det.detect_stream(cuda, refine_mode=1, keep_undetected_mask=True, textheight=48, device_results=True))
        n_crops = 0
        for page, (mask, mask_refined, blk_list, crops) in zip(pages, got):
            rmask, rref, rblk = det(page.copy(), refine_mode=1, keep_undetected_mask=True)
            assert np.array_equal(mask.cpu().numpy(), rmask) and np.array_equal(mask_refined.cpu().numpy(), rref)
            assert [_key(a) for a in blk_list] == [_key(b) for b in rblk]
            if any(c is None for blk in crops for c in blk):
                continue   # a line the reference's crop raises on: get_transformed_regions refuses the whole page
            ref_crops = det.get_transformed_regions(page, rblk, 48)
            for blk, ref_blk in zip(crops, ref_crops):
                for c, r in zip(blk, ref_blk):
                    assert np.array_equal(c.cpu().numpy(), r)
                    n_crops += 1
        assert n_crops > 0
    finally:
        det.close()


def test_same_kernel_launches_as_pt_detector():
    page = synth.structured_page(3400, NET, NET)[None]
    counts = []
    for model in (_ref_file("ctd_%d.onnx" % NET), synth.make_checkpoint(0)):
        det = ctd_b200.TextDetector(model, input_size=NET)
        try:
            det.net.forward(page)
            counts.append(det.net.last_launch_count())
        finally:
            det.close()
    assert counts[0] == counts[1] and counts[0] > 0, counts
