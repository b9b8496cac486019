"""Captures tests/golden/refine_finding.npz on an H100: the inputs of refine_undetected_mask's second refine_mask on
structured_page(42, 413, 292) at input size 256, REFINEMASK_ANNOTATION -- the page mask after the in-place edit and
the blocks -- from the fp16 engine's network maps and the oracle chain at the page's scale (tests/pages_ref.py).  The
page itself is regenerated from its seed.  The reference's answer on the fixture is added afterwards where the
reference tree exists (oracle/make_refine_finding_ref.py).  Also prints, per window, the pixels in which the engine's
refine_mask differs from the oracle's, with the oracle run with and without OpenCV's IPP code paths.

    python scripts/capture_refine_finding.py OUT.npz
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(out):
    import cv2
    import ctd_b200
    from ctd_b200.inference import letterbox, letterbox_geometry
    from oracle import pipeline_ref, postproc_ref, synth, textblock_ref
    from pages_ref import postprocess_page_any_size
    from util import get_checkpoint

    net = 256
    page = synth.structured_page(42, 413, 292)
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=net, act="leaky", max_batch=2)
    try:
        eng = det.net
        _r, (uw, uh), _dw, _dh = letterbox_geometry(page.shape[:2], (net, net))
        eng.forward(letterbox(page, (net, net))[0][None])
        blks, mask, lines = eng.net_outputs()
        m, refined, blk_list = postprocess_page_any_size(page.copy(), (net, net), (uh, uw), blks[0], mask[0, 0], lines[0],
                                                         textblock_ref.group_output, refine_mode=1)
        blocks = pipeline_ref.undetected_blocks(m, refined, [b.xyxy for b in blk_list])
        wins = [postproc_ref.expand_textwindow(page.shape, b, expand_r=16) for b in blocks]
        got = eng.refine_mask(page, m, wins, 1)
        ref = postproc_ref.refine_mask(page, m, blocks, 1)
        cv2.ipp.setUseIPP(False)
        ref_noipp = postproc_ref.refine_mask(page, m, blocks, 1)
        cv2.ipp.setUseIPP(True)
        print("%d blocks; engine vs oracle: %d px, vs oracle without IPP: %d px, oracle with vs without IPP: %d px"
              % (len(blocks), int((got != ref).sum()), int((got != ref_noipp).sum()), int((ref != ref_noipp).sum())))
        print("differing pixels (y, x):", np.argwhere(got != ref).tolist()[:20])
        for w in wins:
            g1 = eng.refine_mask(page, m, [w], 1)
            x1, y1, x2, y2 = w
            im = np.ascontiguousarray(page[y1:y2, x1:x2])
            msk = np.ascontiguousarray(m[y1:y2, x1:x2])
            r1 = np.zeros_like(m)
            r1[y1:y2, x1:x2] = postproc_ref.merge_masks(postproc_ref.candidate_masks(im, msk), msk, 1)
            if not np.array_equal(g1, r1):
                cands = postproc_ref.candidate_masks(im, msk)
                print("window", w, "differs in", int((g1 != r1).sum()), "px; candidate xor sums", [int(s) for _, s in cands])
        np.savez_compressed(out, mask=m, blocks=np.asarray(blocks, np.int32))
        print("wrote", out)
    finally:
        det.close()


if __name__ == "__main__":
    main(sys.argv[1])
