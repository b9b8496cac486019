"""TEST INFRASTRUCTURE ONLY (oracle): the golden of the reference's post-processing on float16 network outputs.

tests/golden/half_ref_256.npz holds the crafted float16 outputs of oracle/postproc_half_ref.golden_inputs and what the
UNMODIFIED reference computes from them on CPU half tensors: non_max_suppression (yolov5_utils.py:124-218),
postprocess_mask (inference.py:85-99) and SegDetectorRepresenter(thresh=0.3) (db_utils.py:40-72).

Needs the reference tree (oracle/ref_shim.py).  Usage, from the repository root:
    python -m oracle.make_golden_half_ref
"""
import os

import numpy as np
import torch

from oracle import postproc_half_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "half_ref_256.npz")


def reference_outputs(ns, blks, mask, lines):
    """(det float32 [n][6], mask u8, line boxes int16 [k][4][2], line scores f32 [k]) of the reference on half
    tensors"""
    det = ns.yolov5_utils.non_max_suppression(torch.from_numpy(blks)[None], 0.4, 0.35)[0]
    m = ns.inference.postprocess_mask(torch.from_numpy(mask)[None].clone())
    boxes, scores = ns.db_utils.SegDetectorRepresenter(thresh=0.3)(None, torch.from_numpy(lines)[None])
    return det.numpy(), m, np.asarray(boxes[0]), np.asarray(scores[0])


def main():
    from oracle import ref_shim
    assert ref_shim.available(), "needs the reference tree (see oracle/ref_shim.py)"
    ns = ref_shim.load()
    blks, mask, lines = postproc_half_ref.golden_inputs()
    det, m, boxes, scores = reference_outputs(ns, blks, mask, lines)
    np.savez_compressed(GOLD, blks=blks, mask=mask, lines=lines, det=det, mask_u8=m, line_boxes=boxes,
                        line_scores=scores)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes;", len(det), "detections,", len(boxes), "line boxes")


if __name__ == "__main__":
    main()
