"""TEST INFRASTRUCTURE ONLY (oracle): adds to tests/golden/refine_finding.npz (captured on an H100 by
scripts/capture_refine_finding.py: the page mask after refine_undetected_mask's in-place edit and the blocks of its
second refine_mask on structured_page(42, 413, 292)) the UNMODIFIED reference's `utils.textmask.refine_mask` on those
inputs, REFINEMASK_ANNOTATION, as `reference`.  Needs the reference tree (oracle/ref_shim.py).  Usage, from the
repository root:
    python -m oracle.make_refine_finding_ref
"""
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "refine_finding.npz")


class _Blk:
    def __init__(self, xyxy):
        self.xyxy = xyxy


def main():
    from oracle import ref_shim, synth
    assert ref_shim.available(), "needs the reference tree (see oracle/ref_shim.py)"
    ns = ref_shim.load()
    d = dict(np.load(GOLD))
    page = synth.structured_page(42, 413, 292)
    d["reference"] = ns.textmask.refine_mask(page, d["mask"].copy(), [_Blk(b) for b in d["blocks"].tolist()],
                                             refine_mode=1)
    np.savez_compressed(GOLD, mask=d["mask"], blocks=d["blocks"], reference=d["reference"])
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes;", int(np.count_nonzero(d["reference"])), "px set")


if __name__ == "__main__":
    main()
