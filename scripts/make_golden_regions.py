"""Writes tests/golden/regions_ref.npz: the crops the UNMODIFIED reference's `TextBlock.get_transformed_region`
(utils/textblock.py:162-194) returns for the cases of tests/region_cases.py, so that the crop tests compare with the
reference where its tree is absent.

Keys: `p{case}_{block}_{line}` for the synthetic pages of PAGE_CASES (at their textheight), `h{textheight}_{block}_{line}`
for the hand-made blocks at textheight 32 and 48, and `raises{textheight}` = the block indices of raising_blocks() on
which the reference raises.

Needs the reference tree (oracle/ref_shim.py) and the built library.  From the repository root:
    python scripts/make_golden_regions.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def ref_crop(ns, b, page, idx, th):
    tb = ns.textblock.TextBlock([0, 0, 0, 0], lines=b.lines, language=b.language, vertical=b.vertical,
                                font_size=b.font_size)
    return tb.get_transformed_region(page, idx, th)


def main():
    from oracle import ref_shim
    import region_cases as rc
    assert ref_shim.available(), "needs the reference tree (see oracle/ref_shim.py)"
    ns = ref_shim.load()
    out = {}
    for i in range(len(rc.PAGE_CASES)):
        page, blks, th = rc.page_case(i)
        for b, blk in enumerate(blks):
            for l in range(len(blk.lines)):
                out["p%d_%d_%d" % (i, b, l)] = ref_crop(ns, blk, page, l, th)
    page = rc.hand_page()
    for th in (32, 48):
        for b, blk in enumerate(rc.hand_blocks()):
            for l in range(len(blk.lines)):
                out["h%d_%d_%d" % (th, b, l)] = ref_crop(ns, blk, page, l, th)
        raises = []
        for b, blk in enumerate(rc.raising_blocks()):
            try:
                ref_crop(ns, blk, page, 0, th)
            except Exception:
                raises.append(b)
        out["raises%d" % th] = np.array(raises, np.int32)
    np.savez_compressed(rc.GOLD, **out)
    print("wrote", rc.GOLD, os.path.getsize(rc.GOLD), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
