"""Inputs shared by the text-line crop tests (tests/test_cpu_regions.py, tests/test_gpu_regions.py) and the script that
writes their golden fixture (scripts/make_golden_regions.py): synthetic pages with the blocks `group_output` makes
of random line sets, and hand-made blocks that reach every branch of `get_transformed_region`
(utils/textblock.py:162-194)."""
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import synth  # noqa: E402
from test_cpu_textblock import make_case  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "regions_ref.npz")

# (page seed, page h, page w, group_output case seed, textheight)
PAGE_CASES = [(41, 1024, 1024, 3, 32), (42, 1024, 1024, 5, 48), (43, 768, 1280, 7, 48), (44, 1170, 1654, 11, 32)]
HAND_PAGE = (45, 600, 800)   # seed, h, w of the page the hand-made blocks sit on


def blk(lines, language, vertical, font_size):
    """a block-like record with the fields get_transformed_region reads"""
    return types.SimpleNamespace(lines=[np.asarray(q).tolist() for q in lines], language=language,
                                 vertical=bool(vertical), font_size=font_size)


def page_case(i):
    """(page, blocks, textheight) of PAGE_CASES[i]; the blocks are what the native group_output (equal to the
    reference's, tests/test_cpu_textblock.py) makes of a random line set"""
    from ctd_b200 import textblock as tb
    seed, h, w, case_seed, th = PAGE_CASES[i]
    page = synth.structured_page(seed, h, w)
    blks, lines, _, _, mask = make_case(case_seed, w, h)
    if mask.shape != (h, w):   # make_case's mask covers whole 8 x 8 cells only
        mask = None
    return page, tb.group_output(blks, lines, w, h, mask), th


def rect(x0, y0, x1, y1):
    return [[x0, y0], [x1, y0], [x1, y1], [x0, y1]]


def hand_blocks():
    """one block per branch; the page is HAND_PAGE (800 wide, 600 high)"""
    tilt = [[100, 300], [330, 318], [326, 362], [96, 344]]
    return [
        blk([rect(3, 2, 220, 30)], "eng", False, 24),                  # expansion clipped at 0 (x and y)
        blk([rect(560, 575, 798, 599)], "eng", False, 27),             # clipped at im_w = 800 and im_h = 600 exactly
        blk([rect(300, 100, 520, 131), tilt], "unknown", False, 17.5),  # float font_size (a merged block), expansion
        blk([rect(40, 200, 75, 520)], "unknown", True, 30),             # vertical 'unknown': no expansion, rotated
        blk([tilt, rect(420, 420, 700, 452)], "ja", False, 22),         # no expansion
        blk([rect(700, 60, 736, 420), [[640, 80], [668, 84], [650, 330], [622, 326]]], "ja", True, 25),   # vertical
        blk([rect(120, 380, 152, 590)], "eng", True, 26),               # vertical 'eng': expansion + rotation
        blk([rect(500, 200, 502, 590)], "ja", False, 10),               # w rounds to 0: page-sized crop
        blk([rect(150, 560, 700, 562)], "ja", True, 10),                # h rounds to 0: page-sized crop, rotated
        blk([[[-60, 150], [260, 140], [270, 190], [-50, 200]], [[640, -30], [860, -20], [850, 40], [630, 30]],
             [[620, 560], [900, 570], [890, 640], [610, 630]]], "ja", False, 20),   # quads crossing the page borders
    ]


def raising_blocks():
    """lines on which the reference raises (findHomography returns None: a 1 px side; a degenerate quad)"""
    return [
        blk([rect(400, 100, 402, 160)], "ja", False, 10),   # ratio 30: w = round(32 / 30) = 1 at textheight 32
        blk([rect(100, 100, 160, 102)], "ja", True, 10),    # ratio 1/30: h = round(32 / 30) = 1 at textheight 32
        blk([rect(100, 100, 160, 100)], "ja", False, 10),   # zero height: textheight / 0.0
    ]


def hand_page():
    seed, h, w = HAND_PAGE
    return synth.structured_page(seed, h, w)
