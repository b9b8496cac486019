"""conv_tc_kernel's fp16 epilogue: the staged tile stored through the destination tensor map, pinned exactly.

The fp16 epilogue writes its tile into shared memory and one thread stores it with TMA; an in-place residual is
loaded through the same map.  The cases below are the store shapes the routing tables of tests/test_gpu_conv_tc.py
and tests/test_gpu_conv_tc_tiles.py do not reach: two 64-channel store boxes with the second clipped at the op's
cout inside a wider destination buffer, a residual at 16x8 tiles and BN = 128, and the four DECONV4 phase maps with
two boxes each.  The one-hot construction of test_routing_exact makes every output exactly one input value, and the
comparison covers the whole destination buffer, so a write into a neighbouring channel, a padding column or a pixel
beyond the grid fails with zero tolerance.
"""
import pytest

import test_gpu_conv_tc as base
import test_gpu_conv_tc_tiles as tiles
from util import cc, PREC_FP16_TC

F16 = PREC_FP16_TC

# (name, precision, source channels, kind, k, stride, cout, act, residual, down, n, h, w, dst): as ROUTING_CASES
STORE_CASES = [
    # TH = 16, BN = 128: cout 120 into channels 8 .. 127 of a 136-channel buffer, in-place residual; grid 184 x 184
    # (x- and y-partial tiles)
    ("st_1x1_cout120_res", F16, [128], "conv", 1, 1, 120, cc.ACT_RELU, True, 8, 1, 1472, 1472, (136, 8)),
    # TH = 8, BN = 128 (64 tiles of 16x16, fewer than one per SM), residual; grid 64 x 120 (x-partial)
    ("st_3x3_res_th8_bn128", F16, [64], "conv", 3, 1, 128, cc.ACT_NONE, True, 8, 2, 512, 960, (136, 8)),
    # cout 21 into a slice of a 40-channel buffer: the last 5 columns lie in a 16-byte granule the map leaves out
    ("st_1x1_cout21_res", F16, [64], "conv", 1, 1, 21, cc.ACT_RELU, True, 8, 2, 512, 960, (40, 8)),
    # DECONV4 256 -> 128 at TH = 16, BN = 128: four phase maps x two store boxes
    ("st_deconv4_bn128", F16, [256], "deconv", 4, 2, 128, cc.ACT_RELU, False, 8, 1, 1024, 1024, None),
]


def test_store_cases_plans():
    plans = {c[0]: tiles.case_plan16(c) for c in STORE_CASES}
    got = {k: (p["bn"], p["th"], p["partial"]) for k, p in plans.items()}
    assert got == {"st_1x1_cout120_res": (128, 16, True), "st_3x3_res_th8_bn128": (128, 8, True),
                   "st_1x1_cout21_res": (32, 8, True), "st_deconv4_bn128": (128, 16, False)}, got


@pytest.mark.gpu
@pytest.mark.parametrize("case", STORE_CASES, ids=tiles._case_id)
def test_routing_exact_store(case):
    base.test_routing_exact(case)
