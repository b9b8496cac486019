"""conv_tc_kernel at 16x16-pixel tiles (TH = 16, M = 256): the routing of every N-block width pinned exactly, and the
launch-plan rule that picks the tile height.

* CPU: a replica of conv_tc_plan's tile-height rule.  The routing cases below run at TH = 16 at every BN
  (16 / 32 / 64 / 128), with full and partial tiles, y-partial tiles with gh % 8 == 0 and gh % 8 != 0, and one case
  loops each persistent CTA over more than 3 tiles.  The number of benchmark ops that run at TH = 16 is pinned.
* GPU: the one-hot routing construction of tests/test_gpu_conv_tc.py (every output is exactly one input value or a
  zero from the padding), so a wrong row block, tile origin, halo row, parity map, deconvolution phase, K block,
  residual or epilogue column fails with zero tolerance.  A TH = 16 tile accumulates every output element in the
  same K order as a 16x8 tile, so the float results of the real program do not change either
  (test_bench_plans_per_op holds them to the same bound).
"""
import pytest

import test_gpu_conv_tc as base
from util import cc, PREC_FP16_TC, PREC_SPLIT_TC, H100_SMS, TILE_W, tc_plan, get_checkpoint

F16 = PREC_FP16_TC

# (name, precision, source channels, kind, k, stride, cout, act, residual, down, n, h, w, dst): as ROUTING_CASES
TILE16_CASES = [
    # 2048 tiles: 16 per persistent CTA
    ("t16_1x1_many", F16, [128], "conv", 1, 1, 128, cc.ACT_RELU, False, 1, 2, 512, 512, None),
    # grid 72 x 128: the last tile row holds 8 of 16 pixel rows; 2 sources of 64-channel K blocks, in-place residual
    ("t16_3x3_res_2src_ypartial8", F16, [64, 64], "conv", 3, 1, 128, cc.ACT_NONE, True, 8, 4, 576, 1024, (136, 8)),
    # grid 20 x 128: 4 of 16 rows in the last tile row (20 % 8 != 0), three N blocks of 64
    ("t16_3x3_ypartial4", F16, [64], "conv", 3, 1, 192, cc.ACT_RELU, False, 16, 8, 320, 2048, None),
    # stride 2: dy = -1 reads the parity-1 map one row above the tile, zero-filled above the first row
    ("t16_3x3s2", F16, [32], "conv", 3, 2, 32, cc.ACT_NONE, False, 1, 2, 512, 512, None),
    # stride 2 on a grid of 72 x 136: y- and x-partial tiles
    ("t16_3x3s2_partial", F16, [32], "conv", 3, 2, 32, cc.ACT_RELU, False, 4, 4, 576, 1088, None),
    # three sources -> 16-channel K blocks
    ("t16_3x3_3src_kb16", F16, [64, 32, 16], "conv", 3, 1, 64, cc.ACT_NONE, False, 1, 1, 256, 512, None),
    # two sources -> 32-channel K blocks, residual into a destination slice
    ("t16_3x3_res_2src_kb32", F16, [32, 64], "conv", 3, 1, 32, cc.ACT_RELU, True, 1, 1, 256, 256, (72, 8)),
    # cout 40: three N blocks of 16, the last one 8 columns wide
    ("t16_3x3_cout40", F16, [32], "conv", 3, 1, 40, cc.ACT_RELU, False, 1, 1, 512, 512, (48, 8)),
    # every deconvolution phase; grid 20 x 64 (y-partial)
    ("t16_deconv4_ypartial4", F16, [128], "deconv", 4, 2, 16, cc.ACT_NONE, False, 16, 6, 320, 1024, None),
    ("t16_deconv4", F16, [64], "deconv", 4, 2, 64, cc.ACT_RELU, False, 8, 3, 512, 512, None),
]


def tile_h(cout, gh, gw, n_img, n_phase=1, split=False, nhwc_store=True, num_sms=H100_SMS):
    """conv_tc_plan's tile height: 16 for fp16 NHWC-store ops (CONV, DECONV4) whose layer has at least one 16x16
    tile per SM at the N-block width tc_plan picks (from the 16x8 tile count), else 8."""
    bn = tc_plan(cout, gh, gw, n_img, n_phase, split, num_sms)["bn"]
    cout_pad = (cout + 15) // 16 * 16
    tiles16 = n_img * -(-gw // TILE_W) * -(-gh // 16) * n_phase * (cout_pad // bn)
    return 16 if not split and nhwc_store and tiles16 >= num_sms else 8


def case_grid(case):
    _, _, _, kind, _, stride, _, _, _, down, _, h, w, _ = case
    gh, gw = h // down, w // down
    if kind == "conv":
        gh, gw = gh // stride, gw // stride
    return gh, gw


def case_plan16(case):
    _, prec, _, kind, _, _, cout, _, _, _, n, _, _, _ = case
    gh, gw = case_grid(case)
    n_phase = 4 if kind == "deconv" else 1
    p = dict(tc_plan(cout, gh, gw, n, n_phase, split=prec == PREC_SPLIT_TC))
    th = tile_h(cout, gh, gw, n, n_phase, split=prec == PREC_SPLIT_TC)
    p.update(th=th, tiles=n * -(-gw // TILE_W) * -(-gh // th) * n_phase * ((cout + 15) // 16 * 16 // p["bn"]),
             partial=gw % TILE_W != 0 or gh % th != 0)
    p["tiles_per_cta"] = -(-p["tiles"] // min(p["tiles"], H100_SMS))
    return p


def _case_id(case):
    p = case_plan16(case)
    return "%s-bn%d-th%d%s" % (case[0], p["bn"], p["th"], "-partial" if p["partial"] else "")


def bench_th16_counts(prog, n, h, w):
    """(ops at TH = 16, CONV / DECONV4 / DETECT ops) of the program at batch shape n x h x w."""
    k16 = total = 0
    for op in prog.ops:
        if op["kind"] not in (cc.OP_CONV, cc.OP_DECONV4, cc.OP_DETECT):
            continue
        total += 1
        down = prog.bufs[op["src_buf"][0]][1]
        gh, gw = h // down, w // down
        if op["kind"] == cc.OP_DECONV4:
            th = tile_h(op["cout"], gh, gw, n, 4)
        else:
            s = op["stride"]
            th = tile_h(op["cout"], gh // s, gw // s, n, 1, nhwc_store=op["kind"] == cc.OP_CONV)
        k16 += th == 16
    return k16, total


# ---------------------------------------------------------------------------------------------------------------
# CPU
def test_tile16_cases_cover_every_block_n():
    plans = [(case_plan16(c), case_grid(c)) for c in TILE16_CASES]
    assert all(p["th"] == 16 for p, _ in plans), [c[0] for c, (p, _) in zip(TILE16_CASES, plans) if p["th"] != 16]
    have = {(p["bn"], p["partial"]) for p, _ in plans}
    want = {(bn, part) for bn in (16, 32, 64, 128) for part in (False, True)}
    assert want <= have, "uncovered (BN, partial) at TH = 16: %s" % sorted(want - have)
    gh = [g[0] for _, g in plans]
    assert any(y % 16 and y % 8 == 0 for y in gh) and any(y % 8 for y in gh)         # both kinds of y-partial tile
    assert max(p["tiles_per_cta"] for p, _ in plans) > 3
    assert any(c[3] == "deconv" for c in TILE16_CASES) and any(c[3] == "conv" and c[5] == 2 for c in TILE16_CASES)
    assert any(c[8] for c in TILE16_CASES) and any(len(c[2]) == 3 for c in TILE16_CASES)
    kb = {64 if all(s % 64 == 0 for s in c[2]) else 32 if all(s % 32 == 0 for s in c[2]) else 16 for c in TILE16_CASES}
    assert kb == {16, 32, 64}


def test_tile_h_rule():
    assert tile_h(128, 512, 512, 1) == 16
    assert tile_h(128, 512, 512, 1, split=True) == 8
    assert tile_h(255, 64, 64, 1, nhwc_store=False) == 8       # Detect
    assert tile_h(128, 64, 128, 4) == 8                         # 128 tiles of 16x16 < 132 SMs
    assert tile_h(128, 64, 128, 5) == 16                        # 160
    # the existing routing cases keep running at 16x8 except the two large ones
    th16 = sorted(c[0] for c in base.ROUTING_CASES if case_plan16(c)["th"] == 16)
    assert th16 == ["f16_1x1_many", "f16_3x3s2_many"], th16


def test_benchmark_ops_at_tile16():
    """How many of the 92 CONV / DECONV4 / DETECT ops run at 16x16 tiles at the benchmarked shapes; the rest (the
    small late layers and Detect) keep 16x8.  The N-block width of every op is still tests/util.py's tc_plan."""
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    got = {shape: bench_th16_counts(prog, *shape) for shape in [(16, 1024, 1024), (8, 640, 640), (8, 1536, 1536)]}
    print("ops at TH = 16:", got)
    assert got == {(16, 1024, 1024): (71, 92), (8, 640, 640): (51, 92), (8, 1536, 1536): (81, 92)}


# ---------------------------------------------------------------------------------------------------------------
# GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", TILE16_CASES, ids=_case_id)
def test_routing_exact_tile16(case):
    base.test_routing_exact(case)
