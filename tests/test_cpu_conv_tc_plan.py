"""CPU: the launch-plan replica and the elementwise error bound that tests/test_gpu_conv_tc.py relies on.

* The routing cases cover every (precision, N-block width) pair conv_tc_kernel has, with full and partial tiles, and
  at least one case loops each persistent CTA over several tiles.
* The bound accepts a float64 reference carrying fp32 (and, for the fp16 engine, fp16) output rounding, and rejects
  typical kernel faults on a fixed random 3x3 convolution by at least 16x.
"""
import numpy as np
import pytest
import torch

from util import (cc, PREC_FP16_TC, PREC_SPLIT_TC, tc_plan, program_tc_plans, get_checkpoint, fp16_tc_ab, split_tc_ab,
                  bound_ratio, conv_ref_mag)
from test_gpu_conv_tc import ROUTING_CASES, case_plan


def test_routing_cases_cover_every_block_n():
    want = {(PREC_FP16_TC, bn, part) for bn in (16, 32, 64, 128) for part in (False, True)}
    want |= {(PREC_SPLIT_TC, bn, part) for bn in (16, 32, 64) for part in (False, True)}
    have = set()
    for case in ROUTING_CASES:
        p = case_plan(case)
        have.add((case[1], p["bn"], p["partial"]))
    assert want <= have, "uncovered (precision, BN, partial): %s" % sorted(want - have)
    for prec in (PREC_FP16_TC, PREC_SPLIT_TC):
        loops = [case_plan(c)["tiles"] for c in ROUTING_CASES if c[1] == prec]
        assert max(loops) > 3 * 132, "no %d case with more than 3 tiles per CTA" % prec
    for prec in (PREC_FP16_TC, PREC_SPLIT_TC):
        assert any(c[10] >= 2 for c in ROUTING_CASES if c[1] == prec)                 # batch
        assert any(len(c[2]) == 3 for c in ROUTING_CASES if c[1] == prec)             # three sources
        assert any(c[8] for c in ROUTING_CASES if c[1] == prec)                       # residual
        assert any(c[3] == "deconv" for c in ROUTING_CASES if c[1] == prec)
        assert any(c[3] == "conv" and c[5] == 2 for c in ROUTING_CASES if c[1] == prec)
        assert any(c[6] % 16 for c in ROUTING_CASES if c[1] == prec)                  # ncols tail


def test_plan_replica_matches_kernel_rules():
    # conv_tc_plan: 128 only for multiples of 128, narrowed to 64 while the whole layer has <= 66 tiles
    assert tc_plan(128, 64, 64, 1)["bn"] == 64            # 32 tiles
    assert tc_plan(128, 64, 128, 2)["bn"] == 128          # 128 tiles
    assert tc_plan(384, 8, 16, 1)["bn"] == 64             # 3 tiles of 128 -> 6 of 64
    assert tc_plan(192, 512, 512, 1)["bn"] == 64
    assert tc_plan(48, 64, 64, 1)["bn"] == 16
    assert tc_plan(21, 64, 64, 1)["bn"] == 32             # cout_pad 32
    assert tc_plan(512, 512, 512, 4, split=True)["bn"] == 64
    p = tc_plan(64, 12, 20, 2)
    assert p["partial"] and p["tiles"] == 2 * 2 * 2 and p["grid"] == 8


def test_benchmark_plans_differ_from_the_small_shapes():
    """The benchmark's shapes reach BN = 128 on most ops and loop each CTA over hundreds of tiles; the small shapes
    the interpreter test runs do not, which is why the per-op test at the benchmarked plans exists."""
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    stats = {}
    for n, h, w, split in [(2, 256, 320, 0), (1, 192, 448, 0), (16, 1024, 1024, 0), (8, 640, 640, 0),
                           (8, 1536, 1536, 0), (1, 1024, 1024, 1)]:
        P = program_tc_plans(prog, n, h, w, bool(split))
        stats[(n, h, w, split)] = (len(P), sum(p["bn"] == 128 for p in P.values()),
                                   max(p["tiles_per_cta"] for p in P.values()))
    assert stats[(2, 256, 320, 0)] == (92, 4, 3)
    assert stats[(1, 192, 448, 0)] == (92, 0, 2)
    assert stats[(16, 1024, 1024, 0)] == (92, 69, 249)
    assert stats[(8, 640, 640, 0)] == (92, 65, 49)
    assert stats[(8, 1536, 1536, 0)] == (92, 73, 280)
    assert stats[(1, 1024, 1024, 1)] == (92, 0, 16)


# ---------------------------------------------------------------------------------------------------------------
# the bound against mutants of a fixed random 3x3 convolution
N, C, CO, H, W = 2, 16, 24, 24, 40      # K = 144; W = 40: the last 16-wide tile column is partial


def _case():
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.standard_normal((N, C, H, W)).astype(np.float32)).double()
    w = torch.from_numpy((rng.standard_normal((CO, C, 3, 3)) / 12).astype(np.float32)).double()
    b = torch.from_numpy((rng.standard_normal(CO) * 0.5).astype(np.float32)).double()
    r = torch.from_numpy(rng.standard_normal((N, CO, H, W)).astype(np.float32)).double()
    ref, mag = conv_ref_mag(x, w, b, 1, 1)
    return x, w, b, r, ref + r, mag


def _f32(t):
    return t.float().double()


def _mutants():
    x, w, b, r, ref, mag = _case()
    F = torch.nn.functional
    out = {}
    # one K block (16 channels of the centre tap) never accumulated
    wk = torch.zeros_like(w)
    wk[:, 0:16, 1, 1] = w[:, 0:16, 1, 1]
    out["missing_k_block"] = ref - F.conv2d(x, wk, None, 1, 1)
    # tap (0, 0) read one pixel to the right
    wt = torch.zeros_like(w)
    wt[:, :, 0, 0] = w[:, :, 0, 0]
    xs = F.pad(x, (0, 1))[..., 1:]
    out["tap_shifted"] = ref - F.conv2d(x, wt, None, 1, 1) + F.conv2d(xs, wt, None, 1, 1)
    # last column of the partial tile (x = 39) not written
    z = ref.clone()
    z[..., W - 1] = 0
    out["partial_tile_column_zeroed"] = z
    out["residual_dropped"] = ref - r
    # activation lo plane dropped: x carried as fp16(x) only
    out["lo_dropped"] = conv_ref_mag(x.half().double(), w, b, 1, 1)[0] + r
    return ref, mag, {k: _f32(v) for k, v in out.items()}


@pytest.mark.parametrize("engine", ["fp16_tc", "split_tc"])
def test_bound_accepts_rounded_reference(engine):
    _, _, _, _, ref, mag = _case()
    K = 9 * C
    a, b = fp16_tc_ab(K) if engine == "fp16_tc" else split_tc_ab(K)
    assert float(bound_ratio(_f32(ref), ref, mag, a, b).max()) <= 1.0
    if engine == "fp16_tc":
        assert float(bound_ratio(ref.half().double(), ref, mag, a, b).max()) <= 1.0


MUTANTS = [(e, m) for e in ("fp16_tc", "split_tc")
           for m in ("missing_k_block", "tap_shifted", "partial_tile_column_zeroed", "residual_dropped")]
MUTANTS.append(("split_tc", "lo_dropped"))      # the fp16 engine has no lo plane


@pytest.mark.parametrize("engine,mutant", MUTANTS, ids=["%s-%s" % m for m in MUTANTS])
def test_bound_rejects_mutant(engine, mutant):
    ref, mag, muts = _mutants()
    a, b = fp16_tc_ab(9 * C) if engine == "fp16_tc" else split_tc_ab(9 * C)
    worst = float(bound_ratio(muts[mutant], ref, mag, a, b).max())
    assert worst >= 16.0, "%s: worst err/bound only %.3g" % (mutant, worst)
