"""not-gpu: the crafted NMS boundary cases of tests/nms_cases.py, their properties and the oracle on them, and the IoU
threshold the binding gives the device.

  * every case builds (each builder asserts its property in float32 / float16 arithmetic), and the oracle (torchvision's
    CPU nms, double threshold) keeps exactly the rows the numpy restatement of that rule keeps;
  * for every threshold that float32 rounds up, some case is decided differently by `IoU > t` in double and by
    `IoU > float32(t)`, so the GPU tests can tell the two rules apart; for the others no case is;
  * the binding passes RD_f32(t), and `x > RD_f32(t)` equals `x > t` for float32 x around every threshold;
  * torch CPU's `half_tensor > t` equals `x > half(float32(t))` (what the kernel compares) on every finite half."""
import numpy as np
import pytest
import torch

from ctd_b200 import binding
import nms_cases as nc

ALL_HALF = np.arange(65536, dtype=np.uint16).view(np.float16)
FINITE_HALF = ALL_HALF[np.isfinite(ALL_HALF)]


def _assert_oracle_keeps(rows, conf, t, what):
    ref = nc.oracle_nms(rows, conf, t)
    exp = nc.expected_rows(rows, conf, nc.kept_double(rows, conf, t))
    assert ref.shape == exp.shape and np.array_equal(ref.view(np.uint32), exp.view(np.uint32)), what


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_tie_cases_and_oracle(t):
    cases = nc.tie_rows(t)
    assert {k for k in cases if k.startswith("f32_pair")} == {"f32_pair_%s_c%d" % (n, c) for n in ("at", "below", "above")
                                                              for c in (0, 1)}
    assert "f32_chain_at_c1" in cases and "f16_pair_at_c0" in cases and "f32_survivor" in cases
    for name, rows in cases.items():
        _assert_oracle_keeps(rows, 0.4, t, name)
    # the survivor chain: A suppresses B, so C (which B would have suppressed) survives
    assert nc.kept_double(cases["f32_survivor"], 0.4, t) == [0, 2]


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_rounding_up_thresholds_split_the_rules(t):
    cases = nc.tie_rows(t)
    split = [k for k, rows in cases.items() if nc.kept_double(rows, 0.4, t) != nc.kept_float(rows, 0.4, t)]
    if nc.rounds_up(t):
        # at IoU exactly float32(t): suppressed by the double rule, kept by the float one
        assert {"f32_pair_at_c0", "f32_pair_at_c1", "f16_pair_at_c0", "f32_survivor", "f16_survivor"} <= set(split)
        assert nc.kept_double(cases["f32_pair_at_c0"], 0.4, t) == [0]
        assert nc.kept_float(cases["f32_pair_at_c0"], 0.4, t) == [0, 1]
    else:
        assert split == []
    # the float rule on RD_f32(t) is the double rule, on every case
    rd = binding.iou_thresh_f32(t)
    for k, rows in cases.items():
        assert nc.greedy(rows, 0.4, lambda v: v > np.float32(rd)) == nc.kept_double(rows, 0.4, t), k


def test_integer_pair_of_the_issue():
    rows = nc.tie_rows(0.4)["f32_integer_pair"]
    assert len(nc.oracle_nms(rows, 0.4, 0.4)) == 1
    assert nc.kept_float(rows, 0.4, 0.4) == [0, 1]


def test_binding_threshold_conversion():
    rng = np.random.default_rng(0)
    ts = list(nc.THRESHOLDS) + list(rng.uniform(0, 1, 200)) + [0.0, 1.0, 0.1, 0.2, 0.55, 1e-40]
    for t in ts:
        rd = binding.iou_thresh_f32(t)
        assert rd == float(nc.rd_f32(t)) and rd <= t and float(np.float32(rd)) == rd, t
        assert float(np.nextafter(np.float32(rd), np.float32(np.inf))) > t, t
        f = np.float32(t)
        xs = (f.view(np.uint32) + np.arange(-4, 5, dtype=np.int64)).astype(np.uint32).view(np.float32)
        assert [float(x) > t for x in xs] == [bool(x > np.float32(rd)) for x in xs], t
    # the default 0.35 rounds down: the device gets what it got before
    assert binding.iou_thresh_f32(0.35) == float(np.float32(0.35))
    for t in (0.3, 0.4, 0.6, 0.8, 0.1, 0.2, 0.55):
        assert nc.rounds_up(t) and binding.iou_thresh_f32(t) < float(np.float32(t))
    assert not nc.rounds_up(0.35) and not nc.rounds_up(0.45) and not nc.rounds_up(0.5)


def test_half_conf_rule_every_value():
    """torch CPU's `half_tensor > t` is `x > half(float32(t))` for every finite half, for 315 thresholds: the kernel
    compares with round_half(the float32 conf_thresh)"""
    x = torch.from_numpy(FINITE_HALF.copy())
    xf = FINITE_HALF.astype(np.float32)
    rng = np.random.default_rng(3)
    ts = list(np.linspace(0.005, 0.995, 199)) + list(rng.uniform(0, 1, 100)) + \
        [0.3, 0.4, 0.35, 0.45, 0.55, 0.6, 0.8, 0.1, 0.2, 0.25, 0.5, 0.7, 0.75, 0.9, 0.95, 0.05]
    assert len(ts) == 315
    for t in ts:
        assert np.array_equal((x > float(t)).numpy(), xf > np.float32(np.float16(np.float32(t)))), t
    # and a float32 tensor compares with float32(t)
    f = torch.from_numpy(np.float32(0.4) + np.arange(-3, 4, dtype=np.float32) * np.spacing(np.float32(0.4)))
    assert np.array_equal((f > 0.4).numpy(), f.numpy() > np.float32(0.4))


def test_degenerate_cases_and_oracle():
    for dtype in (np.float32, np.float16):
        rows = nc.degenerate_rows(dtype)
        for t in nc.THRESHOLDS:
            _assert_oracle_keeps(rows, 0.4, t, (dtype, t))


@pytest.mark.parametrize("conf", nc.CONFS)
def test_score_cases_and_oracle(conf):
    for k in (1, 2, 3):
        rows, expect = nc.score_rows_f32(conf, k)
        ref = nc.oracle_nms(rows, conf, 0.35)
        kept = [i for i in range(len(rows)) if expect[i] >= 0]
        assert np.array_equal(ref, nc.expected_rows(rows, conf, sorted(kept, key=lambda i: -nc.scores(rows, conf)[1][i])))
        assert list(ref[:, 5].astype(int)) == [expect[i] for i in sorted(kept, key=lambda i: -nc.scores(rows, conf)[1][i])]
    rows = nc.score_rows_f16(conf)
    _assert_oracle_keeps(rows, conf, 0.35, "f16")


def test_half_corner_and_cap_cases_and_oracle():
    rows = nc.half_corner_rows()
    _assert_oracle_keeps(rows, 0.4, 0.35, "corners")
    assert len(nc.oracle_nms(rows, 0.4, 0.35)) == len(rows)   # every box apart: every row survives
    rows = nc.max_det_rows()
    ref = nc.oracle_nms(rows, 0.4, 0.35)
    exp = nc.expected_rows(rows, 0.4, nc.kept_double(rows, 0.4, 0.35)[:nc.MAX_DET])
    assert np.array_equal(ref, exp) and len(ref) == nc.MAX_DET
    rows = nc.overflow_rows()
    assert len(nc.capped(rows, 0.4)) == nc.CAP and len(nc.oracle_nms(rows, 0.4, 0.35)) == nc.MAX_DET
