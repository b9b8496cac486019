"""-m gpu: the NMS at its decision boundaries (tests/nms_cases.py) against the oracle, raw rows bit for bit and in
order, at every IoU threshold of nms_cases.THRESHOLDS, through every entry that feeds it:

  * `Engine.nms` (ctd_nms_dtype) on float32 and float16 rows;
  * `Engine(conf_thresh=, nms_thresh=)` and `debug_postprocess`: one case per page, many pages per batch in a seeded
    shuffled order;
  * `PostProcessor(nms_thresh=, half=True)` with float32 and float16 pages in one batch, through its blocks;
  * sweeps of the half rules over every half value of their operand near the boundary, and a seeded sample elsewhere,
    a few hundred disjoint boxes per call."""
import numpy as np
import pytest

import ctd_b200
from ctd_b200.textblock import kernels_only_engine
from oracle import postproc_half_ref, synth, textblock_ref
from pages_ref import postprocess_page_any_size
import nms_cases as nc

pytestmark = pytest.mark.gpu

S = 512   # page side of the batched tests: rows_per_image(512) = 16128 rows per page


def rows_per_image(s):
    return 3 * ((s // 8) ** 2 + (s // 16) ** 2 + (s // 32) ** 2)


def same_rows(got, ref):
    return got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


@pytest.fixture(scope="module")
def engines():
    """Engine.nms on pages of up to 16128 rows, one engine per nc"""
    es = {k: kernels_only_engine(0, 1, max_size=(S, S), nc=k) for k in (1, 2, 3)}
    yield es
    for e in es.values():
        e.close()


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_engine_nms_ties(engines, t):
    bad = []
    for name, rows in nc.tie_rows(t).items():
        got = engines[2].nms(rows, 0.4, t)
        ref = nc.oracle_nms(rows, 0.4, t)
        if not same_rows(got, ref):
            bad.append((name, len(got), len(ref)))
    assert bad == [], (t, bad)


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_engine_nms_degenerate_and_caps(engines, t):
    cases = {"f32_degenerate": nc.degenerate_rows(np.float32), "f16_degenerate": nc.degenerate_rows(np.float16),
             "max_det": nc.max_det_rows(), "overflow": nc.overflow_rows()}
    for name, rows in cases.items():
        got = engines[2].nms(rows, 0.4, t)
        assert same_rows(got, nc.oracle_nms(rows, 0.4, t)), (t, name)
    tot, cap = engines[2].nms_status()
    assert cap == nc.CAP and int(tot[0]) > nc.CAP   # the last call was the overflow page
    assert len(engines[2].nms(cases["max_det"], 0.4, t)) == nc.MAX_DET


@pytest.mark.parametrize("conf", nc.CONFS)
def test_engine_nms_scores(engines, conf):
    for k in (1, 2, 3):
        rows, expect = nc.score_rows_f32(conf, k)
        got = engines[k].nms(rows, conf, 0.35)
        assert same_rows(got, nc.oracle_nms(rows, conf, 0.35)), ("f32", k)
        assert len(got) == sum(v >= 0 for v in expect.values())
    rows = nc.score_rows_f16(conf)
    assert same_rows(engines[2].nms(rows, conf, 0.35), nc.oracle_nms(rows, conf, 0.35)), "f16"
    rows = nc.half_corner_rows()
    assert same_rows(engines[2].nms(rows, conf, 0.35), nc.oracle_nms(rows, conf, 0.35)), "f16 corners"


def _sweep(eng, values, place, conf=0.4):
    """every value through the half rows' rules, 300 rows per call on disjoint boxes: place(rows, chunk) writes the
    values into the rows"""
    for i in range(0, len(values), nc.MAX_DET):
        chunk = values[i:i + nc.MAX_DET]
        rows = nc._spaced(len(chunk), 2, np.float16, pitch=40.0)
        rows[:, 2:4] = 8
        rows[:, 4] = np.float16(0.9)
        rows[:, 5] = 1
        place(rows, chunk)
        got, ref = eng.nms(rows, conf, 0.35), nc.oracle_nms(rows, conf, 0.35)
        assert same_rows(got, ref), (i, len(got), len(ref))


def test_half_rules_sweep(engines):
    eng = engines[2]
    rng = np.random.default_rng(11)
    unit = np.arange(0x3c01, dtype=np.uint16).view(np.float16)                   # +0 .. 1
    c = np.float16(np.float32(0.4))
    near = unit[np.abs(unit.astype(np.float32) - np.float32(c)) < 0.05]           # every half near half(0.4)
    sample = rng.choice(unit, 600, replace=False)

    def obj(rows, v):
        rows[:, 4] = v

    def cls(rows, v):
        rows[:, 4] = np.float16(0.875)
        rows[:, 5], rows[:, 6] = v, np.flip(v)

    _sweep(eng, np.concatenate([near, sample]), obj)
    _sweep(eng, np.concatenate([near * np.float16(1.125), sample]), cls)   # products around half(0.4) / 0.875
    small = np.arange(1, 0x2400, 7, dtype=np.uint16).view(np.float16)        # subnormal and small widths

    def width(rows, v):
        rows[:, 2] = v
        rows[:, 3] = np.flip(v)

    _sweep(eng, small, width)
    big = (np.arange(0x6000, 0x6800, 3, dtype=np.uint16)).view(np.float16)   # cx in [512, 2048): sums that round

    def centre(rows, v):
        rows[:, 0] = v
        rows[:, 2] = rng.uniform(1, 30, len(v)).astype(np.float16)
        rows[:, 1] = (np.arange(len(v)) * 40 + 20).astype(np.float16)

    _sweep(eng, big, centre)


def _page(rows, rng, s=S):
    """rows at a seeded offset in a page of empty Detect rows (obj 0: no candidates)"""
    p = np.zeros((rows_per_image(s), rows.shape[1]), rows.dtype)
    at = int(rng.integers(0, len(p) - len(rows) + 1))
    p[at:at + len(rows)] = rows
    return p


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_forward_postprocess_batch(t):
    """the forward's NMS (the handle's nms_thresh) on a batch of crafted pages, one case per page, shuffled"""
    cases = {k: v for k, v in nc.tie_rows(t).items() if k.startswith("f32")}
    cases.update(degenerate=nc.degenerate_rows(), max_det=nc.max_det_rows(), overflow=nc.overflow_rows())
    rng = np.random.default_rng(int(t * 1000))
    names = sorted(cases)
    rng.shuffle(names)
    blks = np.stack([_page(cases[k], rng) for k in names])
    lines = np.zeros((len(names), 2, S, S), np.float32)
    eng = kernels_only_engine(0, len(names), max_size=(S, S), conf_thresh=0.4, nms_thresh=t, skip_postproc=False)
    try:
        eng.debug_postprocess(blks, lines)
        det = eng.detections()
    finally:
        eng.close()
    bad = [(i, k) for i, k in enumerate(names) if not same_rows(det[i], nc.oracle_nms(blks[i], 0.4, t))]
    assert bad == [], (t, bad)


def _key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


@pytest.mark.parametrize("t", nc.THRESHOLDS)
def test_postprocessor_mixed_dtypes(t):
    """PostProcessor(nms_thresh=t, half=True) on float32 and float16 tie pages in one batch: every detection is a block
    (the mask is text everywhere), so the blocks show which boxes the NMS kept"""
    cases = {k: v for k, v in nc.tie_rows(t).items() if "_pair_at_" in k or "survivor" in k}
    rng = np.random.default_rng(int(t * 1000) + 1)
    names = sorted(cases)
    rng.shuffle(names)
    page = synth.structured_page(7, S, S)
    items, refs = [], []
    for k in names:
        rows = cases[k]
        blks = _page(rows, rng)
        mask = np.ones((1, S, S), rows.dtype)
        lines = np.zeros((2, S, S), rows.dtype)
        items.append((page, blks, mask, lines))
        if rows.dtype == np.float16:
            refs.append(postproc_half_ref.postprocess_page_half(page.copy(), blks, mask[0], lines,
                                                                textblock_ref.group_output, 0.4, t))
        else:
            refs.append(postprocess_page_any_size(page.copy(), (S, S), (S, S), blks, mask[0], lines,
                                                  textblock_ref.group_output, 0.4, t, 0, False))
    post = ctd_b200.PostProcessor(input_size=S, max_batch=len(items), nms_thresh=t, half=True)
    try:
        got = post.postprocess_batch(items)
    finally:
        post.close()
    for k, g, r in zip(names, got, refs):
        n_kept = len(nc.oracle_nms(cases[k], 0.4, t))
        assert len(r[2]) == n_kept, (t, k)
        assert [_key(b) for b in g[2]] == [_key(b) for b in r[2]], (t, k)
        assert np.array_equal(g[0], r[0]) and np.array_equal(g[1], r[1]), (t, k)
