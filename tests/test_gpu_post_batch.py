"""-m gpu: the post-processing stage (NMS, connected components, text-line boxes) on whole batches at the benchmarked
shapes -- 16 pages of 1024^2 and 8 of 1536^2 -- against the oracle page by page, and at the sizes where its index
arithmetic runs out: 2048^2 contour maps, connected components past 4096 scan segments, an A4 page at 600 dpi.

Crafted batches go through `Engine.debug_postprocess`, which runs the forward's own NMS and DB post-processing on given
network outputs.  Every page kind and Detect-row kind asserts on the CPU the property it exists for; the kinds sit in
one batch in a seeded shuffled order, so that every page offset past page 0 is exercised by a different kind of page.
Each page must also equal itself run alone (n = 1)."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import compiler as cc
from ctd_b200.inference import letterbox, letterbox_geometry
from lattice_polygon import fill_exact, many_vertex_polygon
from oracle import postproc_ref, synth, textblock_ref
from pages_ref import postprocess_page_any_size
import seg_geometry as sg
import stress_maps
from util import get_checkpoint

pytestmark = pytest.mark.gpu

T = np.float32(0.3)       # db_thresh
CONF = np.float32(0.4)    # conf_thresh
CAP = 4096                # NMS candidate workspace per page


def rows_per_image(s):
    return 3 * ((s // 8) ** 2 + (s // 16) ** 2 + (s // 32) ** 2)


def n_contours(m):
    cs, _ = cv2.findContours((m > T).astype(np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_SIMPLE)
    return cs


# ---- page kinds: (DB shrink map f32 [s][s], property asserted on the CPU) -----------------------------------------
def page_empty(s, rng):
    m = np.zeros((s, s), np.float32)
    assert len(n_contours(m)) == 0
    return m


def page_full(s, rng):
    m = np.full((s, s), 0.9, np.float32)
    assert len(n_contours(m)) == 1
    return m


def page_blobs(s, rng):
    m = stress_maps.blobs(int(rng.integers(1 << 30)), s, s, s // 8)
    assert len(n_contours(m)) > 50
    return m


def page_rings(s, rng):
    m = np.zeros((s, s), np.float32)
    for cx, cy in ((s // 4, s // 4), (3 * s // 4, s // 3), (s // 2, 3 * s // 4)):
        for k, r in enumerate(range(s // 5, 4, -s // 60)):
            cv2.circle(m, (cx, cy), r, 0.9 if k % 2 == 0 else 0.05, -1)
    cs = n_contours(m)
    assert len(cs) > 20   # outer borders and hole borders, nested several deep
    return m


def page_checker(s, rng):
    m = np.zeros((s, s), np.float32)
    m[s // 4:s // 4 + 160, s // 3:s // 3 + 160] = stress_maps.checkerboard(160, 160, 1)
    assert len(n_contours(m)) > 1000   # one 8-connected component with thousands of holes
    return m


def _squares(s, count):
    m = np.zeros((s, s), np.float32)
    pitch = (s - 8) // 32
    for i in range(count):
        y, x = 4 + (i // 32) * pitch, 4 + (i % 32) * pitch
        m[y:y + pitch // 2, x:x + pitch // 2] = 0.8
    return m


def page_squares1000(s, rng):
    m = _squares(s, 1000)
    assert len(n_contours(m)) == 1000
    return m


def page_squares1001(s, rng):
    # OpenCV lists contours in reverse discovery order and the reference keeps the first 1000: the top-left square,
    # found first, is the one dropped
    m = _squares(s, 1001)
    assert len(n_contours(m)) == 1001
    return m


def page_disc(s, rng):
    m = np.zeros((s, s), np.float32)
    cv2.circle(m, (s // 2, s // 2), 260, 0.95, -1)
    cv2.circle(m, (s // 2 + 40, s // 2 - 30), 60, 0.1, -1)   # a hole, so the disc is scored with its ring
    cs = n_contours(m)
    assert max(len(cv2.convexHull(c)) for c in cs) > 128   # the second, large-hull pass of contour_kernel
    return m


def page_edges(s, rng):
    m = np.zeros((s, s), np.float32)
    m[0:40, 0:40] = m[0:40, s - 40:] = m[s - 40:, 0:40] = m[s - 40:, s - 40:] = 0.9     # every corner
    m[0:5, 100:400] = m[s - 5:, 200:500] = m[300:600, 0:5] = m[400:700, s - 5:] = 0.8  # every edge
    m[s - 1, :] = 0.7                                                                     # the whole last row
    m[:, s - 120] = 0.7                                                                   # a full-height column
    cs = n_contours(m)
    touch = [c.reshape(-1, 2) for c in cs]
    assert any((c[:, 0] == 0).any() for c in touch) and any((c[:, 1] == 0).any() for c in touch)
    assert any((c[:, 0] == s - 1).any() for c in touch) and any((c[:, 1] == s - 1).any() for c in touch)
    return m


def page_noise(s, rng):
    m = np.where(rng.random((s, s)) < 0.08, rng.uniform(0.31, 1.0, (s, s)), rng.uniform(0, 0.29, (s, s)))
    m = m.astype(np.float32)
    assert len(n_contours(m)) > 1000
    return m


def page_at_thresh(s, rng):
    # exactly float32(0.3) is background, the next float up is foreground
    m = stress_maps.blobs(int(rng.integers(1 << 30)), s, s, s // 16)
    up = np.nextafter(T, np.float32(1))
    m = np.where(m > 0.2, np.where(rng.random((s, s)) < 0.5, T, up), np.float32(0)).astype(np.float32)
    assert (m == T).sum() > 1000 and (m == up).sum() > 1000
    assert len(n_contours(m)) > 10
    return m


PAGE_KINDS = {"empty": page_empty, "full": page_full, "blobs": page_blobs, "rings": page_rings, "checker": page_checker,
              "squares1000": page_squares1000, "squares1001": page_squares1001, "disc": page_disc, "edges": page_edges,
              "noise": page_noise, "at_thresh": page_at_thresh}


# ---- Detect-row kinds: (blks f32 [rows][7], property asserted on the CPU) ------------------------------------------
def _score(p):
    return (p[:, 5:] * p[:, 4:5]).max(1)


def _n_cand(p):
    return int(((p[:, 4] > CONF) & (_score(p) > CONF)).sum())


def _base_rows(rows, s, rng):
    p = np.zeros((rows, 7), np.float32)
    p[:, 0] = rng.uniform(0, s, rows)
    p[:, 1] = rng.uniform(0, s, rows)
    p[:, 2] = rng.uniform(4, 300, rows)
    p[:, 3] = rng.uniform(4, 300, rows)
    p[:, 4] = rng.uniform(0, 0.39, rows)
    p[:, 5:] = rng.uniform(0, 1, (rows, 2))
    return p


def _hot(p, n, rng):
    hot = rng.choice(len(p), n, replace=False)
    p[hot, 4] = rng.uniform(0.41, 1.0, n)
    for k in hot[: n // 2]:   # near-duplicates, so that suppression really happens
        j = int(rng.integers(0, len(p)))
        p[j] = p[k]
        p[j, :4] += rng.normal(0, 3, 4).astype(np.float32)
        p[j, 4] = min(1.0, p[k, 4] * float(rng.uniform(0.8, 1.2)))
    return p


def rows_none(rows, s, rng):
    p = _base_rows(rows, s, rng)
    assert _n_cand(p) == 0
    return p


def rows_overflow(rows, s, rng):
    p = _hot(_base_rows(rows, s, rng), 9000, rng)
    p[:, 4] = np.round(p[:, 4], 2)   # many exact ties straddling the 4096 cut: the lowest rows must win
    p[:, 5:] = 1.0
    sc = _score(p)
    cand = np.where((p[:, 4] > CONF) & (sc > CONF))[0]
    order = cand[np.lexsort((cand, -sc[cand]))]
    assert len(cand) > CAP and sc[order[CAP - 1]] == sc[order[CAP]]
    return p


def rows_max_det(rows, s, rng):
    # 2000 small boxes on a jittered grid: hardly any overlap, so the 300-detection cut ends the scan
    p = _base_rows(rows, s, rng)
    hot = rng.choice(rows, 2000, replace=False)
    g = np.arange(2000)
    p[hot, 0] = (g % 45) * (s / 45) + 8 + rng.uniform(-1, 1, 2000)
    p[hot, 1] = (g // 45) * (s / 45) + 8 + rng.uniform(-1, 1, 2000)
    p[hot, 2:4] = 6
    p[hot, 4] = rng.uniform(0.5, 1.0, 2000)
    p[hot, 5:] = rng.uniform(0.8, 1.0, (2000, 2))
    ref = postproc_ref.non_max_suppression(torch.from_numpy(p)[None], 0.4, 0.35)[0]
    assert len(ref) == 300
    return p


def rows_ties(rows, s, rng):
    p = _hot(_base_rows(rows, s, rng), 1200, rng)
    p[:, 4] = np.round(p[:, 4], 1)   # exact score ties: the stable order must decide
    p[:, 5:] = 1.0
    sc = _score(p)[p[:, 4] > CONF]
    assert 0 < _n_cand(p) <= CAP and len(np.unique(sc)) < len(sc) // 50
    return p


def rows_obj_at_conf(rows, s, rng):
    p = _hot(_base_rows(rows, s, rng), 800, rng)
    at = rng.choice(rows, 800, replace=False)
    p[at, 4] = CONF                                   # obj exactly at conf_thres: not a candidate
    p[at[:400], 4] = np.nextafter(CONF, np.float32(1))   # the next float up is one if its class score stays above
    p[at, 5:] = 1.0
    assert (p[:, 4] == CONF).sum() >= 300 and 0 < _n_cand(p) <= CAP
    return p


ROW_KINDS = {"none": rows_none, "overflow": rows_overflow, "max_det": rows_max_det, "ties": rows_ties,
             "obj_at_conf": rows_obj_at_conf}


def crafted_batch(n, s, seed, page_kinds=tuple(PAGE_KINDS)):
    """n pages of s x s: every kind of `page_kinds` and every row kind at least once (row kinds cycle independently
    of page kinds), in a seeded shuffled order.
    -> (blks f32 [n][rows][7], lines f32 [n][2][s][s], page kinds, row kinds)"""
    rng = np.random.default_rng(seed)
    pk = (list(page_kinds) * (n // len(page_kinds) + 1))[:n]
    rk = (list(ROW_KINDS) * (n // len(ROW_KINDS) + 1))[:n]
    assert set(pk) == set(page_kinds) and set(rk) == set(ROW_KINDS)
    rng.shuffle(pk)
    rng.shuffle(rk)
    rows = rows_per_image(s)
    blks = np.stack([ROW_KINDS[k](rows, s, rng) for k in rk])
    lines = np.zeros((n, 2, s, s), np.float32)
    for i, k in enumerate(pk):
        lines[i, 0] = PAGE_KINDS[k](s, rng)
        lines[i, 1] = rng.uniform(0, 1, (s, s)).astype(np.float32)   # the threshold map: not read by this stage
    return blks, lines, pk, rk


# ---- the oracle, page by page ---------------------------------------------------------------------------------------
def ref_nms(p):
    """the reference NMS; past the 4096-candidate workspace, on the 4096 best rows by (score desc, row asc)"""
    sc = _score(p)
    cand = np.where((p[:, 4] > CONF) & (sc > CONF))[0]
    if len(cand) > CAP:
        p = p[np.sort(cand[np.lexsort((cand, -sc[cand]))][:CAP])]
    return postproc_ref.non_max_suppression(torch.from_numpy(p)[None], 0.4, 0.35)[0].numpy(), len(cand)


def assert_boxes_match(geom, gb, gs, pred, what):
    """the rule of tests/seg_geometry.py: every box equals the host build of csrc/geom.h on cv2's contours bit for bit,
    skipped rows included (the host equals the oracle but on cv2's start-vertex ties, which are counted); scores equal
    cv2's bit for bit on a map quantised to 2^-24, else within one float32 ulp and bit for bit on >= 99.9 %"""
    n = sg.assert_text_lines(sg.Reference(geom, pred), gb, gs, what)
    print(what, "host-vs-oracle residuals", n)


def results(eng):
    bm, lab, nl = eng.db_components()
    boxes, scores = eng.text_lines()
    return dict(det=eng.detections(), bitmap=bm, labels=lab, n_labels=nl, boxes=boxes, scores=scores)


def check_page_against_oracle(geom, r, i, blks_i, shrink_i, what):
    ref_det, n_cand = ref_nms(blks_i)
    assert r["det"][i].shape == ref_det.shape and np.array_equal(r["det"][i], ref_det), (what, "NMS")
    assert np.array_equal(r["bitmap"][i], (shrink_i > T).astype(np.uint8)), (what, "bitmap")
    n_ref, lab_ref, _, _ = postproc_ref.connected_components_cv2(r["bitmap"][i])
    assert int(r["n_labels"][i]) == n_ref and np.array_equal(r["labels"][i], lab_ref), (what, "CCL")
    assert_boxes_match(geom, r["boxes"][i], r["scores"][i], shrink_i, what)
    return n_cand


def assert_same_results(a, i, b, j, what):
    """page i of result set a equals page j of b: bit for bit, except scores (double sums in another order: one ulp)"""
    assert np.array_equal(a["det"][i], b["det"][j]), (what, "NMS")
    for k in ("bitmap", "labels", "n_labels", "boxes"):
        assert np.array_equal(a[k][i], b[k][j]), (what, k)
    sg.assert_scores_within_ulp(a["scores"][i], b["scores"][j], (what, "scores"))


# ---- engines ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return sg.build_host_geom(tmp_path_factory.mktemp("geom"))


@pytest.fixture(scope="module")
def prog():
    return ctd_b200.compiler.compile_checkpoint(get_checkpoint(0, True))


@pytest.fixture(scope="module")
def eng16(prog):
    """the bench's engine: 16 pages of 1024^2, CUDA graph"""
    e = ctd_b200.Engine(prog, max_batch=16, max_h=1024, max_w=1024, use_graph=True)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng8(prog):
    """the bench's config 5 engine: 8 pages of 1536^2, CUDA graph"""
    e = ctd_b200.Engine(prog, max_batch=8, max_h=1536, max_w=1536, use_graph=True)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng2048():
    """stage-isolated kernels on 2048^2 maps (ctd_seg_represent's limit) and on large pages"""
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    e = ctd_b200.Engine(P, max_batch=1, max_h=2048, max_w=2048, skip_postproc=True)
    yield e
    e.close()


# ---- 2: crafted batches through the forward's post-processing --------------------------------------------------------
# 8 pages cannot hold every kind: the ones whose indexing differs most at 1536^2 (1152 scan segments per page)
KINDS_1536 = ("blobs", "rings", "checker", "squares1001", "disc", "edges", "noise", "at_thresh")


@pytest.mark.parametrize("n,s,seed", [(16, 1024, 0), (8, 1536, 1)])
def test_crafted_batch_matches_oracle_and_single_pages(request, geom, n, s, seed):
    eng = request.getfixturevalue("eng16" if s == 1024 else "eng8")
    blks, lines, pk, rk = crafted_batch(n, s, seed, tuple(PAGE_KINDS) if s == 1024 else KINDS_1536)
    eng.debug_postprocess(blks, lines)
    r = results(eng)
    tot, cap = eng.nms_status(n)
    assert cap == CAP
    over = []
    for i in range(n):
        what = (i, pk[i], rk[i])
        n_cand = check_page_against_oracle(geom, r, i, blks[i], lines[i, 0], what)
        assert int(tot[i]) == n_cand, (what, int(tot[i]), n_cand)
        over.append(n_cand > CAP)
    assert any(over) and not all(over)
    # every page equals itself run alone
    for i in range(n):
        eng.debug_postprocess(blks[i:i + 1], lines[i:i + 1])
        assert_same_results(r, i, results(eng), 0, (i, pk[i], rk[i], "alone"))
        assert int(eng.nms_status(1)[0][0]) == int(tot[i])


def test_debug_postprocess_refuses_bad_shapes(eng16, eng2048):
    z = lambda n, s: (np.zeros((n, rows_per_image(s), 7), np.float32), np.zeros((n, 2, s, s), np.float32))
    with pytest.raises(ctd_b200.CtdError, match="max_batch"):
        eng16.debug_postprocess(*z(17, 64))
    with pytest.raises(ctd_b200.CtdError, match="multiple of 64"):
        eng16.debug_postprocess(*z(1, 200))
    with pytest.raises(ctd_b200.CtdError, match="full pipeline"):
        eng2048.debug_postprocess(*z(1, 64))


# ---- 3: benchmark batches end to end --------------------------------------------------------------------------------
@pytest.mark.parametrize("n,s", [(16, 1024), (8, 1536)])
def test_bench_batch_matches_oracle_and_serial_order(request, geom, n, s):
    """The forward as bench.py runs it (graph, post-processing on two side streams under the rest of the network)
    against the oracle on the engine's own network outputs; then the same batch through profile_forward, which runs
    the post-processing serially on one stream, must give the same results."""
    eng = request.getfixturevalue("eng16" if s == 1024 else "eng8")
    pages = np.stack([synth.structured_page((1000 if s == 1024 else 500) + i, s, s) for i in range(n)])
    eng.forward(pages)
    blks, _mask, lines = eng.net_outputs(want_mask=False)
    r = results(eng)
    n_det = n_lines = 0
    for i in range(n):
        check_page_against_oracle(geom, r, i, blks[i], lines[i, 0], (i, "bench"))
        n_det += len(r["det"][i])
        n_lines += int((r["scores"][i] > 0).sum())
    assert n_det > 10 * n and n_lines > 10 * n, (n_det, n_lines)
    eng.profile_forward(pages)
    blks2, _m, lines2 = eng.net_outputs(want_mask=False)
    assert np.array_equal(blks2, blks) and np.array_equal(lines2, lines)
    r2 = results(eng)
    for i in range(n):
        assert_same_results(r2, i, r, i, (i, "serial"))


# ---- 4: sizes at the limits -----------------------------------------------------------------------------------------
def _map_polygon():
    m = fill_exact(many_vertex_polygon(), 2048, 2048, 20, 25)
    cs = n_contours(m)
    assert len(cs) == 1 and len(cv2.convexHull(cs[0])) == 560
    return m


def _map_blobs2048():
    return stress_maps.blobs(7, 2048, 2048, 400)


def _map_discs2048():
    m = np.zeros((2048, 2048), np.float32)
    for k, (x, y) in enumerate(((400, 400), (1500, 600), (800, 1600))):
        cv2.circle(m, (x, y), 250 + 40 * k, 0.9, -1)
    assert min(len(cv2.convexHull(c)) for c in n_contours(m)) > 128
    return m


MAPS_2048 = {"polygon560": _map_polygon, "blobs": _map_blobs2048, "discs": _map_discs2048}


@pytest.mark.parametrize("name", list(MAPS_2048))
def test_seg_represent_2048(eng2048, geom, name):
    """2048^2 maps: 2048 scan segments in the contour-order scan, hulls of up to 560 vertices"""
    pred = MAPS_2048[name]()
    gb, gs = eng2048.seg_represent(pred, 0.3)
    assert_boxes_match(geom, gb, gs, pred, name)
    if name == "polygon560":
        rb, rs = postproc_ref.seg_represent(pred, 0.3)
        assert rs[0] > 0 and gs[0] == rs[0] and np.array_equal(gb[0], rb[0]), (gb, gs, rb, rs)


@pytest.mark.parametrize("h,w", [(3508, 2480), (4096, 8194), (7016, 4960)])
def test_connected_components_large(eng2048, h, w):
    """A4 at 300 dpi (1062 scan segments), just past 4096 segments, A4 at 600 dpi (4249): labels, count and stats"""
    rng = np.random.default_rng(h + w)
    img = (rng.random((h, w)) < 0.3).astype(np.uint8)
    img[h // 3:h // 3 + 500, :] = 1          # one component across the whole width, met in many segments
    img[:, w // 2] = 0
    n_ref, lab_ref, stats_ref, _ = postproc_ref.connected_components_cv2(img)
    n, lab, stats = eng2048.connected_components(img, stats_cap=n_ref + 4)
    assert n == n_ref
    assert np.array_equal(lab, lab_ref)
    assert np.array_equal(stats[:n_ref], stats_ref)


def test_detect_page_a4_600dpi_keep_undetected():
    """refine_undetected_mask labels the whole page: 7016 x 4960 has 8 699 840 2x2 blocks, 4249 scan segments"""
    net = 1024
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=net, act="leaky", max_batch=1)
    try:
        page = cv2.resize(synth.structured_page(31, 1403, 992), (4960, 7016), interpolation=cv2.INTER_NEAREST)
        got = d(page.copy(), refine_mode=1, keep_undetected_mask=True)
        _r, (uw, uh), _dw, _dh = letterbox_geometry(page.shape[:2], (net, net))
        eng = d.net
        eng.forward(letterbox(page, (net, net))[0][None])
        blks, mask, lines = eng.net_outputs()
        rmask, rref, rblk = postprocess_page_any_size(page.copy(), (net, net), (uh, uw), blks[0], mask[0, 0], lines[0],
                                                      textblock_ref.group_output, refine_mode=1, keep_undetected_mask=True)
    finally:
        d.close()
    key = lambda b: (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
                     float(b.font_size), int(b.angle))
    assert len(rblk) > 0
    assert [key(a) for a in got[2]] == [key(b) for b in rblk]
    assert np.array_equal(got[0], rmask), int((got[0] != rmask).sum())
    assert np.array_equal(got[1], rref), int((got[1] != rref).sum())
