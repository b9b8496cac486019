"""-m gpu: `ctd_b200.PostProcessor`, the detector's post-processing on a caller's network outputs (`ctd_submit_outputs`).

  * identity with the detector: host letterbox -> `TextDetBase` -> `postprocess_batch` equals `TextDetector.detect_batch`
    on the same pages, byte for byte, for every page form, refine mode and result form;
  * against the oracle on outputs this engine never produced: the reference goldens, stress maps, masks on the exact
    k/255 boundaries and outside [0, 1], tied scores and more candidates than the NMS cap;
  * caller tensor forms (batched slices, channel views, permuted strides, mixed batches, a side stream);
  * refusals before any GPU work, a NaN failing its batch, and an abandoned stream."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200.inference import letterbox, letterbox_geometry
from oracle import synth, textblock_ref
from pages_ref import postprocess_page_any_size
from stress_maps import blobs, checkerboard, nested, tiny_components
from util import get_checkpoint, page_to_net_input

pytestmark = pytest.mark.gpu

NET = 256


def _pages(sizes, seed=700):
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _same_value(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return (isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype
                and np.array_equal(a, b, equal_nan=a.dtype.kind == "f"))
    return type(a) is type(b) and a == b


def _same_blocks(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        dg, dr = vars(g), vars(r)
        assert list(dg) == list(dr)
        for k in dr:
            assert _same_value(dg[k], dr[k]), (k, dg[k], dr[k])


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same_result(got, ref):
    assert len(got) == len(ref)
    assert np.array_equal(_host(got[0]), _host(ref[0])), int((_host(got[0]) != _host(ref[0])).sum())
    assert np.array_equal(_host(got[1]), _host(ref[1])), int((_host(got[1]) != _host(ref[1])).sum())
    _same_blocks(got[2], ref[2])
    if len(ref) > 3:
        for gb, rb in zip(got[3], ref[3]):
            assert len(gb) == len(rb)
            for g, r in zip(gb, rb):
                assert (g is None) == (r is None)
                if r is not None:
                    assert np.array_equal(_host(g), _host(r))


def _key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


def _net_outputs(base, pages, net):
    """the outputs of TextDetBase on the host-letterboxed pages: (blks, mask, lines) CUDA tensors, batched"""
    boxed = np.stack([letterbox(p, (net, net))[0] for p in pages])
    return base(page_to_net_input(boxed).cuda())


@pytest.fixture(scope="module")
def env():
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=4)
    base = ctd_b200.TextDetBase(ck, max_batch=8, max_size=NET)
    post = ctd_b200.PostProcessor(input_size=NET, max_batch=4)
    yield det, base, post
    det.close()
    post.close()


SIZES = [(NET, NET), (361, 251), (2 * NET, 2 * NET), (200, 150), (96, 1500), (1, 300), (300, 1)]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("keep", [False, True])
def test_identity_with_detector(env, mode, keep):
    det, base, post = env
    pages = _pages(SIZES)
    blks, mask, lines = _net_outputs(base, pages, NET)
    got = post.postprocess_batch([(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)], mode, keep)
    ref = det.detect_batch([p.copy() for p in pages], refine_mode=mode, keep_undetected_mask=keep)
    for g, r in zip(got, ref):
        _same_result(g, r)
    assert sum(len(r[2]) for r in ref) > 5
    one = post(pages[1], blks[1], mask[1], lines[1], mode, keep)
    _same_result(one, ref[1])


@pytest.mark.parametrize("form", ["numpy", "cuda", "encoded", "textheight", "device_results"])
def test_identity_page_forms(env, form):
    det, base, post = env
    pages = _pages(SIZES[:5], seed=900)
    blks, mask, lines = _net_outputs(base, pages, NET)
    th = 48 if form in ("textheight", "device_results") else None
    dr = form == "device_results"
    imgs = list(pages)
    if form == "cuda":
        imgs = [torch.from_numpy(p).cuda().permute(2, 0, 1).contiguous().permute(1, 2, 0) for p in pages]
    elif form == "encoded":
        imgs = [cv2.imencode(".png" if i % 2 else ".jpg", p)[1].tobytes() for i, p in enumerate(pages)]
    items = [(img, blks[i], mask[i], lines[i]) for i, img in enumerate(imgs)]
    if form == "encoded":   # the decoded pages are what the detector sees
        pages = [cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) for b in imgs]
        blks, mask, lines = _net_outputs(base, pages, NET)
        items = [(img, blks[i], mask[i], lines[i]) for i, img in enumerate(imgs)]
    got = list(post.postprocess_stream(items, 1, True, textheight=th, device_results=dr))
    ref = det.detect_batch(imgs, refine_mode=1, keep_undetected_mask=True, textheight=th, device_results=dr)
    for g, r in zip(got, ref):
        if dr:
            assert g[0].is_cuda and g[1].is_cuda
        _same_result(g, r)


def test_identity_16_pages_1024():
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=1024, act="leaky", max_batch=16)
    base = ctd_b200.TextDetBase(ck, max_batch=16, max_size=1024)
    post = ctd_b200.PostProcessor(input_size=1024, max_batch=16)
    try:
        pages = [synth.structured_page(3000 + i, 1024, 1024) for i in range(16)]
        blks, mask, lines = base(page_to_net_input(np.stack(pages)).cuda())
        got = post.postprocess_batch([(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)])
        ref = det.detect_batch(pages)
        for g, r in zip(got, ref):
            _same_result(g, r)
        assert sum(len(r[2]) for r in ref) > 16
    finally:
        det.close()
        post.close()


# ---- against the oracle ----------------------------------------------------------------------------------------------
def _oracle(page, net_hw, blks, mask, lines, mode=0, keep=False, conf=0.4, iou=0.35):
    # a net-sized page too: its letterbox is the identity, and this form skips the blocks whose window is empty
    unpad = letterbox_geometry(page.shape[:2], net_hw)[1][::-1]
    return postprocess_page_any_size(page.copy(), net_hw, unpad, blks, mask, lines, textblock_ref.group_output, conf,
                                     iou, mode, keep)


def _check_oracle(post, net_hw, items, mode=0, keep=False):
    got = post.postprocess_batch(items, mode, keep)
    n_blocks = 0
    for (page, blks, mask, lines), g in zip(items, got):
        b = blks.reshape(-1, blks.shape[-1])
        rm, rr, rb = _oracle(page, net_hw, b, mask.reshape(net_hw), lines.reshape((-1,) + tuple(net_hw)), mode, keep,
                             post.conf_thresh, post.nms_thresh)
        assert np.array_equal(g[0], rm), int((g[0] != rm).sum())
        gk, rk = [_key(a) for a in g[2]], [_key(r) for r in rb]
        bad = next((i for i, (x, y) in enumerate(zip(gk, rk)) if x != y), None)
        assert len(gk) == len(rk) and bad is None, (len(gk), len(rk), bad, bad is not None and (gk[bad], rk[bad]))
        assert np.array_equal(g[1], rr), int((g[1] != rr).sum())
        n_blocks += len(rb)
    return n_blocks


@pytest.mark.xfail(strict=True, reason="on the 312 blocks of this golden, block 291 (9 lines) differs between the "
                   "native group_output and the oracle's textblock_ref: a group_output finding, not one of the ingest")
def test_oracle_reference_golden():
    z = np.load("tests/golden/net_ref_128x192.npz")
    post = ctd_b200.PostProcessor(input_size=(128, 192), max_batch=2)
    try:
        pages = [synth.structured_page(11, 128, 192), _pages([(300, 200)], seed=12)[0]]
        items = [(p, z["blks"], z["mask"], z["lines"]) for p in pages]
        for mode, keep in ((0, False), (1, True)):
            _check_oracle(post, (128, 192), items, mode, keep)
    finally:
        post.close()


@pytest.mark.parametrize("name", ["net_rough_256", "net_smooth_256"])
def test_oracle_goldens_sub_maps(name):
    z = np.load("tests/golden/%s.npz" % name)
    post = ctd_b200.PostProcessor(input_size=64, max_batch=2)
    try:
        items = [(synth.structured_page(20 + i, 128, 128)[:64, :64].copy(), z["blks_sub"][i], z["mask_sub"][i],
                  z["lines_sub"][i]) for i in range(2)]
        _check_oracle(post, (64, 64), items, 0, True)
    finally:
        post.close()


def _det_rows(rng, a, net, n_cand, tie=False):
    """blks rows [a][7]: n_cand candidates (obj, cls above conf) of small boxes spread over the net, the rest below"""
    b = np.zeros((a, 7), np.float32)
    b[:, 0:2] = rng.uniform(8, net - 8, (a, 2))
    b[:, 2:4] = rng.uniform(4, 24, (a, 2))
    b[:, 4] = rng.uniform(0, 0.35, a)
    b[:, 5:7] = rng.uniform(0, 1, (a, 2))
    idx = rng.choice(a, n_cand, replace=False)
    b[idx, 4] = 0.5 + 0.5 * rng.uniform(0, 1, n_cand) if not tie else 0.75
    b[idx, 5] = 1.0
    return b


def test_oracle_stress_maps_boundaries_ties_overflow():
    net = 512
    post = ctd_b200.PostProcessor(input_size=net, max_batch=3)
    rng = np.random.default_rng(5)
    a = ctd_b200.postprocess.workspace_rows(net, net)
    try:
        k = np.arange(-600, 600, dtype=np.float32)
        edge = np.concatenate([k / np.float32(255), np.nextafter(k / np.float32(255), np.float32(2)),
                               np.array([1.2, 300 / 255, -0.5, -1 / 255, 3e9 / 255, -3e9 / 255], np.float32)])
        maps = [cv2.resize(blobs(1), (net, net)), np.resize(edge, (net, net)).astype(np.float32),
                np.pad(nested(2), 128).astype(np.float32), np.pad(checkerboard(), 192).astype(np.float32),
                cv2.resize(tiny_components(), (net, net), interpolation=cv2.INTER_NEAREST)]
        items = []
        for i, m in enumerate(maps):
            page = _pages([(net, net) if i % 2 == 0 else (700, 400)], seed=40 + i)[0]
            # the boundary mask is not a probability map: its lines_map is a stress map of its own
            l0 = cv2.resize(blobs(3), (net, net)) if i == 1 else m
            lines = np.stack([l0, rng.uniform(0, 1, m.shape).astype(np.float32)])[None]
            n_cand = [50, 5000, 300, 4200, 20][i]   # 5000 and 4200: more candidates than the NMS cap of 4096
            blks = _det_rows(rng, a - 17 * i, net, n_cand, tie=(i == 2))
            if i == 4:
                blks[10:20] = blks[9]   # exactly tied rows
            items.append((page, blks[None], m[None, None], lines))
        assert _check_oracle(post, (net, net), items, 1, True) > 0
    finally:
        post.close()


# ---- caller tensor forms -------------------------------------------------------------------------------------------
def test_tensor_forms(env):
    det, base, post = env
    pages = _pages(SIZES[:4], seed=300)
    blks, mask, lines = _net_outputs(base, pages, NET)
    want = post.postprocess_batch([(p, blks[i].contiguous(), mask[i].contiguous(), lines[i].contiguous())
                                   for i, p in enumerate(pages)])
    cl = mask.contiguous(memory_format=torch.channels_last)
    lt = lines.transpose(2, 3).contiguous().transpose(2, 3)         # column-major planes
    bt = blks.transpose(1, 2).contiguous().transpose(1, 2)          # column-major rows
    forms = [
        [(p, blks[i:i + 1], mask[i:i + 1], lines[i:i + 1, :1]) for i, p in enumerate(pages)],
        [(p, bt[i], cl[i], lt[i]) for i, p in enumerate(pages)],
        [(p, blks[i].cpu().numpy() if i % 2 else blks[i], mask[i] if i % 2 else mask[i].cpu().numpy(),
          lines[i].cpu().numpy()) for i, p in enumerate(pages)],
        [(torch.from_numpy(p).cuda(), blks[i][:, :].cpu(), mask[i, 0].cpu(), lines[i]) for i, p in enumerate(pages)],
    ]
    for items in forms:
        for g, r in zip(post.postprocess_batch(items), want):
            _same_result(g, r)


def test_outputs_written_on_side_stream(env):
    det, base, post = env
    pages = _pages(SIZES[:3], seed=310)
    blks, mask, lines = _net_outputs(base, pages, NET)
    want = post.postprocess_batch([(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        b2, m2, l2 = torch.zeros_like(blks), torch.zeros_like(mask), torch.zeros_like(lines)
        torch.cuda._sleep(20_000_000)
        b2.copy_(blks)
        m2.copy_(mask)
        l2.copy_(lines)
        got = list(post.postprocess_stream([(p, b2[i], m2[i], l2[i]) for i, p in enumerate(pages)]))
    for g, r in zip(got, want):
        _same_result(g, r)


# ---- refusals, non-finite values, early stop --------------------------------------------------------------------------
def test_refusals_then_usable(env):
    det, base, post = env
    pages = _pages(SIZES[:2], seed=320)
    blks, mask, lines = _net_outputs(base, pages, NET)
    good = [(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)]
    want = post.postprocess_batch(good)
    bad = [
        (pages[1], blks[1].half(), mask[1], lines[1]),
        (pages[1], blks[1], mask[1, :, :128], lines[1]),
        (pages[1], blks[1], mask[1].bfloat16(), lines[1]),
        (pages[1], blks[1], mask[1], lines[1, :0]),
        (np.zeros((1, 100000, 3), np.uint8), blks[1], mask[1], lines[1]),
        (pages[1], np.zeros((1, 99999, 7), np.float32), mask[1], lines[1]),
        (pages[1][..., 0], blks[1], mask[1], lines[1]),
    ]
    for item in bad:
        with pytest.raises(ValueError, match="item 1: "):
            post.postprocess_batch([good[0], item])
        with pytest.raises(ValueError, match="item 1: "):
            list(post.postprocess_stream([good[0], item]))
    for g, r in zip(post.postprocess_batch(good), want):
        _same_result(g, r)


@pytest.mark.parametrize("where", ["blks", "mask", "lines_map"])
def test_nonfinite_fails_its_batch(env, where):
    det, base, post = env
    pages = _pages(SIZES[:4], seed=330)
    blks, mask, lines = _net_outputs(base, pages, NET)
    good = [(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)]
    want = post.postprocess_batch(good)
    b, m, ln = blks[2].clone(), mask[2].clone(), lines[2].clone()
    {"blks": b, "mask": m, "lines_map": ln}[where].view(-1)[77] = float("nan") if where != "mask" else float("inf")
    items = list(good)
    items[2] = (pages[2], b, m, ln)
    with pytest.raises(ValueError, match="item 2: a non-finite value .*%s" % where):
        list(post.postprocess_stream(items))
    for g, r in zip(post.postprocess_batch(good), want):
        _same_result(g, r)


def test_abandoned_stream(env):
    det, base, post = env
    pages = _pages(SIZES[:5], seed=340)
    blks, mask, lines = _net_outputs(base, pages, NET)
    items = [(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)] * 3
    want = post.postprocess_batch(items[:5])
    gen = post.postprocess_stream(items)
    next(gen)
    gen.close()   # batches in flight are drained
    for g, r in zip(post.postprocess_batch(items[:5]), want):
        _same_result(g, r)
