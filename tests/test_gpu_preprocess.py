"""-m gpu: the detector's pre-processing on the GPU (`ctd_preprocess_pages`): `Preprocessor.preprocess_batch` and
`preprocess_img` against the oracle's restatement of the reference's `preprocess_img` (oracle/preprocess_ref.py), bit
for bit, in all three layouts and both channel orders, for every page form; stream order; refusals before any GPU
work; and `NetworkDetector` against `TextDetector` (through `TextDetBase`) and against `PostProcessor` on the oracle's
pre-processing (through a network that is not the engine's)."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding
from oracle import preprocess_ref, synth
from util import get_checkpoint

pytestmark = pytest.mark.gpu

FLAGS = [(True, False, True), (False, False, True), (True, True, True), (False, True, True), (True, False, False),
         (False, False, False)]   # (bgr2rgb, half, to_tensor)


def _page(h, w, seed=0):
    return np.ascontiguousarray(synth.structured_page(seed, max(h, 128), max(w, 128))[:h, :w])


def _noise(h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


# at 1024 x 1024: net-sized (every u8 value), exact 2x decimation, upscaling, 1 x N and N x 1, half-to-even unpad sizes
# (5 * 0.5 = 2.5 -> 2, 7 * 0.5 = 3.5 -> 4), a downscale
SHAPES_1024 = [(1024, 1024), (2048, 2048), (361, 251), (1, 300), (300, 1), (2048, 5), (2048, 7), (1654, 1170)]
# a non-square net input (h, w) = (384, 640)
SHAPES_NS = [(384, 640), (768, 1280), (100, 70), (1, 300), (300, 1), (640, 5), (900, 1600)]


def _pages(shapes, seed=0):
    return [_noise(h, w, seed + i) if i % 2 == 0 else _page(h, w, seed + i) for i, (h, w) in enumerate(shapes)]


def _same(got, ref, half, to_tensor, what=""):
    """got (a CUDA tensor [..]) and the oracle's value (tensor or numpy) have the same dtype, shape and bits"""
    ref = torch.from_numpy(ref) if isinstance(ref, np.ndarray) else ref
    got = got.cpu()
    assert got.dtype == ref.dtype and tuple(got.shape) == tuple(ref.shape), (what, got.dtype, ref.dtype, got.shape)
    view = (torch.int16 if half else torch.int32) if to_tensor else torch.uint8
    eq = got.view(view) == ref.view(view)
    assert bool(eq.all()), (what, int((~eq).sum()))


def _check_batch(pre, pages, refs_src, flags):
    bgr2rgb, half, to_tensor = flags
    img_in, ratios, dws, dhs = pre.preprocess_batch(pages, bgr2rgb, half, to_tensor)
    assert img_in.is_cuda and img_in.shape[0] == len(pages)
    for i, src in enumerate(refs_src):
        r_in, r_ratio, r_dw, r_dh = preprocess_ref.preprocess_img(src.copy(), pre.input_size, 'cpu', bgr2rgb, half,
                                                                  to_tensor)
        _same(img_in[i], r_in[0] if to_tensor else r_in, half, to_tensor, "page %d %s" % (i, src.shape))
        assert ratios[i] == r_ratio and type(ratios[i][0]) is float
        assert (dws[i], dhs[i]) == (r_dw, r_dh) and type(dws[i]) is int and type(dhs[i]) is int


@pytest.fixture(scope="module")
def pre1024():
    p = ctd_b200.Preprocessor(1024, max_batch=4)
    yield p
    p.close()


@pytest.fixture(scope="module")
def pre_ns():
    p = ctd_b200.Preprocessor((384, 640), max_batch=16)
    yield p
    p.close()


@pytest.mark.parametrize("flags", FLAGS)
def test_shapes_1024(pre1024, flags):
    pages = _pages(SHAPES_1024)
    _check_batch(pre1024, pages, pages, flags)


@pytest.mark.parametrize("flags", FLAGS)
def test_shapes_non_square(pre_ns, flags):
    pages = _pages(SHAPES_NS, seed=50)
    _check_batch(pre_ns, pages, pages, flags)


@pytest.mark.parametrize("flags", FLAGS)
def test_every_u8_value(pre_ns, flags):
    """a net-sized page holding every u8 value in every channel, as is (no resize)"""
    v = np.arange(384 * 640 * 3, dtype=np.int64).reshape(384, 640, 3)
    page = ((v * 7 + v // 640) % 256).astype(np.uint8)
    _check_batch(pre_ns, [page], [page], flags)


def _cuda_forms(pages):
    """contiguous, a crop of a larger tensor, and a channels-first tensor permuted back"""
    out = []
    for i, p in enumerate(pages):
        t = torch.from_numpy(p).cuda()
        if i % 3 == 1:
            big = torch.zeros((p.shape[0] + 5, p.shape[1] + 9, 3), dtype=torch.uint8, device="cuda")
            big[3:3 + p.shape[0], 7:7 + p.shape[1]] = t
            t = big[3:3 + p.shape[0], 7:7 + p.shape[1]]
        elif i % 3 == 2:
            t = t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
        out.append(t)
    return out


@pytest.mark.parametrize("form", ["cuda", "jpeg", "png", "paths", "mixed"])
@pytest.mark.parametrize("flags", [FLAGS[0], FLAGS[3], FLAGS[5]])
def test_page_forms(pre_ns, form, flags, tmp_path):
    src = _pages(SHAPES_NS[:6], seed=90)
    if form == "cuda":
        pages = _cuda_forms(src)
    elif form in ("jpeg", "png", "paths"):
        ext = ".png" if form == "png" else ".jpg"
        pages = [cv2.imencode(ext if form != "paths" or i % 2 else ".png", p)[1].tobytes() for i, p in enumerate(src)]
        if form == "paths":
            paths = []
            for i, b in enumerate(pages):
                f = tmp_path / ("p%d.bin" % i)
                f.write_bytes(b)
                paths.append(str(f))
            pages = paths
            src = [cv2.imdecode(np.fromfile(f, np.uint8), cv2.IMREAD_COLOR) for f in paths]
        else:
            src = [cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) for b in pages]
    else:
        cuda = _cuda_forms(src)
        enc = [cv2.imencode(".jpg", p)[1].tobytes() for p in src]
        pages = [src[0], cuda[1], enc[2], cuda[3], src[4], cv2.imencode(".png", src[5])[1].tobytes()]
        src = list(src)
        src[2] = cv2.imdecode(np.frombuffer(enc[2], np.uint8), cv2.IMREAD_COLOR)
    _check_batch(pre_ns, pages, src, flags)


def test_batch_of_one_and_max_batch(pre_ns, pre1024):
    pages = _pages([(500 + 13 * i, 300 + 29 * i) for i in range(16)], seed=300)
    _check_batch(pre_ns, pages, pages, FLAGS[0])            # one launch of max_batch = 16 pages
    _check_batch(pre_ns, pages[:1], pages[:1], FLAGS[0])
    _check_batch(pre1024, pages[:11], pages[:11], FLAGS[2])  # three launches of up to 4 pages into one tensor


@pytest.mark.parametrize("flags", FLAGS)
def test_preprocess_img_drop_in(flags):
    bgr2rgb, half, to_tensor = flags
    for shape, size in (((361, 251), (1024, 1024)), ((700, 1200), (384, 640)), ((1024, 1024), 1024)):
        page = _page(*shape, seed=shape[0])
        got = ctd_b200.preprocess_img(page, size, 'cuda', bgr2rgb, half, to_tensor)
        ref = preprocess_ref.preprocess_img(page.copy(), size, 'cpu', bgr2rgb, half, to_tensor)
        if to_tensor:
            assert got[0].is_cuda and got[0].device == torch.device("cuda", 0)
        else:
            assert isinstance(got[0], np.ndarray)
        _same(torch.from_numpy(got[0]) if not to_tensor else got[0], ref[0], half, to_tensor)
        assert got[1:] == ref[1:]
    got = ctd_b200.preprocess_img(torch.from_numpy(page).cuda(), device=torch.device("cuda", 0))
    _same(got[0], preprocess_ref.preprocess_img(page.copy())[0], False, True)


def test_side_stream_writer(pre_ns):
    """a page written by a kernel queued on the current (side) stream right before the call is read after it, and
    the call's result there has the same bits"""
    src = _page(700, 500, seed=5)
    side = torch.cuda.Stream()
    base = torch.from_numpy(src).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)   # keeps the writer below queued when the call is made
        page = torch.empty_like(base)
        page.copy_(base.flip(0).flip(0))
        img_in = pre_ns.preprocess_batch([page])[0]
    side.synchronize()
    _same(img_in[0], preprocess_ref.preprocess_img(src.copy(), (384, 640))[0][0], False, True)


def test_non_default_stream_same_bits(pre_ns):
    pages = _pages(SHAPES_NS, seed=77)
    want = pre_ns.preprocess_batch(pages, half=True)[0]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = pre_ns.preprocess_batch(_cuda_forms(pages), half=True)[0]
    s.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_host_pages_through_input_host(pre_ns):
    """the C entry's input_host path: numpy pages packed into a pinned buffer, a mixed batch with CUDA pages"""
    pages = _pages(SHAPES_NS[:4], seed=11)
    mixed = [pages[0], torch.from_numpy(pages[1]).cuda(), pages[2], torch.from_numpy(pages[3]).cuda()]
    _ent, in_bytes, _ = binding.pages_plan([p.shape[:2] for p in pages], 384, 640)
    host = torch.empty((in_bytes,), dtype=torch.uint8, pin_memory=True)
    out = torch.empty((4, 3, 384, 640), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream()
    pre_ns.net.preprocess_pages(mixed, 384, 640, binding.PRE_F32_NCHW, False, out.data_ptr(), stream.cuda_stream,
                                input_host=host)
    torch.cuda.synchronize()
    for i, p in enumerate(pages):
        _same(out[i], preprocess_ref.preprocess_img(p.copy(), (384, 640))[0][0], False, True)


def test_refusals_before_gpu_work():
    pre = ctd_b200.Preprocessor((384, 640), max_batch=2)
    try:
        lib = binding.load_library()
        page = torch.from_numpy(_page(300, 200)).cuda()
        ent, _, _ = binding.pages_plan([(300, 200)], 384, 640)
        ent3, _, _ = binding.pages_plan([(300, 200)] * 3, 384, 640)
        ent_thin, _, _ = binding.pages_plan([(1, 300)], 384, 640)   # fine at 384 x 640, 0 px high at 64 x 64
        moved = ent.copy()
        moved[0]["page_off"] = 256
        dst = torch.full((3, 3, 384, 640), -7.0, device="cuda")
        host_dst = torch.zeros((3 * 384 * 640,), dtype=torch.float32, pin_memory=True)
        st = torch.cuda.current_stream().cuda_stream

        def call(entries, n, net_h, net_w, pages, fmt=0, out=dst.data_ptr()):
            dev = (binding.CtdDevicePage * n)()
            for i in range(n):
                p = pages[i]
                dev[i] = binding.CtdDevicePage(p if isinstance(p, int) else p.data_ptr(), 600, 3, 1, None)
            return lib.ctd_preprocess_pages(pre.net.h, binding._ptr(entries), n, net_h, net_w, None,
                                            C.cast(dev, C.c_void_p), fmt, 0, C.c_void_p(out), C.c_void_p(st))

        cases = [
            ("max_batch", call(ent3, 3, 384, 640, [page] * 3), -5),
            ("net side", call(ent, 1, 384, 600, [page]), -4),
            ("letterbox", call(ent_thin, 1, 64, 64, [page]), -4),
            ("not the plan", call(moved, 1, 384, 640, [page]), -1),
            ("host page", call(ent, 1, 384, 640, [host_dst.data_ptr()]), -1),
            ("format", call(ent, 1, 384, 640, [page], fmt=3), -1),
            ("dst alignment", call(ent, 1, 384, 640, [page], out=dst.data_ptr() + 4), -1),
            ("host dst", call(ent, 1, 384, 640, [page], out=host_dst.data_ptr()), -1),
        ]
        for what, rc, want in cases:
            assert rc == want, (what, rc, lib.ctd_last_error(pre.net.h))
        torch.cuda.synchronize()
        assert bool((dst == -7.0).all()), "a refused call wrote dst"
        assert bool((host_dst == 0).all())
        # the handle is usable afterwards
        img_in = pre.preprocess_batch([page, page.cpu().numpy()])[0]
        ref = preprocess_ref.preprocess_img(page.cpu().numpy(), (384, 640))[0][0]
        _same(img_in[0], ref, False, True)
        _same(img_in[1], ref, False, True)
        with pytest.raises(ValueError, match="item 1: a page must be a uint8"):
            pre.preprocess_batch([page, np.zeros((5, 5), np.uint8)])
    finally:
        pre.close()


# ---- NetworkDetector ---------------------------------------------------------------------------------------------

NET = 256
SIZES = [(NET, NET), (361, 251), (2 * NET, 2 * NET), (200, 150), (96, 1500), (1, 300), (300, 1)]


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same_value(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return (isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype
                and np.array_equal(a, b, equal_nan=a.dtype.kind == "f"))
    return type(a) is type(b) and a == b


def _same_result(got, ref):
    assert len(got) == len(ref)
    assert np.array_equal(_host(got[0]), _host(ref[0]))
    assert np.array_equal(_host(got[1]), _host(ref[1]))
    assert len(got[2]) == len(ref[2])
    for g, r in zip(got[2], ref[2]):
        dg, dr = g.to_dict(), r.to_dict()
        assert list(dg) == list(dr)
        for k in dr:
            assert _same_value(dg[k], dr[k]), (k, dg[k], dr[k])
    if len(ref) > 3:
        for gb, rb in zip(got[3], ref[3]):
            assert len(gb) == len(rb)
            for g, r in zip(gb, rb):
                assert (g is None) == (r is None)
                if r is not None:
                    assert np.array_equal(_host(g), _host(r))


@pytest.fixture(scope="module")
def env():
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=3)
    base = ctd_b200.TextDetBase(ck, max_batch=3, max_size=NET)
    nd = ctd_b200.NetworkDetector(base, NET, max_batch=3)
    yield det, base, nd
    det.close()
    nd.close()
    base.close()


def _mixed(pages):
    cuda = _cuda_forms(pages)
    return [pages[0], cuda[1], cv2.imencode(".jpg", pages[2])[1].tobytes(), cuda[3], pages[4],
            cv2.imencode(".png", pages[5])[1].tobytes(), cuda[6]]


@pytest.mark.parametrize("mode", [
    dict(), dict(refine_mode=1, keep_undetected_mask=True), dict(textheight=48), dict(textheight=48, device_results=True)])
def test_network_detector_is_text_detector(env, mode):
    det, _base, nd = env
    pages = _pages(SIZES, seed=400)
    imgs = _mixed(pages)
    got = nd.detect_batch(imgs, **mode)
    ref = det.detect_batch(imgs, **mode)
    assert sum(len(r[2]) for r in ref) > 5
    for g, r in zip(got, ref):
        if mode.get("device_results"):
            assert g[0].is_cuda and g[1].is_cuda
        _same_result(g, r)
    _same_result(nd(pages[1]), det(pages[1].copy()))
    _same_result(list(nd.detect_stream(iter(imgs[:4]), **mode))[3], ref[3])


def test_network_detector_other_net(env):
    """a network that is not the engine (TextDetBase, then a fixed perturbation of its outputs): NetworkDetector
    equals PostProcessor on the oracle's pre-processing through the same network"""
    _det, base, _nd = env

    def net(x):
        blks, mask, lines = base(x)
        blks = blks.clone()
        blks[..., 4] = blks[..., 4] * 0.9 + 0.08
        return blks, (mask * 0.8 + 0.15).clamp(0, 1), lines.flip(-1) * 0.97 + 0.02

    nd = ctd_b200.NetworkDetector(net, NET, max_batch=3)
    post = ctd_b200.PostProcessor(NET, max_batch=3)
    try:
        pages = _pages(SIZES, seed=600)
        got = nd.detect_batch(pages, textheight=32)
        items = []
        for a in range(0, len(pages), 3):
            chunk = pages[a:a + 3]
            x = torch.cat([preprocess_ref.preprocess_img(p.copy(), (NET, NET))[0] for p in chunk]).cuda()
            blks, mask, lines = net(x)
            items += [(p, blks[i], mask[i], lines[i]) for i, p in enumerate(chunk)]
        ref = post.postprocess_batch(items, textheight=32)
        assert sum(len(r[2]) for r in ref) > 3
        for g, r in zip(got, ref):
            _same_result(g, r)
    finally:
        nd.close()
        post.close()


def test_network_detector_refusals(env):
    _det, _base, nd = env
    with pytest.raises(ValueError, match="item 2: "):
        nd.detect_batch([_page(100, 100), _page(100, 100), np.zeros((4, 4), np.uint8)])
    with pytest.raises(ValueError, match="item 0: blks"):
        bad = ctd_b200.NetworkDetector(lambda x: (torch.zeros((x.shape[0], 5, 3), device="cuda"),) * 3, NET)
        try:
            bad.detect_batch([_page(100, 100)])
        finally:
            bad.close()
    assert len(nd.detect_batch([_page(120, 90)])) == 1
