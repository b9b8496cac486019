"""-m gpu: pages and results in GPU memory for the batched stream (`TextDetector.detect_stream` / `detect_batch` with
torch.uint8 CUDA pages and `device_results=True`; ctd_submit_pages with device pages, the batched strided page gather,
ctd_collect_device).  The numpy stream is the reference (it is pinned against the reference's goldens elsewhere): every
mask, mask_refined, block and crop must be byte-identical to what it gives for the same pages."""
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding
from oracle import synth
from util import get_checkpoint

pytestmark = pytest.mark.gpu

NET = 256
# the mixed sizes of test_gpu_stream_regions.py: 6 pages at max_batch 4 give a full and a partial batch
SIZES = [(NET, NET), (361, 251), (414, 292), (2 * NET, 2 * NET), (200, 150), (96, 1500)]


def _pages(sizes, seed=500):
    return [np.ascontiguousarray(synth.structured_page(seed + i, max(h, 128), max(w, 128))[:h, :w])
            for i, (h, w) in enumerate(sizes)]


def _detector(max_batch, net=NET):
    return ctd_b200.TextDetector(get_checkpoint(0, True), input_size=net, act="leaky", max_batch=max_batch)


@pytest.fixture(scope="module")
def det():
    d = _detector(4)
    yield d
    d.close()


def _cuda(pages, device=0):
    return [torch.from_numpy(p).to("cuda:%d" % device) for p in pages]


def _host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same_value(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)
    return type(a) is type(b) and a == b


def _same_item(got, ref, device=None):
    """one yielded item against the numpy stream's; device: the results must be CUDA tensors on that GPU, every tensor
    of the page a view into one allocation.  Returns the page's storage pointer (device) or None."""
    assert len(got) == len(ref)
    tensors = [got[0], got[1]] + ([c for blk in got[3] for c in blk if c is not None] if len(got) == 4 else [])
    storage = None
    if device is not None:
        for t in tensors:
            assert isinstance(t, torch.Tensor) and t.is_cuda and t.device.index == device and t.dtype == torch.uint8
        ptrs = {t.untyped_storage().data_ptr() for t in tensors}
        assert len(ptrs) == 1, ptrs
        storage = ptrs.pop()
    else:
        assert all(isinstance(t, np.ndarray) for t in tensors)
    for k in (0, 1):
        g = _host(got[k])
        assert g.shape == ref[k].shape and np.array_equal(g, ref[k]), (k, int((g != ref[k]).sum()))
    assert len(got[2]) == len(ref[2])
    for g, r in zip(got[2], ref[2]):
        dg, dr = vars(g), vars(r)
        assert list(dg) == list(dr)
        for k in dr:
            assert _same_value(dg[k], dr[k]), (k, dg[k], dr[k])
    if len(got) == 4:
        assert len(got[3]) == len(ref[3])
        for gb, rb in zip(got[3], ref[3]):
            assert len(gb) == len(rb)
            for g, r in zip(gb, rb):
                assert (g is None) == (r is None)
                if r is not None:
                    g = _host(g)
                    assert g.shape == r.shape and np.array_equal(g, r)
    return storage


def _same_stream(got, ref, device=None):
    assert len(got) == len(ref)
    storages = [_same_item(g, r, device) for g, r in zip(got, ref)]
    if device is not None:
        assert len(set(storages)) == len(storages)   # one allocation per page, none shared


@pytest.mark.parametrize("th", [None, 32, 48])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("keep", [False, True])
def test_cuda_pages_and_device_results(det, th, mode, keep):
    pages = _pages(SIZES)
    kw = dict(refine_mode=mode, keep_undetected_mask=keep, textheight=th)
    ref = list(det.detect_stream([p.copy() for p in pages], **kw))
    n_crops = sum(1 for r in ref if th for blk in r[3] for c in blk if c is not None)
    assert th is None or n_crops > 20
    # CUDA pages, host results
    _same_stream(list(det.detect_stream(_cuda(pages), **kw)), ref)
    # CUDA pages, device results
    _same_stream(list(det.detect_stream(_cuda(pages), device_results=True, **kw)), ref, device=0)
    # numpy pages, device results; detect_batch gives the same
    _same_stream(det.detect_batch([p.copy() for p in pages], device_results=True, **kw), ref, device=0)


def test_strided_pages(det):
    pages = _pages([(361, 251), (414, 292), (200, 150), (300, 211), (NET, NET), (123, 457)], seed=1500)
    cuda = []
    # a sub-window of a larger tensor at byte offsets 0, 1, 2 and 4 modulo 16 of the row (every copy path of the
    # gather), with row pitches that are not multiples of 16
    for i, (p, x0) in enumerate(zip(pages[:4], (0, 1, 2, 4))):
        h, w = p.shape[:2]
        big = torch.zeros((h + 7, w + x0 + 3, 3), dtype=torch.uint8, device="cuda:0")
        assert (big.stride(0) % 16) != 0
        big[5:5 + h, x0:x0 + w] = torch.from_numpy(p).cuda()
        cuda.append(big[5:5 + h, x0:x0 + w])
    # a channels-first tensor, permuted
    chw = torch.from_numpy(np.ascontiguousarray(pages[4].transpose(2, 0, 1))).cuda()
    cuda.append(chw.permute(1, 2, 0))
    # a column-major page ([w][h][3] transposed) and a broadcast uniform page (strides 0)
    cuda.append(torch.from_numpy(np.ascontiguousarray(pages[5].transpose(1, 0, 2))).cuda().transpose(0, 1))
    uniform = torch.tensor([30, 90, 200], dtype=torch.uint8, device="cuda:0").expand(150, 220, 3)
    cuda.append(uniform)
    assert not any(t.is_contiguous() for t in cuda)
    host = [t.cpu().numpy() for t in cuda]
    for th in (None, 48):
        ref = list(det.detect_stream([h.copy() for h in host], textheight=th, keep_undetected_mask=True))
        _same_stream(list(det.detect_stream(cuda, textheight=th, keep_undetected_mask=True)), ref)
        _same_stream(list(det.detect_stream(cuda, textheight=th, keep_undetected_mask=True, device_results=True)), ref,
                     device=0)


def test_mixed_batches(det):
    pages = _pages(SIZES + [(333, 222), (222, 333)], seed=2500)
    mixed = [torch.from_numpy(p).cuda() if i % 3 != 1 else p.copy() for i, p in enumerate(pages)]
    for th in (None, 32):
        ref = list(det.detect_stream([p.copy() for p in pages], refine_mode=1, textheight=th))
        _same_stream(list(det.detect_stream(mixed, refine_mode=1, textheight=th)), ref)
        _same_stream(det.detect_batch(mixed, refine_mode=1, textheight=th, device_results=True), ref, device=0)
    # CPU torch tensors still go through np.asarray
    ref = list(det.detect_stream([p.copy() for p in pages[:3]]))
    _same_stream(list(det.detect_stream([torch.from_numpy(p.copy()) for p in pages[:3]])), ref)


def test_stream_ordering(det):
    # pages written on a side stream behind a long sleep: the engine must wait for that stream before reading them
    pages = _pages(SIZES, seed=3500)
    ref = list(det.detect_stream([p.copy() for p in pages], textheight=48))
    src = _cuda(pages)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    for device_results in (False, True):
        with torch.cuda.stream(side):
            filled = []
            for s in src:
                d = torch.zeros_like(s)
                torch.cuda._sleep(20_000_000)
                d.copy_(s)
                filled.append(d)
            got = list(det.detect_stream(filled, textheight=48, device_results=device_results))
            _same_stream(got, ref, device=0 if device_results else None)
    torch.cuda.synchronize()


def test_blank_pages_growth_and_abandoned_stream():
    d = _detector(3)
    try:
        blanks = [np.full((NET, NET, 3), 128, np.uint8), np.full((NET // 2, NET // 2, 3), 144, np.uint8),
                  np.full((2 * NET, 2 * NET, 3), 112, np.uint8)]
        ref = list(d.detect_stream([p.copy() for p in blanks], textheight=32))
        assert any(sum(len(b.lines) for b in r[2]) == 0 for r in ref)
        _same_stream(list(d.detect_stream(_cuda(blanks), textheight=32, device_results=True)), ref, device=0)
        empty = [p for p, r in zip(blanks, ref) if sum(len(b.lines) for b in r[2]) == 0]
        # a batch without a single crop
        ref_e = list(d.detect_stream([p.copy() for p in empty], textheight=32))
        _same_stream(d.detect_batch(_cuda(empty), textheight=32, device_results=True), ref_e, device=0)
        # a later batch larger than every earlier one, then small ones again
        small = _pages([(120, 90), (200, 150), (150, 150)], seed=4000)
        large = _pages([(2000, 3000), (1654, 1170), (3000, 2000)], seed=4100)
        for pages in (small, large + small[:2], small):
            ref = list(d.detect_stream([p.copy() for p in pages], keep_undetected_mask=True, textheight=48))
            _same_stream(list(d.detect_stream(_cuda(pages), keep_undetected_mask=True, textheight=48,
                                              device_results=True)), ref, device=0)
        # a generator abandoned mid-stream, then a normal stream on the same detector
        pages = _pages(SIZES, seed=4500)
        ref = list(d.detect_stream([p.copy() for p in pages], textheight=48))
        g = d.detect_stream(_cuda(pages), textheight=48, device_results=True)
        _same_item(next(g), ref[0], device=0)
        g.close()
        _same_stream(list(d.detect_stream(_cuda(pages), textheight=48, device_results=True)), ref, device=0)
        _same_stream(list(d.detect_stream([p.copy() for p in pages], textheight=48)), ref)
    finally:
        d.close()


def test_device_page_errors(det):
    pages = _pages(SIZES[:3], seed=5500)
    good = _cuda(pages)
    bad = {
        "dtype": torch.from_numpy(pages[0]).cuda().float(),
        "rank": torch.from_numpy(pages[0][..., 0].copy()).cuda(),
        "channels": torch.zeros((64, 64, 4), dtype=torch.uint8, device="cuda:0"),
        "empty": torch.zeros((0, 64, 3), dtype=torch.uint8, device="cuda:0"),
    }
    if torch.cuda.device_count() > 1:
        bad["device"] = torch.from_numpy(pages[0]).to("cuda:1")
    for name, b in bad.items():
        with pytest.raises(ValueError):
            det.detect_batch(good + [b])
        with pytest.raises(ValueError):
            next(det.detect_stream([b] + good))
        with pytest.raises(ValueError):
            ctd_b200.inference.check_page(b, 0)
    # the C ABI: a host pointer given as a device page, a NULL page with no input_host, and ctd_collect_device of a
    # slot whose batch kept its results on the host
    eng = det.net
    ent, ib, rb = binding.pages_plan([p.shape[:2] for p in pages[:2]], NET, NET)
    out = torch.empty((rb,), dtype=torch.uint8, pin_memory=True)
    host = np.ascontiguousarray(pages[0])
    dev = (binding.CtdDevicePage * 2)(binding.CtdDevicePage(host.ctypes.data, host.strides[0], 3, 1, None),
                                      binding.CtdDevicePage(good[1].data_ptr(), good[1].stride(0), 3, 1, None))
    rc = eng.lib.ctd_submit_pages(eng.h, 1, binding._ptr(ent), 2, NET, NET, None, binding.C.cast(dev, binding.C.c_void_p),
                                  0, 0, 0, 1, binding.C.c_void_p(out.data_ptr()))
    assert rc == -1 and b"page 0" in eng.lib.ctd_last_error(eng.h)
    dev[0] = binding.CtdDevicePage(None, 0, 0, 0, None)
    rc = eng.lib.ctd_submit_pages(eng.h, 1, binding._ptr(ent), 2, NET, NET, None, binding.C.cast(dev, binding.C.c_void_p),
                                  0, 0, 0, 1, binding.C.c_void_p(out.data_ptr()))
    assert rc == -1
    eng.submit_pages(1, pages[:2], NET, NET)
    eng.collect_pages(1)
    ptrs = (binding.C.c_void_p * 2)(good[0].data_ptr(), good[1].data_ptr())
    assert eng.lib.ctd_collect_device(eng.h, 1, ptrs) == -1
    # the detector still works after every refusal
    ref = list(det.detect_stream([p.copy() for p in pages], textheight=32))
    _same_stream(det.detect_batch(good, textheight=32, device_results=True), ref, device=0)
