"""-m gpu: the layout stage between the caller's memory and the kernels of a batch, byte for byte.

* gather_pages_kernel (csrc/gather.cu) and copy_host_images: every batch of tests/gather_cases.py runs once with host
  pages (and masks) of the same sizes filled with a sentinel, then once with its own images, through ctd_submit_pages
  or through ctd_submit_refine with no blocks (which leaves the mask plane as gathered).  The packed pages (and the mask
  plane) are read back with ctd_debug_read_slot: every image's bytes at its page_off (mask_off) must equal the numpy
  packing of the image, and every byte outside the images must be what the sentinel batch left there.  The cases
  reach every copy path, head and tail of the kernel (tests/test_cpu_gather_cases.py).
* letterbox_batch_kernel (csrc/resize.cu): after a ctd_submit_pages batch, the engine's net input must equal the host
  letterbox of every page byte for byte, for pages that came from the host and through the gather."""
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200.inference import letterbox
from gather_cases import CASES, MAX_BATCH, NET, SENTINEL, dev, host, is_fast, meta, plan, row_path, window
from util import get_checkpoint

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def det():
    d = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=NET, act="leaky", max_batch=MAX_BATCH)
    yield d
    d.close()


def _images(imgs, ch, seed):
    """per image: (what the submit call takes: a numpy array or a CUDA view, its bytes packed as u8 [h][w](x3))"""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    rng = np.random.default_rng(seed)
    out = []
    for img in imgs:
        if img.view is None:
            a = rng.integers(0, 256, (img.h, img.w, 3) if ch == 3 else (img.h, img.w), dtype=np.uint8)
            out.append((a, a))
            continue
        st = torch.randint(0, 256, (img.view.nbytes,), dtype=torch.uint8, device="cuda", generator=gen)
        assert st.data_ptr() % 512 == 0   # the source phases tests/gather_cases.py assumes
        t = st.as_strided(img.view.size, img.view.stride, img.view.offset)
        out.append((t, np.ascontiguousarray(t.cpu().numpy())))
    return out


def _run(eng, job, pages, masks):
    if job == "pages":
        eng.submit_pages(0, pages, NET, NET)
        eng.collect_pages(0, discard=True)
    else:
        eng.submit_refine(0, pages, masks, [np.zeros((0, 4), np.int32)] * len(pages))
        eng.collect_refine(0, discard=True)


def _row(img, ch, dst_off, y):
    if img.view is None:
        return "host image"
    if not is_fast(img, ch):
        return "generic path"
    path, head, words, tail = row_path((img.view.offset + y * img.view.stride[0]) % 256,
                                       (dst_off + y * img.w * ch) % 256, img.w * ch)
    return "%s, head %d, %d words, tail %d" % (path, head, words, tail)


def _check_plane(name, kind, ch, before, after, imgs, items, offs):
    outside = np.ones(after.shape, bool)
    for i, (img, (_obj, want), off) in enumerate(zip(imgs, items, offs)):
        want = want.reshape(-1)
        got = after[off:off + want.size]
        outside[off:off + want.size] = False
        bad = np.flatnonzero(got != want)
        if bad.size:
            y, b = divmod(int(bad[0]), img.w * ch)
            raise AssertionError("%s: %s %d (%dx%d) has %d wrong bytes, the first at row %d, byte %d of %d (%s)"
                                 % (name, kind, i, img.h, img.w, bad.size, y, b, img.w * ch, _row(img, ch, off, y)))
    bad = np.flatnonzero(after[outside] != before[outside])
    assert bad.size == 0, "%s: %d %s-plane bytes outside the images changed" % (name, bad.size, kind)


def _letterboxed(eng, packed):
    got = eng.debug_read_slot(0, 2, 0, len(packed) * NET * NET * 3).reshape(len(packed), NET, NET, 3)
    want = np.stack([letterbox(p, (NET, NET))[0] for p in packed])
    for i in range(len(packed)):
        assert np.array_equal(got[i], want[i]), (i, packed[i].shape, int((got[i] != want[i]).sum()))


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_gather_bytes(det, case):
    eng = det.net
    entries, page_bytes, mask_bytes = plan(case)
    page_offs = [int(e["page_off"]) for e in entries]
    mask_offs = [int(e["mask_off"]) for e in entries]
    sent_p = [np.full((i.h, i.w, 3), SENTINEL, np.uint8) for i in case.pages]
    sent_m = [np.full((i.h, i.w), SENTINEL, np.uint8) for i in case.pages]
    _run(eng, case.job, sent_p, sent_m)
    before_p = eng.debug_read_slot(0, 0, 0, page_bytes)
    before_m = eng.debug_read_slot(0, 1, 0, mask_bytes)
    for p, off in zip(sent_p, page_offs):
        assert (before_p[off:off + p.size] == SENTINEL).all()
    pages = _images(case.pages, 3, 1)
    masks = _images(case.masks, 1, 2) if case.masks else None
    _run(eng, case.job, [p for p, _ in pages], masks and [m for m, _ in masks])
    _check_plane(case.name, "page", 3, before_p, eng.debug_read_slot(0, 0, 0, page_bytes), case.pages, pages,
                 page_offs)
    if masks:
        _check_plane(case.name, "mask", 1, before_m, eng.debug_read_slot(0, 1, 0, mask_bytes), case.masks, masks,
                     mask_offs)
    if case.job == "pages":
        _letterboxed(eng, [want for _, want in pages])


def test_letterbox_kernel_bytes(det):
    # net-sized (identity), exactly 2x (cv2's INTER_AREA branch of INTER_LINEAR), downscaled, upscaled, a 1-row and a
    # 1-column strip as long as the letterbox takes them; host pages and pages gathered from device views
    imgs = [window(NET, NET, 3, 3, NET * 3 + 5), host(2 * NET, 2 * NET),
            dev(361, 251, 3, meta(3, 361, 251).permute(1, 2, 0)), host(200, 150), window(1, 300, 3, 9, 907),
            dev(300, 1, 3, meta(300, 2, 3)[:, 1:])]
    pages = _images(imgs, 3, 3)
    eng = det.net
    eng.submit_pages(0, [p for p, _ in pages], NET, NET)
    eng.collect_pages(0, discard=True)
    _letterboxed(eng, [want for _, want in pages])
    assert np.array_equal(eng.debug_read_slot(0, 2, 0, NET * NET * 3).reshape(NET, NET, 3), pages[0][1])


def test_read_slot_refusals(det):
    eng = det.net
    page = np.zeros((40, 30, 3), np.uint8)
    eng.submit_pages(1, [page], NET, NET)
    with pytest.raises(ctd_b200.CtdError, match="uncollected"):
        eng.debug_read_slot(1, 0, 0, 16)
    eng.collect_pages(1, discard=True)
    assert eng.debug_read_slot(1, 0, 0, page.size).tolist() == [0] * page.size
    with pytest.raises(ctd_b200.CtdError, match="past its end"):
        eng.debug_read_slot(1, 2, NET * NET * 3 - 1, 2)
    with pytest.raises(ctd_b200.CtdError):
        eng.debug_read_slot(1, 3, 0, 1)
