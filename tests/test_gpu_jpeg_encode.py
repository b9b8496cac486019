"""gpu: JPEG files encoded on the GPU (`ctd_b200.JpegEncoder`, csrc/jpeg_enc.cu) equal cv2.imencode('.jpg', img,
params) byte for byte: the whole corpus of tests/jpeg_enc_corpus.py in one call and one image at a time, numpy and
strided CUDA inputs mixed, 64 images in a call, calls that grow and shrink the buffers, a tensor written on a side
stream just before the call, and a 4096x4096 page."""
import cv2
import numpy as np
import pytest
import torch

import ctd_b200
import jpeg_enc_corpus as jc

pytestmark = pytest.mark.gpu


def _cv2(img, params=()):
    return cv2.imencode(".jpg", img, list(params))[1]


@pytest.fixture(scope="module")
def enc():
    e = ctd_b200.JpegEncoder(0)
    yield e
    e.close()


def test_corpus_in_one_call(enc):
    cases = jc.cases() + jc.golden_page()
    got = enc.encode([img for _n, img, _p in cases], [p for _n, _i, p in cases])
    for (name, img, params), g in zip(cases, got):
        assert np.array_equal(g, _cv2(img, params)), name


def test_corpus_one_by_one_from_cuda(enc):
    for name, img, params in jc.cases(large=False):
        t = torch.from_numpy(img).cuda()
        assert np.array_equal(enc.encode([t], params)[0], _cv2(img, params)), name


def test_mixed_strided_inputs(enc):
    rng = np.random.default_rng(7)
    page = jc.page("text", 301, 517, 3, rng)
    grey = jc.page("gradient", 77, 45, 1, rng)
    dev = torch.from_numpy(page).cuda()
    crop = dev[13:250, 31:480]                                   # row stride of the full page
    chw = torch.from_numpy(np.ascontiguousarray(page.transpose(2, 0, 1))).cuda()
    perm = chw.permute(1, 2, 0)                                  # channel stride h * w
    gcol = torch.from_numpy(np.ascontiguousarray(grey.T)).cuda().t()   # a transposed grey image
    imgs = [page, crop, grey, perm, gcol, page[::2, ::3]]
    refs = [page, page[13:250, 31:480], grey, page, grey, np.ascontiguousarray(page[::2, ::3])]
    params = [[], [jc.Q, 80, jc.SF, jc.SAMPLINGS["422"]], [jc.OPT, 1], [jc.RST, 5, jc.SF, jc.SAMPLINGS["411"]],
              [jc.Q, 30], [jc.SF, jc.SAMPLINGS["440"], jc.OPT, 1]]
    got = enc.encode(imgs, params)
    for k, (g, r, p) in enumerate(zip(got, refs, params)):
        assert np.array_equal(g, _cv2(r, p)), k


def test_64_images_in_one_call(enc):
    rng = np.random.default_rng(64)
    kinds = ("flat", "gradient", "noise", "text")
    imgs, params = [], []
    for k in range(64):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        imgs.append(jc.page(kinds[k % 4], h, w, 1 + 2 * (k % 2), rng))
        params.append([jc.Q, int(rng.integers(0, 101)), jc.SF, list(jc.SAMPLINGS.values())[k % 5], jc.OPT, int(k % 3 == 0),
                       jc.RST, int(rng.choice([0, 1, 2, 7]))])
    got = enc.encode(imgs, params)
    for k, (g, img, p) in enumerate(zip(got, imgs, params)):
        assert np.array_equal(g, _cv2(img, p)), k


def test_calls_grow_then_shrink(enc):
    rng = np.random.default_rng(3)
    for h, w, n in ((8, 8, 1), (640, 480, 4), (1500, 1100, 3), (30, 20, 2), (700, 900, 1), (1, 1, 1)):
        imgs = [jc.page("text", h, w, 3, rng) for _ in range(n)]
        for g, img in zip(enc.encode(imgs, [jc.OPT, 1]), imgs):
            assert np.array_equal(g, _cv2(img, [jc.OPT, 1])), (h, w)


def test_tensor_written_on_a_side_stream(enc):
    """the encode reads a tensor after the work queued on the current stream: a page filled there just before the
    call is encoded as filled"""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.empty((1024, 1536, 3), dtype=torch.uint8, device="cuda")
        for _ in range(4):
            t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda"))
        t[100:900, 200:1300] = 255
        got = enc.encode([t], [jc.Q, 90])[0]
    side.synchronize()
    assert np.array_equal(got, _cv2(t.cpu().numpy(), [jc.Q, 90]))


def test_4096_page(enc):
    rng = np.random.default_rng(4096)
    page = jc.page("text", 4096, 4096, 3, rng)
    for p in ([], [jc.SF, jc.SAMPLINGS["444"], jc.OPT, 1, jc.RST, 64]):
        assert np.array_equal(enc.encode([torch.from_numpy(page).cuda()], p)[0], _cv2(page, p))


def test_refusals_on_device(enc):
    ok = torch.zeros((8, 8), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="image 1.*PROGRESSIVE"):
        enc.encode([ok, ok], [[], [2, 1]])
    with pytest.raises(ValueError, match="image 0.*uint8"):
        enc.encode([torch.zeros((8, 8), dtype=torch.float32, device="cuda")])
    with pytest.raises(ValueError, match="image 0.*empty"):
        enc.encode([torch.zeros((0, 8, 3), dtype=torch.uint8, device="cuda")])
    # the encoder still works after the refusals
    img = np.full((9, 9, 3), 77, np.uint8)
    assert np.array_equal(enc.encode([img])[0], _cv2(img))


def test_side_limit_refused_before_any_event(enc, monkeypatch):
    """a side above 65500 on a CUDA tensor is refused with the shape checks, before an event is recorded"""
    recorded = []
    monkeypatch.setattr(torch.cuda.Event, "record", lambda self, *a, **k: recorded.append(1))
    ok = torch.zeros((8, 8), dtype=torch.uint8, device="cuda")
    tall = torch.zeros((65501, 1), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="image 1.*65500"):
        enc.encode([ok, tall])
    assert recorded == []
