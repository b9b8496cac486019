"""-m gpu: float16 network outputs through the post-processing, `NetworkDetector(half=True)` and
`TextDetBase(half=True)`.

  * torch on CUDA computes the half rules the oracle takes from torch CPU and numpy, for every float16 value;
  * the ingest's mask byte equals numpy's float16 cast of the half product for every finite float16 value;
  * PostProcessor(half=True) equals the half oracle byte for byte on the golden, in every input form, with float32
    pages of the same batch unchanged;
  * TextDetBase(half=True) is `.half()` of its float32 outputs, and the reference's chain with it equals
    NetworkDetector(half=True)."""
import os

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200.binding import PREC_FP16_TC
from oracle import postproc_half_ref, synth, textblock_ref
import region_ref
from pages_ref import postprocess_page_any_size
from util import get_checkpoint

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NET = 256
ALL = np.arange(65536, dtype=np.uint16).view(np.float16)
FINITE = ALL[np.isfinite(ALL)]


def _key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


def _same(got, ref):
    assert np.array_equal(got[0], ref[0]), int((got[0] != ref[0]).sum())
    assert [_key(b) for b in got[2]] == [_key(b) for b in ref[2]]
    assert np.array_equal(got[1], ref[1]), int((got[1] != ref[1]).sum())


def test_torch_cuda_half_rules_every_value():
    t = torch.from_numpy(ALL.copy()).cuda()
    tf = torch.from_numpy(FINITE.copy()).cuda()   # NaN payloads are not kept alike by CUDA and numpy
    with np.errstate(all="ignore"):
        for th in (0.3, 0.4):
            assert np.array_equal((t > th).cpu().numpy(), ALL > np.float16(th))
        assert np.array_equal((tf * 255).cpu().numpy().view(np.uint16), (FINITE * np.float16(255)).view(np.uint16))
        rng = np.random.default_rng(1)
        f = torch.from_numpy(FINITE.copy())
        for other in rng.choice(FINITE, 24):
            o = torch.tensor(float(other), dtype=torch.float16)
            # x[:, 5:] *= x[:, 4:5] and xywh2xyxy's halving, sum and difference, CUDA against CPU
            for op in (lambda a, b: a * b, lambda a, b: a - b / 2, lambda a, b: a + b / 2):
                assert np.array_equal(op(f.cuda(), o.cuda()).cpu().numpy().view(np.uint16),
                                      op(f, o).numpy().view(np.uint16))


@pytest.fixture(scope="module")
def post():
    p = ctd_b200.PostProcessor(input_size=NET, max_batch=4, half=True)
    yield p
    p.close()


def test_mask_byte_every_finite_half(post):
    vals = np.zeros(NET * NET, np.float16)
    vals[:FINITE.size] = FINITE
    mask = vals.reshape(1, NET, NET)
    a = ctd_b200.postprocess.workspace_rows(NET, NET)
    blks = np.zeros((a, 7), np.float16)
    lines = np.zeros((2, NET, NET), np.float16)
    page = synth.structured_page(3, NET, NET)
    got16, got32 = post.postprocess_batch([(page, blks, mask, lines),
                                           (page, blks.astype(np.float32), mask.astype(np.float32),
                                            lines.astype(np.float32))])
    with np.errstate(all="ignore"):
        assert np.array_equal(got16[0], (mask[0] * 255).astype(np.uint8))
        assert np.array_equal(got32[0], (mask[0].astype(np.float32) * 255).astype(np.uint8))


def _golden_page():
    z = np.load(os.path.join(ROOT, "tests", "golden", "half_ref_256.npz"))
    return synth.structured_page(5, NET, NET), z["blks"], z["mask"], z["lines"]


@pytest.mark.parametrize("form", ["numpy", "cuda", "strided", "scalar", "mixed"])
def test_golden_against_half_oracle(post, form):
    page, blks, mask, lines = _golden_page()
    ref = postproc_half_ref.postprocess_page_half(page.copy(), blks, mask[0], lines, textblock_ref.group_output,
                                                  refine_mode=1, keep_undetected_mask=True)
    if form == "numpy":
        items = [(page, blks, mask, lines)]
    elif form == "cuda":
        items = [(page, torch.from_numpy(blks).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(lines).cuda())]
    else:
        # slices of batched outputs: page 1 of [3][...] tensors, mask and lines as channel views of one tensor
        bb = torch.zeros((3,) + blks.shape, dtype=torch.float16, device="cuda")
        bb[1] = torch.from_numpy(blks)
        ml = torch.zeros((3, 4, NET, NET), dtype=torch.float16, device="cuda")
        ml[1, 1] = torch.from_numpy(mask[0])
        ml[1, 2] = torch.from_numpy(lines[0])
        items = [(page, bb[1], ml[1, 1:2], ml[1, 2:4])]
        if form == "scalar":
            # maps the ingest reads one strided element at a time: the mask as a channel of a channels_last tensor
            # (width stride 4), column-major lines planes and blks rows, and a view one element off 8-byte alignment
            cl = ml.contiguous(memory_format=torch.channels_last)
            lt = torch.from_numpy(lines).cuda().transpose(1, 2).contiguous().transpose(1, 2)
            bt = torch.from_numpy(blks).cuda().t().contiguous().t()
            flat = torch.zeros(1 + mask.size, dtype=torch.float16, device="cuda")
            off = flat[1:].view(NET, NET)
            off.copy_(torch.from_numpy(mask[0]))
            assert cl[1, 1].stride(-1) == 4 and lt.stride(-1) == NET and bt.stride(-1) == blks.shape[0]
            items = [(page, bt, cl[1, 1:2], lt), (page, blks, off, lines)]
    if form == "mixed":
        f32 = (blks.astype(np.float32), mask.astype(np.float32), lines.astype(np.float32))
        ref32 = postprocess_page_any_size(page.copy(), (NET, NET), (NET, NET), f32[0], f32[1][0], f32[2],
                                          textblock_ref.group_output, 0.4, 0.35, 1, True)
        items = [(page,) + f32, items[0], (page, torch.from_numpy(f32[0]).cuda()) + f32[1:]]
        got = post.postprocess_batch(items, 1, True)
        _same(got[0], ref32)
        _same(got[1], ref)
        _same(got[2], ref32)
        assert [_key(b) for b in got[0][2]] != [_key(b) for b in got[1][2]] or not np.array_equal(got[0][0], got[1][0])
        return
    got = post.postprocess_batch(items, 1, True)
    for g in got:
        _same(g, ref)
    assert len(ref[2]) > 0


def test_golden_crops_against_oracle(post):
    page, blks, mask, lines = _golden_page()
    ref = postproc_half_ref.postprocess_page_half(page.copy(), blks, mask[0], lines, textblock_ref.group_output)
    th, n = 32, 0
    for items in ([(page, blks, mask, lines)], [(page, torch.from_numpy(blks).cuda(), torch.from_numpy(mask).cuda(),
                                                 torch.from_numpy(lines).cuda())]):
        got = post.postprocess_batch(items, textheight=th)[0]
        _same(got[:3], ref)
        assert len(got[3]) == len(ref[2]) > 0
        for b, blk in enumerate(ref[2]):
            assert len(got[3][b]) == len(blk.lines)
            for i, c in enumerate(got[3][b]):
                try:
                    r = region_ref.transformed_region(blk, page, i, th)
                except Exception:
                    assert c is None, (b, i)
                    continue
                assert c is not None and np.array_equal(c, r), (b, i)
                n += 1
    assert n > 0


def test_overflow_ties_at_the_cap():
    """a 512 x 512 float16 page with 5100 candidates, more than the 4096 NMS slots: 100 with distinct high scores and
    5000 tied at 0.75 in half (their float products differ), so the cut at the cap falls inside the tie and the
    detections past the first 100 come from it in row order"""
    net = 512
    rng = np.random.default_rng(9)
    a = ctd_b200.postprocess.workspace_rows(net, net)
    b = np.zeros((a, 7), np.float16)
    b[:, 0:2] = rng.uniform(8, net - 8, (a, 2))
    b[:, 2:4] = rng.uniform(2, 12, (a, 2))
    b[:, 4] = rng.uniform(0, 0.35, a)
    b[:, 5:7] = rng.uniform(0, 1, (a, 2))
    idx = rng.choice(a, 5100, replace=False)
    b[idx[:100], 4] = rng.uniform(0.9, 1, 100)
    b[idx[:100], 5] = 1
    # (0.75, 1) or (0.75 + 2^-11, 1 - 2^-11): products 0.75 and 0.75 + 2^-13 - 2^-22, both 0.75 in half
    pick = rng.integers(0, 2, 5000).astype(np.float16) * np.float16(2 ** -11)
    b[idx[100:], 4] = np.float16(0.75) + pick
    b[idx[100:], 5] = np.float16(1) - pick
    # the float products differ, the half ones tie
    assert len(np.unique(b[idx[100:], 4].astype(np.float32) * b[idx[100:], 5].astype(np.float32))) == 2
    assert len(np.unique(b[idx[100:], 4] * b[idx[100:], 5])) == 1
    page = synth.structured_page(60, net, net)
    mask = cv2_blobs(net)
    lines = np.stack([mask[0], np.zeros_like(mask[0])])
    ref = postproc_half_ref.postprocess_page_half(page.copy(), b, mask[0], lines, textblock_ref.group_output)
    post = ctd_b200.PostProcessor(input_size=net, max_batch=2, half=True)
    try:
        got = post.postprocess_batch([(page, b, mask, lines), (page, torch.from_numpy(b).cuda(),
                                                               torch.from_numpy(mask).cuda(),
                                                               torch.from_numpy(lines).cuda())])
    finally:
        post.close()
    for g in got:
        _same(g, ref)
    assert len(ref[2]) > 0


def cv2_blobs(net):
    """a float16 [1][net][net] probability map of a few text-line bars"""
    m = np.zeros((net, net), np.float16)
    for k in range(10):
        y = 20 + 45 * k
        m[y:y + 8, 30:30 + 200 + 20 * k] = np.float16(0.9)
    return m[None]


def test_check_outputs_cuda_half_views():
    a = ctd_b200.postprocess.workspace_rows(NET, NET)
    blks = torch.zeros((2, a, 7), dtype=torch.float16, device="cuda")
    ml = torch.zeros((2, 3, NET, NET), dtype=torch.float16, device="cuda")
    b, m, ln = ctd_b200.postprocess.check_outputs(blks[1], ml[1, :1], ml[1, 1:], (NET, NET), device_index=0, half=True)
    assert b.data_ptr() == blks[1].data_ptr() and m.data_ptr() == ml[1, 0].data_ptr()
    assert ln.data_ptr() == ml[1, 1].data_ptr() and b.dtype == m.dtype == ln.dtype == torch.float16
    with pytest.raises(ValueError, match="item 2: mask is torch.float32 but blks is torch.float16"):
        ctd_b200.postprocess.check_outputs(blks[1], ml[1, :1].float(), ml[1, 1:], (NET, NET), what="item 2: ",
                                           half=True)
    with pytest.raises(ValueError, match="lines_map must be float32 or float16, got torch.bfloat16"):
        ctd_b200.postprocess.check_outputs(blks[1], ml[1, :1], ml[1, 1:].bfloat16(), (NET, NET), half=True)


@pytest.mark.parametrize("where", [0, 1, 2])
@pytest.mark.parametrize("value", [np.inf, np.nan])
def test_nonfinite_half_fails_its_item(post, where, value):
    page, blks, mask, lines = _golden_page()
    outs = [blks.copy(), mask.copy(), lines.copy()]
    outs[where].reshape(-1)[123] = value
    with pytest.raises(ValueError, match="item 1: a non-finite value"):
        post.postprocess_batch([(page, blks, mask, lines), (page,) + tuple(outs)])
    post.postprocess_batch([(page, blks, mask, lines)])   # still usable


# ---- TextDetBase(half=True) and NetworkDetector(half=True) --------------------------------------------------------
@pytest.fixture(scope="module")
def base16():
    b = ctd_b200.TextDetBase(get_checkpoint(0, True), max_batch=4, max_size=NET, half=True)
    yield b
    b.close()


def test_textdetbase_half_is_half_of_float(base16):
    g = torch.Generator().manual_seed(7)
    x16 = torch.rand((2, 3, NET, NET), generator=g).half().cuda()
    got = base16(x16)
    ref = base16(x16.float())
    assert all(t.dtype == torch.float16 for t in got) and all(t.dtype == torch.float32 for t in ref)
    for a, b in zip(got, ref):
        assert torch.equal(a.view(torch.int16), b.half().view(torch.int16))
    # x16 = (u8 / 255).half() gives .half() of the u8 path's outputs: the fp16 engine stages u8 / 255 rounded to fp16
    # either way, and for x = u8 / 255 in float32 the outputs are those of Engine.forward on the u8 pages
    pages = np.stack([synth.structured_page(30 + i, NET, NET) for i in range(2)])
    u8 = (torch.from_numpy(pages).cuda().permute(0, 3, 1, 2).float() / 255).contiguous()
    eng = ctd_b200.Engine(ctd_b200.compiler.compile_checkpoint(get_checkpoint(0, True)), precision=PREC_FP16_TC,
                          max_batch=2, max_h=NET, max_w=NET)
    try:
        eng.forward(pages)
        u8_path = eng.net_outputs()
    finally:
        eng.close()
    for a, b, c in zip(base16(u8.half()), base16(u8), u8_path):
        assert torch.equal(a.view(torch.int16), b.half().view(torch.int16))
        assert torch.equal(b.cpu(), torch.from_numpy(c).reshape(b.shape))


def test_network_detector_half_equals_reference_chain(base16):
    pages = [synth.structured_page(40 + i, NET, NET) for i in range(3)]
    det = ctd_b200.NetworkDetector(base16, input_size=NET, max_batch=2, half=True)
    try:
        got = det.detect_batch(pages)
    finally:
        det.close()
    n_blocks = 0
    for page, g in zip(pages, got):
        img_in = ctd_b200.preprocess_img(page, input_size=(NET, NET), half=True)[0]
        assert img_in.dtype == torch.float16
        blks, mask, lines = (t.cpu().numpy() for t in base16(img_in))
        ref = postproc_half_ref.postprocess_page_half(page.copy(), blks[0], mask[0, 0], lines[0],
                                                      textblock_ref.group_output)
        _same(g, ref)
        n_blocks += len(ref[2])
    assert n_blocks > 0
