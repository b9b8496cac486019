"""-m gpu: the network's two ends on the tensor cores (csrc/conv_ends.cu): the stem, which reads the u8 pages itself,
and the seg tail, one halo tile per 16x16 output tile.

* Each op re-runs alone on the engine's own buffers and is compared with a float64 emulation of its fp16 operands
  (the space-to-depth page and window weights; the 3x3 / 4-phase form of the seg tail) under the elementwise bound of
  tests/util.py; the u8 mask is the truncated f32 mask exactly and within one level of the float64 reference.
* Shapes: one 64x64 page (one 2x2 grid of tiles), the smallest grids of a batch, a non-square batch, and pages whose
  border pixels are 255 (a padding mistake at any edge shows there).  The engine takes page sides that are multiples of
  64 only, so every stem and seg-tail grid is a whole number of 16x16 tiles; other sides are rejected.
* The stem writes nothing but its own output: the destination buffer beyond the batch's pixels keeps a sentinel.
"""
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import synth
from util import get_checkpoint, blob_tensor
from test_gpu_conv_tc import _op_ratio

pytestmark = pytest.mark.gpu


def _pages(n, h, w, white_border):
    if h >= 128 and w >= 128:
        pages = np.stack([synth.structured_page(700 + i, h, w) for i in range(n)])
    else:   # too small for the synthetic page layout
        pages = np.random.default_rng(h * w + n).integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    if white_border:
        last = pages[-1]
        last[:3] = 255
        last[-3:] = 255
        last[:, :3] = 255
        last[:, -3:] = 255
    return pages


def _tensor(prog, buf, coff, c):
    return dict(buf=buf, coff=coff, c=c, down=prog.bufs[buf][1])


@pytest.mark.parametrize("n,h,w,white", [(1, 64, 64, True), (2, 128, 192, True), (3, 320, 576, True),
                                         (2, 256, 256, False)],
                         ids=["1x64x64", "2x128x192", "3x320x576", "2x256x256"])
def test_stem_and_seg_tail(n, h, w, white):
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    ops = prog.ops
    stem = 0
    seg = next(i for i, o in enumerate(ops) if o["kind"] == cc.OP_SEG_TAIL)
    assert ops[stem]["kind"] == cc.OP_STEM
    pages = _pages(n, h, w, white)
    eng = ctd_b200.Engine(prog, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
    try:
        eng.forward(pages)
        # stem, alone
        o = ops[stem]
        eng.debug_run_ops(stem, stem, n, h, w, pages=pages)
        got = eng.debug_read(_tensor(prog, o["dst_buf"], o["dst_coff"], o["cout"]))
        for img in range(n):
            r, _ = _op_ratio(prog, o, [], None, got, pages, img, False)
            assert r <= 1.0, "stem, image %d: err/bound %.3g" % (img, r)
        # seg tail, alone, on the input the forward left
        o = ops[seg]
        ins = [eng.debug_read(_tensor(prog, o["src_buf"][0], o["src_coff"][0], o["src_c"][0]))]
        eng.debug_run_ops(seg, seg, n, h, w)
        mask = eng.net_outputs(want_blks=False, want_lines=False)[1]
        mask_u8 = eng.mask_u8()
        for img in range(n):
            r, _ = _op_ratio(prog, o, ins, None, mask, pages, img, False)
            assert r <= 1.0, "seg tail, image %d: err/bound %.3g" % (img, r)
        np.testing.assert_array_equal(mask_u8, (mask[:, 0] * np.float32(255)).astype(np.uint8))
        # u8 within one level of the float64 sigmoid's truncation
        ref = _seg_ref(prog, o, ins[0])
        lvl = np.floor(ref * 255.0)
        assert np.abs(mask_u8.astype(np.float64) - lvl).max() <= 1.0
    finally:
        eng.close()


def _seg_ref(prog, op, x):
    """float64 mask of the seg tail's fp16 3x3 / 4-phase form over its fp16 input x [n][gh][gw][64]."""
    import torch
    c = op["src_c"][0]
    wc = blob_tensor(prog, op["w16_off"], 16 * 9 * c, np.float16).double().cpu()
    wt = wc.view(16, 3, 3, c)[:4].permute(0, 3, 1, 2)
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    y = torch.nn.functional.conv2d(xt, wt, None, 1, 1)
    n, _, gh, gw = y.shape
    ref = torch.zeros(n, 2 * gh, 2 * gw, dtype=torch.float64)
    for p in range(4):
        ref[:, p >> 1::2, p & 1::2] = torch.sigmoid(y[:, p])
    return ref.numpy()


def test_stem_leaves_the_rest_of_its_buffer():
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    o = prog.ops[0]
    buf = o["dst_buf"]
    ch, down = prog.bufs[buf][0], prog.bufs[buf][1]
    N, H, W = 2, 256, 256
    n, h, w = 1, 128, 192
    eng = ctd_b200.Engine(prog, max_batch=N, max_h=H, max_w=W, skip_postproc=True)
    try:
        t = _tensor(prog, buf, 0, ch)
        eng.debug_write(t, np.full((N, H // down, W // down, ch), 7.0, np.float32), N, H, W)
        eng.debug_run_ops(0, 0, n, h, w, pages=_pages(n, h, w, True))
        written = eng.debug_read(t).size
        # the seg tail, which writes only the masks, at the largest shape: debug_read then covers the whole allocation,
        # the stem's batch's pixels first
        seg = next(i for i, op in enumerate(prog.ops) if op["kind"] == cc.OP_SEG_TAIL)
        eng.debug_run_ops(seg, seg, N, H, W)
        flat = eng.debug_read(t).reshape(-1)
        assert np.all(flat[written:] == 7.0), "the stem wrote beyond its batch's pixels"
        out = flat[:written].reshape(n, h // down, w // down, ch)[..., o["dst_coff"]:o["dst_coff"] + o["cout"]]
        assert not np.any(out == 7.0)
    finally:
        eng.close()


def test_page_sides_must_be_multiples_of_64():
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    eng = ctd_b200.Engine(prog, max_batch=1, max_h=128, max_w=128, skip_postproc=True)
    try:
        with pytest.raises(ctd_b200.CtdError):
            eng.forward(_pages(1, 96, 128, False))
    finally:
        eng.close()
