"""-m "not gpu": the oracle of `preprocess_img` (oracle/preprocess_ref.py) against the reference's own function, the
exact float32 division the pre-processing kernel restates, and what `preprocess_img` / `Preprocessor` refuse before
any GPU work."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding, preprocess
from oracle import preprocess_ref, ref_shim, synth

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="/root/reference not present on this box")


def _page(h, w, seed=0):
    return np.ascontiguousarray(synth.structured_page(seed, max(h, 128), max(w, 128))[:h, :w])


# (page size, input_size): net-sized, exact 2x decimation (INTER_AREA), upscaling, 1xN and Nx1, half-to-even unpad
# sizes, non-square input sizes
CASES = [
    ((256, 256), (256, 256)),
    ((512, 512), (256, 256)),
    ((100, 70), (256, 256)),
    ((1, 300), (256, 256)),
    ((300, 1), (256, 256)),
    ((640, 2), (256, 256)),      # 2 * 0.4 = 0.8 -> 1
    ((320, 5), (128, 128)),      # 5 * 0.4 = 2.0; 320 -> 128
    ((200, 5), (64, 64)),        # 5 * 0.32 = 1.6 -> 2
    ((256, 10), (64, 64)),       # 10 * 0.25 = 2.5 -> 2 (half to even)
    ((256, 14), (64, 64)),       # 14 * 0.25 = 3.5 -> 4 (half to even)
    ((361, 251), (256, 384)),
    ((200, 900), (384, 256)),
]


def test_half_to_even_cases_are_hit():
    """the cases include unpad sizes that Python's round takes to even, down and up"""
    exact = [w * min(s[0] / h, s[1] / w) for (h, w), s in CASES]
    assert 2.5 in exact and 3.5 in exact


@needs_ref
@pytest.mark.parametrize("shape, size", CASES)
@pytest.mark.parametrize("bgr2rgb, half, to_tensor", [(True, False, True), (False, False, True), (True, True, True),
                                                      (False, True, True), (True, False, False),
                                                      (False, False, False)])
def test_oracle_matches_reference(shape, size, bgr2rgb, half, to_tensor):
    ref = ref_shim.load().inference.preprocess_img
    page = _page(*shape, seed=shape[0] * 7 + shape[1])
    got = preprocess_ref.preprocess_img(page.copy(), size, 'cpu', bgr2rgb, half, to_tensor)
    want = ref(page.copy(), size, 'cpu', bgr2rgb, half, to_tensor)
    assert type(got[0]) is type(want[0])
    if to_tensor:
        assert got[0].dtype == want[0].dtype and tuple(got[0].shape) == tuple(want[0].shape)
        view = torch.int16 if half else torch.int32
        assert torch.equal(got[0].view(view), want[0].view(view))
    else:
        assert got[0].dtype == want[0].dtype and got[0].shape == want[0].shape
        assert np.array_equal(got[0], want[0])
    assert got[1] == want[1] and type(got[1][0]) is type(want[1][0]) is float
    assert got[2:] == want[2:] and all(type(v) is int for v in got[2:])


def test_oracle_divides_by_255():
    """`astype(float32) / 255` is a correctly rounded float32 division: it differs from the product by float32(1/255)
    on 126 of the 256 u8 values, so the product is not a restatement"""
    v = np.arange(256, dtype=np.float32)
    div = v / np.float32(255)
    mul = v * (np.float32(1) / np.float32(255))
    assert int((div.view(np.int32) != mul.view(np.int32)).sum()) == 126
    page = np.repeat(np.arange(256, dtype=np.uint8), 3).reshape(4, 64, 3)
    x = preprocess_ref.preprocess_img(page, (64, 64), bgr2rgb=False)[0]
    assert torch.equal(x[0, 2, :4].reshape(-1).view(torch.int32), torch.from_numpy(div).view(torch.int32))


def _rn32(x):
    """x (a Fraction) rounded to the nearest float32, ties to even, as a Fraction"""
    if x == 0:
        return Fraction(0)
    s, x = (-1 if x < 0 else 1), abs(x)
    e = math.floor(math.log2(x)) - 23
    while x / Fraction(2) ** e >= 2 ** 24:
        e += 1
    while x / Fraction(2) ** e < 2 ** 23:
        e -= 1
    m = x / Fraction(2) ** e
    q = math.floor(m)
    if m - q > Fraction(1, 2) or (m - q == Fraction(1, 2) and q % 2):
        q += 1
    return s * q * Fraction(2) ** e


def test_kernel_division_is_exact():
    """letterbox_tensor_kernel computes v / 255 as q0 = RN(v * r), r = RN(1 / 255), then RN(RN(v - 255 q0) * r + q0)
    with two fmas (csrc/resize.cu, unit_f32): in exact arithmetic that equals the correctly rounded division, which
    numpy computes, for every u8 value"""
    r = _rn32(Fraction(1, 255))
    assert float(r) == float(np.float32(1) / np.float32(255)) == float.fromhex("0x1.010102p-8")
    for v in range(256):
        q0 = _rn32(v * r)
        q = _rn32(_rn32(v - 255 * q0) * r + q0)
        assert q == _rn32(Fraction(v, 255)) == Fraction(float(np.float32(v) / np.float32(255))), v


def test_exported():
    assert "ctd_preprocess_pages" in binding.EXPORTS
    assert ctd_b200.preprocess_img is preprocess.preprocess_img
    assert ctd_b200.Preprocessor is preprocess.Preprocessor and ctd_b200.NetworkDetector is preprocess.NetworkDetector


@pytest.mark.parametrize("size", [0, 63, 100, (64, 96), (64,), (64, 64, 64), -64, (64.0, 64)])
def test_bad_input_sizes(size):
    with pytest.raises(ValueError, match="multiples of 64"):
        preprocess.net_size(size)
    with pytest.raises(ValueError, match="multiples of 64"):
        ctd_b200.preprocess_img(np.zeros((8, 8, 3), np.uint8), size)


def test_input_sizes():
    assert preprocess.net_size(1024) == (1024, 1024)
    assert preprocess.net_size((640, 1024)) == (640, 1024)
    assert preprocess.net_size([64, 128]) == (64, 128)


@pytest.mark.parametrize("device", ["cpu", torch.device("cpu"), "meta"])
def test_non_cuda_device_refused(device):
    with pytest.raises(ValueError, match="no CPU fallback"):
        ctd_b200.preprocess_img(np.zeros((8, 8, 3), np.uint8), (64, 64), device)


@pytest.mark.parametrize("page", [np.zeros((8, 8), np.uint8), np.zeros((8, 8, 4), np.uint8),
                                  np.zeros((8, 8, 3), np.float32), np.zeros((0, 8, 3), np.uint8),
                                  torch.zeros((8, 8, 3), dtype=torch.int16)])
def test_bad_pages_refused_before_gpu(page):
    """pages_on_device checks every page before it asks for the engine's decoders or uploads anything"""
    pre = preprocess.Preprocessor.__new__(preprocess.Preprocessor)
    pre.input_size, pre.device_index, pre.max_batch = (64, 64), 0, 4
    with pytest.raises(ValueError, match="item 1: "):
        pre.pages_on_device([(0, np.zeros((8, 8, 3), np.uint8)), (1, page)])


def test_page_that_does_not_letterbox_refused():
    """a 1 x 200 page letterboxes to 0 px high in a 64 x 64 input: refused by ctd_pages_plan's arithmetic"""
    pre = preprocess.Preprocessor.__new__(preprocess.Preprocessor)
    pre.input_size, pre.device_index, pre.max_batch = (64, 64), 0, 4
    with pytest.raises(ValueError, match="item 0: a 1x200 page does not letterbox"):
        pre.pages_on_device([(0, np.zeros((1, 200, 3), np.uint8))])
