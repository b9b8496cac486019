"""not-gpu: the JPEG encoder's rules.

The numpy restatement (oracle/jpeg_enc_ref.py) equals cv2.imencode('.jpg', img, params) byte for byte on the seeded
corpus (tests/jpeg_enc_corpus.py: edge sizes, every quality, sampling, optimise and restart setting, flat, gradient,
noise and text-like pages, the golden scan); the corpus reaches the rules it is there for; and the encoder's Python
front end refuses what it does not implement before any GPU work."""
import cv2
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import jpeg
from oracle import jpeg_enc_ref as R
import jpeg_enc_corpus as jc

CASES = jc.cases() + jc.golden_page()
IDS = [n for n, _i, _p in CASES]


@pytest.mark.parametrize("name,img,params", CASES, ids=IDS)
def test_oracle_equals_cv2(name, img, params):
    ref = cv2.imencode(".jpg", img, params)[1]
    got = R.encode(img, params)
    assert got.dtype == np.uint8 and got.ndim == 1
    assert np.array_equal(got, ref), name


def test_params_read_as_cv2_reads_them():
    """the binding's reading of a parameter list (clamps, fallbacks) equals the oracle's, which the corpus pins"""
    for _name, img, params in CASES:
        p = jpeg.jpeg_params(0, params)
        q, hv, opt, rst = R.parse_params(params)
        assert (p.quality, p.optimize, p.restart_interval) == (q, int(opt), rst)
        assert R.SAMPLING[p.sampling] == hv


def test_corpus_reaches_every_rule():
    """top DC / AC categories, FF bytes to stuff, more than eight restart intervals, right and bottom dummy blocks,
    optimised tables that differ from Annex K and code lengths cut to 16 bits never needed here but counted"""
    dc11 = ac10 = dummy_r = dummy_b = False
    ff = 0
    for name, img, params in CASES:
        if img.size > 200000:
            continue
        q, hv, _opt, _rst = R.parse_params(params)
        g, blocks, coef, _qt = R.coefficients(img, q, hv)
        ac10 |= bool((np.abs(coef[:, 1:]) >= 512).any())
        for c in range(g.nc):
            v = coef[blocks[:, 0] == c, 0]
            dc11 |= bool((np.abs(np.diff(v)) >= 1024).any())
        dummy = blocks[:, 3].astype(bool)
        dummy_r |= bool((dummy & (blocks[:, 2] < np.array(g.hib)[blocks[:, 0]])).any())
        dummy_b |= bool((dummy & (blocks[:, 2] >= np.array(g.hib)[blocks[:, 0]])).any())
        if name.startswith("noise_q100"):
            f = cv2.imencode(".jpg", img, params)[1]
            ff = max(ff, int(((f[:-1] == 0xFF) & (f[1:] == 0)).sum()))
    assert dc11 and ac10 and dummy_r and dummy_b and ff > 100


def test_optimal_table_limits_code_lengths():
    """counts in a Fibonacci progression make a Huffman tree deeper than 16 levels: jpeg_gen_optimal_table's
    adjustment brings it to 16 and every code stays a prefix code with no all-ones code"""
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    freq = np.zeros(256, np.int64)
    freq[:30] = fib
    bits, vals = R.gen_optimal_table(freq)
    assert sum(bits) == len(vals) == 30 and bits[15] > 0
    kraft = sum(b * 2.0 ** -(k + 1) for k, b in enumerate(bits))
    assert kraft < 1.0


def _encoder_without_device():
    enc = jpeg.JpegEncoder.__new__(jpeg.JpegEncoder)
    enc.lib = ctd_b200.load_library()
    enc.device_index = 0
    enc.h = None
    return enc


@pytest.mark.parametrize("key", [2, 5, 6, 8, 99])
def test_refuses_unsupported_keys(key):
    """PROGRESSIVE, LUMA_QUALITY, CHROMA_QUALITY and any other key: ValueError naming the image and the key"""
    enc = _encoder_without_device()
    ok = np.zeros((8, 8), np.uint8)
    with pytest.raises(ValueError, match="image 1.*(PROGRESSIVE|LUMA|CHROMA|key %d)" % key):
        enc.encode([ok, ok], [[jc.Q, 90], [key, 1]])


def test_refuses_bad_images_and_lists():
    enc = _encoder_without_device()
    ok = np.zeros((8, 8, 3), np.uint8)
    for bad in (np.zeros((0, 4), np.uint8), np.zeros((4, 4, 4), np.uint8), np.zeros((4, 4), np.uint16),
                np.zeros((4, 4, 1), np.uint8), np.zeros(4, np.uint8), [[1, 2], [3, 4]]):
        with pytest.raises(ValueError, match="image 1"):
            enc.encode([ok, bad])
    with pytest.raises(ValueError, match="image 0"):
        enc.encode([np.zeros((65501, 1), np.uint8)])
    with pytest.raises(ValueError, match="pairs"):
        enc.encode([ok], [jc.Q])
    with pytest.raises(ValueError, match="2 parameter lists for 1 images"):
        enc.encode([ok], [[jc.Q, 5], [jc.Q, 6]])
    import torch
    with pytest.raises(ValueError, match="image 0.*cuda:0"):
        enc.encode([torch.zeros((8, 8), dtype=torch.uint8)])


def test_null_encoder_is_refused_by_the_library():
    """valid input reaches ctd_jpeg_encode, which refuses a NULL encoder (CTD_E_INVALID) without touching a device"""
    enc = _encoder_without_device()
    with pytest.raises(ctd_b200.CtdError, match="ctd_jpeg_encode failed \\(-1\\)"):
        enc.encode([np.zeros((8, 8), np.uint8)])
