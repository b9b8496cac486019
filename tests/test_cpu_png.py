"""not-gpu: the PNG encoder's integer rules.

The numpy restatement (oracle/png_ref.py) equals cv2.imencode('.png') byte for byte on the seeded corpus
(tests/png_corpus.py: window boundaries, runs of 258 k + {0..4}, token counts of 16383 k +- 1, blocks spanning the
window, stored / static / dynamic blocks, the golden scan and a mask of it); cv2 decodes every file back to its
input; and the closed-form tokens equal zlib 1.2.11's deflate_rle loop run as libpng drives it."""
import hashlib
import json
import os

import cv2
import numpy as np
import pytest

from oracle import png_ref
import png_corpus as pc

CASES = pc.corpus() + pc.golden_page()
IDS = [n for n, _ in CASES]
PINS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png_cv2_sha256.json")))


def _cv2(img):
    ref = cv2.imencode(".png", img)[1]
    got = hashlib.sha256(ref.tobytes()).hexdigest()
    return ref, got


@pytest.mark.parametrize("name,img", CASES, ids=IDS)
def test_oracle_equals_cv2(name, img):
    ref, sha = _cv2(img)
    assert sha == PINS["sha256"][name], (
        "cv2's PNG writer differs from the pinned target (libpng 1.6 + zlib 1.2.11 at OpenCV's defaults, cv2 %s): "
        "%s gives another file; this cv2 (%s) links another zlib or libpng" % (PINS["cv2"], name, cv2.__version__))
    got = png_ref.encode(img)
    assert got.dtype == np.uint8 and got.ndim == 1
    assert np.array_equal(got, ref), name


@pytest.mark.parametrize("name,img", CASES, ids=IDS)
def test_file_decodes_to_input(name, img):
    back = cv2.imdecode(png_ref.encode(img), cv2.IMREAD_UNCHANGED)
    assert back.shape == img.shape and np.array_equal(back, img), name


@pytest.mark.parametrize("name,img", CASES, ids=IDS)
def test_closed_form_equals_deflate_rle_loop(name, img):
    s = png_ref.filter_stream(img)
    wbits = png_ref.window_bits(s.size)[0]
    tok, blocks = png_ref.deflate_rle_literal(s, s.size // img.shape[0], wbits)
    assert np.array_equal(png_ref.tokens(s), tok), name
    # blocks of 16383 tokens, the rest (maybe none) in the final one
    T = tok.size
    assert [b[1] for b in blocks] == [png_ref.BLOCK_TOKENS] * (T // png_ref.BLOCK_TOKENS) + [T % png_ref.BLOCK_TOKENS]
    # the loop's exact `buf != NULL` and the closed form's rule make the same stream
    assert png_ref.deflate(s, tok, blocks)[0] == png_ref.deflate(s)[0], name
    for _b0, _n, _start, ln, ok, _last in blocks:
        if ok != png_ref.stored_ok(ln):
            assert ln > 32506


def test_corpus_reaches_every_rule():
    """the corpus holds what random images rarely give: an empty final block, a block whose start left the window,
    stored, static and dynamic blocks, every CINFO"""
    forms, empty_final, slid, cinfo = set(), False, False, set()
    for name, img in CASES:
        s = png_ref.filter_stream(img)
        tok, blocks = png_ref.deflate_rle_literal(s, s.size // img.shape[0], png_ref.window_bits(s.size)[0])
        forms |= set(png_ref.deflate(s)[1])
        empty_final |= blocks[-1][1] == 0
        slid |= any(not b[4] for b in blocks)
        cinfo.add(png_ref.window_bits(s.size)[1])
    assert forms == {0, 1, 2} and empty_final and slid and cinfo == set(range(8))


def test_refuses_other_images():
    for bad in (np.zeros((0, 4), np.uint8), np.zeros((4, 4, 4), np.uint8), np.zeros((4, 4), np.uint16),
                np.zeros((4, 4, 1), np.uint8)):
        with pytest.raises(ValueError):
            png_ref.encode(bad)
