"""-m "not gpu": what `PostProcessor` checks on the host before any GPU work, the ctypes mirror of `ctd_net_output`
against the header, and the numpy cast of `postprocess_mask` the ingest kernel restates."""
import ctypes as C
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding, postprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NET = (256, 192)
A = postprocess.workspace_rows(*NET)


def test_net_output_mirror_matches_header(tmp_path):
    """sizeof and every field offset of ctd_net_output, as a C compiler lays it out from include/ctd_b200.h"""
    fields = [f for f, _t in binding.CtdNetOutput._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ctd_b200.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(ctd_net_output));\n' +
                   "".join('  printf("%%zu\\n", offsetof(ctd_net_output, %s));\n' % f for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(binding.CtdNetOutput) == 96
    assert got[1:] == [getattr(binding.CtdNetOutput, f).offset for f in fields]


def test_submit_outputs_exported():
    assert "ctd_submit_outputs" in binding.EXPORTS
    assert hasattr(C.CDLL(ctd_b200.LIB_PATH), "ctd_submit_outputs")


def _outs(a=A, c=2, h=NET[0], w=NET[1], dtype=np.float32):
    return (np.zeros((1, a, 7), dtype), np.zeros((1, 1, h, w), dtype), np.zeros((1, c, h, w), dtype))


@pytest.mark.parametrize("form", ["batched", "flat"])
def test_accepted_forms_are_views(form):
    blks, mask, lines = _outs()
    if form == "flat":
        blks, mask, lines = blks[0], mask[0, 0], lines[0]
    b, m, ln = postprocess.check_outputs(blks, mask, lines, NET)
    assert b.shape == (A, 7) and m.shape == NET and ln.shape == NET
    assert np.shares_memory(b, blks) and np.shares_memory(m, mask) and np.shares_memory(ln, lines)
    # only channel 0 of lines_map is read
    assert ln.__array_interface__["data"][0] == lines.__array_interface__["data"][0]
    # [1][H][W] masks, lines_map[:, :1], no rows at all
    postprocess.check_outputs(blks[:0] if form == "flat" else blks[:, :0], np.zeros((1,) + NET, np.float32),
                              np.zeros((1, 1) + NET, np.float32), NET)


@pytest.mark.parametrize("case, arg", [
    (lambda o: (o[0][..., :6], o[1], o[2]), "blks"),                                 # 5 + nc columns
    (lambda o: (np.zeros((1, A + 1, 7), np.float32), o[1], o[2]), "blks"),           # A past the workspace
    (lambda o: (np.zeros((2, 10, 7), np.float32), o[1], o[2]), "blks"),              # a batch of two
    (lambda o: (o[0].astype(np.float16), o[1], o[2]), "blks"),                       # fp16
    (lambda o: (o[0], o[1].astype(np.float64), o[2]), "mask"),                       # another dtype
    (lambda o: (o[0], o[1][..., :-64], o[2]), "mask"),                               # not input_size
    (lambda o: (o[0], np.zeros((2,) + NET, np.float32), o[2]), "mask"),              # two channels
    (lambda o: (o[0], np.zeros((1, 1, 1) + NET, np.float32), o[2]), "mask"),         # 5-D
    (lambda o: (o[0], o[1], o[2][:, :0]), "lines_map"),                              # C = 0
    (lambda o: (o[0], o[1], o[2][0, 0]), "lines_map"),                               # [H][W]
    (lambda o: (o[0], o[1], np.zeros((1, 2, NET[1], NET[0]), np.float32)), "lines_map"),   # transposed size
    (lambda o: (o[0], o[1], torch.zeros((1, 2) + NET, dtype=torch.bfloat16)), "lines_map"),
])
def test_refusals_name_item_and_argument(case, arg):
    with pytest.raises(ValueError) as e:
        postprocess.check_outputs(*case(_outs()), NET, what="item 3: ")
    msg = str(e.value)
    assert msg.startswith("item 3: ") and arg in msg, msg


def test_nc_sets_the_columns():
    postprocess.check_outputs(np.zeros((5, 9), np.float32), *_outs()[1:], NET, nc=4)
    with pytest.raises(ValueError):
        postprocess.check_outputs(np.zeros((5, 7), np.float32), *_outs()[1:], NET, nc=4)


def test_page_plan_refusal():
    postprocess.check_plan((1, 300), NET)
    with pytest.raises(ValueError, match="item 0: a 1x100000 page does not letterbox"):
        postprocess.check_plan((1, 100000), NET, "item 0: ")


def test_input_size_refused_before_any_engine():
    with pytest.raises(ValueError, match="multiples of 64"):
        ctd_b200.PostProcessor(input_size=1000)


# postprocess_mask's cast: (p * 255).astype(np.uint8) on float32 p, restated as the ingest kernel computes it
def mask_cast(p):
    v = np.asarray(p, np.float32) * np.float32(255)
    ok = (v >= np.float32(-2 ** 31)) & (v < np.float32(2 ** 31))
    t = np.trunc(np.where(ok, v, 0)).astype(np.int64)
    return np.where(ok, t & 255, 0).astype(np.uint8)


def numpy_cast(p):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return (np.asarray(p, np.float32) * 255).astype(np.uint8)


TABLE = [(1.0, 255), (0.999, 254), (1.2, 50), (300 / 255, 44), (-0.5, 129), (-1 / 255, 255), (3e9 / 255, 0),
         (-3e9 / 255, 0), (1e30, 0), (-1e30, 0)]


def test_cast_table():
    p = np.array([t[0] for t in TABLE], np.float32)
    want = np.array([t[1] for t in TABLE], np.uint8)
    assert mask_cast(p).tolist() == want.tolist()
    assert numpy_cast(p).tolist() == want.tolist()


def test_cast_against_numpy_on_boundaries():
    k = np.arange(-2048, 2048, dtype=np.float32)
    p = np.concatenate([k / np.float32(255), np.nextafter(k / np.float32(255), np.float32(np.inf)),
                        np.nextafter(k / np.float32(255), np.float32(-np.inf)),
                        np.array([2 ** 31 / 255, -2 ** 31 / 255, 2 ** 24, -2 ** 24, 8.4e6, -8.4e6], np.float32),
                        np.random.default_rng(0).uniform(-3, 3, 100000).astype(np.float32)])
    assert np.array_equal(mask_cast(p), numpy_cast(p))
