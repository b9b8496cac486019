"""-m "not gpu": post-processing of float16 network outputs on the host side.

  * the half oracle (oracle/postproc_half_ref.py) equals the unmodified reference on tests/golden/half_ref_256.npz
    (the reference itself where its tree is present), and that golden exercises every half rule: `.float()` and
    today's float32 oracle give another bitmap, mask, scores and boxes;
  * check_outputs(half=True) takes float16 maps as views, refuses mixed pages and bfloat16; half=False keeps refusing;
  * the new entry points and the ctd_dtype values against include/ctd_b200.h."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import binding, postprocess
from oracle import postproc_half_ref, postproc_ref, ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "half_ref_256.npz")
NET = (256, 256)


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _oracle(z):
    det = postproc_half_ref.non_max_suppression_half(z["blks"][None])[0].numpy()
    mask = postproc_half_ref.mask_u8_half(z["mask"][0])
    boxes, scores = postproc_half_ref.seg_represent_half(z["lines"][0])
    return det, mask, boxes, scores


def test_golden_inputs_are_the_recipe(gold):
    blks, mask, lines = postproc_half_ref.golden_inputs()
    assert np.array_equal(gold["blks"].view(np.uint16), blks.view(np.uint16))
    assert np.array_equal(gold["mask"].view(np.uint16), mask.view(np.uint16))
    assert np.array_equal(gold["lines"].view(np.uint16), lines.view(np.uint16))


def test_half_oracle_equals_reference_golden(gold):
    det, mask, boxes, scores = _oracle(gold)
    assert det.dtype == np.float32 and np.array_equal(det, gold["det"])
    assert np.array_equal(mask, gold["mask_u8"])
    assert np.array_equal(boxes, gold["line_boxes"]) and np.array_equal(scores, gold["line_scores"])


@pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")
def test_half_oracle_equals_reference_itself(gold):
    from oracle import make_golden_half_ref
    ref = make_golden_half_ref.reference_outputs(ref_shim.load(), gold["blks"], gold["mask"], gold["lines"])
    got = _oracle(gold)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)


def test_golden_exercises_every_half_rule(gold):
    det, mask, _b, _s = _oracle(gold)
    f32 = {k: gold[k].astype(np.float32) for k in ("blks", "mask", "lines")}
    det32 = postproc_ref.non_max_suppression(torch.from_numpy(f32["blks"])[None], 0.4, 0.35)[0].numpy()
    mask32 = (f32["mask"][0] * 255).astype(np.uint8)
    bitmap = postproc_half_ref.binarize_half(gold["lines"][0])
    bitmap32 = f32["lines"][0] > 0.3
    assert int((mask != mask32).reshape(-1)[:0x3c01].sum()) == 131   # every float16 value in [0, 1]
    assert (bitmap != bitmap32).any()
    # scores: quantised to half in the half path
    assert not np.array_equal(np.sort(det[:, 4]), np.sort(det32[:, 4]))
    assert np.array_equal(det[:, 4], det[:, 4].astype(np.float16).astype(np.float32))
    # at least one box whose corners truncate to other blines: the same detection (class, rounded score) in both
    rows32 = {(r[5], round(float(r[4]), 2), int(r[0] // 8), int(r[1] // 8)): r for r in det32}
    moved = [d for d in det if (k := (d[5], round(float(d[4]), 2), int(d[0] // 8), int(d[1] // 8))) in rows32
             and not np.array_equal(d[:4].astype(np.int32), rows32[k][:4].astype(np.int32))]
    assert moved


# ---- check_outputs --------------------------------------------------------------------------------------------------
def _outs(dtype):
    a = postprocess.workspace_rows(*NET)
    return np.zeros((1, a, 7), dtype), np.zeros((1, 1) + NET, dtype), np.zeros((1, 2) + NET, dtype)


@pytest.mark.parametrize("form", ["numpy", "cpu_tensor"])
def test_check_outputs_half_views(form):
    o = _outs(np.float16)
    if form == "cpu_tensor":
        o = tuple(torch.from_numpy(x) for x in o)
    b, m, ln = postprocess.check_outputs(*o, NET, half=True)
    assert b.dtype == m.dtype == ln.dtype == np.float16
    base = [x.numpy() if form == "cpu_tensor" else x for x in o]
    assert np.shares_memory(b, base[0]) and np.shares_memory(m, base[1]) and np.shares_memory(ln, base[2])
    # float32 pages still pass with half=True
    assert postprocess.check_outputs(*_outs(np.float32), NET, half=True)[0].dtype == np.float32


@pytest.mark.parametrize("which", [1, 2])
def test_check_outputs_refuses_mixed_page(which):
    o = list(_outs(np.float16))
    o[which] = o[which].astype(np.float32)
    name = ["blks", "mask", "lines_map"][which]
    with pytest.raises(ValueError, match="item 3: %s is float32 but blks is float16" % name):
        postprocess.check_outputs(*o, NET, what="item 3: ", half=True)


def test_check_outputs_refuses_bfloat16_and_half_without_half():
    o = [torch.from_numpy(x) for x in _outs(np.float32)]
    o[2] = o[2].bfloat16()
    with pytest.raises(ValueError, match="lines_map must be float32 or float16, got torch.bfloat16"):
        postprocess.check_outputs(*o, NET, half=True)
    with pytest.raises(ValueError, match=r"blks must be float32, got float16"):
        postprocess.check_outputs(*_outs(np.float16), NET)
    with pytest.raises(ValueError, match=r"convert with \.float\(\)"):
        postprocess.check_outputs(*[torch.from_numpy(x) for x in _outs(np.float16)], NET)


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_half_entries_and_dtype_enum_match_header(tmp_path):
    src = tmp_path / "dtype.c"
    src.write_text('#include <stdio.h>\n#include "ctd_b200.h"\nint main(void) {\n'
                   '  int (*a)(ctd_handle*, int32_t, const ctd_page_entry*, int32_t, int32_t, int32_t, const uint8_t*,\n'
                   '           const ctd_device_page*, const ctd_net_output*, const int32_t*, int32_t, int32_t,\n'
                   '           int32_t, int32_t, void*) = ctd_submit_outputs_dtype;\n'
                   '  int (*b)(ctd_handle*, const void*, int32_t, int32_t, int32_t, void*, void*, void*, void*) =\n'
                   '      ctd_forward_tensor_f16;\n'
                   '  printf("%d %d %d\\n", (int)CTD_DTYPE_F32, (int)CTD_DTYPE_F16, CTD_ABI_VERSION);\n'
                   '  return a == 0 || b == 0;\n}\n')
    obj = tmp_path / "dtype.o"
    subprocess.check_call(["cc", "-c", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(obj)])
    exe = tmp_path / "dtype"
    subprocess.check_call(["cc", str(obj), "-o", str(exe), ctd_b200.LIB_PATH, "-Wl,-rpath," + os.path.dirname(ctd_b200.LIB_PATH)])
    f32, f16, abi = (int(v) for v in subprocess.check_output([str(exe)]).split())
    assert (f32, f16) == (binding.DTYPE_F32, binding.DTYPE_F16) == (0, 1)
    assert abi == 3
    lib = C.CDLL(ctd_b200.LIB_PATH)
    for name in ("ctd_submit_outputs_dtype", "ctd_forward_tensor_f16"):
        assert name in binding.EXPORTS and hasattr(lib, name)
