"""not-gpu: the C-ABI shared library loads, exports every symbol include/ctd_b200.h declares, and
refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import compiler as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "ctd_b200.h")).read()
    return sorted(set(re.findall(r"CTD_API\s+[\w\s\*]+?\b(ctd_\w+)\s*\(", src)))


def test_header_symbols_exported():
    names = _declared()
    assert len(names) >= 16, names
    lib = ctypes.CDLL(ctd_b200.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), "libctd_b200.so does not export %s" % n
    assert sorted(ctd_b200.binding.EXPORTS) == names


def test_struct_layouts_match_header():
    # field counts / sizes the ctypes mirrors must agree with (ctd_op: 20 int32 + 4 int64)
    from ctd_b200.binding import CtdOp, CtdBufDesc, CtdConfig
    assert ctypes.sizeof(CtdOp) == 20 * 4 + 4 * 8
    assert ctypes.sizeof(CtdBufDesc) == 8
    assert ctypes.sizeof(CtdConfig) == 12 * 4


def test_stale_abi_version_refused():
    """a caller built against ABI version 2 (where ctd_submit_pages had another signature) is refused by ctd_create
    before any device is probed"""
    from ctd_b200.binding import ABI_VERSION, CtdBufDesc, CtdConfig, CtdOp
    src = open(os.path.join(ROOT, "include", "ctd_b200.h")).read()
    assert int(re.search(r"#define CTD_ABI_VERSION (\d+)", src).group(1)) == ABI_VERSION == 3
    lib = ctd_b200.load_library()
    cfg = CtdConfig(2, 0, 0, 1, 64, 64, 2, 0, 0.4, 0.35, 0.3, 0)
    ops, bufs, blob = (CtdOp * 1)(), (CtdBufDesc * 1)(), ctypes.create_string_buffer(64)
    h = ctypes.c_void_p()
    rc = lib.ctd_create(ctypes.byref(h), ctypes.byref(cfg), ops, 1, bufs, 1, ctypes.cast(blob, ctypes.c_void_p), 64)
    assert rc == -1 and not h   # CTD_E_INVALID
    assert lib.ctd_last_error(None) == b"ABI version mismatch"


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    P._op(cc.OP_AVGPOOL2, [P.tensor(0, 0, 8)], P.tensor(P.newbuf(8, 2), 0, 8))
    with pytest.raises(ctd_b200.CtdError) as e:
        ctd_b200.Engine(P, max_batch=1, max_h=64, max_w=64)
    assert "no CPU fallback" in str(e.value) or "not sm_90" in str(e.value)


def test_nms_dtype_entry():
    """ctd_nms_dtype: the NMS entry with the rows' ctd_dtype, ctd_nms its float32 case; the binding declares it with the
    header's argument list"""
    src = open(os.path.join(ROOT, "include", "ctd_b200.h")).read()
    decl = re.search(r"CTD_API int ctd_nms_dtype\(([^)]*)\)", src).group(1)
    assert [a.split()[-1].lstrip("*") for a in decl.replace("\n", " ").split(",")] == [
        "h", "pred", "rows", "dtype", "conf_thresh", "iou_thresh", "det", "det_count"]
    lib = ctd_b200.load_library()
    assert "ctd_nms_dtype" in ctd_b200.binding.EXPORTS
    assert lib.ctd_nms_dtype.argtypes == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32,
                                          ctypes.c_float, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
    assert lib.ctd_nms_dtype.restype is ctypes.c_int
