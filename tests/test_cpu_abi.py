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


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback():
    P = cc.Program()
    P.nc = 2
    P.newbuf(8, 1)
    P._op(cc.OP_AVGPOOL2, [P.tensor(0, 0, 8)], P.tensor(P.newbuf(8, 2), 0, 8))
    with pytest.raises(ctd_b200.CtdError) as e:
        ctd_b200.Engine(P, max_batch=1, max_h=64, max_w=64)
    assert "no CPU fallback" in str(e.value) or "not sm_90" in str(e.value)
