"""not-gpu: the ctypes mirror of `ctd_device_page` matches the header's layout, and the page check of the batched
stream keeps taking CPU tensors and numpy arrays as before."""
import ctypes

import numpy as np
import pytest
import torch

from ctd_b200 import binding
from ctd_b200.inference import check_page


def test_device_page_layout():
    # const uint8_t* data; int64_t stride_h, stride_w, stride_c; void* event
    P = binding.CtdDevicePage
    assert ctypes.sizeof(P) == 40
    assert [getattr(P, f).offset for f in ("data", "stride_h", "stride_w", "stride_c", "event")] == [0, 8, 16, 24, 32]


def test_check_page_host_inputs():
    a = np.arange(5 * 7 * 3, dtype=np.uint8).reshape(5, 7, 3)
    for page in (a, torch.from_numpy(a), a[:, ::2]):
        got = check_page(page, 0)
        assert isinstance(got, np.ndarray) and got.flags.c_contiguous and np.array_equal(got, np.asarray(page))
    for bad in (a.astype(np.float32), a[..., 0], a[..., :2], a[:0], torch.from_numpy(a).float()):
        with pytest.raises(ValueError):
            check_page(bad, 0)
