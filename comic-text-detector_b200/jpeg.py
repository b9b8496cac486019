"""JPEG pages decoded on the GPU (csrc/jpeg_plan.cpp, csrc/jpeg.cu), equal to what the reference's `io_utils.imread`
reads: `cv2.imdecode(buf, cv2.IMREAD_COLOR)`.

`JpegDecoder.decode(bufs)` decodes every baseline JPEG of a list on the GPU in one call and returns a torch.uint8 CUDA
page for each; every other file (PNG, progressive JPEG, CMYK, a corrupt scan, ...) is decoded by cv2.imdecode on the
host, so each result is exactly what cv2 returns, a numpy page or None.  (PNG files have a GPU decoder of their own,
png.PngDecoder; TextDetector sends each encoded page to the decoder of its format.)  `jpeg_probe(buf)` is the host marker walk that
decides which files the GPU takes.
"""
import ctypes as C
import os

import numpy as np

from .binding import CtdError, CtdJpegInfo, load_library

# ctd_jpeg_status (include/ctd_b200.h)
JPEG_STATUS = ["ok", "not_jpeg", "truncated", "progressive", "arithmetic", "precision", "lossless", "sampling", "color",
               "scans", "exif", "tables", "entropy", "range", "size"]


def as_buffer(buf):
    """bytes / bytearray / memoryview / 1-D np.uint8 array -> a C-contiguous 1-D np.uint8 array over the same bytes"""
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.uint8 or buf.ndim != 1:
            raise ValueError("an encoded page must be a 1-D uint8 array, got %s %s" % (buf.dtype, buf.shape))
        return np.ascontiguousarray(buf)
    if isinstance(buf, (bytes, bytearray, memoryview)):
        return np.frombuffer(buf, np.uint8)
    raise ValueError("an encoded page must be bytes, bytearray, memoryview or a 1-D uint8 array, got %s" % type(buf))


def jpeg_probe(buf):
    """`ctd_jpeg_probe` (host only): dict of the ctd_jpeg_info fields, plus `reason`, the status's name.  status 0:
    the GPU decodes the file, to a page of shape (height, width, 3) (EXIF orientation applied)."""
    a = as_buffer(buf)
    info = CtdJpegInfo()
    rc = load_library().ctd_jpeg_probe(a.ctypes.data_as(C.c_void_p), a.size, C.byref(info))
    if rc != 0:
        raise CtdError("ctd_jpeg_probe failed (%d)" % rc)
    out = {k: int(getattr(info, k)) for k, _t in CtdJpegInfo._fields_}
    out["reason"] = JPEG_STATUS[out["status"]]
    return out


class JpegDecoder:
    """A GPU JPEG decoder on cuda:device_index with a stream of its own.  subsequence_bits: the length of the pieces
    the parallel Huffman decode cuts each restart interval into (0: the default); it changes how the work is split,
    never the result."""

    def __init__(self, device_index=0, subsequence_bits=0):
        self.lib = load_library()
        self.device_index = int(device_index)
        self.h = C.c_void_p()
        rc = self.lib.ctd_jpeg_decoder_create(self.device_index, int(subsequence_bits), C.byref(self.h))
        if rc != 0:
            raise CtdError("ctd_jpeg_decoder_create failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        self._alloc_stream = None
        self.last_status = []

    def close(self):
        if getattr(self, "h", None):
            self.lib.ctd_jpeg_decoder_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def decode(self, bufs):
        """bufs: a list of encoded files (bytes-like or 1-D np.uint8 arrays).  Returns a list with, per file, a
        torch.uint8 CUDA tensor [h][w][3] (BGR) when the GPU decoded it, else `cv2.imdecode(buf, IMREAD_COLOR)`: a
        numpy page or None.  Every result equals cv2.imdecode's.  The tensors are complete on return and marked as
        used on the current stream.  `last_status` keeps each file's ctd_jpeg_status."""
        import torch
        arrs = [as_buffer(b) for b in bufs]
        n = len(arrs)
        if n == 0:
            return []
        dev = torch.device("cuda", self.device_index)
        infos = [jpeg_probe(a) for a in arrs]
        # the pages are allocated on a stream of this decoder's own, so the caching allocator cannot hand out memory
        # that work still queued on the caller's stream uses (the decode does not wait for that stream)
        if self._alloc_stream is None:
            self._alloc_stream = torch.cuda.Stream(dev)
        with torch.cuda.stream(self._alloc_stream):
            pages = [torch.empty((i["height"], i["width"], 3), dtype=torch.uint8, device=dev) if i["status"] == 0
                     else None for i in infos]
        data = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_size_t * n)(*[a.size for a in arrs])
        dst = (C.c_void_p * n)(*[p.data_ptr() if p is not None else None for p in pages])
        status = (C.c_int32 * n)()
        rc = self.lib.ctd_jpeg_decode(self.h, data, lens, n, dst, status)
        if rc != 0:
            raise CtdError("ctd_jpeg_decode failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        self.last_status = list(status)
        cur = torch.cuda.current_stream(dev)
        out = []
        for a, p, s in zip(arrs, pages, status):
            if s == 0:
                p.record_stream(cur)
                out.append(p)
            else:
                out.append(_cv2_decode(a))
        return out


def _cv2_decode(a):
    import cv2
    return cv2.imdecode(a, cv2.IMREAD_COLOR)


def is_encoded(page):
    """True for the forms TextDetector's batch calls read as encoded files: bytes, bytearray, memoryview, a 1-D
    np.uint8 array, a str or os.PathLike path"""
    if isinstance(page, (bytes, bytearray, memoryview, str, os.PathLike)):
        return True
    return isinstance(page, np.ndarray) and page.ndim == 1 and page.dtype == np.uint8


def read_encoded(page):
    """(1-D np.uint8 buffer, path or None) of an encoded page; a path is read as the reference's imread reads it"""
    if isinstance(page, (str, os.PathLike)):
        return np.fromfile(page, dtype=np.uint8), os.fspath(page)
    return as_buffer(page), None
