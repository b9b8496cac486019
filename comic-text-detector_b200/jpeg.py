"""JPEG pages decoded on the GPU (csrc/jpeg_plan.cpp, csrc/jpeg.cu), equal to what the reference's `io_utils.imread`
reads: `cv2.imdecode(buf, cv2.IMREAD_COLOR)`.

`JpegDecoder.decode(bufs)` decodes every baseline JPEG of a list on the GPU in one call and returns a torch.uint8 CUDA
page for each; every other file (PNG, progressive JPEG, CMYK, a corrupt scan, ...) is decoded by cv2.imdecode on the
host, so each result is exactly what cv2 returns, a numpy page or None.  (PNG files have a GPU decoder of their own,
png.PngDecoder; TextDetector sends each encoded page to the decoder of its format.)  `jpeg_probe(buf)` is the host marker walk that
decides which files the GPU takes.

`JpegEncoder.encode(imgs, params)` (csrc/jpeg_enc.cu) writes JPEG files on the GPU, byte for byte what the reference's
`io_utils.imwrite(path, img, '.jpg')` writes: `cv2.imencode('.jpg', img, params)[1]`, for u8 grey [h][w] or BGR
[h][w][3] images, numpy arrays or torch.uint8 CUDA tensors of any strides, many in one call.
"""
import ctypes as C
import os

import numpy as np

from .binding import CtdError, CtdJpegInfo, CtdJpegParams, load_library

# cv2.IMWRITE_JPEG_* keys and the IMWRITE_JPEG_SAMPLING_FACTOR_* values
JPEG_QUALITY, JPEG_PROGRESSIVE, JPEG_OPTIMIZE, JPEG_RST_INTERVAL, JPEG_LUMA_QUALITY, JPEG_CHROMA_QUALITY, \
    JPEG_SAMPLING_FACTOR = 1, 2, 3, 4, 5, 6, 7
JPEG_SAMPLINGS = (0x411111, 0x221111, 0x211111, 0x121111, 0x111111)
_JPEG_KEY_NAMES = {JPEG_PROGRESSIVE: "IMWRITE_JPEG_PROGRESSIVE", JPEG_LUMA_QUALITY: "IMWRITE_JPEG_LUMA_QUALITY",
                   JPEG_CHROMA_QUALITY: "IMWRITE_JPEG_CHROMA_QUALITY"}

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


def jpeg_params(i, params):
    """cv2.imencode's reading of image i's flat [key, value, ...] list, as a CtdJpegParams: quality clamped to
    [0, 100] (default 95), a sampling value other than the five IMWRITE_JPEG_SAMPLING_FACTOR_* constants taken as 4:2:0
    (the default), OPTIMIZE clamped to [0, 1], the restart interval clamped to [0, 65535].  PROGRESSIVE,
    LUMA_QUALITY, CHROMA_QUALITY and every other key raise ValueError naming the image and the key."""
    p = CtdJpegParams(95, 0x221111, 0, 0)
    params = list(params)
    if len(params) % 2:
        raise ValueError("image %d: JPEG params must be [key, value, ...] pairs, got %d values" % (i, len(params)))
    for k, v in zip(params[0::2], params[1::2]):
        k, v = int(k), int(v)
        if k == JPEG_QUALITY:
            p.quality = min(max(v, 0), 100)
        elif k == JPEG_SAMPLING_FACTOR:
            p.sampling = v if v in JPEG_SAMPLINGS else 0x221111
        elif k == JPEG_OPTIMIZE:
            p.optimize = int(v > 0)
        elif k == JPEG_RST_INTERVAL:
            p.restart_interval = min(max(v, 0), 65535)
        else:
            raise ValueError("image %d: JPEG parameter %s is not supported by the GPU encoder"
                             % (i, _JPEG_KEY_NAMES.get(k, "key %d" % k)))
    return p


class JpegEncoder:
    """A GPU JPEG encoder on cuda:device_index with a stream and buffers of its own."""

    def __init__(self, device_index=0):
        self.lib = load_library()
        self.device_index = int(device_index)
        self.h = C.c_void_p()
        rc = self.lib.ctd_jpeg_encoder_create(self.device_index, C.byref(self.h))
        if rc != 0:
            raise CtdError("ctd_jpeg_encoder_create failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.ctd_jpeg_encoder_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def encode(self, imgs, params=None):
        """imgs: a list of u8 images, each a numpy [h][w] / [h][w][3] array or a torch.uint8 CUDA tensor of those
        shapes on this encoder's device (any strides: a crop, `chw.permute(1, 2, 0)`).  A CUDA tensor is read after
        the work already queued on its device's current stream.  params: None, one cv2-style flat list
        ([cv2.IMWRITE_JPEG_QUALITY, 90, ...]) for every image, or a list of such lists, one per image.  Returns one
        1-D np.uint8 array per image, equal to `cv2.imencode('.jpg', img, params)[1]`.  Any other input, a side above
        65500 or an unsupported parameter raises ValueError naming its index, before any GPU work."""
        from .png import files_from, image_descs
        n = len(imgs)
        if params is None:
            params = []
        if len(params) and isinstance(params[0], (list, tuple, np.ndarray)):
            per = list(params)
            if len(per) != n:
                raise ValueError("%d parameter lists for %d images" % (len(per), n))
        else:
            per = [params] * n
        prm = (CtdJpegParams * max(n, 1))(*[jpeg_params(i, p) for i, p in enumerate(per)])
        if n == 0:
            return []
        descs, _keep = image_descs(imgs, self.device_index, "JPEG", max_side=65500)
        files = (C.c_void_p * n)()
        sizes = (C.c_int64 * n)()
        rc = self.lib.ctd_jpeg_encode(self.h, descs, prm, n, files, sizes)
        if rc != 0:
            raise CtdError("ctd_jpeg_encode failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        return files_from(files, sizes, n)
