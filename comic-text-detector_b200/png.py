"""PNG files on the GPU.

Encode (csrc/png.cu), byte for byte what the reference's `io_utils.imwrite` writes: `cv2.imencode('.png', img)[1]`.
`PngEncoder.encode(imgs)` encodes a list of u8 images, grey [h][w] or BGR [h][w][3], numpy arrays or torch.uint8 CUDA
tensors of any strides on the encoder's GPU, in one call, and returns each file as a 1-D np.uint8 array.

Decode (csrc/png_plan.cpp, csrc/png_dec.cu), equal to what the reference's `io_utils.imread` reads:
`cv2.imdecode(buf, cv2.IMREAD_COLOR)`.  `PngDecoder.decode(bufs)` decodes every PNG of a list the GPU takes in one call
and returns a torch.uint8 CUDA page for each; every other file (Adam7, APNG, a bad CRC or corrupt data, a JPEG, ...)
is decoded by cv2.imdecode on the host, so each result is exactly what cv2 returns, a numpy page or None.
`png_probe(buf)` is the host chunk walk that decides which files the GPU takes.
"""
import ctypes as C

import numpy as np

from .binding import CtdError, CtdPngImage, CtdPngInfo, load_library
from .jpeg import _cv2_decode, as_buffer

# ctd_png_status (include/ctd_b200.h)
PNG_STATUS = ["ok", "not_png", "truncated", "header", "interlaced", "apng", "chunks", "exif", "zlib", "size", "crc",
              "data"]
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _check(i, shape, dtype_ok, fmt, max_side):
    if not dtype_ok:
        raise ValueError("image %d: a %s image must be uint8" % (i, fmt))
    if len(shape) not in (2, 3) or (len(shape) == 3 and shape[2] != 3):
        raise ValueError("image %d: a %s image must be [h][w] or [h][w][3], got shape %s" % (i, fmt, tuple(shape)))
    if 0 in tuple(shape):
        raise ValueError("image %d: a %s image must not be empty, got shape %s" % (i, fmt, tuple(shape)))
    if max_side and max(shape[0], shape[1]) > max_side:
        raise ValueError("image %d: a %s image has sides of at most %d, got shape %s" % (i, fmt, max_side, tuple(shape)))


def image_descs(imgs, device_index, fmt, max_side=None):
    """`ctd_png_image` descriptors of u8 images for the encoders (PNG and JPEG): numpy arrays, or torch.uint8 CUDA
    tensors on cuda:device_index of any strides, each tensor with an event recorded on its device's current stream.
    max_side (None: no limit) bounds both sides.  Returns (descs, keep): `keep` holds what the descriptors point to
    (and the events) until the call returns.  Any other input raises ValueError naming its index, before an event is
    recorded."""
    n = len(imgs)
    descs = (CtdPngImage * n)()
    keep = []
    torch = None
    for i, img in enumerate(imgs):
        d = descs[i]
        if isinstance(img, np.ndarray):
            _check(i, img.shape, img.dtype == np.uint8, fmt, max_side)
            a = np.ascontiguousarray(img)
            keep.append(a)
            d.data = a.ctypes.data
            d.on_device = 0
        else:
            if torch is None:
                import torch
            if not isinstance(img, torch.Tensor):
                raise ValueError("image %d: expected a numpy array or a torch CUDA tensor, got %s" % (i, type(img)))
            if not img.is_cuda or img.device.index != device_index:
                raise ValueError("image %d: a tensor must be on cuda:%d, got %s" % (i, device_index, img.device))
            _check(i, img.shape, img.dtype == torch.uint8, fmt, max_side)
            keep.append(img)
            d.data = img.data_ptr()
            d.on_device = 1
            st = img.stride()
            d.stride_h, d.stride_w = st[0], st[1]
            d.stride_c = st[2] if img.dim() == 3 else 0
        d.height, d.width = img.shape[0], img.shape[1]
        d.channels = 3 if len(img.shape) == 3 else 1
        d.bit_depth = 8
    for i, img in enumerate(imgs):
        if descs[i].on_device:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(img.device))
            keep.append(ev)
            descs[i].event = ev.cuda_event
    return descs, keep


def files_from(files, sizes, n):
    """copies of the n files an encoder left in its pinned output"""
    return [np.ctypeslib.as_array(C.cast(files[i], C.POINTER(C.c_uint8)), (sizes[i],)).copy() for i in range(n)]


class PngEncoder:
    """A GPU PNG encoder on cuda:device_index with a stream and buffers of its own."""

    def __init__(self, device_index=0):
        self.lib = load_library()
        self.device_index = int(device_index)
        self.h = C.c_void_p()
        rc = self.lib.ctd_png_encoder_create(self.device_index, C.byref(self.h))
        if rc != 0:
            raise CtdError("ctd_png_encoder_create failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.ctd_png_encoder_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def encode(self, imgs):
        """imgs: a list of u8 images, each a numpy [h][w] / [h][w][3] array or a torch.uint8 CUDA tensor of those
        shapes on this encoder's device (any strides: a crop, `chw.permute(1, 2, 0)`).  A CUDA tensor is read after
        the work already queued on its device's current stream.  Returns one 1-D np.uint8 array per image, equal to
        `cv2.imencode('.png', img)[1]`.  Any other input raises ValueError naming its index, before any GPU work."""
        n = len(imgs)
        if n == 0:
            return []
        descs, _keep = image_descs(imgs, self.device_index, "PNG")
        files = (C.c_void_p * n)()
        sizes = (C.c_int64 * n)()
        rc = self.lib.ctd_png_encode(self.h, descs, n, files, sizes)
        if rc != 0:
            raise CtdError("ctd_png_encode failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        return files_from(files, sizes, n)


def png_probe(buf):
    """`ctd_png_probe` (host only): dict of the ctd_png_info fields, plus `reason`, the status's name.  status 0: the
    GPU decodes the file, to a page of shape (height, width, 3) (eXIf orientation applied), unless its CRCs or its
    image data turn out not to be clean (`PngDecoder.last_status` "crc" / "data")."""
    a = as_buffer(buf)
    info = CtdPngInfo()
    rc = load_library().ctd_png_probe(a.ctypes.data_as(C.c_void_p), a.size, C.byref(info))
    if rc != 0:
        raise CtdError("ctd_png_probe failed (%d)" % rc)
    out = {k: int(getattr(info, k)) for k, _t in CtdPngInfo._fields_}
    out["reason"] = PNG_STATUS[out["status"]]
    return out


def is_png(buf):
    """True when an encoded file (1-D np.uint8 array) starts with the PNG signature"""
    return buf.size >= 8 and buf[:8].tobytes() == PNG_SIGNATURE


class PngDecoder:
    """A GPU PNG decoder on cuda:device_index with a stream of its own.  subsequence_bits (0: the default): the length
    of the pieces the parallel inflate cuts each Huffman block into; it changes how the work is split, never the
    result."""

    def __init__(self, device_index=0, subsequence_bits=0):
        self.lib = load_library()
        self.device_index = int(device_index)
        self.h = C.c_void_p()
        rc = self.lib.ctd_png_decoder_create(self.device_index, int(subsequence_bits), C.byref(self.h))
        if rc != 0:
            raise CtdError("ctd_png_decoder_create failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        self._alloc_stream = None
        self.last_status = []

    def close(self):
        if getattr(self, "h", None):
            self.lib.ctd_png_decoder_destroy(self.h)
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
        used on the current stream.  `last_status` keeps each file's ctd_png_status."""
        import torch
        arrs = [as_buffer(b) for b in bufs]
        n = len(arrs)
        if n == 0:
            return []
        dev = torch.device("cuda", self.device_index)
        infos = [png_probe(a) for a in arrs]
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
        rc = self.lib.ctd_png_decode(self.h, data, lens, n, dst, status)
        if rc != 0:
            raise CtdError("ctd_png_decode failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
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

    def last_stats(self):
        """(deflate blocks, self-synchronisation rounds) of the last decode's files decoded on the GPU"""
        blocks, rounds = C.c_int64(), C.c_int64()
        if self.lib.ctd_png_decoder_stats(self.h, C.byref(blocks), C.byref(rounds)) != 0:
            raise CtdError("ctd_png_decoder_stats failed: %s" % self.lib.ctd_last_error(None).decode())
        return blocks.value, rounds.value
