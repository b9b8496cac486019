"""PNG files encoded on the GPU (csrc/png.cu), byte for byte what the reference's `io_utils.imwrite` writes:
`cv2.imencode('.png', img)[1]`.

`PngEncoder.encode(imgs)` encodes a list of u8 images, grey [h][w] or BGR [h][w][3], numpy arrays or torch.uint8 CUDA
tensors of any strides on the encoder's GPU, in one call, and returns each file as a 1-D np.uint8 array.
"""
import ctypes as C

import numpy as np

from .binding import CtdError, CtdPngImage, load_library


def _check(i, shape, dtype_ok):
    if not dtype_ok:
        raise ValueError("image %d: a PNG image must be uint8" % i)
    if len(shape) not in (2, 3) or (len(shape) == 3 and shape[2] != 3):
        raise ValueError("image %d: a PNG image must be [h][w] or [h][w][3], got shape %s" % (i, tuple(shape)))
    if 0 in tuple(shape):
        raise ValueError("image %d: a PNG image must not be empty, got shape %s" % (i, tuple(shape)))


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
        descs = (CtdPngImage * n)()
        keep, events = [], []
        torch = None
        for i, img in enumerate(imgs):
            d = descs[i]
            if isinstance(img, np.ndarray):
                _check(i, img.shape, img.dtype == np.uint8)
                a = np.ascontiguousarray(img)
                keep.append(a)
                d.data = a.ctypes.data
                d.on_device = 0
            else:
                if torch is None:
                    import torch
                if not isinstance(img, torch.Tensor):
                    raise ValueError("image %d: expected a numpy array or a torch CUDA tensor, got %s" % (i, type(img)))
                if not img.is_cuda or img.device.index != self.device_index:
                    raise ValueError("image %d: a tensor must be on cuda:%d, got %s" % (i, self.device_index, img.device))
                _check(i, img.shape, img.dtype == torch.uint8)
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
                events.append(ev)
                descs[i].event = ev.cuda_event
        files = (C.c_void_p * n)()
        sizes = (C.c_int64 * n)()
        rc = self.lib.ctd_png_encode(self.h, descs, n, files, sizes)
        if rc != 0:
            raise CtdError("ctd_png_encode failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        return [np.ctypeslib.as_array(C.cast(files[i], C.POINTER(C.c_uint8)), (sizes[i],)).copy() for i in range(n)]
