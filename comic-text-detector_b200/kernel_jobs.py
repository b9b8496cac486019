"""What the batched entries share: `TextDetector` (inference.py) on its network engine, and `MaskRefiner`
(textmask.py), `RegionCropper` (regions.py), `PostProcessor` (postprocess.py) and `Preprocessor` (preprocess.py) on a
kernels-only engine of their own, each decode encoded pages with decoders made on first use, and run their batches
through the engine's two slots, two batches in flight, leaving no batch in flight when the caller stops early."""
from collections import deque

import numpy as np

from .jpeg import JpegDecoder, read_encoded
from .png import PngDecoder, is_png
from .textblock import kernels_only_engine


def decode_files(bufs, png_decoder, jpeg_decoder):
    """encoded files (1-D np.uint8 arrays) -> their pages in input order: files with the PNG signature through
    png_decoder() (a function returning a PngDecoder), every other file through jpeg_decoder() (baseline JPEGs on the
    GPU, the rest by cv2); each page is a CUDA tensor or what cv2.imdecode(buf, IMREAD_COLOR) returns.  A decoder is
    asked for only when a file goes to it."""
    pngs = [i for i, b in enumerate(bufs) if is_png(b)]
    others = [i for i, b in enumerate(bufs) if not is_png(b)]
    out = [None] * len(bufs)
    for idx, dec in ((pngs, png_decoder), (others, jpeg_decoder)):
        if idx:
            for i, page in zip(idx, dec().decode([bufs[i] for i in idx])):
                out[i] = page
    return out


def check_page(img, device_index=None):
    """A page as TextDetector's batch calls take it: u8 BGR [h][w][3] with h, w >= 1, else ValueError.  A CUDA tensor
    (torch.uint8 [h][w][3], any strides) is returned as it is; with a device_index it must be on that GPU.  Anything
    else, CPU tensors included, goes through np.asarray and comes back as a C-contiguous array."""
    if getattr(img, "is_cuda", False):
        if img.dtype != _torch().uint8 or img.dim() != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
            raise ValueError("a page must be a uint8 tensor of shape [h][w][3], got %s %s"
                             % (img.dtype, tuple(img.shape)))
        if device_index is not None and img.device.index != device_index:
            raise ValueError("a CUDA page must be on the detector's device cuda:%d, got %s" % (device_index, img.device))
        return img
    a = np.asarray(img)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
        raise ValueError("a page must be a uint8 array of shape [h][w][3], got %s %s" % (a.dtype, a.shape))
    return np.ascontiguousarray(a)


def checked_page(img, what, device_index):
    """check_page with the item named in its ValueError"""
    try:
        return check_page(img, device_index)
    except ValueError as ex:
        raise ValueError("%s%s" % (what, ex)) from None


class _Encoded:
    """an encoded page of a stream, with its index in the stream, until its batch is decoded"""
    __slots__ = ("index", "src")

    def __init__(self, index, src):
        self.index, self.src = index, src


def _page_ready_event(page):
    """for a CUDA page: an event recorded on its device's current torch stream (the engine waits for it); else None"""
    if not getattr(page, "is_cuda", False):
        return None
    torch = _torch()
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(page.device))
    return ev


def _torch():
    import torch
    return torch


class BatchJob:
    """An engine `net` on cuda:device_index for batches of up to max_batch pages, and the decoders of its encoded
    pages.  An undecodable page is named by its index as `<item> <index>`."""
    item = "item"

    def __init__(self, net, device_index, max_batch):
        self.net = net
        self.device_index = int(device_index)
        self.max_batch = int(max_batch)
        self._jpeg = None
        self._png = None

    def jpeg_decoder(self):
        """the JpegDecoder encoded pages are decoded with (made on first use, closed with this object)"""
        if self._jpeg is None:
            self._jpeg = JpegDecoder(self.device_index)
        return self._jpeg

    def png_decoder(self):
        """the PngDecoder PNG pages are decoded with (made on first use, closed with this object)"""
        if self._png is None:
            self._png = PngDecoder(self.device_index)
        return self._png

    def close(self):
        self.net.close()
        for d in (self._jpeg, self._png):
            if d is not None:
                d.close()
        self._jpeg = self._png = None

    def _decode(self, batch, check):
        """the batch (records (item index, page, ...)) with its encoded pages (_Encoded) decoded by decode_files;
        check(record, page, what) gives the record of each decoded page, page checked or raising ValueError"""
        enc = [i for i, b in enumerate(batch) if isinstance(b[1], _Encoded)]
        if not enc:
            return batch
        bufs = [read_encoded(batch[i][1].src) for i in enc]
        pages = decode_files([b for b, _path in bufs], self.png_decoder, self.jpeg_decoder)
        batch = list(batch)
        for i, (_b, path), page in zip(enc, bufs, pages):
            idx = batch[i][0]
            if page is None:
                raise ValueError("%s %d%s could not be decoded (cv2.imdecode returns None)"
                                 % (self.item, idx, "" if path is None else " (%s)" % path))
            what = "%s %d: " % (self.item, idx)
            page = page if getattr(page, "is_cuda", False) else checked_page(page, what, self.device_index)
            batch[i] = check(batch[i], page, what)   # a page decoded on the GPU is complete when decode returns
        return batch

    def _pipeline(self, records, decode, submit, collect):
        """Generator: the records in batches of up to max_batch on the engine's two slots.  decode(batch) gives the
        batch to submit, submit(slot, batch) submits it and returns what collect needs, collect(slot, token, discard)
        waits for the batch and returns its results in record order (discard: only waits)."""
        inflight = deque()   # (slot, token) in submission order
        free = [0, 1]

        def drain():
            slot, token = inflight.popleft()
            res = collect(slot, token, False)
            free.append(slot)
            yield from res

        def run(batch):
            batch = decode(batch)
            if not free:
                yield from drain()
            slot = free.pop(0)
            inflight.append((slot, submit(slot, batch)))

        try:
            batch = []
            for rec in records:
                batch.append(rec)
                if len(batch) == self.max_batch:
                    yield from run(batch)
                    batch = []
            if batch:
                yield from run(batch)
            while inflight:
                yield from drain()
        finally:
            while inflight:   # an error or an abandoned generator: leave the engine with no batch in flight
                slot, token = inflight.popleft()
                try:
                    collect(slot, token, True)
                except Exception:
                    pass


class KernelsOnlyJob(BatchJob):
    """BatchJob on a kernels-only engine of its own."""

    def __init__(self, device_index=0, max_batch=16, **engine_args):
        """engine_args: the workspace and post-processing arguments of kernels_only_engine"""
        super().__init__(kernels_only_engine(int(device_index), int(max_batch), **engine_args), device_index, max_batch)
