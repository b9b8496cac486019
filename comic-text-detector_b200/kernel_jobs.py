"""What the batched jobs that run no network share: `MaskRefiner` (textmask.py), `RegionCropper` (regions.py) and
`PostProcessor` (postprocess.py) each own a kernels-only engine, decode encoded pages with decoders made on first use,
and run their batches through the engine's two slots, two batches in flight, leaving no batch in flight when the caller
stops early."""
from collections import deque

from .inference import _Encoded, check_page, decode_files
from .jpeg import JpegDecoder, read_encoded
from .png import PngDecoder
from .textblock import kernels_only_engine


def checked_page(img, what, device_index):
    """check_page with the item named in its ValueError"""
    try:
        return check_page(img, device_index)
    except ValueError as ex:
        raise ValueError("%s%s" % (what, ex)) from None


class KernelsOnlyJob:
    """A kernels-only engine on cuda:device_index for batches of up to max_batch pages, and the decoders of its
    encoded pages."""

    def __init__(self, device_index=0, max_batch=16, **engine_args):
        """engine_args: the workspace and post-processing arguments of kernels_only_engine"""
        self.device_index = int(device_index)
        self.max_batch = int(max_batch)
        self.net = kernels_only_engine(self.device_index, self.max_batch, **engine_args)
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
                raise ValueError("item %d%s could not be decoded (cv2.imdecode returns None)"
                                 % (idx, "" if path is None else " (%s)" % path))
            what = "item %d: " % idx
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
