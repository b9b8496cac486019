"""Text-line crops for OCR of any block list, many pages at once.

`RegionCropper.crop_stream` cuts every line of every block the caller gives: the detector's blocks after an edit (SFX
blocks dropped, a missed block added), or blocks read back from `model2annotations`'s json with `TextBlock(**d)`.  Each
crop is byte for byte the reference's `blk.get_transformed_region(img, i, textheight)` (utils/textblock.py:162-194),
and a line on which that method raises gets None, as in `TextDetector.detect_stream(textheight=)`.  The batches run
through `ctd_submit_regions` on a kernels-only engine: the lines are planned on the engine's worker threads and every
crop of a batch is cut in one GPU launch, from host pages uploaded once or from CUDA pages read where they are.
"""
import numpy as np

from . import binding
from .inference import _Encoded, _page_ready_event
from .jpeg import is_encoded
from .kernel_jobs import KernelsOnlyJob, checked_page
from .textblock import LANGCLS2IDX, _check_textheight

MAX_SIDE = 32767   # ctd_region_plan takes pages with both sides below this


def check_textheight(textheight):
    """textheight as an int >= 2, else ValueError"""
    th = _check_textheight(textheight)
    if th < 2:
        raise ValueError("textheight must be at least 2 px, got %r" % (textheight,))
    return th


def line_records(blk_list, what=""):
    """(REGION_LINE_DTYPE records of every line of every block, block then line order; the number of lines of each
    block), with the fields `get_transformed_region` reads: `lines`, `language`, `vertical` and `font_size`.  Built a
    column per block, not a record per line.  ValueError naming the block and the line for a line that is not 4 x 2
    numbers."""
    counts, quads, lang, vert, size = [], [], [], [], []
    for b, blk in enumerate(blk_list):
        lines = blk.lines
        n = len(lines)
        counts.append(n)
        if n == 0:
            continue
        try:
            q = np.asarray(lines, np.float64)
        except (TypeError, ValueError):
            q = None
        if q is None or q.shape != (n, 4, 2):
            _raise_bad_line(lines, b, what)
        quads.append(q.reshape(n, 8))
        lang.append(LANGCLS2IDX["eng"] if blk.language == "eng" else
                    LANGCLS2IDX["unknown"] if blk.language == "unknown" else LANGCLS2IDX["ja"])
        vert.append(1 if blk.vertical else 0)
        size.append(float(blk.font_size))
    rec = np.zeros((sum(counts),), binding.REGION_LINE_DTYPE)
    if len(rec):
        per_block = [c for c in counts if c]
        rec["quad"] = np.concatenate(quads)
        rec["language"] = np.repeat(np.asarray(lang, np.int32), per_block)
        rec["vertical"] = np.repeat(np.asarray(vert, np.int32), per_block)
        rec["font_size"] = np.repeat(np.asarray(size, np.float64), per_block)
    return rec, counts


def _raise_bad_line(lines, b, what):
    for i, line in enumerate(lines):
        try:
            ok = np.asarray(line, np.float64).shape == (4, 2)
        except (TypeError, ValueError):
            ok = False
        if not ok:
            raise ValueError("%sblock %d, line %d: a line must be 4 x 2 numbers, got %r" % (what, b, i, line))
    raise ValueError("%sblock %d: its lines must be 4 x 2 numbers each" % (what, b))


def _check_side(page, what):
    h, w = int(page.shape[0]), int(page.shape[1])
    if h >= MAX_SIDE or w >= MAX_SIDE:
        raise ValueError("%sthe page is %dx%d; crops are cut from pages with both sides below %d px"
                         % (what, h, w, MAX_SIDE))
    return page


class RegionCropper(KernelsOnlyJob):
    """The OCR crops of caller block lists for many pages on cuda:device_index, in batches of up to max_batch pages
    with two batches in flight, on a kernels-only engine of its own (no network, no checkpoint)."""

    def crop_batch(self, items, textheight, device_results=False):
        """list(crop_stream(...)), with every item checked before any GPU work"""
        th = check_textheight(textheight)
        items = list(items)
        for i, (img, blk_list) in enumerate(items):
            what = "item %d: " % i
            line_records(blk_list, what)
            if not is_encoded(img):
                _check_side(checked_page(img, what, self.device_index), what)
        return list(self.crop_stream(items, th, device_results))

    def crop_stream(self, items, textheight, device_results=False):
        """Generator over an iterable of (img, blk_list): yields `crops` for each item in input order, where
        crops[b][i] is line i of blk_list[b] cut out as the reference's `blk_list[b].get_transformed_region(img, i,
        textheight)` cuts it, byte for byte, and None where that method raises (a crop side of 1 px, a degenerate quad;
        or a side of 32767 px or more), so one such line does not end the stream.

        img: a page as `TextDetector.detect_stream` takes it: u8 BGR [h][w][3] numpy, a torch.uint8 CUDA tensor on
        cuda:device_index with any strides (an event is recorded on the current stream when the item is read and the
        GPU waits for it; the tensor is read where it is and must not be written until the item is yielded), or an
        encoded file or path (decoded with its batch).  blk_list: blocks with the fields the reference's method reads,
        `lines`, `language`, `vertical` and `font_size` (TextBlock objects, including `TextBlock(**d)` from json).

        Each item's crops are views into one array of its own; with device_results=True, torch.uint8 CUDA tensors
        viewing one CUDA allocation of the item's own, complete when yielded.  An item without a crop allocates nothing.

        textheight (an integer >= 2) is checked before any item is read.  A page of the wrong type or shape, a page with
        a side of 32767 px or more, or a line that is not 4 x 2 numbers raises ValueError naming the item (and the block
        and the line) before its batch reaches the GPU (for an encoded page: once its batch is decoded)."""
        return self._stream(items, check_textheight(textheight), bool(device_results))

    def _stream(self, items, th, device_results):
        def records():
            for idx, (img, blk_list) in enumerate(items):
                what = "item %d: " % idx
                rec, counts = line_records(blk_list, what)
                if is_encoded(img):
                    page = _Encoded(idx, img)   # decoded, and its size checked, with its batch
                else:
                    page = _check_side(checked_page(img, what, self.device_index), what)
                yield (idx, page, rec, counts, _page_ready_event(page))

        def submit(slot, batch):
            self.net.submit_regions(slot, [b[1] for b in batch], np.concatenate([b[2] for b in batch]),
                                    [len(b[2]) for b in batch], th, [b[4] for b in batch], device_results)
            return [b[3] for b in batch]   # each page's lines per block

        def collect(slot, counts, discard):
            return self.net.collect_crops(slot, counts, discard)

        decoded = lambda rec, page, what: (rec[0], _check_side(page, what)) + tuple(rec[2:])
        return self._pipeline(records(), lambda batch: self._decode(batch, decoded), submit, collect)
