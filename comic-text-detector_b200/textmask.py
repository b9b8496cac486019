"""Text masks for any block list: the reference's `utils/textmask.py` library functions and a batched form.

`refine_mask(img, pred_mask, blk_list, refine_mode)` and `refine_undetected_mask(img, mask_pred, mask_refined,
blk_list, refine_mode)` (textmask.py:135-169) take the block list from the caller, so code that edits the detector's
blocks (drops SFX blocks, adds a missed block, merges or moves blocks) or reads them back from `model2annotations`'s
json refines the mask on the GPU, byte for byte what the reference computes (with refine_mask's histogram ties broken by
ascending bin, as everywhere in this package).  Both run as one-page batches of `ctd_submit_refine` on the kernels-only
engine of `TextBlock.get_transformed_region`.  `MaskRefiner.refine_stream` runs many pages in batches, two in flight,
with pages and masks in host or GPU memory and pages also as encoded files, as `TextDetector.detect_stream` takes them.

Only `blk.xyxy` of a block is read: the reference's `merge_mask_list` reads the rest of the block only when it filters
with the text lines, which `refine_mask` never asks for.
"""
import operator

import numpy as np

from . import binding
from .inference import REFINEMASK_INPAINT, _Encoded, _page_ready_event, _torch
from .jpeg import is_encoded
from .kernel_jobs import KernelsOnlyJob, checked_page
from .textblock import _region_engine


def block_boxes(blk_list):
    """int32 [k][4] of each block's xyxy; ValueError naming a block whose xyxy is not 4 integers that fit int32"""
    out = np.zeros((len(blk_list), 4), np.int32)
    for b, blk in enumerate(blk_list):
        try:
            xy = [operator.index(v) for v in blk.xyxy]
        except (TypeError, AttributeError):
            raise ValueError("block %d: xyxy must be 4 integers, got %r" % (b, getattr(blk, "xyxy", None))) from None
        if len(xy) != 4 or any(not -2 ** 31 <= v < 2 ** 31 for v in xy):
            raise ValueError("block %d: xyxy must be 4 integers that fit int32, got %r" % (b, xy))
        out[b] = xy
    return out


def check_blocks(shape, boxes, what=""):
    """ValueError naming the first block of `boxes` (int32 [k][4]) on which the reference's refine_mask raises on an
    ih x iw page, or whose window does not fit int32 (ctd_refine_plan's status)"""
    _e, win, status, _ib, _rb = binding.refine_plan([shape], boxes, [len(boxes)])
    bad = np.flatnonzero(status)
    if len(bad):
        b = int(bad[0])
        why = "its window %s is empty, and the reference raises on it" % win[b].tolist() if status[b] == 1 else \
              "its window does not fit int32"
        raise ValueError("%sblock %d (xyxy %s) on a %dx%d page: %s" % (what, b, boxes[b].tolist(), shape[0], shape[1],
                                                                       why))


def check_mask(mask, shape, what="", device_index=None):
    """a mask as the refine calls take it: u8 [h][w] of the page's size (numpy, or a CUDA tensor of any strides on
    cuda:device_index), else ValueError"""
    if getattr(mask, "is_cuda", False):
        if mask.dtype != _torch().uint8 or tuple(mask.shape) != tuple(shape):
            raise ValueError("%sthe mask must be a uint8 tensor of shape %s, got %s %s"
                             % (what, tuple(shape), mask.dtype, tuple(mask.shape)))
        if device_index is not None and mask.device.index != device_index:
            raise ValueError("%sa CUDA mask must be on cuda:%d, got %s" % (what, device_index, mask.device))
        return mask
    a = np.asarray(mask)
    if a.dtype != np.uint8 or a.shape != tuple(shape):
        raise ValueError("%sthe mask must be a uint8 array of shape %s, got %s %s" % (what, tuple(shape), a.dtype, a.shape))
    return a


def _one(img, pred_mask, blk_list, refine_mode, keep_undetected, refined):
    """one page through ctd_submit_refine on the process-wide kernels-only engine: (mask, mask_refined)"""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError("the page must be a uint8 array of shape [h][w][3], got %s %s" % (img.dtype, img.shape))
    shape = img.shape[:2]
    pred_mask = check_mask(pred_mask, shape)
    if getattr(pred_mask, "is_cuda", False):
        raise ValueError("the mask must be a numpy array")
    if refined is not None:
        refined = check_mask(refined, shape, "mask_refined: ")
        if getattr(refined, "is_cuda", False):
            raise ValueError("mask_refined must be a numpy array")
    boxes = block_boxes(blk_list)
    if refined is None:
        check_blocks(shape, boxes)
    eng, lock = _region_engine()
    with lock:
        eng.submit_refine(0, [img], [pred_mask], [boxes], refine_mode, keep_undetected,
                          None if refined is None else [refined])
        return eng.collect_refine(0)[0]


def refine_mask(img, pred_mask, blk_list, refine_mode=REFINEMASK_INPAINT):
    """The reference's `refine_mask` (utils/textmask.py:159-169) on the GPU: img u8 BGR [h][w][3], pred_mask u8 [h][w]
    (numpy) -> the refined mask, a new u8 [h][w] array.  ValueError before any GPU work for a block on which the
    reference raises (its window is empty after Python's slice normalisation, e.g. y2 <= y1) and for a mask that is not
    u8 [h][w] of the page's size."""
    return _one(img, pred_mask, blk_list, refine_mode, False, None)[1]


def refine_undetected_mask(img, mask_pred, mask_refined, blk_list, refine_mode=REFINEMASK_INPAINT):
    """The reference's `refine_undetected_mask` (utils/textmask.py:135-156) on the GPU: refines the parts of the
    predicted mask that no block of `blk_list` covers and returns mask_refined OR those parts, a new array.  As in the
    reference, mask_pred (numpy u8 [h][w]) is modified in place: its pixels under mask_refined > 30 are cleared.
    mask_refined may be any u8 [h][w] mask, not only refine_mask's result."""
    mask, refined = _one(img, mask_pred, blk_list, refine_mode, True, mask_refined)
    mask_pred[...] = mask
    return refined


class MaskRefiner(KernelsOnlyJob):
    """refine_mask (and refine_undetected_mask) for many pages on cuda:device_index, in batches of up to max_batch
    pages with two batches in flight, on a kernels-only engine of its own (no network)."""

    def refine_batch(self, items, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, device_results=False):
        """list(refine_stream(...)), with every item checked before any GPU work"""
        items = list(items)
        for i, (img, mask, blk_list) in enumerate(items):
            if not is_encoded(img):
                page = checked_page(img, "item %d: " % i, self.device_index)
                check_mask(mask, tuple(page.shape[:2]), "item %d: " % i, self.device_index)
                check_blocks(tuple(page.shape[:2]), block_boxes(blk_list), "item %d: " % i)
        return list(self.refine_stream(items, refine_mode, keep_undetected_mask, device_results))

    def refine_stream(self, items, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, device_results=False):
        """Generator over an iterable of (img, mask, blk_list): yields (mask, mask_refined) for each item in input
        order, where mask_refined is `refine_mask(img, mask, blk_list, refine_mode)`, and with keep_undetected_mask
        `refine_undetected_mask(img, mask, that, blk_list, refine_mode)`, as `TextDetector.__call__` chains them.

        img: a page as `TextDetector.detect_stream` takes it: u8 BGR [h][w][3] numpy, a torch.uint8 CUDA tensor on
        cuda:device_index with any strides, or an encoded file (decoded on the GPU with its batch where the GPU
        takes it, else by cv2).  mask: u8 [h][w] of the page's size, numpy or a CUDA tensor with any strides (such as
        `page[..., 0]`).  For CUDA pages and masks an event is recorded on the current stream when the item is read,
        and the GPU waits for it before reading them; they must not be written until the item's result is yielded.

        Output: without keep_undetected_mask, `mask` is the caller's own object, untouched; with it, a new array holding
        the predicted mask as refine_undetected_mask leaves it (the caller's input is not modified).  device_results:
        the new masks are torch.uint8 CUDA tensors, one allocation per item, complete when yielded.

        A page or mask of the wrong type or shape, or a block on which the reference's refine_mask raises, raises
        ValueError naming the item before its batch reaches the GPU (for an encoded page: once its batch is decoded)."""
        return self._stream(items, refine_mode, bool(keep_undetected_mask), bool(device_results))

    def _stream(self, items, refine_mode, keep, device_results):
        def records():
            for idx, (img, mask, blk_list) in enumerate(items):
                what = "item %d: " % idx
                boxes = block_boxes(blk_list)
                if is_encoded(img):
                    page = _Encoded(idx, img)   # decoded, and its mask and blocks checked, with its batch
                else:
                    page = checked_page(img, what, self.device_index)
                    mask = check_mask(mask, tuple(page.shape[:2]), what, self.device_index)
                    check_blocks(tuple(page.shape[:2]), boxes, what)
                cuda = page if getattr(page, "is_cuda", False) else mask if getattr(mask, "is_cuda", False) else None
                yield (idx, page, mask, boxes, _page_ready_event(cuda))

        def decoded(rec, page, what):
            idx, _e, mask, boxes, ev = rec
            mask = check_mask(mask, tuple(page.shape[:2]), what, self.device_index)
            check_blocks(tuple(page.shape[:2]), boxes, what)
            return (idx, page, mask, boxes, ev)

        def submit(slot, batch):
            self.net.submit_refine(slot, [b[1] for b in batch], [b[2] for b in batch], [b[3] for b in batch],
                                   refine_mode, keep, None, [b[4] for b in batch], device_results)
            return [b[2] for b in batch]   # the caller's masks

        def collect(slot, masks, discard):
            res = self.net.collect_refine(slot, discard=discard)
            return None if discard else [((mask if keep else m), refined) for m, (mask, refined) in zip(masks, res)]

        return self._pipeline(records(), lambda batch: self._decode(batch, decoded), submit, collect)
