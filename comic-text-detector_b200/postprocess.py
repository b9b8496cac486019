"""The detector's post-processing on any network's outputs: everything the reference's `TextDetector.__call__` does
after `blks, mask, lines_map = self.net(img_in)` (inference.py:148-178), on the GPU, for outputs the caller computed.

The outputs may come from this engine's `TextDetBase`, from a checkpoint `compiler.py` does not take run in torch, from
TensorRT or from `torch.compile`: `PostProcessor` runs non_max_suppression, postprocess_mask, SegDetectorRepresenter
and the box_thresh filter, the mask crop and resize back to the page, the line rescale, group_output, refine_mask and
refine_undetected_mask, and with a textheight the text-line crops, byte for byte what the reference computes from the
same outputs.  It batches pages with `ctd_submit_outputs`, two batches in flight, on a kernels-only engine of its own
sized for max_batch pages of input_size.  The reference's CPU code takes about 0.9 s per page for these stages
(SURVEY §8a).
"""
import re

import numpy as np

from . import binding
from .binding import CtdError
from .inference import REFINEMASK_INPAINT, _Encoded, _page_ready_event, _torch
from .jpeg import is_encoded
from .kernel_jobs import KernelsOnlyJob, checked_page
from .textblock import _check_textheight, blocks_from_records


def workspace_rows(net_h, net_w):
    """the largest A a blks output may have at (net_h, net_w): 3 * (H/8 * W/8 + H/16 * W/16 + H/32 * W/32)
    (yolo.py:44), the Detect rows of one page of the engine's workspace"""
    return 3 * ((net_h // 8) * (net_w // 8) + (net_h // 16) * (net_w // 16) + (net_h // 32) * (net_w // 32))


def _float_map(x, name, what, device_index, half=False):
    """x as a float32 numpy array or a float32 CUDA tensor on cuda:device_index (with half also float16), else
    ValueError"""
    if getattr(x, "is_cuda", None) is not None:   # a torch tensor
        ok = (_torch().float32, _torch().float16) if half else (_torch().float32,)
        if x.dtype not in ok:
            raise ValueError("%s%s must be %s, got %s%s" % (what, name, " or ".join(str(d)[6:] for d in ok), x.dtype,
                                                           "" if half else " (convert with .float())"))
        if not x.is_cuda:
            return x.detach().numpy()
        if device_index is not None and x.device.index != device_index:
            raise ValueError("%sa CUDA %s must be on cuda:%d, got %s" % (what, name, device_index, x.device))
        return x
    a = np.asarray(x)
    if a.dtype != np.float32 and not (half and a.dtype == np.float16):
        raise ValueError("%s%s must be %s, got %s" % (what, name, "float32 or float16" if half else "float32", a.dtype))
    return a


def check_outputs(blks, mask, lines_map, input_size, nc=2, device_index=None, what="", half=False):
    """The network outputs of one page as PostProcessor takes them -> (blks [A][5 + nc], mask [H][W], lines channel 0
    [H][W]), views of the caller's arrays or tensors (never copies), else ValueError naming `what` and the argument.
    blks: [1][A][5 + nc] or [A][5 + nc] with A <= workspace_rows(H, W); mask: [1][1][H][W], [1][H][W] or [H][W];
    lines_map: [1][C][H][W] or [C][H][W] with C >= 1, of which only channel 0 is read (db_utils.py:54); (H, W) =
    input_size; float32 numpy arrays or float32 CUDA tensors on cuda:device_index.  With half, all three may instead
    be float16 (numpy, CPU or CUDA tensors), never a mix within the page.  Needs no GPU."""
    net_h, net_w = input_size
    no = 5 + int(nc)
    b = _float_map(blks, "blks", what, device_index, half)
    m = _float_map(mask, "mask", what, device_index, half)
    ln = _float_map(lines_map, "lines_map", what, device_index, half)
    for name, x in (("mask", m), ("lines_map", ln)):
        if binding._is_f16(x) != binding._is_f16(b):
            raise ValueError("%s%s is %s but blks is %s: the three outputs of a page must share one dtype" % (
                what, name, x.dtype, b.dtype))
    bs, ms, ls = tuple(b.shape), tuple(m.shape), tuple(ln.shape)
    if len(bs) == 3 and bs[0] == 1:
        b = b[0]
    if b.ndim != 2 or b.shape[1] != no:
        raise ValueError("%sblks must be [1][A][%d] or [A][%d], got %s" % (what, no, no, bs))
    if b.shape[0] > workspace_rows(net_h, net_w):
        raise ValueError("%sblks has %d rows, more than the %d a %dx%d input has" % (
            what, b.shape[0], workspace_rows(net_h, net_w), net_h, net_w))
    while m.ndim > 2 and m.shape[0] == 1:
        m = m[0]
    if m.ndim != 2 or len(ms) > 4 or tuple(m.shape) != (net_h, net_w):
        raise ValueError("%smask must be [1][1][%d][%d], [1][%d][%d] or [%d][%d], got %s" % (
            what, net_h, net_w, net_h, net_w, net_h, net_w, ms))
    if len(ls) == 4 and ls[0] == 1:
        ln = ln[0]
    if ln.ndim != 3 or ln.shape[0] < 1 or tuple(ln.shape[1:]) != (net_h, net_w):
        raise ValueError("%slines_map must be [1][C][%d][%d] or [C][%d][%d] with C >= 1, got %s" % (
            what, net_h, net_w, net_h, net_w, ls))
    return b, m, ln[0]


def check_plan(shape, input_size, what=""):
    """ValueError naming `what` for a page ctd_pages_plan refuses at input_size (a side that letterboxes to 0 px).
    Needs no GPU."""
    try:
        binding.pages_plan([tuple(shape)], input_size[0], input_size[1])
    except CtdError:
        raise ValueError("%sa %dx%d page does not letterbox into a %dx%d input" % (
            what, shape[0], shape[1], input_size[0], input_size[1])) from None


_NONFINITE = re.compile(r"page (\d+) of the batch: (a non-finite value .*)")


class PostProcessor(KernelsOnlyJob):
    """`TextDetector.__call__` without its network, for many pages on cuda:device_index: the caller's
    `blks, mask, lines_map` in, `(mask, mask_refined, blk_list)` out.  input_size (an int or (h, w), multiples of 64)
    means what it means for `TextDetector`: the net input the outputs were computed on, the page letterboxed into it
    (`ctd_pages_plan`).  max_batch sizes the engine's workspace; nc, conf_thresh and nms_thresh are those of the
    reference's TextDetector and Detect head.  half: a page's outputs may also be float16 (all three of one page in
    one dtype); such a page is post-processed with the reference's arithmetic on half tensors, as its
    `TextDetector(half=True)` does on a float16 network's outputs (include/ctd_b200.h, ctd_submit_outputs_dtype)."""

    def __init__(self, input_size=1024, device_index=0, max_batch=16, nc=2, conf_thresh=0.4, nms_thresh=0.35,
                 half=False):
        if isinstance(input_size, int):
            input_size = (input_size, input_size)
        self.input_size = tuple(int(v) for v in input_size)
        if len(self.input_size) != 2 or any(v < 64 or v % 64 for v in self.input_size):
            raise ValueError("input_size must be positive multiples of 64, got %r" % (input_size,))
        self.nc = int(nc)
        self.conf_thresh, self.nms_thresh = conf_thresh, nms_thresh
        self.half = bool(half)
        super().__init__(device_index, max_batch, max_size=self.input_size, nc=self.nc, conf_thresh=conf_thresh,
                         nms_thresh=nms_thresh, skip_postproc=False)

    def __call__(self, img, blks, mask, lines_map, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False):
        """inference.py:148-178 for one page: (mask, mask_refined, blk_list), as `TextDetector(img)` returns them when
        its network gives (blks, mask, lines_map)"""
        return self.postprocess_batch([(img, blks, mask, lines_map)], refine_mode, keep_undetected_mask)[0]

    def postprocess_batch(self, items, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                          device_results=False):
        """list(postprocess_stream(...)), with every item checked before any GPU work"""
        items = list(items)
        for i, (img, blks, mask, lines_map) in enumerate(items):
            what = "item %d: " % i
            check_outputs(blks, mask, lines_map, self.input_size, self.nc, self.device_index, what, self.half)
            if not is_encoded(img):
                page = checked_page(img, what, self.device_index)
                check_plan(page.shape[:2], self.input_size, what)
        return list(self.postprocess_stream(items, refine_mode, keep_undetected_mask, textheight, device_results))

    def postprocess_stream(self, items, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                           device_results=False):
        """Generator over an iterable of (img, blks, mask, lines_map): yields for each item in input order what
        `TextDetector.detect_stream` yields for the page img when its network gives those outputs on the letterboxed
        page: `(mask, mask_refined, blk_list)`, with a textheight `(mask, mask_refined, blk_list, crops)`, and with
        device_results the masks and crops as CUDA tensors.

        img: a page as detect_stream takes it (u8 BGR numpy, a torch.uint8 CUDA tensor with any strides, or an encoded
        file).  blks, mask, lines_map: see check_outputs; float32 (with half also float16) numpy arrays or CUDA
        tensors on cuda:device_index with any strides (a slice `blks[i]` of a batched output is read where it is).  For CUDA
        pages and outputs an event is recorded on the device's current stream when the item is read, and the GPU
        waits for it before reading them; they are referenced until the item's batch is collected and must not be
        written before.

        A page or an output of the wrong type, dtype, shape or device, or a page that does not letterbox into
        input_size, raises ValueError naming the item before its batch reaches the GPU (an encoded page: once its batch
        is decoded).  A NaN or inf in an output fails its batch with a ValueError naming the item when the batch is
        collected."""
        th = 0
        if textheight is not None:
            th = _check_textheight(textheight)
            if th < 2:
                raise ValueError("textheight must be at least 2 px, got %r" % (textheight,))
        return self._stream(items, refine_mode, bool(keep_undetected_mask), th, bool(device_results))

    def _stream(self, items, refine_mode, keep, th, device_results):
        net_h, net_w = self.input_size

        def records():
            for idx, (img, blks, mask, lines_map) in enumerate(items):
                what = "item %d: " % idx
                outs = check_outputs(blks, mask, lines_map, self.input_size, self.nc, self.device_index, what, self.half)
                if is_encoded(img):
                    page = _Encoded(idx, img)   # decoded, and its plan checked, with its batch
                else:
                    page = checked_page(img, what, self.device_index)
                    check_plan(page.shape[:2], self.input_size, what)
                cuda = next((x for x in (page,) + outs if getattr(x, "is_cuda", False)), None)
                yield (idx, page, outs, _page_ready_event(cuda))

        def decoded(rec, page, what):
            check_plan(page.shape[:2], self.input_size, what)
            return (rec[0], page, rec[2], rec[3])

        def submit(slot, batch):
            self.net.submit_outputs(slot, [b[1] for b in batch], [b[2] for b in batch], net_h, net_w, refine_mode,
                                    keep, th, [b[3] for b in batch], device_results)
            return [b[0] for b in batch]

        def collect(slot, idxs, discard):
            try:
                pages = self.net.collect_pages(slot, discard=discard)
            except CtdError as ex:
                m = _NONFINITE.search(str(ex))
                if m is None:
                    raise
                raise ValueError("item %d: %s" % (idxs[int(m.group(1))], m.group(2))) from None
            if discard:
                return None
            return [(mask, mask_refined, blocks_from_records(rec, lines, dist)) + tuple(crops)
                    for mask, mask_refined, rec, lines, dist, *crops in pages]

        return self._pipeline(records(), lambda batch: self._decode(batch, decoded), submit, collect)
