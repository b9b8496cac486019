"""Drop-in `TextDetector` over the H100 engine.

Same constructor and call signature as the reference's `inference.TextDetector`
(inference.py:116-178): `TextDetector(model_path, input_size=1024, device=..., half=False, nms_thresh=0.35,
conf_thresh=0.4, mask_thresh=0.3, act='leaky')` and
`detector(img, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False) -> (mask, mask_refined, blk_list)`.
A `.onnx` model_path is read as the reference's OpenCV-DNN backend reads it (onnx_model.py): same engine, same calls.
`detect_batch` / `detect_stream` give the same results for many pages of any sizes, batched on the GPU, and with a
`textheight` also the OCR crops of every text line (`get_transformed_regions`), cut in the same batches; their pages may
be torch.uint8 CUDA tensors or encoded files (JPEGs and PNGs decoded on the GPU, jpeg.py, png.py), and with `device_results=True` the
masks and crops come back as CUDA tensors.

Everything runs in libctd_b200.so: network, NMS, mask u8, DB binarize, connected components, contour boxes + scores,
refine_mask on the GPU; ratio scaling, `group_output` and the window expansion in host C++ (csrc/group.cpp,
csrc/pipeline.cu).  This module is the reference-shaped Python surface over `ctd_detect_page` and, for batches,
`ctd_submit_pages`.
"""
from pathlib import Path
from typing import List

import numpy as np

from . import compiler, onnx_model
from .binding import Engine, PREC_FP16_TC, PREC_FP32_SIMT
from .jpeg import is_encoded
from .kernel_jobs import BatchJob, _Encoded, _page_ready_event, check_page
from .textblock import (TextBlock, blocks_from_records, check_textheight, group_output, overlap_area,  # noqa: F401
                        transformed_regions)

REFINEMASK_INPAINT = 0
REFINEMASK_ANNOTATION = 1


def letterbox_geometry(shape_hw, new_shape=(1024, 1024)):
    """The size arithmetic of `letterbox(im, new_shape, auto=False)` (utils/imgproc_utils.py:86-117): aspect-preserving
    scale r, resized size (w, h) = round(size * r) (Python's round), bottom/right padding (dw, dh)."""
    r = min(new_shape[0] / shape_hw[0], new_shape[1] / shape_hw[1])
    new_unpad = int(round(shape_hw[1] * r)), int(round(shape_hw[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    return r, new_unpad, int(dw), int(dh)


def letterbox(im, new_shape=(1024, 1024)):
    """Host restatement of the reference's `letterbox` (kept for tests / tools; the detector itself letterboxes on the
    GPU inside `ctd_detect_page` and `ctd_submit_pages`, bit-exact with cv2.INTER_LINEAR)."""
    r, new_unpad, dw, dh = letterbox_geometry(im.shape[:2], new_shape)
    if im.shape[:2][::-1] != new_unpad:
        import cv2
        im = cv2.resize(im, new_unpad, interpolation=cv2.INTER_LINEAR)
    if dw or dh:
        padded = np.zeros((new_shape[0], new_shape[1], 3), np.uint8)
        padded[:im.shape[0], :im.shape[1]] = im
        im = padded
    return im, (r, r), (dw, dh)


class TextDetector(BatchJob):
    lang_list = ['eng', 'ja', 'unknown']
    langcls2idx = {'eng': 0, 'ja': 1, 'unknown': 2}
    item = "page"   # an undecodable page of detect_stream is "page <index>"

    def __init__(self, model_path, input_size=1024, device='cuda', half=False, nms_thresh=0.35, conf_thresh=0.4,
                 mask_thresh=0.3, act='leaky', precision=None, device_index=0, max_batch=1):
        if isinstance(input_size, int):
            input_size = (input_size, input_size)
        if isinstance(model_path, (str, Path)) and Path(model_path).suffix == '.onnx':
            # the reference's OpenCV-DNN backend (inference.py:124-130): the activation comes from the graph, `act` is
            # ignored as there, and the network sees RGB (onnx_model.py reverses the stem's input channels)
            ckpt, act, net_size = onnx_model.load_checkpoint(str(model_path))
            if tuple(input_size) != (net_size, net_size):
                raise ValueError("%s was exported for %d x %d input, input_size is %s"
                                 % (model_path, net_size, net_size, tuple(input_size)))
        elif isinstance(model_path, (str, Path)):
            import torch
            ckpt = torch.load(str(model_path), map_location='cpu')  # reference basemodel.py:212
        else:
            ckpt = model_path  # already a checkpoint dict
        self.input_size = input_size
        self.device = device
        self.half = half
        self.conf_thresh = conf_thresh
        self.nms_thresh = nms_thresh
        self.backend = 'b200'
        if precision is None:
            precision = PREC_FP16_TC
        self.program = compiler.compile_checkpoint(ckpt, head_act=act)
        # DB threshold is hard-coded 0.3 in the reference (inference.py:139 ignores mask_thresh)
        # max_batch: pages per GPU batch of detect_batch / detect_stream (the workspace is sized for it)
        super().__init__(Engine(self.program, device=device_index, precision=precision, max_batch=int(max_batch),
                                max_h=input_size[0], max_w=input_size[1], conf_thresh=conf_thresh,
                                nms_thresh=nms_thresh, db_thresh=0.3), device_index, max_batch)

    def __call__(self, img, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False):
        """reference inference.py:141-178.  One native call (`ctd_detect_page`): letterbox (cv2-exact INTER_LINEAR) +
        network + NMS + mask u8 + DB boxes on the GPU, postprocess_yolo casts / box_thresh / group_output on the host
        in C++, refine_mask (and refine_undetected_mask) on the GPU with the page and its mask resident in HBM; this
        method only turns the block records into `TextBlock` objects."""
        img = np.ascontiguousarray(img)
        mask, mask_refined, rec, lines, dist = self.net.detect_page(img, self.input_size[0], self.input_size[1], refine_mode,
                                                                    keep_undetected_mask)
        return mask, mask_refined, blocks_from_records(rec, lines, dist)

    def get_transformed_regions(self, img, blk_list, textheight):
        """The OCR crops of every line of every block: per block, a list of u8 arrays in line order, each equal byte
        for byte to the reference's `blk.get_transformed_region(img, idx, textheight)` (utils/textblock.py:162-194).
        One host plan (csrc/region_plan.cpp), one page upload, one GPU launch and one copy back for the whole page,
        on this detector's engine.  img: u8 BGR [h][w][3], the page `blk_list` was detected on.  Raises CtdError,
        naming the block and the line, before any GPU work if the reference would raise on a line."""
        return transformed_regions(self.net, img, blk_list, textheight)

    def detect_batch(self, imgs, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                     device_results=False):
        """`[self(img, refine_mode, keep_undetected_mask) for img in imgs]`, with the same results byte for byte, computed
        in GPU batches of up to `max_batch` pages of any sizes (see detect_stream, which also describes CUDA-tensor
        pages and device_results).  Every page is checked before any GPU work: a page that is not u8 [h][w][3], or a
        CUDA tensor on another device, raises ValueError.  An encoded page (see detect_stream) is decoded with its
        batch; one cv2 cannot decode raises ValueError then.  With a textheight, each result is the 4-tuple
        detect_stream yields, crops included."""
        imgs = [img if is_encoded(img) else check_page(img, self.device_index) for img in imgs]
        return list(self.detect_stream(imgs, refine_mode, keep_undetected_mask, textheight, device_results))

    def detect_stream(self, imgs, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                      device_results=False):
        """Generator over an iterable of pages: yields `(mask, mask_refined, blk_list)` for each page in input order,
        equal to `self(img, refine_mode, keep_undetected_mask)`.  Pages are grouped into batches of up to `max_batch`
        and two batches are kept in flight (`ctd_submit_pages`): while one batch runs on the GPU and in the engine's
        host stage, the next one is read from `imgs` and packed.  A page that is not u8 [h][w][3] raises ValueError
        before it reaches the GPU.

        A page may also be a torch.uint8 CUDA tensor [h][w][3], BGR, on cuda:device_index, with any strides (a crop
        `big[y0:y1, x0:x1]`, `chw.permute(1, 2, 0)`): it is read on the GPU where it is, without a copy through the
        host, and one batch may mix such pages with numpy pages.  When the page is read from `imgs`, an event is
        recorded on the current torch stream of its device, and the engine waits for it before reading the page, so
        a page written by work still queued on that stream is read correctly.  The stream keeps a reference to the
        tensor until its batch is collected; do not write into it before its result has been yielded.  The results
        are the same as for `page.cpu().numpy()`.

        A page may also be an encoded file, read as the reference's `io_utils.imread` reads it, i.e. as
        `cv2.imdecode(buf, cv2.IMREAD_COLOR)`: bytes, bytearray, memoryview or a 1-D np.uint8 array of the file, or a
        str / os.PathLike path, read with np.fromfile.  The encoded pages of a batch are decoded right before the batch
        is submitted, in one `PngDecoder.decode` call for the files with the PNG signature and one `JpegDecoder.decode`
        call for the others: baseline JPEGs and the PNGs the GPU takes on the GPU into CUDA pages (which then enter as
        CUDA-tensor pages do), every other file by cv2 on the host into a numpy page.  The results are
        byte for byte those for the `cv2.imdecode` pages of the same files.  A file cv2 cannot decode raises ValueError
        naming its index in `imgs` (and its path), when its batch is decoded.

        textheight (an integer >= 2; checked here, before any page is read): yields `(mask, mask_refined, blk_list,
        crops)` instead, where crops[b][i] is line i of blk_list[b] cut out as `get_transformed_regions(img, blk_list,
        textheight)` cuts it, byte for byte, except that a line on which the reference's `get_transformed_region`
        raises (a crop side of 1 px, a degenerate quad; or a side of 32767 px or more) gets None instead of raising,
        so one such line does not end the stream.  The crops are planned on the engine's worker threads and cut in
        one GPU launch per batch from the pages already in device memory (`ctd_submit_pages`).  Each page's
        crops are views into one array of that page's own.

        device_results=True: mask, mask_refined and every crop are torch.uint8 CUDA tensors on cuda:device_index
        ([ih][iw], [ih][iw], [h][w][3]; None where the numpy stream gives None), byte for byte what the numpy stream
        gives, never copied to the host; blk_list stays the host TextBlock list.  A page's tensors are views into one
        allocation of that page's own, complete when yielded, and marked as used on the current stream; like any
        tensor made on another stream, call `record_stream` before using one on a different stream."""
        th = 0 if textheight is None else check_textheight(textheight)
        net_h, net_w = self.input_size

        def records():
            for idx, img in enumerate(imgs):
                # an encoded page is decoded with its batch
                page = _Encoded(idx, img) if is_encoded(img) else check_page(img, self.device_index)
                yield (idx, page, _page_ready_event(page))

        def submit(slot, batch):
            self.net.submit_pages(slot, [b[1] for b in batch], net_h, net_w, refine_mode, keep_undetected_mask, th,
                                  [b[2] for b in batch], bool(device_results))

        def collect(slot, _token, discard):
            pages = self.net.collect_pages(slot, discard=discard)
            if discard:
                return None
            return [(mask, mask_refined, blocks_from_records(rec, lines, dist)) + tuple(crops)
                    for mask, mask_refined, rec, lines, dist, *crops in pages]

        decoded = lambda rec, page, what: (rec[0], page, rec[2])
        return self._pipeline(records(), lambda batch: self._decode(batch, decoded), submit, collect)
