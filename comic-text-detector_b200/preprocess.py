"""The detector's pre-processing on the GPU: everything the reference's `TextDetector.__call__` does before
`self.net(img_in)`, i.e. `preprocess_img` (inference.py:72-83): the letterbox (cv2.resize INTER_LINEAR, bit-exact, zero
padding at the bottom and the right), the channel order, and `astype(float32) / 255` (or `.half()` of it), for many
pages in one launch (`ctd_preprocess_pages`), enqueued on the current torch stream with no host wait.

  * `preprocess_img(img, input_size, device, bgr2rgb, half, to_tensor)`: the reference's signature and return value,
    bit for bit, for one page: a drop-in for `from inference import preprocess_img`.
  * `Preprocessor.preprocess_batch(pages, ...)`: the same for many pages, into one [n][3][H][W] tensor.
  * `NetworkDetector(net, ...)`: `TextDetector.detect_stream` around a caller's network: this pre-processing, then
    `net(img_in)`, then `PostProcessor`, batch after batch, with no CPU work per page.
"""
import threading

import numpy as np

from .binding import PRE_F16_NCHW, PRE_F32_NCHW, PRE_U8_NHWC
from .inference import REFINEMASK_INPAINT, _Encoded, _torch, letterbox_geometry
from .jpeg import is_encoded
from .kernel_jobs import KernelsOnlyJob, checked_page
from .postprocess import PostProcessor, check_plan


def net_size(input_size):
    """input_size (an int or (h, w)) as (h, w), else ValueError: the sides must be positive multiples of 64"""
    size = (input_size, input_size) if isinstance(input_size, int) else tuple(input_size)
    if len(size) != 2 or any(not isinstance(v, (int, np.integer)) or v < 64 or v % 64 for v in size):
        raise ValueError("input_size must be positive multiples of 64, got %r" % (input_size,))
    return int(size[0]), int(size[1])


def upload_pages(pages, device_index):
    """the pages with every numpy page replaced by a CUDA copy on cuda:device_index: one pinned staging buffer and one
    host-to-device copy on the current stream for all of them (the pinned block is released to torch's host allocator,
    which keeps it until the copy ran); CUDA pages as they are"""
    torch = _torch()
    host = [i for i, p in enumerate(pages) if not getattr(p, "is_cuda", False)]
    if not host:
        return list(pages)
    offs = [0]
    for i in host:
        offs.append(offs[-1] + (pages[i].size + 255) // 256 * 256)
    pinned = torch.empty((offs[-1],), dtype=torch.uint8, pin_memory=True)
    buf = pinned.numpy()
    for i, o in zip(host, offs):
        np.copyto(buf[o:o + pages[i].size].reshape(pages[i].shape), pages[i])
    dev = pinned.to(torch.device("cuda", device_index), non_blocking=True)
    out = list(pages)
    for i, o in zip(host, offs):
        out[i] = dev[o:o + pages[i].size].view(pages[i].shape)
    return out


class Preprocessor(KernelsOnlyJob):
    """`preprocess_img` for many pages on cuda:device_index: input_size (an int or (h, w), multiples of 64) is the net
    input the pages are letterboxed into, max_batch the pages of one launch (a batch of more pages takes several)."""

    def __init__(self, input_size=1024, device_index=0, max_batch=16):
        self.input_size = net_size(input_size)
        super().__init__(device_index, max_batch)

    def preprocess_batch(self, pages, bgr2rgb=True, half=False, to_tensor=True):
        """-> (img_in, ratios, dws, dhs): what `preprocess_img(page, input_size, bgr2rgb=bgr2rgb, half=half,
        to_tensor=to_tensor)` returns for each page, the tensors stacked.  img_in is a fresh CUDA tensor:
        [n][3][H][W] float32 (float16 with half), or with to_tensor=False the letterboxed u8 pixels [n][H][W][3] in
        the order preprocess_img gives them; ratios[i] = (r, r), dws[i] and dhs[i] the padding, as Python numbers.

        pages: u8 BGR [h][w][3] numpy arrays, torch.uint8 CUDA tensors [h][w][3] on cuda:device_index with any strides
        (read in place), or encoded files (JPEG / PNG bytes or paths, decoded as detect_stream decodes them).  The
        work is enqueued on the current stream of the device, like any torch op; the CUDA pages are marked as used on
        it (record_stream).  A page of the wrong type, dtype, shape or device, or one that does not letterbox into
        input_size, raises ValueError naming the item before any GPU work (an encoded page: once it is decoded)."""
        pages = self.pages_on_device(list(enumerate(pages)))
        return self.run(pages, bgr2rgb, half, to_tensor)

    def pages_on_device(self, items):
        """(index, page) items -> the pages as CUDA tensors on cuda:device_index: numpy pages uploaded once
        (upload_pages), encoded ones decoded; ValueError naming the index for a page that is not one, before any GPU
        work (an encoded page: once it is decoded)"""
        recs = []
        for idx, page in items:
            what = "item %d: " % idx
            if is_encoded(page):
                recs.append((idx, _Encoded(idx, page)))
            else:
                page = checked_page(page, what, self.device_index)
                check_plan(page.shape[:2], self.input_size, what)
                recs.append((idx, page))

        def decoded(rec, page, what):
            check_plan(page.shape[:2], self.input_size, what)
            return (rec[0], page)

        recs = self._decode(recs, decoded)
        return upload_pages([r[1] for r in recs], self.device_index)

    def run(self, pages, bgr2rgb=True, half=False, to_tensor=True):
        """preprocess_batch on pages that are checked CUDA tensors of this device"""
        torch = _torch()
        net_h, net_w = self.input_size
        dev = torch.device("cuda", self.device_index)
        stream = torch.cuda.current_stream(dev)
        n = len(pages)
        if to_tensor:
            fmt = PRE_F16_NCHW if half else PRE_F32_NCHW
            out = torch.empty((n, 3, net_h, net_w), dtype=torch.float16 if half else torch.float32, device=dev)
            reverse = not bgr2rgb   # cvtColor then transpose(...)[::-1]: the page's order with bgr2rgb
        else:
            fmt = PRE_U8_NHWC
            out = torch.empty((n, net_h, net_w, 3), dtype=torch.uint8, device=dev)
            reverse = bool(bgr2rgb)
        page_bytes = 3 * net_h * net_w * out.element_size()
        for a in range(0, n, self.max_batch):
            batch = pages[a:a + self.max_batch]
            for p in batch:
                p.record_stream(stream)
            self.net.preprocess_pages(batch, net_h, net_w, fmt, reverse, out.data_ptr() + a * page_bytes,
                                      stream.cuda_stream)
        geo = [letterbox_geometry(p.shape[:2], self.input_size) for p in pages]
        return out, [(g[0], g[0]) for g in geo], [g[2] for g in geo], [g[3] for g in geo]


_PREPROCESSORS = {}   # (device index, input size) -> the Preprocessor behind preprocess_img
_PREPROCESSORS_LOCK = threading.Lock()


def preprocess_img(img, input_size=(1024, 1024), device='cuda', bgr2rgb=True, half=False, to_tensor=True):
    """The reference's `preprocess_img` (inference.py:72-83) on the GPU, bit for bit: -> (img_in, ratio, dw, dh) with
    img_in a float32 (float16 with half) [1][3][H][W] CUDA tensor on `device`, or with to_tensor=False the letterboxed
    u8 [H][W][3] page as numpy, ratio = (r, r), dw and dh ints.  img: a page as Preprocessor takes it.  `device` must
    be a CUDA device (there is no CPU fallback: anything else raises ValueError).  Runs on a Preprocessor per device
    and input size, created at the first call and kept for the process."""
    torch = _torch()
    size = net_size(input_size)
    dev = torch.device(device)
    if dev.type != 'cuda':
        raise ValueError("preprocess_img runs on a CUDA device (there is no CPU fallback), got %s" % (device,))
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), size)
    with _PREPROCESSORS_LOCK:
        pre = _PREPROCESSORS.get(key)
        if pre is None:
            pre = _PREPROCESSORS[key] = Preprocessor(size, key[0], max_batch=1)
        img_in, ratios, dws, dhs = pre.preprocess_batch([img], bgr2rgb, half, to_tensor)
    if not to_tensor:
        img_in = img_in[0].cpu().numpy()
    return img_in, ratios[0], dws[0], dhs[0]


class NetworkDetector:
    """`TextDetector` around a caller's network: `net(img_in) -> (blks, mask, lines_map)` is any callable on the
    float32 BGR tensor preprocess_img makes ([n][3][H][W], n <= max_batch), e.g. this engine's `TextDetBase`, a
    torch module, a TensorRT engine or a `torch.compile`d model, whose outputs are those of the reference's network
    (float32; see PostProcessor).  Each page's result is byte for byte what the reference's `TextDetector.__call__`
    returns when its `self.net` is `net`.

    It composes a `Preprocessor` and a `PostProcessor` on cuda:device_index for max_batch pages of input_size (nc,
    conf_thresh and nms_thresh as for PostProcessor): per batch one pre-processing launch and one `net` call on the
    current stream, then the batch goes to the post-processing, which keeps two batches in flight, so batch k + 1's
    pre-processing and network are enqueued while batch k is post-processed.  Each page is uploaded or decoded once,
    and both stages read that CUDA page.

    half: the reference's `TextDetector(half=True)` for a float16 network (a `.half()` module, a TensorRT fp16
    engine, `TextDetBase(half=True)`): `net` gets the float16 tensor `preprocess_img(half=True)` makes, and float16
    outputs are post-processed with the reference's half arithmetic (PostProcessor(half=True))."""

    def __init__(self, net, input_size=1024, device_index=0, max_batch=16, nc=2, conf_thresh=0.4, nms_thresh=0.35,
                 half=False):
        self.net = net
        self.half = bool(half)
        self.pre = Preprocessor(input_size, device_index, max_batch)
        self.post = PostProcessor(self.pre.input_size, device_index, max_batch, nc, conf_thresh, nms_thresh,
                                  half=self.half)
        self.input_size = self.pre.input_size
        self.device_index = self.pre.device_index
        self.max_batch = self.pre.max_batch

    def close(self):
        self.pre.close()
        self.post.close()

    def __call__(self, img, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False):
        """(mask, mask_refined, blk_list) of one page, as the reference's `TextDetector(img)` returns them"""
        return self.detect_batch([img], refine_mode, keep_undetected_mask)[0]

    def detect_batch(self, imgs, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                     device_results=False):
        """list(detect_stream(...)), with every page that is not an encoded file checked before any GPU work"""
        imgs = list(imgs)
        for i, img in enumerate(imgs):
            if not is_encoded(img):
                what = "item %d: " % i
                check_plan(checked_page(img, what, self.device_index).shape[:2], self.input_size, what)
        return list(self.detect_stream(imgs, refine_mode, keep_undetected_mask, textheight, device_results))

    def detect_stream(self, imgs, refine_mode=REFINEMASK_INPAINT, keep_undetected_mask=False, textheight=None,
                      device_results=False):
        """Generator over an iterable of pages: yields for each page in input order what `TextDetector.detect_stream`
        yields, `(mask, mask_refined, blk_list)` (with a textheight also the crops, with device_results the masks and
        crops as CUDA tensors), computed from `net`'s outputs.  Pages in every form detect_stream takes (numpy, CUDA
        tensors with any strides, encoded files); a bad page raises ValueError naming its index before its batch
        reaches the GPU."""
        return self.post.postprocess_stream(self._items(imgs), refine_mode, keep_undetected_mask, textheight,
                                            device_results)

    def _items(self, imgs):
        """(page, blks, mask, lines_map) per page: the pages of each batch of max_batch on the device, pre-processed
        in one launch and run through net"""
        def run(batch):
            pages = self.pre.pages_on_device(batch)
            img_in = self.pre.run(pages, half=self.half)[0]
            blks, mask, lines_map = self.net(img_in)
            for i, page in enumerate(pages):
                yield page, blks[i], mask[i], lines_map[i]

        batch = []
        for item in enumerate(imgs):
            batch.append(item)
            if len(batch) == self.max_batch:
                yield from run(batch)
                batch = []
        if batch:
            yield from run(batch)
