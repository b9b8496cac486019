"""`TextBlock` records, the line -> block grouping of the drop-in detector and the text-line crops for OCR.

The grouping itself (`group_output`, reference utils/textblock.py:421-508 and its callees) is native code:
`ctd_group_output` in libctd_b200.so (csrc/group.cpp, declared in include/ctd_b200.h).  This module only converts
between the reference's python types -- the `(boxes, cls, conf)` tuple of `postprocess_yolo`, the int32 line quads,
the `TextBlock` objects callers of `TextDetector.__call__` receive (field names of utils/textblock.py:12-85) -- and the
flat C arrays of that call.

The crops (`get_transformed_region`, utils/textblock.py:162-194) are native too: `ctd_region_plan` (host C++,
csrc/region_plan.cpp) computes every line's output shape and cv2-identical homography, `ctd_transform_regions`
(csrc/region.cu) warps all of them out of the page in one GPU launch.
"""
import copy
import ctypes as C
import numbers
import threading

import numpy as np

from . import binding

LANG_LIST = ["eng", "ja", "unknown"]
LANGCLS2IDX = {"eng": 0, "ja": 1, "unknown": 2}


class TextBlock(object):
    """Result record with the reference's field names (textblock.py:12-85).  Of the reference class's helpers it has
    `get_transformed_region`, the per-line OCR crop (on the GPU); the UI helpers (min_rect, alignment, colours ...)
    are not part of it."""

    def __init__(self, xyxy, lines=None, language="unknown", vertical=False, font_size=-1, distance=None, angle=0,
                 vec=None, norm=-1, merged=False, weight=-1, text=None, translation="", fg_r=0, fg_g=0, fg_b=0,
                 bg_r=0, bg_g=0, bg_b=0, line_spacing=1., font_family="", bold=False, underline=False, italic=False,
                 alignment=-1, alpha=255, rich_text="", _bounding_rect=None, accumulate_color=True,
                 default_stroke_width=0.2, target_lang="", **kwargs):
        self.xyxy = [int(v) for v in xyxy]
        self.lines = [] if lines is None else lines
        self.vertical = vertical
        self.language = language
        self.font_size = font_size
        self.distance = None if distance is None else np.array(distance, np.float64)
        self.angle = angle
        self.vec = None if vec is None else np.array(vec, np.float64)
        self.norm = norm
        self.merged = merged
        self.weight = weight
        self.text = text if text is not None else []
        self.prob = 1
        self.translation = translation
        self.fg_r, self.fg_g, self.fg_b = fg_r, fg_g, fg_b
        self.bg_r, self.bg_g, self.bg_b = bg_r, bg_g, bg_b
        self.font_family = font_family
        self.bold, self.underline, self.italic = bold, underline, italic
        self.alpha = alpha
        self.rich_text = rich_text
        self.line_spacing = line_spacing
        self._alignment = alignment
        self._target_lang = target_lang
        self._bounding_rect = _bounding_rect
        self.default_stroke_width = default_stroke_width
        self.accumulate_color = accumulate_color

    def lines_array(self, dtype=np.float64):
        return np.array(self.lines, dtype=dtype)

    def __len__(self):
        return len(self.lines)

    def __getitem__(self, idx):
        return self.lines[idx]

    def to_dict(self):
        return copy.deepcopy(vars(self))

    def get_transformed_region(self, img, idx, textheight) -> np.ndarray:
        """Line `idx` cut out of `img` (u8 BGR [h][w][3]) straightened to `textheight` px, equal byte for byte to the
        reference's method (utils/textblock.py:162-194): horizontal lines come out textheight px high, vertical ones
        textheight px wide and rotated 90 degrees counter-clockwise.  Runs on a small kernels-only engine that is
        created on cuda:0 at the first call and kept for the process; every call uploads the whole page, so for
        several lines use `TextDetector.get_transformed_regions`, which crops all lines of a page in one launch.
        Raises CtdError where the reference raises (a line whose crop would be 1 px wide or high, a degenerate quad)."""
        eng, lock = _region_engine()
        with lock:
            return transformed_regions(eng, img, [self], textheight, line_index=idx)[0][0]


def blocks_from_records(blocks, lines, dist):
    """ctd_block records (+ the flat line / distance arrays they index) -> list of TextBlock.  The record fields are
    converted column-wise (one numpy call per field): indexing a structured array row by row costs ~1 us per field and
    was a third of the single-page latency of `TextDetector.__call__` at 256 blocks."""
    n = len(blocks)
    if n == 0:
        return []
    lo, nl = blocks["line_off"].tolist(), blocks["n_lines"].tolist()
    d0, nd = blocks["dist_off"].tolist(), blocks["n_dist"].tolist()
    fs, fif = blocks["font_size"].tolist(), blocks["font_is_float"].tolist()
    xy, lang = blocks["xyxy"].tolist(), blocks["language"].tolist()
    vert, ang, mrg = blocks["vertical"].tolist(), blocks["angle"].tolist(), blocks["merged"].tolist()
    vec = np.ascontiguousarray(blocks["vec"], np.float64)
    norm = np.ascontiguousarray(blocks["norm"], np.float64)
    weight = np.ascontiguousarray(blocks["weight"], np.float64)
    ll = np.asarray(lines).reshape(-1, 4, 2).tolist()     # every line quad as python ints, once
    dist = np.asarray(dist, np.float64)
    tpl = _template()
    out = []
    for i in range(n):
        # same attributes, in the same order, as TextBlock.__init__ would set (to_dict / the json writer depend on it)
        d = tpl.copy()
        d["xyxy"] = xy[i]
        d["lines"] = ll[lo[i]:lo[i] + nl[i]]
        d["vertical"] = bool(vert[i])
        d["language"] = LANG_LIST[lang[i]]
        d["font_size"] = float(fs[i]) if fif[i] else int(fs[i])
        d["distance"] = dist[d0[i]:d0[i] + nd[i]].copy()
        d["angle"] = int(ang[i])
        d["vec"] = vec[i].copy()
        d["norm"] = norm[i]
        d["merged"] = bool(mrg[i])
        d["weight"] = weight[i]
        d["text"] = []
        blk = TextBlock.__new__(TextBlock)
        blk.__dict__ = d
        out.append(blk)
    return out


_TEMPLATE = None


def _template():
    """attribute dict of a default TextBlock (insertion order = the order __init__ assigns them)"""
    global _TEMPLATE
    if _TEMPLATE is None:
        _TEMPLATE = dict(vars(TextBlock([0, 0, 0, 0], distance=[0.0], vec=[0.0, 0.0])))
    return _TEMPLATE


def group_output(blks, lines, im_w, im_h, mask=None, sort_blklist=True):
    """`group_output` (textblock.py:421-508) through the native library.  blks = (boxes int32 [n,4], cls int32 [n],
    conf f32 [n]); lines = int32 [m,4,2] (or []); mask = u8 page mask [im_h, im_w] or None."""
    lib = binding.load_library()
    boxes = np.ascontiguousarray(np.asarray(blks[0], np.int32).reshape(-1, 4))
    cls = np.ascontiguousarray(np.asarray(blks[1], np.int32).reshape(-1))
    ln = np.ascontiguousarray(np.asarray(lines, np.int32).reshape(-1, 4, 2))
    nb, nl = len(boxes), len(ln)
    if mask is not None:
        mask = np.ascontiguousarray(mask, np.uint8)
        assert mask.shape == (im_h, im_w), (mask.shape, im_h, im_w)
    cap_b, cap_l = nb + nl + 1, nb + nl + 1
    cap_d = cap_l * max(nl, 1) + 1
    rec = np.zeros((cap_b,), binding.BLOCK_DTYPE)
    lout = np.zeros((cap_l, 8), np.int32)
    dout = np.zeros((cap_d,), np.float64)
    n = C.c_int32()
    rc = lib.ctd_group_output(binding._ptr(boxes), binding._ptr(cls), nb, binding._ptr(ln), nl, int(im_w), int(im_h),
                              binding._ptr(mask), int(bool(sort_blklist)), binding._ptr(rec), cap_b, binding._ptr(lout),
                              cap_l, binding._ptr(dout), cap_d, C.byref(n))
    if rc != 0:
        raise binding.CtdError("ctd_group_output failed (%d)" % rc)
    return blocks_from_records(rec[:n.value], lout, dout)


_KERNELS_ONLY = {}   # nc -> the program with no ops
_REGION_ENGINE = None
_REGION_LOCK = threading.Lock()


def kernels_only_engine(device_index, max_batch, max_size=(64, 64), nc=2, conf_thresh=0.4, nms_thresh=0.35,
                        skip_postproc=True):
    """an engine on cuda:device_index that runs no network (the program has no ops): the stand-alone kernels and the
    batched jobs of caller blocks take it with the defaults (a 64x64 workspace, no post-processing workspaces in use).
    `PostProcessor` sizes it for max_batch pages of max_size (h, w) with skip_postproc=False, so NMS (nc classes,
    conf_thresh, nms_thresh), the DB tail and the result arena run on it.  The program is built once per process."""
    if nc not in _KERNELS_ONLY:
        from . import compiler
        P = compiler.Program()
        P.nc = int(nc)
        P.newbuf(8, 1)
        _KERNELS_ONLY[nc] = P
    return binding.Engine(_KERNELS_ONLY[nc], device=device_index, max_batch=max_batch, max_h=int(max_size[0]),
                          max_w=int(max_size[1]), conf_thresh=conf_thresh, nms_thresh=nms_thresh,
                          skip_postproc=skip_postproc)


def _region_engine():
    """the process-wide kernels-only engine behind TextBlock.get_transformed_region, created on device 0 at first use;
    its handle is not thread-safe, so calls hold the returned lock"""
    global _REGION_ENGINE
    with _REGION_LOCK:
        if _REGION_ENGINE is None:
            _REGION_ENGINE = kernels_only_engine(0, 1)
    return _REGION_ENGINE, _REGION_LOCK


def _check_textheight(textheight):
    if isinstance(textheight, numbers.Integral) and not isinstance(textheight, bool):
        return int(textheight)
    if isinstance(textheight, numbers.Real) and float(textheight).is_integer():
        return int(textheight)
    raise ValueError("textheight must be an integer number of pixels, got %r" % (textheight,))


def region_lines(blk_list, line_index=None):
    """REGION_LINE_DTYPE records for every line of every block (or line `line_index` of each), and (block, line) of
    each record"""
    keys = []
    for b, blk in enumerate(blk_list):
        for i in (range(len(blk.lines)) if line_index is None else [line_index]):
            keys.append((b, i))
    rec = np.zeros((len(keys),), binding.REGION_LINE_DTYPE)
    for r, (b, i) in zip(rec, keys):
        blk = blk_list[b]
        r["quad"] = np.asarray(blk.lines[i], np.float64).reshape(8)
        r["language"] = LANGCLS2IDX["eng"] if blk.language == "eng" else (
            LANGCLS2IDX["unknown"] if blk.language == "unknown" else LANGCLS2IDX["ja"])
        r["vertical"] = 1 if blk.vertical else 0
        r["font_size"] = float(blk.font_size)
    return rec, keys


def transformed_regions(engine, img, blk_list, textheight, line_index=None, page_shape=None):
    """Crops of every line of every block (or of line `line_index` of each block) as per-block lists of u8 arrays:
    one plan, one page upload, one launch, one copy back.  img: u8 [h][w][3] host array, or a device pointer (int)
    with page_shape = (h, w).  Raises CtdError, naming the block and the line, where the reference would raise; that
    check runs before any GPU work."""
    textheight = _check_textheight(textheight)
    if page_shape is None:
        img = np.ascontiguousarray(img)
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError("the page must be uint8 [h][w][3], got %s %s" % (img.dtype, img.shape))
        im_h, im_w = img.shape[:2]
    else:
        im_h, im_w = page_shape
    rec, keys = region_lines(blk_list, line_index)
    plan, total = binding.region_plan(rec, im_w, im_h, textheight)
    for (b, i), st in zip(keys, plan["status"].tolist()):
        if st != 0:
            why = "the reference raises on it (crop side of 1 px or a degenerate quad)" if st == 1 else \
                  "its crop has a side of %d px or more" % 32767
            raise binding.CtdError("block %d, line %d: no crop at textheight %d: %s" % (b, i, textheight, why))
    out = np.empty((total,), np.uint8)
    if len(plan):
        engine.transform_regions(img, plan, out=out, page_shape=page_shape)
    res = [[] for _ in blk_list]
    for (b, _i), r in zip(keys, plan):
        o, hh, ww = int(r["offset"]), int(r["out_h"]), int(r["out_w"])
        res[b].append(out[o:o + hh * ww * 3].reshape(hh, ww, 3))
    return res


def overlap_area(a, b):
    """`union_area` of the reference (imgproc_utils.py:13-20): the INTERSECTION area, -1 when disjoint."""
    x1, y1 = max(a[0], b[0]), max(a[1], b[1])
    x2, y2 = min(a[2], b[2]), min(a[3], b[3])
    if y2 < y1 or x2 < x1:
        return -1
    return (y2 - y1) * (x2 - x1)
