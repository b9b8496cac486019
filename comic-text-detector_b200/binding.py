"""ctypes binding of libctd_b200.so (include/ctd_b200.h).  Thin: numpy arrays in/out, every
non-zero return code becomes a Python exception carrying ctd_last_error().  There is no CPU
fallback: if the library is missing or no sm_90 GPU is visible, construction raises."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctd_b200.so")
MAX_SRC = 3
ABI_VERSION = 3
PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC = 0, 1, 2, 3


class CtdOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_src", C.c_int32), ("src_buf", C.c_int32 * MAX_SRC),
                ("src_coff", C.c_int32 * MAX_SRC), ("src_c", C.c_int32 * MAX_SRC), ("dst_buf", C.c_int32),
                ("dst_coff", C.c_int32), ("cout", C.c_int32), ("cout_pad", C.c_int32), ("ksize", C.c_int32),
                ("stride", C.c_int32), ("act", C.c_int32), ("residual", C.c_int32), ("aux", C.c_int32),
                ("w16_off", C.c_int64), ("w32_off", C.c_int64), ("b_off", C.c_int64), ("p_off", C.c_int64)]


class CtdBufDesc(C.Structure):
    _fields_ = [("channels", C.c_int32), ("down", C.c_int32)]


class CtdConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("precision", C.c_int32), ("max_batch", C.c_int32),
                ("max_h", C.c_int32), ("max_w", C.c_int32), ("nc", C.c_int32), ("use_graph", C.c_int32),
                ("conf_thresh", C.c_float), ("nms_thresh", C.c_float), ("db_thresh", C.c_float),
                ("debug_skip_postproc", C.c_int32)]


# numpy mirror of `ctd_block` (include/ctd_b200.h)
BLOCK_DTYPE = np.dtype([("xyxy", np.int32, (4,)), ("language", np.int32), ("vertical", np.int32), ("angle", np.int32),
                        ("merged", np.int32), ("n_lines", np.int32), ("line_off", np.int32), ("n_dist", np.int32),
                        ("dist_off", np.int32), ("font_is_float", np.int32), ("reserved", np.int32),
                        ("font_size", np.float64), ("vec", np.float64, (2,)), ("norm", np.float64),
                        ("weight", np.float64)], align=True)

class CtdResultsLayout(C.Structure):
    _fields_ = [("max_batch", C.c_int32), ("max_h", C.c_int32), ("max_w", C.c_int32), ("reserved", C.c_int32)] + \
               [(k, C.c_size_t) for k in ("total_bytes", "phase_a_bytes", "mask_u8", "det", "det_count", "n_labels",
                                          "line_boxes", "line_scores", "line_count", "mask_refined", "blocks",
                                          "blocks_stride", "blk_records_off", "blk_lines_off", "blk_dist_off")]


MAX_BLOCKS, MAX_BLOCK_DIST = 1300, 8192   # CTD_MAX_BLOCKS / CTD_MAX_BLOCK_DIST

# numpy mirror of `ctd_page_entry` (include/ctd_b200.h)
PAGE_ENTRY_DTYPE = np.dtype([("ih", np.int32), ("iw", np.int32), ("unpad_h", np.int32), ("unpad_w", np.int32),
                             ("page_off", np.int64), ("mask_off", np.int64), ("refined_off", np.int64),
                             ("blocks_off", np.int64)], align=True)

# numpy mirrors of `ctd_region_line` / `ctd_region` (include/ctd_b200.h)
REGION_LINE_DTYPE = np.dtype([("quad", np.float64, (8,)), ("language", np.int32), ("vertical", np.int32),
                              ("font_size", np.float64)], align=True)
REGION_DTYPE = np.dtype([("out_h", np.int32), ("out_w", np.int32), ("rotate", np.int32), ("status", np.int32),
                         ("offset", np.int64), ("homography", np.float64, (9,)), ("inverse", np.float64, (9,))],
                        align=True)


class CtdJpegInfo(C.Structure):
    """ctypes mirror of `ctd_jpeg_info` (include/ctd_b200.h)"""
    _fields_ = [(k, C.c_int32) for k in ("status", "height", "width", "frame_height", "frame_width", "components",
                                         "h_samp", "v_samp", "orientation", "restart_interval")] + \
               [("ecs_bytes", C.c_int64)]


class CtdPngInfo(C.Structure):
    """ctypes mirror of `ctd_png_info` (include/ctd_b200.h)"""
    _fields_ = [(k, C.c_int32) for k in ("status", "height", "width", "image_height", "image_width", "bit_depth",
                                         "color_type", "orientation", "palette_entries")] + [("zlib_bytes", C.c_int64)]


class CtdPngImage(C.Structure):
    """ctypes mirror of `ctd_png_image` (include/ctd_b200.h)"""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32),
                ("bit_depth", C.c_int32), ("on_device", C.c_int32), ("stride_h", C.c_int64), ("stride_w", C.c_int64),
                ("stride_c", C.c_int64), ("event", C.c_void_p)]


class CtdDevicePage(C.Structure):
    """ctypes mirror of `ctd_device_page` (include/ctd_b200.h)"""
    _fields_ = [("data", C.c_void_p), ("stride_h", C.c_int64), ("stride_w", C.c_int64), ("stride_c", C.c_int64),
                ("event", C.c_void_p)]


class CtdNetOutput(C.Structure):
    """ctypes mirror of `ctd_net_output` (include/ctd_b200.h)"""
    _fields_ = [("blks", C.c_void_p), ("blks_stride_r", C.c_int64), ("blks_stride_c", C.c_int64),
                ("mask", C.c_void_p), ("mask_stride_h", C.c_int64), ("mask_stride_w", C.c_int64),
                ("lines", C.c_void_p), ("lines_stride_h", C.c_int64), ("lines_stride_w", C.c_int64),
                ("rows", C.c_int32), ("blks_on_device", C.c_int32), ("mask_on_device", C.c_int32),
                ("lines_on_device", C.c_int32), ("event", C.c_void_p)]


EXPORTS = ["ctd_create", "ctd_destroy", "ctd_last_error", "ctd_forward", "ctd_get_net_outputs", "ctd_get_mask_u8",
           "ctd_get_detections", "ctd_get_db_components", "ctd_last_forward_ms", "ctd_last_launch_count",
           "ctd_debug_read_buffer", "ctd_debug_write_buffer", "ctd_connected_components", "ctd_nms",
           "ctd_timer_start", "ctd_timer_stop", "ctd_profile_forward", "ctd_get_text_lines", "ctd_seg_represent",
           "ctd_refine_mask", "ctd_collect", "ctd_join", "ctd_resize_linear_u8", "ctd_debug_run_ops",
           "ctd_get_nms_status", "ctd_group_output", "ctd_detect_page", "ctd_results_layout", "ctd_submit_full",
           "ctd_device_arena", "ctd_region_plan", "ctd_transform_regions", "ctd_pages_plan", "ctd_submit_pages",
           "ctd_collect_regions", "ctd_collect_device", "ctd_forward_tensor", "ctd_jpeg_probe",
           "ctd_jpeg_decoder_create", "ctd_jpeg_decoder_destroy", "ctd_jpeg_decode", "ctd_debug_postprocess",
           "ctd_png_encoder_create", "ctd_png_encoder_destroy", "ctd_png_encode", "ctd_png_probe",
           "ctd_png_decoder_create", "ctd_png_decoder_destroy", "ctd_png_decode", "ctd_png_decoder_stats",
           "ctd_refine_plan", "ctd_submit_refine", "ctd_submit_regions", "ctd_debug_read_slot", "ctd_submit_outputs",
           "ctd_preprocess_pages", "ctd_submit_outputs_dtype", "ctd_forward_tensor_f16"]
PRE_F32_NCHW, PRE_F16_NCHW, PRE_U8_NHWC = 0, 1, 2   # ctd_pre_format
DTYPE_F32, DTYPE_F16 = 0, 1   # ctd_dtype

_lib = None


class CtdError(RuntimeError):
    pass


def _is_f16(m):
    """a float16 numpy array or torch tensor"""
    return str(m.dtype) in ("float16", "torch.float16")


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise CtdError("libctd_b200.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "-- there is no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32 = C.c_void_p, C.c_int32
    lib.ctd_create.argtypes = [C.POINTER(vp), C.POINTER(CtdConfig), C.POINTER(CtdOp), i32, C.POINTER(CtdBufDesc), i32,
                               vp, C.c_size_t]
    lib.ctd_create.restype = C.c_int
    lib.ctd_destroy.argtypes = [vp]
    lib.ctd_destroy.restype = None
    lib.ctd_last_error.argtypes = [vp]
    lib.ctd_last_error.restype = C.c_char_p
    lib.ctd_forward.argtypes = [vp, vp, i32, i32, i32, i32]
    lib.ctd_get_net_outputs.argtypes = [vp, vp, vp, vp]
    lib.ctd_forward_tensor.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
    lib.ctd_forward_tensor_f16.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
    lib.ctd_get_mask_u8.argtypes = [vp, vp]
    lib.ctd_get_detections.argtypes = [vp, vp, vp]
    lib.ctd_get_db_components.argtypes = [vp, vp, vp, vp]
    lib.ctd_last_forward_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.ctd_last_launch_count.argtypes = [vp, C.POINTER(i32)]
    lib.ctd_debug_read_buffer.argtypes = [vp, i32, vp, C.c_size_t]
    lib.ctd_debug_write_buffer.argtypes = [vp, i32, vp, i32, i32, i32]
    lib.ctd_connected_components.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp]
    lib.ctd_nms.argtypes = [vp, vp, i32, C.c_float, C.c_float, vp, vp]
    lib.ctd_get_text_lines.argtypes = [vp, vp, vp, vp]
    lib.ctd_seg_represent.argtypes = [vp, vp, i32, i32, C.c_float, vp, vp, vp]
    lib.ctd_refine_mask.argtypes = [vp, vp, vp, i32, i32, vp, i32, i32, vp]
    lib.ctd_timer_start.argtypes = [vp]
    lib.ctd_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    lib.ctd_profile_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, i32]
    lib.ctd_collect.argtypes = [vp, i32]
    lib.ctd_join.argtypes = [vp, vp]
    lib.ctd_resize_linear_u8.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32]
    lib.ctd_debug_run_ops.argtypes = [vp, vp, i32, i32, i32, i32, i32]
    lib.ctd_debug_postprocess.argtypes = [vp, vp, vp, i32, i32, i32]
    lib.ctd_get_nms_status.argtypes = [vp, vp, C.POINTER(i32)]
    lib.ctd_group_output.argtypes = [vp, vp, i32, vp, i32, i32, i32, vp, i32, vp, i32, vp, i32, vp, i32, C.POINTER(i32)]
    lib.ctd_detect_page.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, i32, vp, i32, vp, i32, C.POINTER(i32)]
    lib.ctd_results_layout.argtypes = [vp, C.POINTER(CtdResultsLayout)]
    lib.ctd_submit_full.argtypes = [vp, i32, vp, i32, i32, i32, i32, i32, vp]
    lib.ctd_device_arena.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(vp)]
    lib.ctd_region_plan.argtypes = [vp, i32, i32, i32, i32, vp, C.POINTER(C.c_size_t)]
    lib.ctd_transform_regions.argtypes = [vp, vp, i32, i32, i32, vp, i32, vp, C.c_size_t]
    lib.ctd_pages_plan.argtypes = [vp, i32, i32, i32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.ctd_submit_pages.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp, i32, i32, i32, i32, vp]
    lib.ctd_collect_regions.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(i32), C.POINTER(vp), C.POINTER(vp),
                                        C.POINTER(C.c_size_t)]
    lib.ctd_collect_device.argtypes = [vp, i32, vp]
    lib.ctd_refine_plan.argtypes = [vp, i32, vp, vp, vp, vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.ctd_submit_refine.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.ctd_submit_regions.argtypes = [vp, i32, vp, i32, vp, vp, i32, vp, vp, i32]
    lib.ctd_debug_read_slot.argtypes = [vp, i32, i32, C.c_size_t, vp, C.c_size_t]
    lib.ctd_submit_outputs.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.ctd_submit_outputs_dtype.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.ctd_preprocess_pages.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i32, vp, vp]
    lib.ctd_jpeg_probe.argtypes = [vp, C.c_size_t, C.POINTER(CtdJpegInfo)]
    lib.ctd_jpeg_decoder_create.argtypes = [i32, i32, C.POINTER(vp)]
    lib.ctd_jpeg_decoder_destroy.argtypes = [vp]
    lib.ctd_jpeg_decode.argtypes = [vp, vp, vp, i32, vp, vp]
    for name in EXPORTS[3:]:
        getattr(lib, name).restype = C.c_int
    lib.ctd_jpeg_decoder_destroy.restype = None
    lib.ctd_png_encoder_create.argtypes = [i32, C.POINTER(vp)]
    lib.ctd_png_encoder_destroy.argtypes = [vp]
    lib.ctd_png_encode.argtypes = [vp, C.POINTER(CtdPngImage), i32, vp, vp]
    lib.ctd_png_encoder_destroy.restype = None
    lib.ctd_png_probe.argtypes = [vp, C.c_size_t, C.POINTER(CtdPngInfo)]
    lib.ctd_png_decoder_create.argtypes = [i32, i32, C.POINTER(vp)]
    lib.ctd_png_decoder_destroy.argtypes = [vp]
    lib.ctd_png_decode.argtypes = [vp, vp, vp, i32, vp, vp]
    lib.ctd_png_decoder_stats.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.ctd_png_decoder_destroy.restype = None
    _lib = lib
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def region_plan(lines, im_w, im_h, textheight):
    """`ctd_region_plan` (host C++, no GPU): lines = REGION_LINE_DTYPE records -> (REGION_DTYPE records, packed bytes)"""
    lib = load_library()
    lines = np.ascontiguousarray(lines, REGION_LINE_DTYPE)
    plan = np.zeros((len(lines),), REGION_DTYPE)
    total = C.c_size_t()
    rc = lib.ctd_region_plan(_ptr(lines), len(lines), int(im_w), int(im_h), int(textheight), _ptr(plan), C.byref(total))
    if rc != 0:
        raise CtdError("ctd_region_plan failed (%d): page %dx%d, textheight %d" % (rc, im_w, im_h, textheight))
    return plan, int(total.value)


def pages_plan(shapes, net_h, net_w):
    """`ctd_pages_plan` (host C++, no GPU): page sizes [(ih, iw), ...] -> (PAGE_ENTRY_DTYPE records, input bytes,
    results bytes) of one batch for `Engine.submit_pages`."""
    lib = load_library()
    pages = np.zeros((len(shapes),), PAGE_ENTRY_DTYPE)
    for i, (ih, iw) in enumerate(shapes):
        pages[i]["ih"], pages[i]["iw"] = ih, iw
    ib, rb = C.c_size_t(), C.c_size_t()
    rc = lib.ctd_pages_plan(_ptr(pages), len(pages), int(net_h), int(net_w), C.byref(ib), C.byref(rb))
    if rc != 0:
        raise CtdError("ctd_pages_plan failed (%d): pages %s do not letterbox into a %dx%d net input"
                       % (rc, list(shapes), net_h, net_w))
    return pages, int(ib.value), int(rb.value)


def refine_plan(shapes, xyxy, n_blocks):
    """`ctd_refine_plan` (host C++, no GPU): page sizes [(ih, iw), ...], every page's block boxes (int32 [k][4], page
    0's first) and the number of boxes of each page -> (PAGE_ENTRY_DTYPE records, windows int32 [k][4], status int32
    [k], input bytes, results bytes) of one batch for `Engine.submit_refine`."""
    lib = load_library()
    pages = np.zeros((len(shapes),), PAGE_ENTRY_DTYPE)
    for i, (ih, iw) in enumerate(shapes):
        pages[i]["ih"], pages[i]["iw"] = ih, iw
    xyxy = np.ascontiguousarray(np.asarray(xyxy, np.int32).reshape(-1, 4))
    counts = np.ascontiguousarray(n_blocks, np.int32).reshape(-1)
    assert len(counts) == len(pages) and int(counts.sum()) == len(xyxy), (len(counts), len(pages), len(xyxy))
    win = np.zeros((len(xyxy), 4), np.int32)
    status = np.zeros((len(xyxy),), np.int32)
    ib, rb = C.c_size_t(), C.c_size_t()
    rc = lib.ctd_refine_plan(_ptr(pages), len(pages), _ptr(xyxy), _ptr(counts), _ptr(win), _ptr(status), C.byref(ib),
                             C.byref(rb))
    if rc != 0:
        raise CtdError("ctd_refine_plan failed (%d): pages %s" % (rc, list(shapes)))
    return pages, win, status, int(ib.value), int(rb.value)


def _device_images(items, on_dev, events, channels):
    """ctd_device_page entries of the CUDA images of a batch (NULL entries for the host ones), or None if none is"""
    if not any(on_dev):
        return None
    dev = (CtdDevicePage * len(items))()
    for i, p in enumerate(items):
        if on_dev[i]:
            ev = events[i] if events is not None else None
            st = p.stride()   # uint8: element strides are byte strides
            dev[i] = CtdDevicePage(p.data_ptr(), st[0], st[1], st[2] if channels == 3 else 0,
                                   ev.cuda_event if ev is not None else None)
    return dev


def decode_block_section(sec, layout):
    """One page's block section (u8 bytes, see ctd_results_layout) -> (header i32 [4] = n_blocks, n_lines, n_dist,
    flags; block records; line quads i32 [MAX_BLOCKS, 8]; distances f64 [MAX_BLOCK_DIST]), views into `sec`."""
    hdr = sec[:16].view(np.int32)
    ro, lo, do = layout["blk_records_off"], layout["blk_lines_off"], layout["blk_dist_off"]
    rec = sec[ro:ro + MAX_BLOCKS * BLOCK_DTYPE.itemsize].view(BLOCK_DTYPE)[:int(hdr[0])]
    lines = sec[lo:lo + MAX_BLOCKS * 32].view(np.int32).reshape(-1, 8)
    dist = sec[do:do + MAX_BLOCK_DIST * 8].view(np.float64)
    return hdr, rec, lines, dist


class _BatchPlan:
    """The concatenated crop plan of a collected batch (ctd_collect_regions): page p's entries are
    [first[p], first[p + 1]), its crops the bytes page_range(p) of the batch's packed crops."""

    def __init__(self, plan, first, pixels, total):
        self.first, self.pixels, self.total = first, pixels, total
        self.off, self.oh, self.ow = plan["offset"].tolist(), plan["out_h"].tolist(), plan["out_w"].tolist()
        self.ok = (plan["status"] == 0).tolist()

    def page_range(self, p):
        a, b = self.first[p], self.first[p + 1]
        if b == a:
            return 0, 0
        return self.off[a], self.off[b - 1] + self.oh[b - 1] * self.ow[b - 1] * 3

    def page_crops(self, p, counts, view):
        """page p's crops: per block (counts = its lines) a list of [h][w][3] arrays, view(o, h, w) for the crop at
        byte o from the page's first crop, None where the planner gives no crop"""
        a, b = self.first[p], self.first[p + 1]
        counts = np.asarray(counts).tolist()
        assert sum(counts) == b - a, (p, sum(counts), b - a)
        off, oh, ow, ok = self.off, self.oh, self.ow, self.ok
        lo = off[a] if b > a else 0
        page, k = [], a
        for c in counts:
            page.append([view(off[j] - lo, oh[j], ow[j]) if ok[j] else None for j in range(k, k + c)])
            k += c
        return page


class Engine:
    """One engine handle = one GPU + one stream + one compiled program."""

    def __init__(self, program, device=0, precision=PREC_FP16_TC, max_batch=1, max_h=1024, max_w=1024, use_graph=False,
                 conf_thresh=0.4, nms_thresh=0.35, db_thresh=0.3, skip_postproc=False):
        self.lib = load_library()
        self.h = C.c_void_p()
        self.device = int(device)
        self.program = program
        self.nc = int(getattr(program, "nc", 2))
        ops = (CtdOp * len(program.ops))()
        for o, d in zip(ops, program.ops):
            for k, v in d.items():
                if k in ("src_buf", "src_coff", "src_c"):
                    for i in range(MAX_SRC):
                        getattr(o, k)[i] = int(v[i])
                else:
                    setattr(o, k, int(v))
        bufs = (CtdBufDesc * len(program.bufs))(*[CtdBufDesc(c, d) for c, d in program.bufs])
        cfg = CtdConfig(ABI_VERSION, device, precision, max_batch, max_h, max_w, self.nc, int(use_graph), conf_thresh,
                        nms_thresh, db_thresh, int(skip_postproc))
        blob = (C.c_char * len(program.blob)).from_buffer(program.blob)
        rc = self.lib.ctd_create(C.byref(self.h), C.byref(cfg), ops, len(program.ops), bufs, len(program.bufs),
                                 C.cast(blob, C.c_void_p), len(program.blob))
        if rc != 0:
            raise CtdError("ctd_create failed (%d): %s" % (rc, self.lib.ctd_last_error(None).decode()))
        self.shape = None

    def _ck(self, rc):
        if rc != 0:
            raise CtdError("ctd error %d: %s" % (rc, self.lib.ctd_last_error(self.h).decode()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.ctd_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- forward ------------------------------------------------------------------------
    def forward(self, pages):
        """pages: uint8 [n][h][w][3] BGR (host numpy) -> runs the whole device pipeline."""
        pages = np.ascontiguousarray(pages, dtype=np.uint8)
        if pages.ndim == 3:
            pages = pages[None]
        n, h, w, c = pages.shape
        assert c == 3
        self._ck(self.lib.ctd_forward(self.h, _ptr(pages), n, h, w, 0))
        self.shape = (n, h, w)

    def resize_linear_u8(self, src, dsize_wh):
        """`cv2.resize(src, dsize_wh, interpolation=cv2.INTER_LINEAR)` for uint8 [H,W] / [H,W,3] (bit-exact)."""
        src = np.ascontiguousarray(src, dtype=np.uint8)
        ch = 1 if src.ndim == 2 else src.shape[2]
        dw, dh = int(dsize_wh[0]), int(dsize_wh[1])
        out = np.empty((dh, dw) if src.ndim == 2 else (dh, dw, ch), np.uint8)
        self._ck(self.lib.ctd_resize_linear_u8(self.h, _ptr(src), src.shape[0], src.shape[1], ch, _ptr(out), dh, dw))
        return out

    def forward_device(self, dev_ptr, n, h, w):
        """pages already resident in HBM (device pointer as int)."""
        self._ck(self.lib.ctd_forward(self.h, C.c_void_p(dev_ptr), n, h, w, 1))
        self.shape = (n, h, w)

    def forward_tensor(self, x_ptr, n, h, w, stream, blks_ptr, mask_ptr, lines_ptr, half=False):
        """`ctd_forward_tensor`: the forward of a float32 NCHW [n][3][h][w] device tensor (pointer as int, 16-byte
        aligned) into caller-allocated device outputs (pointers as int, or None), ordered after the work enqueued on
        `stream` (a cudaStream_t as int; 0 is the legacy default stream), which then waits for the outputs.  No host
        synchronisation.  half: the input and the outputs are float16 (`ctd_forward_tensor_f16`)."""
        vp = C.c_void_p
        fn = self.lib.ctd_forward_tensor_f16 if half else self.lib.ctd_forward_tensor
        self._ck(fn(self.h, vp(x_ptr), n, h, w, vp(stream), vp(blks_ptr), vp(mask_ptr), vp(lines_ptr)))
        self.shape = (n, h, w)

    def rows_per_image(self):
        n, h, w = self.shape
        return 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32))

    def net_outputs(self, want_blks=True, want_mask=True, want_lines=True):
        n, h, w = self.shape
        blks = np.empty((n, self.rows_per_image(), 5 + self.nc), np.float32) if want_blks else None
        mask = np.empty((n, 1, h, w), np.float32) if want_mask else None
        lines = np.empty((n, 2, h, w), np.float32) if want_lines else None
        self._ck(self.lib.ctd_get_net_outputs(self.h, _ptr(blks), _ptr(mask), _ptr(lines)))
        return blks, mask, lines

    def mask_u8(self):
        n, h, w = self.shape
        m = np.empty((n, h, w), np.uint8)
        self._ck(self.lib.ctd_get_mask_u8(self.h, _ptr(m)))
        return m

    def detections(self):
        n = self.shape[0]
        det = np.empty((n, 300, 6), np.float32)
        cnt = np.empty((n,), np.int32)
        self._ck(self.lib.ctd_get_detections(self.h, _ptr(det), _ptr(cnt)))
        return [det[i, :cnt[i]].copy() for i in range(n)]

    def nms_status(self, n=1):
        """(candidates per page before the capacity cut, capacity): see ctd_get_nms_status."""
        tot = np.zeros((n,), np.int32)
        cap = C.c_int32()
        self._ck(self.lib.ctd_get_nms_status(self.h, _ptr(tot), C.byref(cap)))
        return tot, cap.value

    def db_components(self, want_bitmap=True, want_labels=True):
        n, h, w = self.shape
        bm = np.empty((n, h, w), np.uint8) if want_bitmap else None
        lab = np.empty((n, h, w), np.int32) if want_labels else None
        nl = np.empty((n,), np.int32)
        self._ck(self.lib.ctd_get_db_components(self.h, _ptr(bm), _ptr(lab), _ptr(nl)))
        return bm, lab, nl

    def text_lines(self):
        """per page (boxes int16 [k,4,2], scores f32 [k]) exactly as SegDetectorRepresenter returns them."""
        n = self.shape[0]
        boxes = np.empty((n, 1000, 4, 2), np.int16)
        scores = np.empty((n, 1000), np.float32)
        cnt = np.empty((n,), np.int32)
        self._ck(self.lib.ctd_get_text_lines(self.h, _ptr(boxes), _ptr(scores), _ptr(cnt)))
        return [boxes[i, :cnt[i]].copy() for i in range(n)], [scores[i, :cnt[i]].copy() for i in range(n)]

    def seg_represent(self, pred, thresh=0.3):
        pred = np.ascontiguousarray(pred, np.float32)
        h, w = pred.shape
        boxes = np.empty((1000, 4, 2), np.int16)
        scores = np.empty((1000,), np.float32)
        cnt = np.zeros((1,), np.int32)
        self._ck(self.lib.ctd_seg_represent(self.h, _ptr(pred), h, w, thresh, _ptr(boxes), _ptr(scores), _ptr(cnt)))
        k = int(cnt[0])
        return boxes[:k].copy(), scores[:k].copy()

    def refine_mask(self, img, mask, windows, refine_mode=0):
        """windows: int32 [k,4] already-expanded xyxy windows (expand_textwindow of every block)."""
        img = np.ascontiguousarray(img, np.uint8)
        mask = np.ascontiguousarray(mask, np.uint8)
        win = np.ascontiguousarray(np.asarray(windows, np.int32).reshape(-1, 4))
        out = np.empty(mask.shape, np.uint8)
        self._ck(self.lib.ctd_refine_mask(self.h, _ptr(img), _ptr(mask), mask.shape[0], mask.shape[1], _ptr(win), len(win),
                                          int(refine_mode), _ptr(out)))
        return out

    def last_forward_ms(self):
        ms = C.c_float()
        self._ck(self.lib.ctd_last_forward_ms(self.h, C.byref(ms)))
        return ms.value

    def last_launch_count(self):
        v = C.c_int32()
        self._ck(self.lib.ctd_last_launch_count(self.h, C.byref(v)))
        return v.value

    def debug_read(self, tensor):
        """tensor: dict(buf, coff, c, down) from the compiler -> float32 [n][h/down][w/down][c]."""
        n, h, w = self.shape
        ch = self.program.bufs[tensor["buf"]][0]
        d = tensor["down"]
        out = np.empty((n, h // d, w // d, ch), np.float32)
        self._ck(self.lib.ctd_debug_read_buffer(self.h, tensor["buf"], _ptr(out), out.size))
        return out[..., tensor["coff"]:tensor["coff"] + tensor["c"]]

    def timer_start(self):
        self._ck(self.lib.ctd_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float()
        self._ck(self.lib.ctd_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def profile_forward(self, pages=None, dev_ptr=None, shape=None):
        """per-op device milliseconds of one un-graphed forward: (op_ms[n_ops], nms_ms, ccl_ms)."""
        nops = len(self.program.ops)
        out = np.zeros((nops + 2,), np.float32)
        if pages is not None:
            pages = np.ascontiguousarray(pages, dtype=np.uint8)
            n, h, w, _ = pages.shape
            self._ck(self.lib.ctd_profile_forward(self.h, _ptr(pages), n, h, w, 0, _ptr(out), out.size))
        else:
            n, h, w = shape
            self._ck(self.lib.ctd_profile_forward(self.h, C.c_void_p(dev_ptr), n, h, w, 1, _ptr(out), out.size))
        self.shape = (n, h, w)
        return out[:nops], float(out[nops]), float(out[nops + 1])

    # ---- batch pipeline: two batches in flight, copies under compute -----------------------------
    def results_layout(self):
        """byte offsets of the result arena (ctd_results_layout): dict of ints."""
        lay = CtdResultsLayout()
        self._ck(self.lib.ctd_results_layout(self.h, C.byref(lay)))
        return {k: int(getattr(lay, k)) for k, _t in CtdResultsLayout._fields_}

    def submit_full(self, slot, pages_ptr, n, h, w, results_ptr, refine_mode=0, pages_on_device=False):
        """asynchronous full pipeline (network + post-processing + group_output + refine_mask) of a batch of
        net-sized pages into HOST `results` (results_layout()['total_bytes'] bytes, pinned): see ctd_submit_full."""
        self._ck(self.lib.ctd_submit_full(self.h, slot, C.c_void_p(pages_ptr), n, h, w, int(bool(pages_on_device)),
                                          int(refine_mode), C.c_void_p(results_ptr)))
        self.shape = (n, h, w)

    def device_arena(self, slot):
        """(device pointer of slot's complete result arena copy, cudaStream_t its last writes were enqueued on)."""
        base, st = C.c_void_p(), C.c_void_p()
        self._ck(self.lib.ctd_device_arena(self.h, slot, C.byref(base), C.byref(st)))
        return base.value, st.value

    def detect_page(self, page, net_h, net_w, refine_mode=0, keep_undetected=False):
        """the whole of TextDetector.__call__ for one page of any size (ctd_detect_page): returns
        (mask u8 [ih,iw], mask_refined u8 [ih,iw], block records, lines i32 [.,8], distances f64)."""
        page = np.ascontiguousarray(page, dtype=np.uint8)
        ih, iw, c = page.shape
        assert c == 3
        mask = np.empty((ih, iw), np.uint8)
        refined = np.empty((ih, iw), np.uint8)
        rec = np.zeros((MAX_BLOCKS,), BLOCK_DTYPE)
        lines = np.zeros((MAX_BLOCKS, 8), np.int32)
        dist = np.zeros((MAX_BLOCK_DIST,), np.float64)
        nb = C.c_int32()
        self._ck(self.lib.ctd_detect_page(self.h, _ptr(page), ih, iw, net_h, net_w, int(refine_mode), int(bool(keep_undetected)),
                                          _ptr(mask), _ptr(refined), _ptr(rec), MAX_BLOCKS, _ptr(lines), MAX_BLOCKS, _ptr(dist),
                                          MAX_BLOCK_DIST, C.byref(nb)))
        self.shape = (1, net_h, net_w)
        return mask, refined, rec[:nb.value], lines, dist

    def collect(self, slot):
        self._ck(self.lib.ctd_collect(self.h, slot))

    def submit_pages(self, slot, pages, net_h, net_w, refine_mode=0, keep_undetected=False, textheight=0, events=None,
                     device_results=False):
        """asynchronous `detect_page` of a batch of pages of any size (ctd_submit_pages).  A page is a u8
        [h][w][3] numpy array, packed into this slot's pinned input buffer (which like the pinned results buffer belongs
        to the engine and grows on demand), or a torch.uint8 CUDA tensor [h][w][3] on this engine's GPU with any
        strides, gathered on the GPU without a host copy; events[i] (a recorded torch.cuda.Event, or None) is waited on
        before CUDA page i is read.  The CUDA pages are referenced until the slot is collected and must not be written
        before.  textheight >= 2 also crops every text line of every page on the GPU (0: no crops).  device_results:
        masks and crops stay on the GPU (see collect_pages).  Collect with collect_pages(slot)."""
        import torch
        if not hasattr(self, "_pg_bufs"):
            self._pg_bufs = [[None, None], [None, None]]   # per slot: pinned input, pinned results
            self._pg_inflight = [None, None]
        if self._pg_inflight[slot] is not None:
            raise CtdError("slot %d has an uncollected submission" % slot)
        entries, in_bytes, res_bytes = pages_plan([tuple(p.shape[:2]) for p in pages], net_h, net_w)
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in pages]
        bufs = self._pg_bufs[slot]
        for k, need in ((0, 0 if all(on_dev) else in_bytes), (1, res_bytes)):
            if need and (bufs[k] is None or bufs[k].numel() < need):
                bufs[k] = torch.empty((need * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        dev = _device_images(pages, on_dev, events, 3)
        if not all(on_dev):
            inp = bufs[0].numpy()
            for e, p, d in zip(entries, pages, on_dev):
                if not d:
                    o = int(e["page_off"])
                    np.copyto(inp[o:o + p.size].reshape(p.shape), p)
        self._ck(self.lib.ctd_submit_pages(self.h, slot, _ptr(entries), len(entries), net_h, net_w,
                                           None if all(on_dev) else C.c_void_p(bufs[0].data_ptr()),
                                           None if dev is None else C.cast(dev, C.c_void_p), int(refine_mode),
                                           int(bool(keep_undetected)), int(textheight), int(bool(device_results)),
                                           C.c_void_p(bufs[1].data_ptr())))
        kept = [(p, None if events is None else events[i]) for i, p in enumerate(pages) if on_dev[i]]
        self._pg_inflight[slot] = (entries, int(textheight), bool(device_results), kept)
        self.shape = (len(entries), net_h, net_w)

    def collect_pages(self, slot, discard=False):
        """blocks until the batch of submit_pages(slot) is done -> per page the 5-tuple detect_page returns
        (mask, mask_refined, block records, lines, distances), copied out of the slot's pinned buffer.  With a
        textheight, each tuple has a sixth element, the page's crops (see collect_regions).  With device_results, mask,
        mask_refined and the crops are torch.uint8 CUDA tensors, views into one allocation of that page's own (filled by
        ctd_collect_device; complete on return).  discard: only wait for the batch and return None."""
        inflight = self._pg_inflight[slot] if hasattr(self, "_pg_inflight") else None
        if inflight is None:
            raise CtdError("slot %d has no submit_pages batch in flight" % slot)
        entries, textheight, device_results, _kept = inflight
        self._pg_inflight[slot] = None
        self.collect(slot)
        if discard:
            return None
        res = self._pg_bufs[slot][1].numpy()
        lay = self.results_layout()
        stride = lay["blocks_stride"]
        blocks = []
        for e in entries:
            bo = int(e["blocks_off"])
            _hdr, rec, lines, dist = decode_block_section(res[bo:bo + stride], lay)
            blocks.append((rec.copy(), lines.copy(), dist.copy()))
        n_lines = [b[0]["n_lines"] for b in blocks]
        if device_results:
            return self._collect_device(slot, entries, blocks, n_lines if textheight else None)
        out = []
        for e, b in zip(entries, blocks):
            ih, iw = int(e["ih"]), int(e["iw"])
            mo, ro = int(e["mask_off"]), int(e["refined_off"])
            out.append((res[mo:mo + ih * iw].reshape(ih, iw).copy(), res[ro:ro + ih * iw].reshape(ih, iw).copy()) + b)
        if textheight:
            crops = self.collect_regions(slot, n_lines)
            out = [o + (c,) for o, c in zip(out, crops)]
        return out

    def submit_outputs(self, slot, pages, outs, net_h, net_w, refine_mode=0, keep_undetected=False, textheight=0,
                       events=None, device_results=False):
        """asynchronous post-processing of a batch of pages from the caller's network outputs
        (ctd_submit_outputs_dtype): pages as submit_pages takes them; outs[i] = (blks [A][5 + nc], mask [net_h][net_w],
        lines [net_h][net_w]) of page i, each a numpy array (copied into this slot's pinned output buffer) or a CUDA
        tensor on this engine's GPU with any strides (read where it is), all three float32 or all three float16 (the
        page is then post-processed with the reference's half arithmetic).  events[i] (a recorded torch.cuda.Event, or None) is
        waited on before CUDA page i and CUDA outputs i are read; the CUDA pages and outputs are referenced until the
        slot is collected and must not be written before.  Collect with collect_pages(slot)."""
        import torch
        if not hasattr(self, "_pg_bufs"):
            self._pg_bufs = [[None, None], [None, None]]
            self._pg_inflight = [None, None]
        if self._pg_inflight[slot] is not None:
            raise CtdError("slot %d has an uncollected submission" % slot)
        entries, in_bytes, res_bytes = pages_plan([tuple(p.shape[:2]) for p in pages], net_h, net_w)
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in pages]
        o_dev = [[isinstance(m, torch.Tensor) and m.is_cuda for m in o] for o in outs]
        # the host maps, packed contiguous into the slot's pinned output buffer, 256-byte aligned each
        offs, need = [], 0
        for o, d in zip(outs, o_dev):
            page = []
            for m, md in zip(o, d):
                page.append(None if md else need)
                need += 0 if md else (m.size * m.itemsize + 255) // 256 * 256
            offs.append(page)
        if not hasattr(self, "_out_bufs"):
            self._out_bufs = [None, None]
        bufs = self._pg_bufs[slot]
        for k, n_bytes in ((0, 0 if all(on_dev) else in_bytes), (1, res_bytes)):
            if n_bytes and (bufs[k] is None or bufs[k].numel() < n_bytes):
                bufs[k] = torch.empty((n_bytes * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        if need and (self._out_bufs[slot] is None or self._out_bufs[slot].numel() < need):
            self._out_bufs[slot] = torch.empty((need * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        if not all(on_dev):
            inp = bufs[0].numpy()
            for e, p, d in zip(entries, pages, on_dev):
                if not d:
                    o = int(e["page_off"])
                    np.copyto(inp[o:o + p.size].reshape(p.shape), p)
        rec = (CtdNetOutput * len(outs))()
        dtypes = (C.c_int32 * len(outs))(*[DTYPE_F16 if _is_f16(o[0]) else DTYPE_F32 for o in outs])
        obuf = self._out_bufs[slot].numpy() if need else None
        base = self._out_bufs[slot].data_ptr() if need else 0
        for i, (o, d, off) in enumerate(zip(outs, o_dev, offs)):
            fields = []
            for m, md, mo in zip(o, d, off):
                if md:
                    st = m.stride()
                    fields.append((m.data_ptr(), st[0], st[1] if len(st) > 1 else 1, 1))
                else:
                    np.copyto(obuf[mo:mo + m.size * m.itemsize].view(m.dtype).reshape(m.shape), m)
                    fields.append((base + mo, m.shape[1] if m.ndim > 1 else 1, 1, 0))
            (bp, bsr, bsc, bd), (mp, msh, msw, md_), (lp, lsh, lsw, ld) = fields
            ev = events[i] if events is not None else None
            rec[i] = CtdNetOutput(bp, bsr, bsc, mp, msh, msw, lp, lsh, lsw, int(o[0].shape[0]), bd, md_, ld,
                                  ev.cuda_event if ev is not None else None)
        dev = _device_images(pages, on_dev, events, 3)
        self._ck(self.lib.ctd_submit_outputs_dtype(self.h, slot, _ptr(entries), len(entries), net_h, net_w,
                                                   None if all(on_dev) else C.c_void_p(bufs[0].data_ptr()),
                                                   None if dev is None else C.cast(dev, C.c_void_p),
                                                   C.cast(rec, C.c_void_p), C.cast(dtypes, C.c_void_p),
                                                   int(refine_mode), int(bool(keep_undetected)), int(textheight),
                                                   int(bool(device_results)), C.c_void_p(bufs[1].data_ptr())))
        kept = [(p, None if events is None else events[i]) for i, p in enumerate(pages) if on_dev[i]] + \
               [(m, None if events is None else events[i]) for i, o in enumerate(outs) for m, md in zip(o, o_dev[i])
                if md]
        self._pg_inflight[slot] = (entries, int(textheight), bool(device_results), kept)
        self.shape = (len(entries), net_h, net_w)

    def preprocess_pages(self, pages, net_h, net_w, fmt, reverse, dst_ptr, stream, events=None, input_host=None):
        """`ctd_preprocess_pages`: the letterboxed network input of a batch (fmt: PRE_*; reverse: output channel k is
        page channel 2 - k) into dst_ptr (a device pointer as int, 16-byte aligned), enqueued on `stream` (a
        cudaStream_t as int) with no host wait.  A page is a torch.uint8 CUDA tensor [h][w][3] on this engine's GPU
        with any strides (events[i]: a recorded torch.cuda.Event or None, waited on before page i is read), or a u8
        [h][w][3] numpy array, packed at its page_off into input_host: a pinned torch.uint8 tensor of at least the
        plan's input bytes, which the caller keeps unwritten until the stream has run the call.  Returns the
        ctd_pages_plan entries of the batch."""
        import torch
        entries, in_bytes, _res = pages_plan([tuple(p.shape[:2]) for p in pages], net_h, net_w)
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in pages]
        host = None
        if not all(on_dev):
            if input_host is None or input_host.numel() < in_bytes:
                raise CtdError("numpy pages need a pinned input_host of %d bytes" % in_bytes)
            inp = input_host.numpy()
            for e, p, d in zip(entries, pages, on_dev):
                if not d:
                    o = int(e["page_off"])
                    np.copyto(inp[o:o + p.size].reshape(p.shape), p)
            host = C.c_void_p(input_host.data_ptr())
        dev = _device_images(pages, on_dev, events, 3)
        self._ck(self.lib.ctd_preprocess_pages(self.h, _ptr(entries), len(entries), int(net_h), int(net_w), host,
                                               None if dev is None else C.cast(dev, C.c_void_p), int(fmt),
                                               int(bool(reverse)), C.c_void_p(dst_ptr), C.c_void_p(stream)))
        return entries

    def submit_refine(self, slot, pages, masks, boxes, refine_mode=0, keep_undetected=False, refined=None,
                      events=None, device_results=False):
        """asynchronous refine_mask of a batch (ctd_submit_refine): per page a u8 [h][w][3] page and a u8 [h][w] mask,
        each a numpy array (packed into this slot's pinned input buffer) or a torch.uint8 CUDA tensor on this engine's
        GPU with any strides (gathered on the GPU), and its block boxes (int32 [k][4]).  events[i] (a recorded
        torch.cuda.Event, or None) is waited on before CUDA page i and CUDA mask i are read; the CUDA images are
        referenced until the slot is collected and must not be written before.  refined: None, or per page a numpy
        u8 [h][w] mask_refined to run refine_undetected_mask alone on (needs keep_undetected).  Collect with
        collect_refine(slot)."""
        import torch
        if not hasattr(self, "_pg_bufs"):
            self._pg_bufs = [[None, None], [None, None]]
            self._pg_inflight = [None, None]
        if self._pg_inflight[slot] is not None:
            raise CtdError("slot %d has an uncollected submission" % slot)
        counts = [len(b) for b in boxes]
        xyxy = np.concatenate([np.asarray(b, np.int32).reshape(-1, 4) for b in boxes]) if boxes else np.zeros((0, 4))
        entries, _win, _st, in_bytes, res_bytes = refine_plan([tuple(p.shape[:2]) for p in pages], xyxy, counts)
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in pages]
        m_dev = [isinstance(m, torch.Tensor) and m.is_cuda for m in masks]
        host = refined is not None or not all(on_dev) or not all(m_dev)
        bufs = self._pg_bufs[slot]
        for k, need in ((0, in_bytes if host else 0), (1, res_bytes)):
            if need and (bufs[k] is None or bufs[k].numel() < need):
                bufs[k] = torch.empty((need * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        if host:
            inp = bufs[0].numpy()
            frame = in_bytes // 5 * 3
            for e, p, d, m, md in zip(entries, pages, on_dev, masks, m_dev):
                ih, iw = int(e["ih"]), int(e["iw"])
                if not d:
                    o = int(e["page_off"])
                    np.copyto(inp[o:o + ih * iw * 3].reshape(ih, iw, 3), p)
                if not md:
                    o = frame + int(e["mask_off"])
                    np.copyto(inp[o:o + ih * iw].reshape(ih, iw), m)
            for e, r in zip(entries, refined or []):
                o = frame + int(e["refined_off"])
                np.copyto(inp[o:o + r.size].reshape(r.shape), r)
        dev_p = _device_images(pages, on_dev, events, 3)
        dev_m = _device_images(masks, m_dev, events, 1)
        self._ck(self.lib.ctd_submit_refine(self.h, slot, _ptr(entries), len(entries), _ptr(xyxy), _ptr(np.asarray(
            counts, np.int32)), C.c_void_p(bufs[0].data_ptr()) if host else None,
            None if dev_p is None else C.cast(dev_p, C.c_void_p), None if dev_m is None else C.cast(dev_m, C.c_void_p),
            int(refine_mode), int(bool(keep_undetected)), int(refined is not None), int(bool(device_results)),
            C.c_void_p(bufs[1].data_ptr())))
        kept = [x for i in range(len(pages)) for x, d in ((pages[i], on_dev[i]), (masks[i], m_dev[i])) if d]
        self._pg_inflight[slot] = ("refine", entries, bool(keep_undetected), bool(device_results), kept, events)

    def collect_refine(self, slot, discard=False):
        """blocks until the batch of submit_refine(slot) is done -> per page (mask, mask_refined): mask is the mask
        refine_undetected_mask modified (keep_undetected), else None.  numpy arrays copied out of the slot's pinned
        buffer, or with device_results torch.uint8 CUDA tensors, views into one allocation of the page's own
        (ctd_collect_device, complete on return, marked as used on the current stream).  discard: only wait."""
        inflight = self._pg_inflight[slot] if hasattr(self, "_pg_inflight") else None
        if inflight is None or inflight[0] != "refine":
            raise CtdError("slot %d has no submit_refine batch in flight" % slot)
        _kind, entries, keep, device_results, _kept, _events = inflight
        self._pg_inflight[slot] = None
        self.collect(slot)
        if discard:
            return None
        shapes = [(int(e["ih"]), int(e["iw"])) for e in entries]
        if device_results:
            import torch
            dev = torch.device("cuda", self.device)
            if getattr(self, "_alloc_stream", None) is None:
                self._alloc_stream = torch.cuda.Stream(dev)
            with torch.cuda.stream(self._alloc_stream):
                bufs = [torch.empty((2 * ih * iw,), dtype=torch.uint8, device=dev) for ih, iw in shapes]
            self._ck(self.lib.ctd_collect_device(self.h, slot, (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])))
            cur = torch.cuda.current_stream(dev)
            out = []
            for b, (ih, iw) in zip(bufs, shapes):
                b.record_stream(cur)
                out.append((b[:ih * iw].view(ih, iw) if keep else None, b[ih * iw:].view(ih, iw)))
            return out
        res = self._pg_bufs[slot][1].numpy()
        out = []
        for e, (ih, iw) in zip(entries, shapes):
            mo, ro = int(e["mask_off"]), int(e["refined_off"])
            out.append((res[mo:mo + ih * iw].reshape(ih, iw).copy() if keep else None,
                        res[ro:ro + ih * iw].reshape(ih, iw).copy()))
        return out

    def submit_regions(self, slot, pages, lines, n_lines, textheight, events=None, device_results=False):
        """asynchronous crops of caller lines (ctd_submit_regions): per page a u8 [h][w][3] numpy page (packed into this
        slot's pinned input buffer) or a torch.uint8 CUDA tensor on this engine's GPU with any strides (read where it
        is), lines = REGION_LINE_DTYPE records of every page's lines, page 0's first, n_lines[i] of page i.
        events[i] (a recorded torch.cuda.Event, or None) is waited on before CUDA page i is read; the CUDA pages are
        referenced until the slot is collected and must not be written before.  Collect with collect_crops(slot)."""
        import torch
        if not hasattr(self, "_pg_bufs"):
            self._pg_bufs = [[None, None], [None, None]]
            self._pg_inflight = [None, None]
        if self._pg_inflight[slot] is not None:
            raise CtdError("slot %d has an uncollected submission" % slot)
        shapes = [tuple(p.shape[:2]) for p in pages]
        entries, _win, _st, in_bytes, _rb = refine_plan(shapes, np.zeros((0, 4), np.int32), [0] * len(pages))
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in pages]
        host = not all(on_dev)
        need = in_bytes // 5 * 3 if host else 0   # the page plane of the layout
        bufs = self._pg_bufs[slot]
        if need and (bufs[0] is None or bufs[0].numel() < need):
            bufs[0] = torch.empty((need * 5 // 4,), dtype=torch.uint8, pin_memory=True)
        if host:
            inp = bufs[0].numpy()
            for e, p, d in zip(entries, pages, on_dev):
                if not d:
                    o = int(e["page_off"])
                    np.copyto(inp[o:o + p.size].reshape(p.shape), p)
        lines = np.ascontiguousarray(lines, REGION_LINE_DTYPE)
        counts = np.ascontiguousarray(n_lines, np.int32)
        dev = _device_images(pages, on_dev, events, 3)
        self._ck(self.lib.ctd_submit_regions(self.h, slot, _ptr(entries), len(entries), _ptr(lines), _ptr(counts),
                                             int(textheight), C.c_void_p(bufs[0].data_ptr()) if host else None,
                                             None if dev is None else C.cast(dev, C.c_void_p), int(bool(device_results))))
        kept = [(p, None if events is None else events[i]) for i, p in enumerate(pages) if on_dev[i]]
        self._pg_inflight[slot] = ("regions", len(entries), bool(device_results), kept)

    def collect_crops(self, slot, counts, discard=False):
        """blocks until the batch of submit_regions(slot) is done -> per page, per block (counts[p]: the number of lines
        of each block of page p) a list of u8 [h][w][3] crops in line order, None where the planner gives no crop.  Each
        page's crops are views into one array of that page's own (collect_regions), or with device_results into one
        CUDA allocation of its own (ctd_collect_device; complete on return, marked as used on the current stream); a
        page without a crop allocates nothing.  discard: only wait for the batch and return None."""
        inflight = self._pg_inflight[slot] if hasattr(self, "_pg_inflight") else None
        if inflight is None or inflight[0] != "regions":
            raise CtdError("slot %d has no submit_regions batch in flight" % slot)
        _kind, n_pages, device_results, _kept = inflight
        self._pg_inflight[slot] = None
        self.collect(slot)
        if discard:
            return None
        if not device_results:
            return self.collect_regions(slot, counts)
        import torch
        dev = torch.device("cuda", self.device)
        if getattr(self, "_alloc_stream", None) is None:
            self._alloc_stream = torch.cuda.Stream(dev)
        plan = self._collected_plan(slot, n_pages)
        ranges = [plan.page_range(p) for p in range(n_pages)]
        with torch.cuda.stream(self._alloc_stream):
            bufs = [torch.empty((hi - lo,), dtype=torch.uint8, device=dev) if hi > lo else None for lo, hi in ranges]
        ptrs = (C.c_void_p * n_pages)(*[None if b is None else b.data_ptr() for b in bufs])
        self._ck(self.lib.ctd_collect_device(self.h, slot, ptrs))
        cur = torch.cuda.current_stream(dev)
        out = []
        for p, buf in enumerate(bufs):
            if buf is not None:
                buf.record_stream(cur)
            out.append(plan.page_crops(p, counts[p], lambda c, h, w, buf=buf: buf.as_strided((h, w, 3), (w * 3, 3, 1), c)))
        return out

    def _collect_device(self, slot, entries, blocks, n_lines):
        """collect_pages of a device_results batch: one CUDA allocation per page, [mask | mask_refined | crops]
        (ctd_collect_device).  The allocations are made on a stream of the engine's own, so the caching allocator
        cannot hand out memory that work still queued on the caller's stream uses (the copies do not wait for that
        stream), and are marked as used on the caller's current stream."""
        import torch
        dev = torch.device("cuda", self.device)
        if getattr(self, "_alloc_stream", None) is None:
            self._alloc_stream = torch.cuda.Stream(dev)
        plan = self._collected_plan(slot, len(entries)) if n_lines is not None else None
        sizes = []
        for p, e in enumerate(entries):
            px = int(e["ih"]) * int(e["iw"])
            lo, hi = plan.page_range(p) if plan is not None else (0, 0)
            sizes.append((px, lo, hi))
        with torch.cuda.stream(self._alloc_stream):
            bufs = [torch.empty((2 * px + hi - lo,), dtype=torch.uint8, device=dev) for px, lo, hi in sizes]
        ptrs = (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
        self._ck(self.lib.ctd_collect_device(self.h, slot, ptrs))
        cur = torch.cuda.current_stream(dev)
        out = []
        for p, (e, b, buf, (px, _lo, _hi)) in enumerate(zip(entries, blocks, bufs, sizes)):
            buf.record_stream(cur)
            ih, iw = int(e["ih"]), int(e["iw"])
            o = (buf[:px].view(ih, iw), buf[px:2 * px].view(ih, iw)) + b
            if plan is not None:
                # as_strided on the fresh allocation (storage offset 0): the cheapest view torch makes, which matters
                # at thousands of crops per batch
                o += (plan.page_crops(p, n_lines[p], lambda c, h, w, buf=buf, px=px:
                                      buf.as_strided((h, w, 3), (w * 3, 3, 1), 2 * px + c)),)
            out.append(o)
        return out

    def _collected_plan(self, slot, n_pages):
        """the plan of the collected ctd_submit_pages batch of `slot` (ctd_collect_regions)"""
        plan_p, n_reg, first_p, pix_p, nbytes = C.c_void_p(), C.c_int32(), C.c_void_p(), C.c_void_p(), C.c_size_t()
        self._ck(self.lib.ctd_collect_regions(self.h, slot, C.byref(plan_p), C.byref(n_reg), C.byref(first_p),
                                              C.byref(pix_p), C.byref(nbytes)))
        n = int(n_reg.value)
        first = np.ctypeslib.as_array(C.cast(first_p, C.POINTER(C.c_int32)), (n_pages + 1,)).tolist()
        plan = np.frombuffer((C.c_char * (n * REGION_DTYPE.itemsize)).from_address(plan_p.value), REGION_DTYPE) \
            if n else np.zeros((0,), REGION_DTYPE)
        return _BatchPlan(plan, first, pix_p.value, int(nbytes.value))

    def collect_regions(self, slot, n_lines):
        """the crops of the collected ctd_submit_pages batch of `slot` (ctd_collect_regions): per page, per
        block a list of u8 [h][w][3] arrays in line order, None for a line the planner gives no crop (status != 0).
        n_lines: per page the block records' n_lines.  Each page's crops are views into one fresh array of that page
        (copied out of the engine's pinned buffer by torch's multi-threaded CPU copy: a single-threaded copy into fresh
        memory was most of the cost of this call)."""
        import torch
        plan = self._collected_plan(slot, len(n_lines))
        total = plan.total
        pix = torch.from_numpy(np.ctypeslib.as_array(C.cast(C.c_void_p(plan.pixels), C.POINTER(C.c_uint8)), (total,))) \
            if total else None
        out = []
        for p, counts in enumerate(n_lines):
            lo, hi = plan.page_range(p)
            buf = torch.empty((hi - lo,), dtype=torch.uint8).copy_(pix[lo:hi]).numpy() if hi > lo else None
            out.append(plan.page_crops(p, counts, lambda o, h, w, buf=buf: buf[o:o + h * w * 3].reshape(h, w, 3)))
        return out

    def join(self, other):
        """everything enqueued so far on `other`'s stream becomes a dependency of this engine's stream."""
        self._ck(self.lib.ctd_join(self.h, other.h))

    def debug_write(self, tensor, arr, n, h, w):
        """fill a whole buffer (all its channels) from float32 [n][h/down][w/down][channels]."""
        arr = np.ascontiguousarray(arr, np.float32)
        ch = self.program.bufs[tensor["buf"]][0]
        assert arr.shape == (n, h // tensor["down"], w // tensor["down"], ch), arr.shape
        self._ck(self.lib.ctd_debug_write_buffer(self.h, tensor["buf"], _ptr(arr), n, h, w))

    def debug_run_ops(self, first, last, n, h, w, pages=None):
        """run ops [first, last] only, on the current buffer contents (see ctd_debug_run_ops)."""
        if pages is not None:
            pages = np.ascontiguousarray(pages, dtype=np.uint8)
        self._ck(self.lib.ctd_debug_run_ops(self.h, _ptr(pages), n, h, w, first, last))
        self.shape = (n, h, w)

    def debug_read_slot(self, slot, plane, offset, nbytes):
        """u8 [nbytes] at byte `offset` of a collected slot's device plane (ctd_debug_read_slot): 0 the packed pages,
        1 the results frame, 2 the net input of the last forward"""
        out = np.empty((nbytes,), np.uint8)
        self._ck(self.lib.ctd_debug_read_slot(self.h, slot, plane, offset, _ptr(out), nbytes))
        return out

    def debug_postprocess(self, blks, lines):
        """the forward's NMS and DB post-processing on given network outputs (ctd_debug_postprocess): blks f32
        [n][rows_per_image][5 + nc], lines f32 [n][2][h][w].  Read the results with detections(), nms_status(n),
        db_components() and text_lines()."""
        blks = np.ascontiguousarray(blks, np.float32)
        lines = np.ascontiguousarray(lines, np.float32)
        n, c, h, w = lines.shape
        assert c == 2 and blks.shape == (n, 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32)),
                                         5 + self.nc), (blks.shape, lines.shape)
        self._ck(self.lib.ctd_debug_postprocess(self.h, _ptr(blks), _ptr(lines), n, h, w))
        self.shape = (n, h, w)

    # ---- text-line crops (ctd_transform_regions) -------------------------------------------
    def transform_regions(self, page, plan, out=None, page_shape=None):
        """warp every plan entry with status 0 out of `page` in one launch -> packed u8 bytes (plan layout).
        page: u8 [ih][iw][3] host array, or a device pointer (int) with page_shape = (ih, iw).  out: optional host
        u8 buffer of at least the plan's total bytes."""
        plan = np.ascontiguousarray(plan, REGION_DTYPE)
        total = int(max((int(r["offset"]) + int(r["out_h"]) * int(r["out_w"]) * 3 for r in plan), default=0))
        if out is None:
            out = np.empty((total,), np.uint8)
        if page_shape is None:
            page = np.ascontiguousarray(page, np.uint8)
            ih, iw, c = page.shape
            assert c == 3
            ptr, on_dev = _ptr(page), 0
        else:
            (ih, iw), ptr, on_dev = page_shape, C.c_void_p(int(page)), 1
        self._ck(self.lib.ctd_transform_regions(self.h, ptr, int(ih), int(iw), on_dev, _ptr(plan), len(plan), _ptr(out),
                                                out.nbytes))
        return out

    # ---- stand-alone array kernels --------------------------------------------------------
    def connected_components(self, img, stats_cap=0):
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        labels = np.empty((h, w), np.int32)
        nl = np.zeros((1,), np.int32)
        stats = np.empty((stats_cap, 5), np.int32) if stats_cap else None
        self._ck(self.lib.ctd_connected_components(self.h, _ptr(img), h, w, _ptr(labels), _ptr(stats), stats_cap, _ptr(nl)))
        n = int(nl[0])
        return n, labels, (stats[:n] if stats is not None else None)

    def nms(self, pred, conf_thresh=0.4, iou_thresh=0.35):
        pred = np.ascontiguousarray(pred, np.float32)
        det = np.empty((300, 6), np.float32)
        cnt = np.zeros((1,), np.int32)
        self._ck(self.lib.ctd_nms(self.h, _ptr(pred), pred.shape[0], conf_thresh, iou_thresh, _ptr(det), _ptr(cnt)))
        return det[:int(cnt[0])].copy()
