/*
 * ctd_b200.h -- C ABI of libctd_b200.so, the H100 (sm_90a) engine behind the reference's
 * inference path  page -> (block boxes, text-line map, segmentation mask).
 *
 * The reference is pure Python and has no FFI; the seam this library replaces is the
 * backend object built in `inference.TextDetector.__init__` (reference inference.py:124-130:
 * `self.net = TextDetBase(...)` / `TextDetBaseDNN(...)`, a callable
 * `net(img_in) -> (blks, mask, lines_map)`, basemodel.py:240-244) plus the array-level
 * post-processing calls made from `TextDetector.__call__` (inference.py:141-178).
 * Each entry point cites the reference interface it stands in for.  Plain C types only:
 * no torch, no C++ types, nothing thrown across the boundary.  Every function returns 0 on
 * success or a negative CTD_E_* code; `ctd_last_error()` gives the message.
 *
 * Threading: a handle is bound to one CUDA device and one internal stream and is NOT
 * thread-safe; independent handles (one per GPU / per process) are independent.
 */
#ifndef CTD_B200_H_
#define CTD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTD_ABI_VERSION 3
#if defined(__GNUC__)
#define CTD_API __attribute__((visibility("default")))
#else
#define CTD_API
#endif

/* ---- error codes ---------------------------------------------------------------------- */
#define CTD_OK 0
#define CTD_E_INVALID (-1)   /* bad argument / malformed program                            */
#define CTD_E_CUDA (-2)      /* CUDA runtime/driver error (message has the CUDA string)     */
#define CTD_E_NO_DEVICE (-3) /* no sm_90 GPU visible: the engine has NO CPU fallback       */
#define CTD_E_SHAPE (-4)     /* page size not a multiple of 64 (basemodel.py:62-78 stride)  */
#define CTD_E_CAPACITY (-5)  /* batch larger than the reserved workspace                    */

/* ---- network program ------------------------------------------------------------------
 * The Python host (comic-text-detector_b200/compiler.py) plays the role of the reference's
 * `parse_model` + `load_state_dict` + `fuse` (models/yolov5/yolo.py:208-259,285-311;
 * utils/yolov5_utils.py:23-43; basemodel.py:211-220): it walks the checkpoint's cfg, folds
 * every BatchNorm and emits a flat list of ops over numbered NHWC activation buffers plus one
 * weight blob.  The engine owns no architecture knowledge beyond these op kinds.           */

enum ctd_op_kind {
  CTD_OP_STEM = 0,      /* 6x6 s2 p2 conv on the u8 BGR page (/255 fused), common.py:30-49 cfg L0;
                           w32_off: direct form, w16_off: 3x3 window form over the 2x2 space-to-depth page
                           (tensor cores, built per tile in shared memory; src_buf[0], the 16-channel
                           space-to-depth buffer older engines staged it in, is no longer read)  */
  CTD_OP_CONV = 1,      /* k in {1,3}, stride in {1,2}, pad k/2; K-concatenated sources     */
  CTD_OP_DECONV4 = 2,   /* ConvTranspose2d 4x4 s2 p1 (basemodel.py:26) as 4 sub-pixel phases */
  CTD_OP_AVGPOOL2 = 3,  /* AvgPool2d(2,2)                (basemodel.py:38)                  */
  CTD_OP_SPPF_POOL = 4, /* 3 chained MaxPool2d(5,1,2)    (common.py:188-196)                */
  CTD_OP_UPSAMPLE2 = 5, /* nn.Upsample(x2, nearest)      (cfg layers 11,15)                 */
  CTD_OP_DETECT = 6,    /* Detect 1x1 conv + sigmoid + box decode (yolo.py:23-44)           */
  CTD_OP_SEG_TAIL = 7,  /* ConvT4x4s2 64->1 + sigmoid    (basemodel.py:57-60); p_off: fp32 [C][4][4],
                           w16_off: fp16 3x3 conv with the 4 sub-pixel phases as outputs, cout_pad 16 */
  CTD_OP_DB_TAIL = 8    /* ConvT2x2s2+BN+ReLU -> ConvT2x2s2 -> sigmoid, both branches
                           (basemodel.py:99-103,138-142)                                    */
  /* 9 is reserved (a retired op kind)                                                      */
};

enum ctd_act { CTD_ACT_NONE = 0, CTD_ACT_SILU = 1, CTD_ACT_LEAKY = 2, CTD_ACT_RELU = 3, CTD_ACT_SIGMOID = 4 };

#define CTD_MAX_SRC 3

typedef struct ctd_op {
  int32_t kind;                  /* enum ctd_op_kind                                        */
  int32_t n_src;                 /* 1..CTD_MAX_SRC K-concatenated inputs (torch.cat on dim 1) */
  int32_t src_buf[CTD_MAX_SRC];  /* activation buffer ids                                   */
  int32_t src_coff[CTD_MAX_SRC]; /* first channel read in that buffer                       */
  int32_t src_c[CTD_MAX_SRC];    /* channels read                                           */
  int32_t dst_buf;               /* activation buffer id (-1 for ops writing engine outputs) */
  int32_t dst_coff;              /* first channel written                                   */
  int32_t cout;                  /* true output channels                                    */
  int32_t cout_pad;              /* rows in the packed weight matrix (multiple of 16)       */
  int32_t ksize;                 /* 1, 3 (conv), 4 (deconv), 6 (stem)                       */
  int32_t stride;                /* 1 or 2                                                  */
  int32_t act;                   /* enum ctd_act                                            */
  int32_t residual;              /* 1: dst = act(conv)+dst in place (Bottleneck.add, common.py:104) */
  int32_t aux;                   /* DETECT: pyramid level (0,1,2)                           */
  int64_t w16_off;               /* blob offset: fp16 weights [phase][cout_pad][taps*Cin] K-major */
  int64_t w32_off;               /* blob offset: fp32 weights, same layout                  */
  int64_t b_off;                 /* blob offset: fp32 bias[cout_pad] (BN folded); STEM, CONV, DECONV4, DETECT */
  int64_t p_off;                 /* blob offset: extra fp32 params (DETECT anchors, tails)  */
} ctd_op;

typedef struct ctd_bufdesc {
  int32_t channels; /* total channels of the NHWC buffer                                   */
  int32_t down;     /* spatial size = page size / down                                     */
} ctd_bufdesc;

enum ctd_precision {
  CTD_PREC_FP16_TC = 0,   /* fp16 storage, wgmma implicit GEMM, fp32 accumulate (default) */
  CTD_PREC_FP32_SIMT = 1, /* fp32 storage + CUDA-core fp32 kernels ("vs reference fp32" config) */
  CTD_PREC_FP16_SIMT = 2, /* fp16 storage + CUDA-core kernels (bisecting aid)               */
  CTD_PREC_SPLIT_TC = 3   /* fp32 storage; wgmma with every operand split into fp16 hi + lo planes
                             (hi*hi + lo*hi + hi*lo, fp32 accumulate: ~22 significant bits) -- the
                             tensor-core path that meets the 1e-3 "vs reference fp32" tolerance  */
};

typedef struct ctd_config {
  int32_t abi_version; /* CTD_ABI_VERSION                                                  */
  int32_t device;      /* CUDA device ordinal                                              */
  int32_t precision;   /* enum ctd_precision                                               */
  int32_t max_batch;   /* pages per ctd_infer call the workspace is sized for              */
  int32_t max_h, max_w; /* largest page (multiples of 64)                                  */
  int32_t nc;          /* classes of the Detect head (reference: 2, inference.py:117-118)  */
  int32_t use_graph;   /* 1: capture the op list into a CUDA graph per (n,h,w)             */
  float conf_thresh;   /* 0.4  (inference.py:120)                                          */
  float nms_thresh;    /* 0.35 (inference.py:120).  A box is suppressed where its float32
                          IoU > nms_thresh in float32; torchvision's CPU nms (the reference's
                          default device) compares with a double t, which is this rule with
                          nms_thresh = RD_f32(t), t rounded toward -inf to float32            */
  float db_thresh;     /* 0.3  (inference.py:139 -> db_utils.py:71-72)                     */
  int32_t debug_skip_postproc; /* 1: ctd_forward stops after the op list (kernel unit tests)  */
} ctd_config;

typedef struct ctd_handle ctd_handle;

/* Replaces TextDetBase.__init__ / get_base_det_models (basemodel.py:211-227).
 * `blob` is copied to the device; the arrays may be freed after the call.                 */
CTD_API int ctd_create(ctd_handle** out, const ctd_config* cfg, const ctd_op* ops, int32_t n_ops,
               const ctd_bufdesc* bufs, int32_t n_bufs, const void* blob, size_t blob_bytes);
CTD_API void ctd_destroy(ctd_handle* h);
CTD_API const char* ctd_last_error(const ctd_handle* h); /* h may be NULL: last create() error     */

/* ---- the forward pass --------------------------------------------------------------------
 * Replaces `TextDetBase.forward` (basemodel.py:240-244) fed by `preprocess_img` for
 * net-sized pages (inference.py:72-83: BGR u8 HWC -> BGR f32 NCHW /255; the /255 and the
 * layout change are fused into the stem kernel).
 *
 * pages : n*h*w*3 bytes, BGR, HWC, u8.  `pages_on_device` != 0 means a device pointer.
 * The result stays on the device inside the handle; fetch what you need with ctd_get_*.   */
CTD_API int ctd_forward(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw, int32_t pages_on_device);

/* Net-level outputs (the tuple TextDetBase.forward returns), copied to HOST memory.
 * blks  : f32 [n][A][5+nc], A = 3*(h/8*w/8 + h/16*w/16 + h/32*w/32)     (yolo.py:44)
 * mask  : f32 [n][h][w] in (0,1)                                        (basemodel.py:57-60)
 * lines : f32 [n][2][h][w] = (shrink, threshold)                        (basemodel.py:125)
 * Any pointer may be NULL to skip it.                                                      */
CTD_API int ctd_get_net_outputs(ctd_handle* h, float* blks, float* mask, float* lines);

/* `TextDetBase.forward(img_in) -> (blks, mask, lines_map)` (basemodel.py:240-244) on DEVICE memory, in stream order.
 * x     : DEVICE f32 [n][3][ph][pw], contiguous NCHW, 16-byte aligned: the BGR tensor preprocess_img makes (values
 *         in [0, 1] for a page; any float is taken).  The engine reads it as it is, rounded to fp16 in
 *         CTD_PREC_FP16_TC and exact in the other precisions; for x = float(u8) / 255 the outputs are bit-identical
 *         to ctd_forward on the u8 pages.
 * stream: the caller's cudaStream_t (NULL: the legacy default stream).  The engine stream first waits for the work
 *         enqueued on it so far, then runs an input pre-pass into the engine's staging page, the forward (its CUDA
 *         graph with use_graph), and device-to-device copies into blks / mask / lines (DEVICE, the layouts of
 *         ctd_get_net_outputs; any may be NULL to skip it); `stream` then waits for those copies.  No host
 *         synchronisation.  Post-processing runs as ctd_config::debug_skip_postproc says.  Shape and batch limits are
 *         ctd_forward's.                                                                        */
CTD_API int ctd_forward_tensor(ctd_handle* h, const float* x, int32_t n, int32_t ph, int32_t pw, void* stream,
                               float* blks, float* mask, float* lines);

/* ctd_forward_tensor for a float16 network: x is DEVICE f16 [n][3][ph][pw] (contiguous NCHW, 16-byte aligned; the
 * tensor `preprocess_img(half=True)` makes) and blks / mask / lines are DEVICE f16 in the layouts of
 * ctd_get_net_outputs.  The engine widens every input value exactly to float and runs what ctd_forward_tensor runs on
 * that float32 tensor; each output is that forward's float32 output rounded to nearest even, written by a conversion
 * kernel in place of the device-to-device copy.  Stream order, limits and NULL outputs as ctd_forward_tensor.          */
CTD_API int ctd_forward_tensor_f16(ctd_handle* h, const void* x, int32_t n, int32_t ph, int32_t pw, void* stream,
                                   void* blks, void* mask, void* lines);

/* `postprocess_mask` (inference.py:85-99): (mask*255) truncated to u8, [n][h][w], HOST.   */
CTD_API int ctd_get_mask_u8(ctd_handle* h, uint8_t* mask_u8);

/* `postprocess_yolo` up to the numpy conversion (inference.py:101-105) =
 * `non_max_suppression(det, conf, iou)[i]` (utils/yolov5_utils.py:124-218): rows
 * [x1,y1,x2,y2,conf,cls] f32, score-descending, at most 300 per page.
 * det: HOST f32 [n][300][6]; det_count: HOST i32 [n].                                      */
CTD_API int ctd_get_detections(ctd_handle* h, float* det, int32_t* det_count);
/* Candidate capacity of the NMS stage.  The reference keeps up to max_nms = 30000 candidates per page
 * (yolov5_utils.py:143,191-194); this engine holds *cap = 4096.  A page with more rows above conf_thresh keeps
 * exactly the 4096 best by (score descending, row ascending) -- deterministic, and identical to the reference
 * whenever the reference's own 300-detection cut (max_det) is reached inside those rows.  cand_total: HOST i32 [n],
 * the number of candidates each page of the last forward (or the last ctd_nms call, n = 1) really had, so a caller
 * can detect cand_total[i] > *cap.  Either pointer may be NULL.                                */
CTD_API int ctd_get_nms_status(ctd_handle* h, int32_t* cand_total, int32_t* cap);

/* `SegDetectorRepresenter.binarize` + connected components of the shrink map
 * (db_utils.py:71-72 and the labelling findContours/connectedComponents imply):
 * bitmap u8 [n][h][w] (0/1), labels i32 [n][h][w] numbered like
 * cv2.connectedComponents(connectivity=8) (0 = background), n_labels i32 [n] (incl. bg).
 * Any pointer may be NULL.  The forward counts the components; the label plane is numbered
 * by this call, on the engine's stream, only when `labels` is given.                       */
CTD_API int ctd_get_db_components(ctd_handle* h, uint8_t* bitmap, int32_t* labels, int32_t* n_labels);

/* `SegDetectorRepresenter.__call__` -> `boxes_from_bitmap` (db_utils.py:40-69,123-166) on the shrink map of
 * the last forward: per page the contours in OpenCV's findContours(RETR_LIST) order, capped at 1000
 * (max_candidates); rows of skipped contours (short side < 2) are zero with score 0 exactly like the
 * reference.  boxes: HOST i16 [n][1000][4][2] (x,y; order TL,TR,BR,BL), scores: HOST f32 [n][1000],
 * counts: HOST i32 [n] = min(#contours, 1000).  The box_thresh (0.6) filter of inference.py:159-161 is
 * left to the caller, as in the reference.                                                        */
CTD_API int ctd_get_text_lines(ctd_handle* h, int16_t* boxes, float* scores, int32_t* counts);

/* Stand-alone `cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)` for u8 images with 1 or 3 channels
 * (HOST in, HOST out); bit-exact with OpenCV 4.x, see csrc/resize.cu.                                            */
CTD_API int ctd_resize_linear_u8(ctd_handle* h, const uint8_t* src, int32_t sh, int32_t sw, int32_t channels, uint8_t* dst,
                                 int32_t dh, int32_t dw);

/* Several handles on ONE GPU (one workspace each) let independent batches overlap: the kernels of batch i+1 fill the
 * tails and dependency gaps of batch i (+8 % pages/s with two handles, bench.py).  ctd_join makes everything
 * enqueued so far on `other`'s stream a dependency of `h`'s stream (device-side, no host wait) -- used to close a
 * timed region or to hand results over.                                                         */
CTD_API int ctd_join(ctd_handle* h, ctd_handle* other);

/* Device-side timing of the last ctd_forward (CUDA events on the engine stream), ms.       */
CTD_API int ctd_last_forward_ms(ctd_handle* h, float* ms);
/* Number of kernels the last ctd_forward launched (graph nodes when captured).             */
CTD_API int ctd_last_launch_count(ctd_handle* h, int32_t* launches);
/* Debug/bisect: copy activation buffer `buf` of the last forward to HOST as f32 NHWC.      */
CTD_API int ctd_debug_read_buffer(ctd_handle* h, int32_t buf, float* out, size_t out_elems);
/* Debug/unit tests: fill activation buffer `buf` (f32 NHWC on the host, converted to the engine's
 * storage type) for a forward of shape (n, ph, pw); used with programs that have no STEM op.  */
CTD_API int ctd_debug_write_buffer(ctd_handle* h, int32_t buf, const float* in, int32_t n, int32_t ph, int32_t pw);

/* Debug/unit tests: run only ops [first_op, last_op] of the program on the CURRENT buffer contents (fill sources
 * with ctd_debug_write_buffer, read the result with ctd_debug_read_buffer): one launch plan of the real network at
 * the real shape, checked in isolation.  `pages` (HOST u8 [n][ph][pw][3]) may be NULL unless the range contains
 * the STEM op.  Synchronous, never graph-captured, no post-processing.                              */
CTD_API int ctd_debug_run_ops(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw, int32_t first_op,
                              int32_t last_op);

/* Debug/unit tests: the post-processing stage of a forward on caller-supplied network outputs.  blks HOST f32
 * [n][rows_per_image][5 + nc] (the Detect rows), lines HOST f32 [n][2][ph][pw] (the DB maps); (n, ph, pw) obey
 * ctd_forward's shape rules.  Uploads both, writes the bitmap as lines[:, 0] > db_thresh (the DB tail's comparison)
 * and runs the forward's own NMS and DB post-processing (CCL + text-line boxes) on the engine stream, then
 * synchronises: ctd_get_detections, ctd_get_nms_status, ctd_get_db_components and ctd_get_text_lines read the
 * results.  Refused (CTD_E_INVALID) on a debug_skip_postproc engine.                                      */
CTD_API int ctd_debug_postprocess(ctd_handle* h, const float* blks, const float* lines, int32_t n, int32_t ph, int32_t pw);

/* Test hook: copies `bytes` bytes at `offset` of one of a collected slot's device buffers to host memory `out`,
 * synchronously.  plane 0: the packed pages (pg_in); 1: the results frame (pg_res: masks | mask_refined);
 * 2: the engine's net input of its last forward (d_pages, n x net_h x net_w x 3).  CTD_E_INVALID while the slot
 * has an uncollected submission, or for a range past the buffer's current size. */
CTD_API int ctd_debug_read_slot(ctd_handle* h, int32_t slot, int32_t plane, size_t offset, uint8_t* out, size_t bytes);

/* ---- measurement / interop ------------------------------------------------------------------
 * CUDA-event timer on the ENGINE stream (bench.py times K forwards between start and stop).    */
CTD_API int ctd_timer_start(ctd_handle* h);
CTD_API int ctd_timer_stop(ctd_handle* h, float* ms); /* synchronises the engine stream          */
/* One un-graphed forward with an event after every op: op_ms[i] = device ms of op i; the two
 * entries after the last op are the NMS and the CCL stage.  cap >= n_ops + 2.                   */
CTD_API int ctd_profile_forward(ctd_handle* h, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw,
                                int32_t pages_on_device, float* op_ms, int32_t cap);

/* ---- stand-alone array kernels (stage-isolated parity; same kernels the pipeline uses) --
 * cv2.connectedComponentsWithStats(img, connectivity=8, ltype=CV_32S) as the reference
 * effectively calls it (utils/textmask.py:93,113,138; SURVEY App. D #16).
 * img u8 [h][w] (non-zero = foreground), HOST pointers.  labels i32 [h][w];
 * stats i32 [n_labels][5] = x,y,w,h,area (row 0 = background); returns count in *n_labels.
 * `stats_cap` = rows available in `stats`.  Images of at most 2^28 pixels (CTD_E_SHAPE beyond).     */
CTD_API int ctd_connected_components(ctd_handle* h, const uint8_t* img, int32_t ih, int32_t iw, int32_t* labels,
                             int32_t* stats, int32_t stats_cap, int32_t* n_labels);

/* Stage-isolated form of the above on a caller-supplied probability map (HOST f32 [ih][iw]):
 * binarize(pred > thresh) -> contours -> boxes/scores, as `SegDetectorRepresenter(thresh).__call__`
 * would return for one image.  boxes i16 [1000][4][2], scores f32 [1000], *count = rows used.  Maps of at most
 * 2048 x 2048 that fit the engine's max_h * max_w pixels (CTD_E_CAPACITY beyond).                        */
CTD_API int ctd_seg_represent(ctd_handle* h, const float* pred, int32_t ih, int32_t iw, float thresh, int16_t* boxes,
                              float* scores, int32_t* count);

/* `refine_mask(img, pred_mask, blk_list, refine_mode)` (utils/textmask.py:159-169): img HOST u8 [ih][iw][3]
 * BGR, mask HOST u8 [ih][iw], windows HOST i32 [n_win][4] = `expand_textwindow(img.shape, blk.xyxy, 16)` of
 * every block (python slice semantics), refine_mode 0 = REFINEMASK_INPAINT, 1 = REFINEMASK_ANNOTATION.
 * out HOST u8 [ih][iw] = mask_refined.  Windows follow python slice semantics (negative bounds wrap).          */
CTD_API int ctd_refine_mask(ctd_handle* h, const uint8_t* img, const uint8_t* mask, int32_t ih, int32_t iw,
                            const int32_t* windows, int32_t n_win, int32_t refine_mode, uint8_t* out);

/* ---- line -> block grouping (host C++, no GPU needed) ---------------------------------------------
 * `group_output(blks, lines, im_w, im_h, mask, sort_blklist)` (utils/textblock.py:421-508) with its callees
 * examine_textblk / split_textblk / try_merge_textline / merge_textlines / sort_textblk_list (267-419) and
 * TextBlock.adjust_bbox / sort_lines (87-105).  One record per resulting TextBlock, field for field
 * (utils/textblock.py:12-85; only the fields group_output assigns are carried).                      */
typedef struct ctd_block {
  int32_t xyxy[4];       /* TextBlock.xyxy                                                  */
  int32_t language;      /* index into LANG_LIST = ['eng', 'ja', 'unknown'] (textblock.py:9) */
  int32_t vertical;      /* TextBlock.vertical                                              */
  int32_t angle;         /* TextBlock.angle (degrees)                                       */
  int32_t merged;        /* TextBlock.merged                                                */
  int32_t n_lines;       /* len(TextBlock.lines); rows line_off .. line_off+n_lines-1 of `lines_out` */
  int32_t line_off;
  int32_t n_dist;        /* len(TextBlock.distance) (differs from n_lines for split blocks: the reference
                            deep-copies the parent's distance array, textblock.py:397,412)   */
  int32_t dist_off;
  int32_t font_is_float; /* python type of font_size: int until try_merge_textline averages it */
  int32_t reserved;
  double font_size;      /* TextBlock.font_size                                             */
  double vec[2];         /* TextBlock.vec                                                   */
  double norm;           /* TextBlock.norm                                                  */
  double weight;         /* TextBlock.weight (reading-order key, -1 when sort_blklist = 0)  */
} ctd_block;

/* Capacity of one page's block section in the result arena / of ctd_detect_page's outputs: the reference produces
 * at most max_det (300) detector blocks + one block per text line left over (<= 1000 lines, db_utils.py max_candidates). */
#define CTD_MAX_BLOCKS 1300
#define CTD_MAX_BLOCK_DIST 8192
/* header of a page's block section (see ctd_results_layout); flags bit 0: the distance arrays did not fit and were
 * dropped (n_dist = 0 in every record), bit 1: group_output failed for the page (n_blocks = 0).                 */
typedef struct ctd_page_blocks {
  int32_t n_blocks, n_lines, n_dist, flags;
} ctd_page_blocks;

/* blk_xyxy i32 [n_blk][4], blk_cls i32 [n_blk]: the detector rows after postprocess_yolo (inference.py:101-114);
 * lines i32 [n_lines][4][2]: the kept text-line quads in page coordinates; mask u8 [im_h][im_w] or NULL.
 * Results: blocks_out[*n_blocks], lines_out i32 [..][4][2], dist_out f64 [..].  Returns CTD_E_CAPACITY (with
 * *n_blocks set) when an output array is too small: blocks <= n_blk + n_lines, lines <= n_lines + n_blk,
 * distances <= (n_lines + n_blk) * max lines per block.  Pure host code, thread-safe, needs no handle. */
CTD_API int ctd_group_output(const int32_t* blk_xyxy, const int32_t* blk_cls, int32_t n_blk, const int32_t* lines,
                             int32_t n_lines, int32_t im_w, int32_t im_h, const uint8_t* mask, int32_t sort_blklist,
                             ctd_block* blocks_out, int32_t blocks_cap, int32_t* lines_out, int32_t lines_cap,
                             double* dist_out, int32_t dist_cap, int32_t* n_blocks);

/* ---- the whole of `TextDetector.__call__` (inference.py:141-178) ---------------------------------------------
 * One page of any size: letterbox + forward + post-processing on the GPU, postprocess_yolo casts / box_thresh /
 * group_output / expand_textwindow on the host (C++), refine_mask (and, with keep_undetected != 0,
 * refine_undetected_mask, textmask.py:135-156) on the GPU with the page and its mask resident in HBM.
 * page HOST u8 [ih][iw][3] BGR; net_h x net_w = the detector's input_size (<= the engine's max shape, multiples of
 * 64); mask_out / mask_refined_out HOST u8 [ih][iw] (mask_out is the page-sized mask, modified in place by
 * refine_undetected_mask exactly like the reference's); blocks / lines_out / dist_out as ctd_group_output.
 * Blocking.  Returns CTD_E_CAPACITY with *n_blocks set when an output array is too small (CTD_MAX_BLOCKS blocks and
 * lines, CTD_MAX_BLOCK_DIST distances always suffice).  With keep_undetected != 0 the page may have at most 2^28
 * pixels (16384 x 16384; an A4 page at 600 dpi has 34.8 M): refine_undetected_mask labels the whole page with the
 * connected-components kernels, whose pixel and label indices are int; a larger page returns CTD_E_CAPACITY.     */
CTD_API int ctd_detect_page(ctd_handle* h, const uint8_t* page, int32_t ih, int32_t iw, int32_t net_h, int32_t net_w,
                            int32_t refine_mode, int32_t keep_undetected, uint8_t* mask_out, uint8_t* mask_refined_out,
                            ctd_block* blocks, int32_t blocks_cap, int32_t* lines_out, int32_t lines_cap, double* dist_out,
                            int32_t dist_cap, int32_t* n_blocks);

/* Batches of NET-SIZED pages through the same chain, two batches in flight per handle (throughput form of the
 * above).  ctd_submit_full returns at once: the H2D of host pages runs on a copy stream, the forward + device
 * post-processing on the engine stream, the D2H of the phase-A section on a second copy stream, and a worker thread of
 * the handle runs the host stage when those results arrive and enqueues refine_mask; ctd_collect(h, slot) blocks until
 * `results_host` is complete.  slot is 0 or 1; a slot must be collected before it is submitted again.  Submissions
 * execute in order; ctd_get_* after a submit refer to the most recently submitted batch.
 * results_host: HOST (pinned) buffer of ctd_results_layout().total_bytes:
 *   [0, phase_a_bytes)  mask_u8 | det | det_count | n_labels | line_boxes | line_scores | line_count
 *   mask_refined        u8 [n][ph][pw]
 *   blocks + i*blocks_stride   page i: ctd_page_blocks header, ctd_block[CTD_MAX_BLOCKS] at +blk_records_off,
 *                       i32 lines [..][4][2] at +blk_lines_off, f64 distances at +blk_dist_off
 * pages: HOST (pinned) pointer, or with pages_on_device != 0 a DEVICE pointer that must stay valid until the slot
 * is collected (refine_mask reads the pages in place).  The same bytes exist on the device (ctd_device_arena) once
 * the slot is collected, so a multi-GPU caller can gather a rank's complete results with one NCCL call.    */
typedef struct ctd_results_layout_t {
  int32_t max_batch, max_h, max_w, reserved;
  size_t total_bytes, phase_a_bytes;
  size_t mask_u8, det, det_count, n_labels, line_boxes, line_scores, line_count;  /* sized for max_batch x max_h x max_w */
  size_t mask_refined, blocks, blocks_stride, blk_records_off, blk_lines_off, blk_dist_off;
} ctd_results_layout_t;
CTD_API int ctd_results_layout(ctd_handle* h, ctd_results_layout_t* out);
CTD_API int ctd_submit_full(ctd_handle* h, int32_t slot, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw,
                            int32_t pages_on_device, int32_t refine_mode, void* results_host);
/* Blocks until the batch submitted on `slot` (ctd_submit_full or ctd_submit_pages) is complete; returns its error.  */
CTD_API int ctd_collect(ctd_handle* h, int32_t slot);
/* Device copy of slot `slot`'s complete results (same layout) and the stream its last writes were enqueued on.   */
CTD_API int ctd_device_arena(ctd_handle* h, int32_t slot, void** base, void** post_stream);

/* Batches of pages of ANY size through the whole chain, two batches in flight per handle: per page the same results
 * as ctd_detect_page, byte for byte.
 *
 * ctd_pages_plan (host code, no handle, thread-safe, needs no GPU) lays a batch out.  The caller fills ih, iw of each
 * entry; the plan fills the rest.  Every offset is a multiple of 256.
 *   input  (*input_bytes):   page i, u8 BGR [ih][iw][3], at page_off
 *   results (*results_bytes): page i's u8 [ih][iw] mask at mask_off and mask_refined at refined_off, and its block
 *                            section (ctd_page_blocks header, ctd_block records at +blk_records_off, i32 lines
 *                            [..][4][2] at +blk_lines_off, f64 distances at +blk_dist_off; ctd_results_layout gives
 *                            these offsets, which do not depend on the handle) at blocks_off
 * The page's pixel offsets inside the image and mask planes agree: page_off / 3 == mask_off - mask_off of page 0.
 * Returns CTD_E_SHAPE where ctd_detect_page does: a page side < 1, a side that letterboxes to 0 px, or a net side
 * that is not a positive multiple of 64.                                                                          */
typedef struct ctd_page_entry {
  int32_t ih, iw;                  /* in : page size (u8 BGR HWC)                                               */
  int32_t unpad_h, unpad_w;        /* out: letterbox size, round(size * r), half to even (imgproc_utils.py:86-117) */
  int64_t page_off;                /* out: byte offset of the page in the packed input buffer                   */
  int64_t mask_off, refined_off;   /* out: page-sized u8 mask / mask_refined in the results buffer              */
  int64_t blocks_off;              /* out: the page's block section in the results buffer                       */
} ctd_page_entry;
CTD_API int ctd_pages_plan(ctd_page_entry* pages, int32_t n, int32_t net_h, int32_t net_w, size_t* input_bytes,
                           size_t* results_bytes);
/* ctd_submit_pages (declared below with ctd_device_page) is asynchronous: the batch runs like a ctd_submit_full batch
 * and is collected with ctd_collect(h, slot), after which `results_host` holds every page's mask (modified by
 * refine_undetected_mask when keep_undetected != 0, as in ctd_detect_page), mask_refined and block section.  pages / n:
 * the planned entries (checked against a fresh plan); input_host: the packed pages (pinned, input_bytes);
 * results_host: pinned, results_bytes.  Both buffers must stay untouched until the slot is collected.  On the GPU: one
 * letterbox launch for the batch, the forward at (n, net_h, net_w), one launch back-projecting every page's mask to
 * its size, one refine_mask launch for every window of every page.  Same checks as ctd_submit_full (slot 0/1 and
 * collected, n <= max_batch, net shape <= the engine's max shape, not a debug_skip_postproc engine), and with
 * keep_undetected != 0 ctd_detect_page's page-size limit (2^28 pixels per page, CTD_E_CAPACITY beyond).           */

/* ---- text-line crops for OCR (SURVEY 8f row f4) ----------------------------------------------------------------
 * `TextBlock.get_transformed_region(img, idx, textheight)` (utils/textblock.py:162-194): line `idx` of a block, pushed
 * out by font_size / 3 for 'eng' (and horizontal 'unknown') blocks and clipped to [0, im_w] x [0, im_h], cut out of the
 * page with `cv2.findHomography(src, dst, RANSAC, 5.0)` + `cv2.warpPerspective(img, M, (w, h))` (INTER_LINEAR,
 * BORDER_CONSTANT 0) at a fixed text height (h = textheight for horizontal lines, w = textheight for vertical ones,
 * the other side from the line's aspect ratio), vertical crops rotated 90 degrees counter-clockwise.
 *
 * ctd_region_plan (host C++, no handle, thread-safe, needs no GPU) does the geometry: for every requested line the
 * output shape, the homography bit-identical to cv2.findHomography's (OpenCV's normalised 4-point DLT with its Jacobi
 * eigen solver) and the inverse cv2.warpPerspective samples with (cv2.invert, DECOMP_LU), plus the crop's offset in one
 * packed u8 buffer (*total_bytes = its size).  A line on which the reference raises (findHomography returns None when
 * w == 1 or h == 1; a zero or non-finite aspect ratio) gets status 1 and no bytes; a crop with a side of 32767 px or more
 * gets status 2 (OpenCV's 16-bit remap coordinates do not reach it).  When the rounded size is 0 the crop has the page's
 * shape, as cv2 gives it for an empty dsize.  Returns CTD_E_INVALID for textheight < 2 (unused by any caller: the
 * reference then either raises or returns that page-sized crop) and for a page side < 1 or >= 32767.               */
typedef struct ctd_region_line {   /* one requested line: TextBlock.lines[idx] + the block fields the method reads */
  double quad[8];                  /* x1 y1 .. x4 y4 (TL, TR, BR, BL)                                                 */
  int32_t language, vertical;      /* LANG_LIST index, TextBlock.vertical                                             */
  double font_size;                /* TextBlock.font_size (an int, or a float after a merge)                          */
} ctd_region_line;
typedef struct ctd_region {
  int32_t out_h, out_w;            /* shape of the returned array (after the rotation, after the dsize-empty rule)    */
  int32_t rotate;                  /* 1: vertical direction                                                           */
  int32_t status;                  /* 0 ok, 1 the reference raises on this line, 2 too large (see above)              */
  int64_t offset;                  /* byte offset of this crop in the packed output (out_h * out_w * 3 bytes, HWC)    */
  double homography[9];            /* as cv2.findHomography returns it                                                */
  double inverse[9];               /* as cv2.invert(M, DECOMP_LU) returns it; what the kernel reads                   */
} ctd_region;
CTD_API int ctd_region_plan(const ctd_region_line* lines, int32_t n, int32_t im_w, int32_t im_h, int32_t textheight,
                            ctd_region* out, size_t* total_bytes);
/* One launch warps every planned crop (status 0) of the page into `pixels_out` (HOST, the plan's packed layout; bytes
 * of regions with status != 0 are not written).  page: u8 BGR [ih][iw][3], a HOST pointer, or with page_on_device != 0
 * a DEVICE pointer on the handle's GPU.  Blocking.  Bit-exact with cv2.warpPerspective(img, M, (w, h)) + cv2.rotate
 * for the plan's `inverse` (csrc/region.cu).  CTD_E_CAPACITY if pixels_bytes is smaller than the plan's total,
 * CTD_E_SHAPE for a bad page size, CTD_E_INVALID for a malformed plan entry.                                       */
CTD_API int ctd_transform_regions(ctd_handle* h, const uint8_t* page, int32_t ih, int32_t iw, int32_t page_on_device,
                                  const ctd_region* plan, int32_t n, uint8_t* pixels_out, size_t pixels_bytes);
/* ctd_submit_pages with a textheight also cuts the OCR crops of every text line of every page of the batch; with
 * textheight = 0 it cuts none.  textheight >= 2 (else CTD_E_INVALID): the handle's worker plans each page's lines with
 * ctd_region_plan right after its group_output, on the same host threads, then one k_warp_regions launch on the post
 * stream cuts every status-0 crop of every page out of the pages where they already are in device memory, and the
 * pixels are copied back into a pinned buffer of the handle before the batch counts as done.  A batch without a single
 * crop launches and allocates nothing.  A page the planner refuses (a side >= 32767) fails the batch, and ctd_collect
 * names the page.
 * After ctd_collect(h, slot) of a ctd_submit_pages batch with textheight > 0: the concatenated ctd_region
 * plans of the batch, *n_regions entries in page, then block, then line order (the order of each page's block
 * section), page i's entries at [(*page_first)[i], (*page_first)[i + 1]) (n + 1 values), and the packed crops,
 * *bytes bytes at *pixels (HOST, NULL when *bytes is 0).  Each entry's offset is relative to *pixels; page i's crops
 * follow page i - 1's.  Entries with status != 0 have no bytes, exactly as ctd_region_plan gives them.  All pointers
 * belong to the handle and stay valid until the slot's next submission or ctd_destroy.  The same after a
 * ctd_submit_regions batch.  CTD_E_INVALID for a slot that is in flight or whose last collected batch did not ask for
 * crops.                                                                                                         */
CTD_API int ctd_collect_regions(ctd_handle* h, int32_t slot, const ctd_region** plan, int32_t* n_regions,
                                const int32_t** page_first, const uint8_t** pixels, size_t* bytes);

/* ---- pages and results in device memory ------------------------------------------------------------------------
 * A page that is already on the GPU (decoded there, or made by an earlier GPU stage) goes into a batch without a trip
 * through host memory, and the masks and crops of a batch can stay on the GPU for the next model (OCR, inpainting).
 *
 * ctd_device_page describes page i of a batch: `data` is the DEVICE address of pixel (0, 0), channel 0 (B) of the u8
 * BGR page, or NULL when the page is in `input_host` at its page_off.  Byte (y, x, c) is at
 * data + y * stride_h + x * stride_w + c * stride_c (each stride >= 0: a sub-window of a larger image, a permuted
 * channels-first image).  `event` (a cudaEvent_t, may be NULL) is waited on by the engine stream before the page is
 * read, so a page still being written by a kernel on the caller's stream is read after that kernel.               */
typedef struct ctd_device_page {
  const uint8_t* data;
  int64_t stride_h, stride_w, stride_c;
  void* event;
} ctd_device_page;
/* The batch entry point (see ctd_pages_plan and the crops above), with pages in device memory and, optionally,
 * results left there.
 *   dev: n entries (NULL: every page is in input_host).  input_host may be NULL when every page is on the device;
 *        then no page byte is copied from the host, and a mixed batch copies only its host pages' byte ranges.  Each
 *        device page must be device memory of the handle's GPU (checked with cudaPointerGetAttributes, else
 *        CTD_E_INVALID naming the page) and must stay unwritten until the slot is collected.  One gather launch on
 *        the engine stream copies every device page into the slot's packed page buffer after the waits on the pages'
 *        events and after the host pages' copy; letterbox, refine_mask and the crops read that buffer as before.
 *   results_on_device != 0: mask_refined, the mask refine_undetected_mask modified (keep_undetected) and the crop
 *        pixels are NOT copied to the host; results_host still gets the phase-A rows, the masks group_output reads
 *        and the block sections, and ctd_collect_regions gives the plan with *pixels = NULL and *bytes = the batch's
 *        crop bytes on the device.  Fetch the device results with ctd_collect_device after ctd_collect.
 * With dev = NULL and results_on_device = 0 the pages come from input_host and every result goes to results_host.   */
CTD_API int ctd_submit_pages(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, int32_t net_h,
                             int32_t net_w, const uint8_t* input_host, const ctd_device_page* dev, int32_t refine_mode,
                             int32_t keep_undetected, int32_t textheight, int32_t results_on_device,
                             void* results_host);
/* After ctd_collect(h, slot) of a results_on_device batch: copies into page_dst[i] (a DEVICE buffer on the handle's
 * GPU, one per page of the batch) page i's [mask ih*iw | mask_refined ih*iw | the page's crops, packed as the plan
 * lays them out, offsets relative to the page's first plan entry].  The mask is the one refine_undetected_mask
 * modified when the batch asked for it.  After a ctd_submit_regions batch page_dst[i] gets only page i's crops, and
 * may be NULL when the page has none.  Blocks until the copies are done, so the buffers may then be used on any
 * stream.  CTD_E_INVALID for a slot in flight or whose last batch was not submitted with results_on_device.       */
CTD_API int ctd_collect_device(ctd_handle* h, int32_t slot, void* const* page_dst);

/* ---- refine_mask on any block list (utils/textmask.py:135-169) ------------------------------------------------------
 * `refine_mask(img, pred_mask, blk_list, refine_mode)` and `refine_undetected_mask(img, mask_pred, mask_refined,
 * blk_list, refine_mode)` for pages, masks and blocks the caller gives: a block list edited after detection (SFX blocks
 * dropped, a missed block added, blocks merged or moved), or one read back from `model2annotations`'s json.
 *
 * ctd_refine_plan (host code, no handle, thread-safe, needs no GPU) lays a batch out and checks its blocks.  The
 * caller fills ih, iw of each entry (any page of at least 1 x 1: there is no letterbox); the plan fills the rest, with
 * the pixel offsets of ctd_pages_plan (unpad_h, unpad_w and blocks_off are 0).  Every offset is a multiple of 256.
 * With T = *results_bytes / 2:
 *   input  (*input_bytes = 5 T): page i, u8 BGR [ih][iw][3], at page_off; then at byte 3 T a frame laid out as the
 *                                results: its u8 [ih][iw] mask at 3 T + mask_off and, for a refined input, its
 *                                mask_refined at 3 T + refined_off
 *   results (*results_bytes):    page i's mask at mask_off, mask_refined at refined_off
 * xyxy: the block boxes, i32 [sum n_blocks][4], page 0's n_blocks[0] blocks first.  For each block it writes the
 * window refine_mask refines, expand_textwindow(img.shape, xyxy, 16) (windows, i32 [.][4], before Python's slice
 * normalisation, clamped to int32), and a status: 0 the window is fine; 1 the reference raises on the block (the window
 * is empty after Python's slice normalisation, e.g. y2 <= y1 or an x2 + pad that wraps negative: cv2.cvtColor raises
 * on the empty crop); 2 a window coordinate does not fit int32.  CTD_E_SHAPE for a page side < 1.                  */
CTD_API int ctd_refine_plan(ctd_page_entry* pages, int32_t n, const int32_t* xyxy, const int32_t* n_blocks,
                            int32_t* windows, int32_t* status, size_t* input_bytes, size_t* results_bytes);
/* ctd_submit_refine runs refine_mask on a planned batch through the schedule of ctd_submit_pages (slots 0 and 1, two
 * batches in flight, collected with ctd_collect and, with results_on_device, ctd_collect_device, which then gives each
 * page's [mask | mask_refined]).  pages / n / xyxy / n_blocks: the planned entries and the boxes they were planned
 * with (checked against a fresh plan).  Pages come from input_host or from device memory (dev_pages, as
 * ctd_submit_pages takes them); masks from input_host's frame or from device memory (dev_masks, NULL or n entries:
 * u8 [ih][iw] at data + y * stride_h + x * stride_w, any strides, stride_c not read, e.g. channel 0 of a page).  One
 * gather launch on the engine stream packs every device page and mask, after the waits on their events.
 * On the GPU: one refine_mask launch over the windows of every block of every page; with keep_undetected != 0 then
 * refine_undetected_mask against the caller's boxes, which modifies the mask in place as the reference does.  With
 * refined_input != 0 (needs keep_undetected and input_host) the frame's mask_refined is an input, refine_mask does not
 * run, and refine_undetected_mask alone modifies both masks.  results_host (pinned, results_bytes): mask_refined, and
 * with keep_undetected the modified mask.  No network runs: a handle of any program (a kernels-only one too) takes it.
 * Refused before any GPU work: a block of status != 0 unless refined_input (CTD_E_INVALID, ctd_last_error names the
 * page and the block), n > max_batch (CTD_E_CAPACITY), and with keep_undetected a page of more than 2^28 pixels
 * (CTD_E_CAPACITY, as ctd_detect_page).  Both buffers and the device images stay untouched until the slot is
 * collected.                                                                                                       */
CTD_API int ctd_submit_refine(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, const int32_t* xyxy,
                              const int32_t* n_blocks, const uint8_t* input_host, const ctd_device_page* dev_pages,
                              const ctd_device_page* dev_masks, int32_t refine_mode, int32_t keep_undetected,
                              int32_t refined_input, int32_t results_on_device, void* results_host);

/* ---- text-line crops of any block list ---------------------------------------------------------------------------
 * ctd_submit_regions cuts the OCR crops of lines the caller gives (a block list edited after detection, or read back
 * from `model2annotations`'s json) through the schedule of ctd_submit_pages (slots 0 and 1, two batches in flight).
 *   pages / n:  the planned entries of ctd_refine_plan for these pages with no blocks (checked against a fresh plan);
 *               any page of at least 1 x 1 with both sides < 32767 (else CTD_E_SHAPE naming the page).
 *   lines:      ctd_region_line records of every line of every block of every page, page 0's first, n_lines[i] of
 *               page i (block then line order within a page, as each page's plan entries are given back).
 *   pages in:   page i from input_host at its page_off (pinned, the first 3 / 5 of ctd_refine_plan's input_bytes), or
 *               from device memory (dev_pages, NULL or n entries as ctd_submit_pages takes them, checked the same way;
 *               the engine waits on each page's event).  A device page is read where it is, with its strides.
 * The handle's worker plans each page's lines with ctd_region_plan on its host threads, then one k_warp_regions launch
 * cuts every status-0 crop of the batch.  Collect with ctd_collect, then ctd_collect_regions (the plan, page_first and,
 * unless results_on_device, the host pixels) or, with results_on_device, ctd_collect_device, which gives page_dst[i]
 * only page i's packed crops (a page without crop bytes may have a NULL page_dst[i]).  Status 1 and 2 lines get no
 * bytes, exactly as ctd_region_plan gives them.  No network runs: a handle of any program takes it.
 * Refused before any GPU work: textheight < 2 (CTD_E_INVALID), n > max_batch (CTD_E_CAPACITY), a page side < 1 or
 * >= 32767 (CTD_E_SHAPE), and a device page that is not memory of the handle's GPU (CTD_E_INVALID).  input_host and
 * the device pages must stay untouched until the slot is collected.                                               */
CTD_API int ctd_submit_regions(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n,
                               const ctd_region_line* lines, const int32_t* n_lines, int32_t textheight,
                               const uint8_t* input_host, const ctd_device_page* dev_pages, int32_t results_on_device);

/* ---- the detector's post-processing on a caller's network outputs ------------------------------------------------
 * ctd_submit_outputs runs everything TextDetector.__call__ does after `self.net(img_in)` (inference.py:148-178) on
 * outputs the caller computed (this engine's TextDetBase, or any other runtime): NMS, postprocess_mask, the DB
 * threshold, connected components and text-line boxes, the box_thresh filter, the mask crop and resize back to the
 * page, the line rescale, group_output, refine_mask and refine_undetected_mask, and with a textheight the crops.  It
 * takes the arguments of ctd_submit_pages (the same ctd_pages_plan entries for (net_h, net_w), page buffers, slots and
 * collect calls: ctd_collect, ctd_collect_regions, ctd_collect_device) plus one ctd_net_output per page, and its results
 * are laid out as theirs.  Instead of the letterbox and the forward, one launch stages every page's outputs into the
 * handle's post-processing workspace; the rest of the batch is that of ctd_submit_pages.
 *
 * ctd_net_output describes the outputs of page i, float32 with element strides (each >= 0):
 *   blks:  element (r, c), r < rows, c < 5 + nc, at blks + r * blks_stride_r + c * blks_stride_c; 0 <= rows <=
 *          3 * (net_h/8 * net_w/8 + net_h/16 * net_w/16 + net_h/32 * net_w/32)
 *   mask:  the [net_h][net_w] segmentation map, (y, x) at mask + y * mask_stride_h + x * mask_stride_w
 *   lines: channel 0 of lines_map, [net_h][net_w], (y, x) at lines + y * lines_stride_h + x * lines_stride_w
 * *_on_device: 1 when the map is device memory of the handle's GPU (its first and last element are checked with
 * cudaPointerGetAttributes), 0 when it is host memory; host maps are copied on the copy stream at submission (pinned
 * memory keeps that copy asynchronous) and, like device maps, must stay unwritten until the slot is collected.
 * `event` (a cudaEvent_t, may be NULL) is waited on before the device maps are read.  A non-finite value in any map
 * fails the batch at ctd_collect (CTD_E_INVALID, naming the page of the batch and the map).  Needs a handle created
 * without debug_skip_postproc and with max_h >= net_h, max_w >= net_w; the handle's program may have no ops.         */
typedef struct ctd_net_output {
  const float* blks;
  int64_t blks_stride_r, blks_stride_c;
  const float* mask;
  int64_t mask_stride_h, mask_stride_w;
  const float* lines;
  int64_t lines_stride_h, lines_stride_w;
  int32_t rows;
  int32_t blks_on_device, mask_on_device, lines_on_device;
  void* event;
} ctd_net_output;
CTD_API int ctd_submit_outputs(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, int32_t net_h,
                               int32_t net_w, const uint8_t* input_host, const ctd_device_page* dev_pages,
                               const ctd_net_output* outs, int32_t refine_mode, int32_t keep_undetected,
                               int32_t textheight, int32_t results_on_device, void* results_host);

/* ctd_submit_outputs_dtype is ctd_submit_outputs with the element type of each page's maps in dtypes[i]
 * (ctd_submit_outputs is this call with every page CTD_DTYPE_F32):
 *   CTD_DTYPE_F32: the three maps of page i are float32, post-processed as above;
 *   CTD_DTYPE_F16: they are float16 (the ctd_net_output pointers point at float16 elements, strides count them; host
 *                  maps are copied at 2 bytes per element), post-processed with the reference's arithmetic on half
 *                  tensors (inference.py:101-114, 85-99, 158; yolov5_utils.py:136-182; db_utils.py:54-72):
 *                  candidates `obj > half(conf_thresh)`; class scores RN_half(cls * obj), the first maximal class kept
 *                  where `> half(conf_thresh)`; box corners RN_half(cx -/+ RN_half(w / 2)) and the same in y, widened
 *                  exactly to float32 before the class offset and NMS; the mask byte numpy's float16 -> uint8 cast
 *                  of RN_half(p * 255); the DB bitmap `p > half(0.3)`; contour scores on the map widened exactly to
 *                  float32 (db_utils.py:209-210).  half(x) is the handle's float32 threshold rounded to nearest even.
 * Pages of both dtypes may share a batch.  Any other dtype fails the call (CTD_E_INVALID) before any GPU work.       */
enum ctd_dtype { CTD_DTYPE_F32 = 0, CTD_DTYPE_F16 = 1 };
CTD_API int ctd_submit_outputs_dtype(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n,
                                     int32_t net_h, int32_t net_w, const uint8_t* input_host,
                                     const ctd_device_page* dev_pages, const ctd_net_output* outs,
                                     const int32_t* dtypes, int32_t refine_mode, int32_t keep_undetected,
                                     int32_t textheight, int32_t results_on_device, void* results_host);

/* ---- the detector's pre-processing: the network input preprocess_img makes ---------------------------------------
 * ctd_preprocess_pages writes, for every page of a batch, what the reference's `preprocess_img(img, (net_h, net_w))`
 * (inference.py:72-83) makes of it, into the caller's device buffer `dst`, in one launch: the letterbox (cv2.resize
 * INTER_LINEAR when the size changes, bit-exact, zero padding at the bottom and the right) in one of three layouts
 *   CTD_PRE_F32_NCHW: float32 [n][3][net_h][net_w], each u8 value v as v / 255 (the correctly rounded float32 division)
 *   CTD_PRE_F16_NCHW: float16 [n][3][net_h][net_w], that float32 value rounded to nearest even (`.half()`)
 *   CTD_PRE_U8_NHWC:  u8 [n][net_h][net_w][3], the letterboxed pixels (`to_tensor=False`)
 * reverse_channels != 0: output channel k is channel 2 - k of the page.  preprocess_img's planes come out in the page's
 * order with bgr2rgb (cvtColor, then `[::-1]`) and reversed without it; its to_tensor=False pixels the other way round.
 *   pages / n:  the ctd_pages_plan entries for (net_h, net_w) (checked against a fresh plan); page i from input_host at
 *               its page_off (pinned: input_bytes of the plan) or from device memory (dev, NULL or n entries, as
 *               ctd_submit_pages takes them; the stream waits on each page's event), packed by one gather launch.
 *   dst:        device memory of the handle's GPU, 16-byte aligned, n * 3 * net_h * net_w elements, contiguous.
 *   stream:     a cudaStream_t of the handle's GPU (NULL: the legacy default stream).
 * Everything is enqueued on `stream`: the host pages' copy, the waits, the gather and the letterbox; nothing waits on
 * the host, and the call returns before the GPU work runs.  input_host and the device pages must stay unwritten until
 * the stream has run it.  The handle's page buffer and tables are reused by the next call after an event wait on the
 * stream of this one.  No network runs: a handle of any program (a kernels-only one too) takes it.  Refused before any
 * GPU work: n > max_batch (CTD_E_CAPACITY), a net side that is not a positive multiple of 64 and a page that
 * letterboxes to 0 px (CTD_E_SHAPE), entries that are not the plan's, a device page or a dst that is not memory of
 * the handle's GPU, a dst that is not 16-byte aligned and a format that is not CTD_PRE_* (CTD_E_INVALID).          */
enum ctd_pre_format { CTD_PRE_F32_NCHW = 0, CTD_PRE_F16_NCHW = 1, CTD_PRE_U8_NHWC = 2 };
CTD_API int ctd_preprocess_pages(ctd_handle* h, const ctd_page_entry* pages, int32_t n, int32_t net_h, int32_t net_w,
                                 const uint8_t* input_host, const ctd_device_page* dev, int32_t format,
                                 int32_t reverse_channels, void* dst, void* stream);

/* utils/yolov5_utils.py:124-218 on a caller-supplied prediction tensor (HOST f32
 * [rows][5+nc]); output as ctd_get_detections for one page.  The device suppresses a box when its float32 IoU with
 * a kept box is > iou_thresh, compared in float32 (as ctd_config::nms_thresh).  torchvision's CPU nms compares the
 * float32 IoU with a double threshold t; a caller who wants that rule passes RD_f32(t), t rounded toward -inf to
 * float32 (the Python binding does).                                                        */
CTD_API int ctd_nms(ctd_handle* h, const float* pred, int32_t rows, float conf_thresh, float iou_thresh, float* det,
            int32_t* det_count);
/* ctd_nms with the element type of the rows in dtype (enum ctd_dtype; ctd_nms is this call with CTD_DTYPE_F32):
 * CTD_DTYPE_F16 rows are HOST f16 [rows][5+nc], widened exactly to float32 and taken with the float16 rules of
 * ctd_submit_outputs_dtype (half(conf_thresh), RN_half class scores and corners).  The output rows are float32 as
 * for ctd_nms.  Any other dtype fails the call (CTD_E_INVALID).                             */
CTD_API int ctd_nms_dtype(ctd_handle* h, const void* pred, int32_t rows, int32_t dtype, float conf_thresh,
                          float iou_thresh, float* det, int32_t* det_count);

/* ---- JPEG pages decoded on the GPU ------------------------------------------------------
 * The reference reads pages with io_utils.imread = cv2.imdecode(np.fromfile(path), IMREAD_COLOR).  These entry points
 * decode baseline JPEG files on the GPU to exactly the u8 BGR page cv2.imdecode returns (cv2 4.13's libjpeg-turbo:
 * ISLOW IDCT, fancy upsampling, EXIF orientation applied).  A file outside the supported set, or one whose entropy
 * data or IDCT range is not certain to decode as libjpeg-turbo's SIMD build decodes it, gets a non-zero status and
 * is left to cv2: the GPU path declines a page, it never returns a different one.
 *
 * Supported: 8-bit sequential Huffman (SOF0/SOF1), one interleaved scan, one component (B = G = R = Y) or three YCbCr
 * components with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1, any restart interval, EXIF orientations 1-8.       */
enum ctd_jpeg_status {
  CTD_JPEG_OK = 0,
  CTD_JPEG_NOT_JPEG = 1,     /* no SOI, or bytes that are not a marker where one must be                    */
  CTD_JPEG_TRUNCATED = 2,    /* ends inside a segment or the scan, no scan, or no EOI after it             */
  CTD_JPEG_PROGRESSIVE = 3,  /* SOF2 / SOF6, or a scan that is not the full spectrum                       */
  CTD_JPEG_ARITHMETIC = 4,   /* SOF9-SOF15, DAC                                                            */
  CTD_JPEG_PRECISION = 5,    /* sample precision other than 8 bits                                         */
  CTD_JPEG_LOSSLESS = 6,     /* SOF3 / SOF5 / SOF7                                                         */
  CTD_JPEG_SAMPLING = 7,     /* 4:4:0, 4:1:1 or any other sampling                                         */
  CTD_JPEG_COLOR = 8,        /* not 1 or 3 components (CMYK, YCCK), Adobe transform other than 1, R/G/B ids */
  CTD_JPEG_SCANS = 9,        /* a second scan or frame, a scan not of every component in frame order, DNL  */
  CTD_JPEG_EXIF = 10,        /* an APP1 Exif block that does not parse cleanly, two of them, or two
                                orientation entries in IFD0                                               */
  CTD_JPEG_TABLES = 11,      /* a missing or invalid Huffman / quantisation table                          */
  CTD_JPEG_ENTROPY = 12,     /* entropy-coded data not clean: restart markers out of order or missing, a
                                marker inside the scan, an invalid code, a run past coefficient 63, too few or
                                too many MCUs in an interval (set by the probe or by the GPU decode)         */
  CTD_JPEG_RANGE = 13,       /* a block whose IDCT leaves the range on which libjpeg-turbo's C and SIMD IDCTs
                                agree (GPU decode)                                                         */
  CTD_JPEG_SIZE = 14         /* a scan of 2^28 bytes or more                                               */
};
typedef struct ctd_jpeg_info {
  int32_t status;              /* ctd_jpeg_status; the fields below are set only for CTD_JPEG_OK          */
  int32_t height, width;       /* the decoded page as cv2.imdecode returns it, i.e. after the orientation   */
  int32_t frame_height, frame_width;
  int32_t components;          /* 1 or 3                                                                   */
  int32_t h_samp, v_samp;      /* luma sampling factors (chroma is 1x1); 1, 1 for one component            */
  int32_t orientation;         /* EXIF orientation 1-8 (1 without an Exif block)                           */
  int32_t restart_interval;    /* MCUs per restart interval, 0 without DRI                                 */
  int64_t ecs_bytes;           /* entropy-coded bytes of the scan, stuffing and RST markers included       */
} ctd_jpeg_info;
/* Marker walk of one file (host only, no handle, thread-safe), including the scan's restart-marker structure and
 * its EOI.  Returns 0, with the verdict in info->status; CTD_E_INVALID only for NULL arguments.                   */
CTD_API int ctd_jpeg_probe(const uint8_t* data, size_t len, ctd_jpeg_info* info);

typedef struct ctd_jpeg_decoder ctd_jpeg_decoder;
/* A decoder bound to one GPU and one stream of its own.  subsequence_bits (>= 1; 0 picks the default): the length of
 * the pieces each restart interval's bits are cut into for the parallel Huffman decode (any value decodes the same
 * pages; it only changes how many threads and rounds the decode takes).  Not thread-safe; errors via
 * ctd_last_error(NULL).                                                                                             */
CTD_API int ctd_jpeg_decoder_create(int32_t device, int32_t subsequence_bits, ctd_jpeg_decoder** out);
CTD_API void ctd_jpeg_decoder_destroy(ctd_jpeg_decoder* dec);
/* Decodes n files at once: data[i] / len[i] (host memory).  Every file whose probe status is CTD_JPEG_OK is decoded
 * into dst[i], a DEVICE buffer of height * width * 3 bytes (u8 BGR [h][w][3], the probe's oriented shape) on the
 * decoder's GPU; dst[i] may be NULL for other files.  status[i] gets the probe status or the decode's verdict
 * (CTD_JPEG_ENTROPY, CTD_JPEG_RANGE); only pages with status 0 have been written, the others are to be decoded by
 * cv2.  Blocks until every page is written, so the buffers may be used on any stream.  Staging, tables and the
 * coefficient buffer belong to the decoder and grow on demand.                                                   */
CTD_API int ctd_jpeg_decode(ctd_jpeg_decoder* dec, const uint8_t* const* data, const size_t* len, int32_t n,
                            uint8_t* const* dst, int32_t* status);

/* ---- PNG pages decoded on the GPU -------------------------------------------------------
 * These entry points decode PNG files on the GPU to exactly the u8 BGR page cv2.imdecode(buf, IMREAD_COLOR) returns
 * (cv2 4.13's libpng 1.6.53 and zlib 1.2.11): 16-bit samples keep their high byte, 1/2/4-bit grey is scaled to 8 bits,
 * grey is replicated to B = G = R, palette indices are looked up ((0, 0, 0) past the PLTE entries), alpha is dropped
 * without compositing, tRNS and gAMA have no effect, and an eXIf orientation is applied.  A file outside the supported
 * set, or one whose data is not clean, gets a non-zero status and is left to cv2: the GPU path declines a file, it
 * never returns a different one.
 *
 * Supported: non-interlaced grey 1/2/4/8/16, RGB 8/16, palette 1/2/4/8, grey+alpha 8/16 and RGBA 8/16 bits, IDAT
 * chunks in one run, at most one eXIf chunk, no APNG chunks.                                                      */
enum ctd_png_status {
  CTD_PNG_OK = 0,
  CTD_PNG_NOT_PNG = 1,     /* no PNG signature, or the first chunk is not IHDR                                  */
  CTD_PNG_TRUNCATED = 2,   /* a chunk past the end of the file, no IDAT or no IEND                              */
  CTD_PNG_HEADER = 3,      /* IHDR invalid: size, colour type / bit depth, compression, filter or interlace method */
  CTD_PNG_INTERLACED = 4,  /* Adam7                                                                             */
  CTD_PNG_APNG = 5,        /* acTL, fcTL or fdAT                                                                */
  CTD_PNG_CHUNKS = 6,      /* IDAT chunks not in one run, PLTE missing, misplaced or invalid, an unknown
                              critical chunk, a bad chunk name, a second IHDR, IEND with data                    */
  CTD_PNG_EXIF = 7,        /* an eXIf chunk that does not parse cleanly, or two of them                         */
  CTD_PNG_ZLIB = 8,        /* zlib header: CM not 8, CINFO above 7, FCHECK wrong or FDICT set                   */
  CTD_PNG_SIZE = 9,        /* a side above 1000000, more than 2^30 pixels, 2^31 or more filtered bytes, or a
                              zlib stream of 2^30 bytes or more                                                  */
  CTD_PNG_CRC = 10,        /* a chunk whose CRC does not match (decode only)                                    */
  CTD_PNG_DATA = 11        /* image data not clean (GPU decode): an invalid block type, stored length, code-length
                              set or code, a distance past the output or the window, data after the final block,
                              too few or too many bytes, a bad Adler-32, a filter type above 4                     */
};
typedef struct ctd_png_info {
  int32_t status;              /* ctd_png_status; the fields below are set only for CTD_PNG_OK               */
  int32_t height, width;       /* the decoded page as cv2.imdecode returns it, i.e. after the orientation      */
  int32_t image_height, image_width;
  int32_t bit_depth, color_type;
  int32_t orientation;         /* eXIf orientation 1-8 (1 without an eXIf chunk)                              */
  int32_t palette_entries;     /* PLTE entries, 0 without PLTE                                                */
  int64_t zlib_bytes;          /* bytes of the zlib stream, the payloads of every IDAT chunk                   */
} ctd_png_info;
/* Chunk walk of one file (host only, no handle, thread-safe); chunk CRCs are checked by ctd_png_decode only.
 * Returns 0, with the verdict in info->status; CTD_E_INVALID only for NULL arguments.                           */
CTD_API int ctd_png_probe(const uint8_t* data, size_t len, ctd_png_info* info);

typedef struct ctd_png_decoder ctd_png_decoder;
/* A decoder bound to one GPU and one stream of its own.  subsequence_bits (>= 1; 0 picks the default, 512): the
 * length of the pieces each Huffman block's bits are cut into for the self-synchronising parallel inflate (any value
 * decodes the same pages; it only changes how many threads and rounds the inflate takes).  Not thread-safe; errors
 * via ctd_last_error(NULL).                                                                                        */
CTD_API int ctd_png_decoder_create(int32_t device, int32_t subsequence_bits, ctd_png_decoder** out);
CTD_API void ctd_png_decoder_destroy(ctd_png_decoder* dec);
/* Decodes n files at once: data[i] / len[i] (host memory).  Every file whose probe status is CTD_PNG_OK is decoded
 * into dst[i], a DEVICE buffer of height * width * 3 bytes (u8 BGR [h][w][3], the probe's oriented shape) on the
 * decoder's GPU; dst[i] may be NULL for other files.  status[i] gets the probe status or the decode's verdict
 * (CTD_PNG_CRC, CTD_PNG_DATA); only pages with status 0 have been written, the others are to be decoded by cv2.
 * Blocks until every page is written, so the buffers may be used on any stream.  Staging and the inflate buffer
 * belong to the decoder and grow on demand.  CTD_E_CAPACITY, before any GPU work, for more than 65535 files the
 * GPU takes in one call.                                                                                          */
CTD_API int ctd_png_decode(ctd_png_decoder* dec, const uint8_t* const* data, const size_t* len, int32_t n,
                           uint8_t* const* dst, int32_t* status);
/* Of the last ctd_png_decode call's files decoded on the GPU: deflate blocks, and self-synchronisation rounds summed
 * over their Huffman chunks (one round per chunk when every guessed start was right).                            */
CTD_API int ctd_png_decoder_stats(const ctd_png_decoder* dec, int64_t* blocks, int64_t* rounds);

/* ---- PNG files encoded on the GPU -------------------------------------------------------
 * The reference writes pages and masks with io_utils.imwrite = cv2.imencode('.png', img).tofile(path).  These entry
 * points encode u8 images on the GPU to exactly the bytes cv2.imencode('.png', img) gives with the libpng and zlib
 * OpenCV 4.13 is built against (libpng 1.6.53, zlib 1.2.11) at OpenCV's PNG defaults: compression level 1, strategy
 * Z_RLE, memLevel 8, filter SUB on every row (NONE for an image 1 pixel wide), IHDR / IDAT / IEND only, IDAT chunks of
 * 8192 bytes of the zlib stream, and libpng's optimize_cmf window field for streams of at most 16 KiB.  The deflate
 * stream restates zlib 1.2.11's deflate_rle parse and trees.c block by block (csrc/png.cu, oracle/png_ref.py).
 *
 * ctd_png_image describes one image: u8, `channels` 1 (grey [h][w]) or 3 (BGR [h][w][3]), bit_depth 8.  With
 * on_device == 0, `data` is HOST memory, C-contiguous.  With on_device != 0, `data` is the DEVICE address of pixel
 * (0, 0), channel 0, on the encoder's GPU, byte (y, x, c) at data + y * stride_h + x * stride_w + c * stride_c (each
 * stride >= 0), and `event` (a cudaEvent_t, may be NULL) is waited on by the encoder's stream before the image is
 * read.                                                                                                            */
typedef struct ctd_png_image {
  const uint8_t* data;
  int32_t height, width, channels, bit_depth;
  int32_t on_device;
  int64_t stride_h, stride_w, stride_c;
  void* event;
} ctd_png_image;
typedef struct ctd_png_encoder ctd_png_encoder;
/* An encoder bound to one GPU and one stream of its own; staging, scratch and output buffers grow on demand.  Not
 * thread-safe; errors via ctd_last_error(NULL).                                                                     */
CTD_API int ctd_png_encoder_create(int32_t device, ctd_png_encoder** out);
CTD_API void ctd_png_encoder_destroy(ctd_png_encoder* enc);
/* Encodes n images at once.  files[i] / sizes[i] get image i's complete PNG file in pinned host memory owned by the
 * encoder, valid until its next call.  Synchronises with the host once, at the end.  CTD_E_INVALID, before any GPU
 * work, for a side < 1, channels other than 1 or 3, bit_depth other than 8, a negative stride or a device image
 * that is not memory of the encoder's GPU; CTD_E_CAPACITY for 2^31 or more filtered bytes (h * (1 + w * channels),
 * summed over the images) in one call.                                                                              */
CTD_API int ctd_png_encode(ctd_png_encoder* enc, const ctd_png_image* images, int32_t n, const uint8_t** files,
                           int64_t* sizes);

/* ---- JPEG files encoded on the GPU ------------------------------------------------------
 * io_utils.imwrite(path, img, '.jpg') writes cv2.imencode('.jpg', img, params).  These entry points encode u8 images
 * on the GPU to exactly the baseline file cv2.imencode('.jpg', img, params) gives with the libjpeg-turbo OpenCV 4.13
 * bundles (3.1): BGR input converted by jccolor.c, jcsample.c's downsampling, jpeg_fdct_islow, the reciprocal
 * quantiser, Annex K.3 or per-image optimal Huffman tables, SOI / APP0 JFIF 1.01 / DQT / SOF0 / DHT / DRI / SOS / EOI
 * (csrc/jpeg_enc.cu, oracle/jpeg_enc_ref.py).  Images are described by ctd_png_image (channels 1: one grey component;
 * channels 3: BGR, coded as YCbCr).
 *
 * ctd_jpeg_params holds one image's parameters, as cv2 leaves them after clamping: quality 0..100 (0 codes as 1),
 * sampling one of cv2's IMWRITE_JPEG_SAMPLING_FACTOR_* values (0x411111, 0x221111, 0x211111, 0x121111, 0x111111: the
 * luma factors H and V in 0xHV1111; a grey image is always 1x1), optimize 0 / nonzero, restart_interval 0..65535 MCUs
 * (0: none).                                                                                                        */
typedef struct ctd_jpeg_params {
  int32_t quality, sampling, optimize, restart_interval;
} ctd_jpeg_params;
typedef struct ctd_jpeg_encoder ctd_jpeg_encoder;
/* An encoder bound to one GPU and one stream of its own; staging, scratch and output buffers grow on demand.  Not
 * thread-safe; errors via ctd_last_error(NULL).                                                                     */
CTD_API int ctd_jpeg_encoder_create(int32_t device, ctd_jpeg_encoder** out);
CTD_API void ctd_jpeg_encoder_destroy(ctd_jpeg_encoder* enc);
/* Encodes n images at once, image i with params[i].  files[i] / sizes[i] get image i's complete JPEG file in pinned
 * host memory owned by the encoder, valid until its next call.  Synchronises with the host once, at the end.
 * CTD_E_INVALID, before any GPU work, for a side < 1 or > 65500, channels other than 1 or 3, bit_depth other than 8,
 * a parameter out of range, a negative stride or a device image that is not memory of the encoder's GPU;
 * CTD_E_CAPACITY when the files' worst case (2048 header bytes and 418 bytes per 8x8 block, MCU padding included, per
 * image) reaches 2^31 bytes in one call.  The output buffer is sized at that worst case.                          */
CTD_API int ctd_jpeg_encode(ctd_jpeg_encoder* enc, const ctd_png_image* images, const ctd_jpeg_params* params,
                            int32_t n, const uint8_t** files, int64_t* sizes);

#ifdef __cplusplus
}
#endif
#endif /* CTD_B200_H_ */
