// Private header of libctd_b200.so: the handle and the helpers shared by engine.cu (network executor, C ABI of the
// forward pass) and pipeline.cu (group_output / refine_mask pipeline around it).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <math.h>

#include <algorithm>
#include <array>
#include <condition_variable>
#include <deque>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "kernels.h"

using ctd::ConvTcPlan;
using ctd::ConvEndsPlan;
using ctd::NmsWorkspace;
using ctd::PFN_encodeTiled;

// byte offsets inside the result arena (one allocation per engine, sized for max_batch pages of max_h x max_w):
// phase-A section (mask_u8 | det | det_count | n_labels | line_boxes | line_scores | line_count) = [0, a_bytes),
// then mask_refined u8 planes, then one fixed-stride block section per page (ctd_page_blocks header, ctd_block
// records, line quads, distances)
struct ArenaLayout {
  size_t det, cnt, nl, lb, ls, lc, a_bytes, refined, blocks, blocks_stride, rec_off, lines_off, dist_off, total;
};

// one page's block section (ctd_page_blocks header, ctd_block records, line quads, distances): offsets inside the
// section and its size, the same for every handle
struct BlockSection {
  size_t rec_off, lines_off, dist_off, stride;
};
inline BlockSection block_section_layout() {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  BlockSection b;
  b.rec_off = 64;
  b.lines_off = b.rec_off + al(size_t(CTD_MAX_BLOCKS) * sizeof(ctd_block));
  b.dist_off = b.lines_off + al(size_t(CTD_MAX_BLOCKS) * 32);
  b.stride = b.dist_off + al(size_t(CTD_MAX_BLOCK_DIST) * 8);
  return b;
}

// letterbox(im, (net_h, net_w), auto=False) (imgproc_utils.py:86-117, python round = half to even) and the
// resize_ratio that maps net coordinates back to the page (inference.py:148).  false: the page does not letterbox into
// the net input (a side < 1 or an unpadded side of 0).
struct Letterbox {
  int unpad_h, unpad_w;
  float ratio_x, ratio_y;
};
inline bool letterbox_of(int ih, int iw, int net_h, int net_w, Letterbox& lb) {
  if (ih < 1 || iw < 1 || net_h < 1 || net_w < 1) return false;
  const double r = std::min(double(net_h) / ih, double(net_w) / iw);
  lb.unpad_w = int(nearbyint(iw * r));
  lb.unpad_h = int(nearbyint(ih * r));
  if (lb.unpad_w < 1 || lb.unpad_h < 1 || lb.unpad_w > net_w || lb.unpad_h > net_h) return false;
  lb.ratio_x = float(double(iw) / double(lb.unpad_w));
  lb.ratio_y = float(double(ih) / double(lb.unpad_h));
  return true;
}

// results of a ctd_submit_pages batch of n pages: the phase-A rows (sized for n pages) at the start of the results
// buffer, then the packed page masks, the mask_refined planes and the block sections at the ctd_page_entry offsets.
// The result arena of ctd_submit_full has its rows at ArenaLayout's offsets and its masks at 0.
struct PagesHead {
  size_t det, cnt, lb, ls, lc, masks;
};
PagesHead pages_head(int n);

// one page of a job as its host and device stages see it
struct JobPage {
  int ih, iw;
  float ratio_x, ratio_y;   // resize_ratio (inference.py:148)
  size_t off;               // pixel offset P_i of the page in the image (x3), mask and mask_refined planes
  char* section;            // with phase-A rows: the block section phase B fills from them and the host mask
  const uint8_t* mask;
  // from the caller or phase B: refine windows (x1 y1 x2 y2), block boxes, lines; the lines' crop plan (textheight)
  std::vector<int32_t> wins, boxes;
  std::vector<ctd_region_line> lines;
  std::vector<ctd_region> plan;
  size_t plan_bytes = 0;
};

// device planes of pages at their pixel offsets, `total` pixels each: image (x3), mask, mask_refined, and the second
// refine output and threshold planes of refine_undetected_mask
struct Planes {
  const uint8_t* img;
  uint8_t *mask, *ref, *ref2, *thr;
  size_t total;
};

// a submitted job: what its host stage and device stage need of it
struct PipeJob {
  int slot = 0, refine_mode = 0;
  char* results_host = nullptr;
  bool rows = false;               // phase-A rows at `head` in results_host: phase B makes the pages' inputs from them
  PagesHead head{};                // phase-A rows and the mask plane in results_host
  size_t refined = 0;              // mask_refined plane in results_host
  std::vector<JobPage> pages;
  Planes pl{};                     // mask and ref NULL without masks; ref2 and thr only with keep_undetected
  // ctd_submit_full: the block sections uploaded here before the refine, so ctd_device_arena holds results_host's
  uint8_t* d_blocks = nullptr;
  size_t blocks_bytes = 0;
  int keep_undetected = 0;
  int textheight = 0;          // > 0: also crop every text line of every page
  int results_on_device = 0;   // mask_refined, the modified mask and the crops stay on the device (ctd_collect_device)
  int refined_input = 0;       // pl.ref holds the caller's mask_refined: only refine_undetected_mask runs
  std::vector<ctd_device_page> dev;   // dev[i].data != NULL: the crops read page i there, else from pl.img
  // ctd_submit_outputs: per page the ingest's non-finite bits (bit 0 blks, 1 mask, 2 lines; host copy, pinned),
  // complete with phase A's results; a set bit fails the batch before phase B
  const int32_t* nonfinite = nullptr;
};

struct ctd_handle;
// a buffer grown on demand and never shrunk (device memory, or pinned host memory): grow() replaces a smaller
// allocation by one of bytes + bytes / headroom, after synchronising `sync`, the stream whose work may still use it
// (none: no enqueued work can use it)
template <bool kPinned>
struct GrowBuf {
  uint8_t* p = nullptr;
  size_t cap = 0;
  int grow(ctd_handle* h, size_t bytes, std::optional<cudaStream_t> sync, size_t headroom = 4);
  void release();
};
using DevBuf = GrowBuf<false>;
using PinnedBuf = GrowBuf<true>;

// one of the two slots of the batch pipeline (ctd_submit_full, ctd_submit_pages, ctd_submit_refine, ctd_submit_regions):
// the staging and events of a batch
// in flight, its hand-over from the worker, and the buffers its results stay in until the next submission
struct Slot {
  // ctd_submit_full staging: the pages, and the device copy of the result arena (ctd_device_arena)
  uint8_t* d_stage_in = nullptr;
  uint8_t* d_stage_out = nullptr;
  cudaEvent_t ev_in_done = nullptr, ev_in_free = nullptr, ev_out_ready = nullptr, ev_out_done = nullptr;
  cudaEvent_t ev_post_done = nullptr;   // phase C of the batch has run (post stream)
  bool busy = false;                    // submitted and not collected
  // what the batch asked for (start()), and whether it was collected without error: the results ctd_collect_regions
  // and ctd_collect_device hand out (masks: the batch has masks, false for ctd_submit_regions)
  bool crops = false, on_device = false, masks = true, collected = false;
  // worker hand-over, under pipe_mu: 0 idle, 1 queued / running, 2 phase C enqueued, 3 failed
  int state = 0;
  int rc = 0;
  std::string err;
  char* pinned = nullptr;   // pinned staging of the refine window tables, pipe_pinned_cap bytes
  // ctd_submit_pages: packed pages | results head, masks, mask_refined | second refine output and threshold planes of
  // refine_undetected_mask (ctd_submit_refine: the same without the results head), grown while the slot is idle; page
  // tables (pinned + device: max_batch PageGeom entries, then at pg_gather_off 2 * max_batch GatherPage entries for
  // the pages and masks gathered from device memory, uploaded together)
  DevBuf pg_in, pg_res, pg_aux;
  DevBuf out_in;   // ctd_submit_outputs: the batch's network outputs that came from host memory
  ctd::PageGeom* h_pg_tab = nullptr;
  ctd::PageGeom* d_pg_tab = nullptr;
  std::vector<ctd_page_entry> dev_pages;   // the page entries of a results_on_device batch (ctd_collect_device)
  // text-line crops, written by the worker: the concatenated plans, the first plan entry of each page (n + 1
  // entries), the device buffer (crop tables | crop pixels) and the pinned host buffer (the same tables staged for
  // upload | the pixels copied back)
  std::vector<ctd_region> crop_plan;
  std::vector<int32_t> crop_first;
  std::vector<size_t> crop_base;   // n + 1 entries: page i's crops are bytes [crop_base[i], crop_base[i + 1])
  DevBuf d_crop;
  PinnedBuf h_crop;
  size_t crop_px_off = 0, crop_bytes = 0;   // pixels at h_crop + crop_px_off, crop_bytes long

  // a submission starts on the slot: the results of its last batch are given up
  void start(bool want_crops, bool want_on_device, bool want_masks = true) {
    crops = want_crops;
    on_device = want_on_device;
    masks = want_masks;
    collected = false;
  }
  void release();   // frees the slot's buffers and events
};

// refine windows of one launch (all pages of a batch) and the chunks they are cut into
struct RefineJob {
  std::vector<ctd::RefineWin> wins;
  std::vector<ctd::RefineChunk> chunks;
  size_t total_px = 0;
  size_t total_words = 0;   // bit-plane words handed to the chunks so far (RefineChunk::woff)
  // window of the iw x ih page whose planes start at pixel page_off; python slice semantics; empty windows dropped
  void add(int x1, int y1, int x2, int y2, size_t page_off, int iw, int ih);
  size_t table_bytes() const;
};

// crops of one k_warp_regions launch (all pages of a batch, or one page) and the tiles they are cut into
struct RegionJob {
  std::vector<ctd::RegionDev> regs;
  std::vector<ctd::RegionTile> tiles;
  size_t out_bytes = 0;   // end of the last crop in the packed output
  // the status-0 entries of plan[0..n), the crops of page `pg`, each written at out_base + its plan offset; returns the
  // index of a malformed entry, or -1
  int add(const ctd_region* plan, int n, const ctd::RegionPage& pg, long long out_base);
  size_t table_bytes() const;   // RegionDev[] | RegionTile[], each 256-aligned
  void write_tables(char* dst) const;
};

// what the stem of a plan reads: the u8 pages (d_pages), or the staging page ctd_forward_tensor's pre-pass writes from
// a float NCHW tensor (in_stage: fp16 in CTD_PREC_FP16_TC, f32 in the other precisions)
enum { INPUT_U8 = 0, INPUT_F32 = 1 };

struct ShapePlan {
  int input = INPUT_U8;
  std::vector<ConvTcPlan> tc;  // index = op index; block_n == 0: the op does not run conv_tc_kernel
  std::vector<ConvEndsPlan> ends;   // index = op index; kind != CTD_END_NONE: the tensor-core stem or seg tail
  cudaGraphExec_t graph = nullptr;
  int launches = 0;
};
struct ctd_handle {
  ctd_config cfg{};
  std::vector<ctd_op> ops;
  std::vector<ctd_bufdesc> bufs;
  std::vector<std::array<float, 7>> detect_prm;   // per op; DETECT: stride, then 3 anchors (w, h) in pixels
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, tev0 = nullptr, tev1 = nullptr;
  std::vector<cudaEvent_t> op_events;
  PFN_encodeTiled enc = nullptr;
  char* d_blob = nullptr;
  size_t blob_bytes = 0;
  std::vector<void*> d_buf;
  // split-fp16 mode (CTD_PREC_SPLIT_TC): d_buf holds the FP32 master copy of every activation; d_buf16[i] holds its
  // fp16 hi | lo planes ([2*n][h][w][C], refreshed after every op that writes the buffer) = the MMA operands;
  // d_wsplit holds per GEMM op the fp16 weight rows hi then lo (wsplit_off[op], bytes).
  std::vector<void*> d_buf16;
  char* d_wsplit = nullptr;
  std::vector<size_t> wsplit_off;
  int elem = 2;  // bytes per activation element
  uint8_t* d_pages = nullptr;
  float* d_blks = nullptr;
  float* d_mask = nullptr;
  uint8_t* d_mask_u8 = nullptr;   // start of the contiguous result arena: mask_u8 | det | det_count | n_labels
  float* d_lines = nullptr;
  uint8_t* d_bitmap = nullptr;
  float* d_det = nullptr;
  int* d_det_count = nullptr;
  int32_t* d_labels = nullptr;
  int32_t* d_nlabels = nullptr;
  int32_t* d_ccl_scratch = nullptr;
  void* d_segrep_scratch = nullptr;
  int2* d_segrep_rows = nullptr;   // segrep_launch's row extents, all 0xff between launches
  DevBuf refine_scratch;   // refine_mask on the engine stream
  DevBuf cc_scratch;       // ctd_connected_components: any image size
  DevBuf io_scratch;       // page and mask staging of the stand-alone entry points and ctd_detect_page
  int16_t* d_line_boxes = nullptr;
  float* d_line_scores = nullptr;
  int32_t* d_line_count = nullptr;
  void* d_nms_ws = nullptr;
  NmsWorkspace nms{};
  std::map<std::tuple<int, int, int, int>, ShapePlan> plans;   // key (n, ph, pw, input)
  // ctd_forward_tensor: the staging page (allocated at its full size on first use, so the plans' tensor maps stay
  // valid), and the events that order the engine stream after the caller's stream and back
  DevBuf in_stage;
  cudaEvent_t ev_tin = nullptr, ev_tout = nullptr;
  // batch pipeline (ctd_submit_full, ctd_submit_pages / ctd_collect): two slots, copy streams either side of compute
  cudaStream_t copy_in = nullptr, copy_out = nullptr;
  Slot slot[2];
  // overlapped schedule (programs with a DB tail): post-processing of the DB maps / the Detect rows runs on side
  // streams under the remaining network ops (see run_ops)
  bool overlap = false;
  cudaStream_t side = nullptr, side2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_fork2 = nullptr, ev_join2 = nullptr;
  cudaEvent_t ev_xjoin = nullptr;   // ctd_join (never part of a captured graph)
  std::vector<char> db_ancestor;   // op feeds the DB tail (computed once in ctd_create)
  // result arena layout (ctd_results_layout) and the full pipeline (pipeline.cu): worker thread + post stream
  ArenaLayout layout{};
  cudaStream_t post = nullptr;
  size_t pipe_pinned_cap = 0;
  std::thread pipe_thread;
  std::mutex pipe_mu;
  std::condition_variable pipe_cv, pipe_done_cv;
  std::deque<PipeJob> pipe_queue;
  bool pipe_quit = false;
  int host_threads = 4;
  size_t pg_gather_off = 0;
  // the OutputGather table, its float16 flags and the non-finite flags in the page tables
  size_t pg_out_off = 0, pg_half_off = 0, pg_flag_off = 0;
  cudaStream_t dev_out = nullptr;   // the stream ctd_collect_device copies on
  // the worker's phase C on the post stream: its own connected-components and refine scratch (refine_scratch and
  // cc_scratch belong to the caller's stream)
  DevBuf pg_cc;
  DevBuf post_refine;
  // ctd_preprocess_pages: the packed pages (stream-ordered allocations) and the page tables of the last call, and an
  // event recorded on its stream after its last read of them, which the next call's stream waits on before it writes
  // them
  uint8_t* pre_in = nullptr;
  size_t pre_in_cap = 0;
  char* d_pre_tab = nullptr;
  cudaEvent_t ev_pre = nullptr;
  // last forward
  int n = 0, ph = 0, pw = 0;
  int last_launches = 0;
  bool have_forward = false;
};


int ctd_fail(ctd_handle* h, int code, const char* fmt, ...);
int prepare_forward(ctd_handle* h, int32_t n, int32_t ph, int32_t pw, ShapePlan** out, int input = INPUT_U8);
int enqueue_forward(ctd_handle* h, int32_t n, int32_t ph, int32_t pw, ShapePlan& sp);
// Detect rows per page of a ph x pw net input (yolo.py:44), the rows of d_blks per page
int rows_per_image(int ph, int pw);
// the forward's post-processing on the engine workspaces, n pages of ph x pw, on stream s (cnt += the launches):
// NMS of d_blks into the arena's detections (half: NULL, or per page the float16 flag of nms_launch), and connected
// components + text-line boxes of d_bitmap / d_lines
int launch_nms(ctd_handle* h, int n, int ph, int pw, cudaStream_t s, int* cnt, const int32_t* half = nullptr);
int launch_db_post(ctd_handle* h, int n, int ph, int pw, cudaStream_t s, int* cnt);
// connected components + stats of a DEVICE u8 image on the engine stream (grow-on-demand scratch): *d_stats points at
// [stats_cap][5] ints on the device, *n_labels is read back (synchronises the stream)
int cc_device(ctd_handle* h, const uint8_t* d_img, int ih, int iw, int stats_cap, int32_t** d_stats, int32_t* n_labels);
int launch_refine(ctd_handle* h, const RefineJob& job, const uint8_t* d_img, const uint8_t* d_mask, int refine_mode,
                  uint8_t* d_out, cudaStream_t st, DevBuf& scratch, char* pinned);
void ctd_pipeline_shutdown(ctd_handle* h);
