// Launch-parameter structs and host entry points of every kernel in the engine.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ctd_b200.h"

namespace ctd {

constexpr int kMaxTaps = 9;

// Split-fp16 lo planes are stored scaled by 2^11.  x - hi is about 2^-11 |x|; unscaled it falls into the fp16
// subnormals (step 2^-24) once |x| < 2^-3 and loses a bit per octave below.  Scaled, lo keeps its 11 bits down to
// |x| ~ 2^-14, so hi + lo holds x to 2^-23 relative (22 significant bits) over the range activations and weights
// take.  |x - hi| * 2^11 <= 2^4 * 2^11 for any fp16-range x, so the scaled lo never overflows.  Both factors are
// powers of two: scaling and unscaling are exact.
constexpr float kSplitLoScale = 2048.0f;
constexpr float kSplitLoUnscale = 1.0f / 2048.0f;
constexpr int kMaxPhases = 4;

// Geometry shared by the tensor-core and CUDA-core convolution kernels.  A "grid" pixel is an
// output pixel for CONV and an input pixel (= one sub-pixel phase output) for DECONV4.
struct ConvGeom {
  int n_img;             // images in the batch
  int gh, gw;            // grid height/width (see above)
  int dst_h, dst_w;      // destination buffer spatial size
  int out_mul;           // 1 (conv) or 2 (deconv): dst pixel = grid pixel * out_mul + phase
  int n_phase;           // 1 or 4
  int taps;              // taps per phase: 1, 9 or 4
  int cin_total;         // sum of src_c
  int k_total;           // taps * cin_total
  int n_src;
  int src_c[CTD_MAX_SRC];
  int src_cstride[CTD_MAX_SRC];  // channels of the source buffer (element stride between pixels)
  int src_h, src_w;              // source spatial size (all sources agree)
  int in_stride;                 // 1 or 2 (conv stride)
  // per phase, per tap: source pixel = grid pixel * in_stride + (dy, dx)
  int8_t tap_dy[kMaxPhases][kMaxTaps];
  int8_t tap_dx[kMaxPhases][kMaxTaps];
  int cout, cout_pad;
  int dst_cstride, dst_coff;
  int act, residual;
};

// Fill taps/offset tables for an op (conv k=1/3 stride 1/2, deconv 4x4 s2 p1).
void fill_conv_geom_taps(ConvGeom& g, int kind, int ksize, int stride);

// ---------------------------------------------------------------------------------------
// wgmma implicit-GEMM convolution (conv_tc.cu)
struct alignas(64) ConvTcParams {
  CUtensorMap a_map[CTD_MAX_SRC][4];  // [source][parity]: parity maps only for stride-2 convs
  CUtensorMap b_map;                  // packed weights [n_phase*cout_pad][k_total], K-major
  // fp16 NHWC destination [phase]: {cout, gw, gh, n_img} over the slice (base at channel dst_coff; a DECONV4 phase
  // map starts at its sub-pixel and steps two pixels).  The epilogue stores its staged tile through it, and an
  // in-place residual is loaded through it; TMA clipping keeps padding columns, neighbouring channels and pixels
  // beyond the grid unwritten.
  CUtensorMap d_map[kMaxPhases];
  ConvGeom g;
  int kb_elems;                       // channels per K block: 64 / 32 / 16 (swizzle 128/64/32 B)
  int src_kblocks[CTD_MAX_SRC];
  int tiles_x, tiles_y;               // 16xTH-pixel tiles per image (TH = ConvTcPlan::tile_h)
  int8_t tap_map[kMaxPhases][kMaxTaps];  // parity map index per tap (stride 2), else 0
  __half* dst;
  // columns [0, dst_map_cols) go through d_map: cout rounded down to 8, since TMA clips the innermost dimension in
  // 16-byte units; the epilogue stores columns [dst_map_cols, cout) from registers
  int dst_map_cols;
  const float* bias;
  // DETECT epilogue (dst == nullptr): decoded rows go to blks
  float* blks;
  int blks_rows_per_img;  // A
  int level_row0;         // first row of this pyramid level
  float det_stride;
  float anchor_wh[6];     // pixels
  int nc;
  // split-fp16 mode (CTD_PREC_SPLIT_TC): every fp32 operand x is carried as two fp16 planes
  // hi = fp16(x), lo = fp16((x - hi) * kSplitLoScale); a K block issues (hi,hi) + (lo,hi) + (hi,lo) into fp32
  // accumulators, the cross terms are merged as cross * kSplitLoUnscale, and the epilogue writes FP32.  Activation
  // planes: image n_img + i of the same tensor map holds the lo plane of image i; weight lo rows follow the hi rows
  // (row + split_row_off).
  int split;
  int split_img_off;
  int split_row_off;
};
static_assert(sizeof(ConvTcParams) <= 4096, "ConvTcParams: kernel parameters are limited to 4 KB");

struct ConvTcPlan {
  ConvTcParams p;
  int block_n;
  int tile_h;   // TH: 8 or 16 pixel rows per tile
  dim3 grid;
  size_t smem_bytes;
};

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Builds tensor maps + launch shape.  Returns nullptr on success, else an error string.
// split != 0: split-fp16 mode (see ConvTcParams::split): src_ptr are the [2*n_img][h][w][C] fp16 hi|lo plane buffers,
// w16 holds hi rows then lo rows, dst is an FP32 NHWC buffer.
const char* conv_tc_plan(ConvTcPlan& plan, PFN_encodeTiled enc, const ConvGeom& g, const void* const src_ptr[],
                         const int src_coff[], const void* w16, const float* bias, __half* dst, int split = 0);
cudaError_t conv_tc_launch(const ConvTcPlan& plan, cudaStream_t s);
cudaError_t conv_tc_init();  // sets max dynamic smem attributes once

// ---------------------------------------------------------------------------------------
// The network's two ends on the tensor cores (conv_ends.cu): the stem, reading the u8 pages itself, and the seg tail.
// Each 16x16-pixel output tile loads its input region once, halo included, into shared memory.
enum { CTD_END_NONE = 0, CTD_END_STEM = 1, CTD_END_SEG = 2, CTD_END_STEM_F16 = 3 };
struct alignas(64) ConvEndsParams {
  CUtensorMap a_map;   // stem: u8 or fp16 pages {3*pw, ph, n}; seg tail: its fp16 NHWC input {64, gw, gh, n}
  CUtensorMap b_map;   // fp16 K-major weights: stem [32][192], seg tail [16][576]
  CUtensorMap d_map;   // stem: fp16 NHWC destination slice {cout, gw, gh, n}
  int n_img, gh, gw;   // output grid (seg tail: input grid; the mask is 2gh x 2gw)
  int tiles_x, tiles_y;
  const float* bias;   // stem: 32 floats
  float* mask_f32;     // seg tail: [n][2gh][2gw]
  uint8_t* mask_u8;
};
struct ConvEndsPlan {
  ConvEndsParams p;
  int kind = CTD_END_NONE;
  dim3 grid;
  size_t smem_bytes;
};
// Stem: Conv 6x6 s2 p2 (3 -> cout <= 32) + SiLU over the BGR pages [n][ph][pw][3] (u8, read as u8 / 255; or, with
// f16_page, fp16 values used as they are), in the space-to-depth window form of the compiler's weights `w16`
// ([32][3 rows][4 pixels][16 channels] fp16, K = 192); output [n][ph/2][pw/2][dst_cstride] fp16 at channel offset
// dst_coff.
const char* conv_ends_plan_stem(ConvEndsPlan& plan, PFN_encodeTiled enc, const void* pages, bool f16_page, int n,
                                int ph, int pw, const void* w16, const float* bias, __half* dst, int dst_cstride,
                                int dst_coff, int cout, int act);
// Seg tail: ConvT 4x4 s2 p1 (64 -> 1) + sigmoid as a 3x3 convolution whose 4 output channels are the sub-pixel phases
// (weights `w16` [16][9 taps][64] fp16, rows 4..15 zero) over the fp16 NHWC input (64 channels at src_coff of a
// src_cstride-channel buffer, gh x gw); writes the f32 and truncated-u8 masks [n][2gh][2gw].
const char* conv_ends_plan_seg(ConvEndsPlan& plan, PFN_encodeTiled enc, const __half* src, int src_cstride,
                               int src_coff, int src_c, int n, int gh, int gw, const void* w16, float* mask_f32,
                               uint8_t* mask_u8);
cudaError_t conv_ends_launch(const ConvEndsPlan& plan, cudaStream_t s);
cudaError_t conv_ends_init();  // sets max dynamic smem attributes once

// ---------------------------------------------------------------------------------------
// CUDA-core kernels (simt.cu): accurate/bisecting path and the thin layers.  T = float | __half.
struct ConvSimtParams {
  ConvGeom g;
  const void* src[CTD_MAX_SRC];  // already offset to the first channel read
  const void* w;                 // [n_phase*cout_pad][k_total] float (T=float) or __half (T=__half)
  const float* bias;
  void* dst;
  float* blks;                   // DETECT
  int blks_rows_per_img, level_row0, nc;
  float det_stride;
  float anchor_wh[6];
};
template <typename T>
cudaError_t conv_simt_launch(const ConvSimtParams& p, cudaStream_t s);

// P = uint8_t: u8 pages, each value read as float(u) / 255; P = float: the f32 staging page of a float input, read as
// it is
template <typename T, typename P>
cudaError_t stem_launch(const P* pages, int n, int h, int w, const float* wgt /*[32][108] (ky,kx,c)*/,
                        const float* bias, T* dst, int dst_cstride, int dst_coff, int cout, int act, cudaStream_t s);
// the input pre-pass of ctd_forward_tensor (X = float) and ctd_forward_tensor_f16 (X = __half): NCHW [n][3][h][w] of
// element X -> the HWC staging page [n][h][w][3] of element S.  Each value is widened exactly to float, then stored as
// S (__half: round to nearest; float: a copy), so an f16 input stages exactly what its float32 copy does.
template <typename X, typename S>
cudaError_t nchw_to_hwc_launch(const X* x, int n, int h, int w, S* dst, cudaStream_t s);
// fp32 NHWC channel slice -> fp16 hi / lo planes (split-fp16 mode): hi = fp16(x), lo = fp16((x - hi) * kSplitLoScale).
// src / hi / lo point at the first channel of the slice; `cstride` elements between pixels (same in all three).
cudaError_t split_planes_launch(const float* src, __half* hi, __half* lo, size_t npix, int c, int cstride,
                                cudaStream_t s);
template <typename T>
cudaError_t avgpool2_launch(const T* src, int n, int h, int w, int c, int src_cstride, T* dst, int dst_cstride,
                            cudaStream_t s);
template <typename T>
cudaError_t sppf_pool_launch(T* buf, int n, int h, int w, int c, int cstride, cudaStream_t s);  // in-place slots
template <typename T>
cudaError_t upsample2_launch(const T* src, int n, int h, int w, int c, int src_cstride, T* dst, int dst_cstride,
                             cudaStream_t s);
// seg tail: ConvT4x4s2p1 C->1 + sigmoid; writes f32 mask [n][2h][2w] and u8 mask (p*255 truncated)
template <typename T>
cudaError_t seg_tail_launch(const T* src, int n, int h, int w, int c, int cstride, const float* wgt /*[c][4][4]*/,
                            float* mask_f32, uint8_t* mask_u8, cudaStream_t s);
// DB tail on the 32-channel (binarize|thresh) map at 1/4 resolution -> lines f32 [n][2][4h][4w]
// and the thresholded bitmap u8 [n][4h][4w] (shrink > db_thresh).
template <typename T>
cudaError_t db_tail_launch(const T* src, int n, int h, int w, int cstride, const float* params, float* lines,
                           uint8_t* bitmap, float db_thresh, cudaStream_t s);

// ---------------------------------------------------------------------------------------
// post-processing (postproc.cu)
struct NmsWorkspace {
  float* cand;     // [n][cap][6]
  int* cand_count; // [n] candidates in `cand` (<= cap after nms_overflow_kernel)
  int* cand_total; // [n] candidates the page really had (> cap: the best `cap` by score were kept)
  float* sorted;   // [n][cap][6]
  unsigned long long* mask;  // [n][cap][cap/64]
  int cap;
};
// half (NULL, or one flag per page): where half[i] != 0 the rows of page i are float16 values widened to float, and its
// candidates follow non_max_suppression on half tensors: `obj > half(conf)`, class scores RN_half(cls * obj), the best
// kept where `> half(conf)`, corners RN_half(cx -/+ RN_half(w / 2)) (yolov5_utils.py:136,169-180 in float16 arithmetic)
cudaError_t nms_launch(const float* blks, int n, int rows, int nc, float conf, float iou, NmsWorkspace& ws,
                       float* det /*[n][300][6]*/, int* det_count, cudaStream_t s, const int32_t* half = nullptr);
constexpr int kNmsLaunches = 5;   // kernels nms_launch enqueues
size_t nms_workspace_bytes(int n, int cap);
void nms_workspace_bind(NmsWorkspace& ws, void* base, int n, int cap);

// 8-connectivity labelling with OpenCV's label numbering; labels i32, n_labels incl. background.
cudaError_t ccl_launch(const uint8_t* img, int n, int h, int w, int32_t* labels, int32_t* scratch /*3*n*h*w ints*/,
                       int32_t* n_labels, cudaStream_t s);
constexpr int kCclLaunches = 8;   // kernels and memsets ccl_launch enqueues
// Largest image ccl_launch + ccl_stats_launch label: the kernels index pixels with int and the stats table with
// 5 ints per label (up to a quarter of the pixels), so 2^28 keeps every index far inside int range.
constexpr size_t kCclMaxPixels = size_t(1) << 28;
cudaError_t ccl_stats_launch(const int32_t* labels, int h, int w, int32_t* stats, int cap, cudaStream_t s);

// SegDetectorRepresenter.boxes_from_bitmap (segrep.cu).  Lf = foreground union-find roots left in the CCL
// scratch by ccl_launch (first n*h*w ints).  boxes i16 [n][max_cand][4][2], scores f32 [n][max_cand].
size_t segrep_scratch_bytes(int n, int h, int w, int max_cand);
cudaError_t segrep_launch(const uint8_t* bitmap, const float* pred, size_t pred_page_stride, const int* Lf, int n, int h,
                          int w, int max_cand, float unclip_ratio, void* scratch, int16_t* boxes, float* scores,
                          int* n_contours, cudaStream_t s);
constexpr int kSegrepLaunches = 15;   // kernels and memsets segrep_launch enqueues
cudaError_t binarize_launch(const float* pred, size_t count, float thresh, uint8_t* bitmap, cudaStream_t s);

// cv2.resize INTER_LINEAR, uint8, 1 or 3 channels, bit-exact (resize.cu).  src rows are `src_pitch` bytes apart; the
// dh x dw result is written at the top-left of a canvas_h x canvas_w canvas whose remaining pixels are zeroed.
cudaError_t resize_linear_u8_launch(const uint8_t* src, int sh, int sw, size_t src_pitch, int channels, uint8_t* dst,
                                    int dh, int dw, int canvas_h, int canvas_w, cudaStream_t s);
// One page of a batch of pages of different sizes (ctd_submit_pages): u8 BGR source at byte `src_off` of the packed
// pages, letterboxed to unpad_h x unpad_w; its page-sized mask starts at byte `dst_off` of the packed mask planes and
// owns rows [row0, row0 + ih) of the batch's stacked mask rows.
struct PageGeom {
  long long src_off, dst_off;
  int ih, iw, unpad_h, unpad_w, row0, pad;
};
// The same resize as resize_linear_u8_launch for every page of a batch in one launch each: the letterbox of page p
// into dst[p] (n x net_h x net_w x 3), and the back-projection of mask[p][:unpad_h, :unpad_w] (n x net_h x net_w u8)
// to ih x iw at dst + dst_off.  total_rows = the sum of ih.
cudaError_t letterbox_batch_launch(const uint8_t* src, const PageGeom* d_tab, int n, uint8_t* dst, int net_h, int net_w,
                                   cudaStream_t s);
cudaError_t backproject_batch_launch(const uint8_t* mask, int net_h, int net_w, const PageGeom* d_tab, int n,
                                     int total_rows, uint8_t* dst, cudaStream_t s);
// The letterbox of every page of a batch as preprocess_img's tensor (ctd_preprocess_pages), written into dst (16-byte
// aligned, net_w a multiple of 16) in one launch: format PRE_F32_NCHW / PRE_F16_NCHW gives [n][3][net_h][net_w] with
// each u8 value v as v / 255 (correctly rounded f32; f16: that f32 rounded to nearest even), PRE_U8_NHWC the u8 pixels
// [n][net_h][net_w][3]; padding is 0.  reverse: output channel k is channel 2 - k of the page.
enum PreFormat { PRE_F32_NCHW = 0, PRE_F16_NCHW = 1, PRE_U8_NHWC = 2 };
cudaError_t letterbox_tensor_launch(const uint8_t* src, const PageGeom* d_tab, int n, void* dst, int net_h, int net_w,
                                    int format, bool reverse, cudaStream_t s);

// Pages (and masks) of a batch that are already in device memory (ctd_submit_pages, ctd_submit_refine), gathered
// into the packed planes of the batch (gather.cu): byte (y, x, c) of the source is at src + y * sh + x * sw + c * sc;
// the packed image is u8 [ih][iw][ch] at dst (ch = 3: a BGR page, ch = 1: a mask; sc is not read then).  The image
// owns rows [row0, row0 + ih) of the stacked rows of the launch's images.  fast: sc == 1 and sw == ch (rows are
// contiguous runs of iw * ch bytes at any pitch), copied with the widest accesses the alignment of source and
// destination allows; else one byte per thread.
struct GatherPage {
  const uint8_t* src;
  long long sh, sw, sc;
  uint8_t* dst;
  int ih, iw, row0, fast, ch, pad;
};
// one CTA per row of the n images of d_tab (total_rows = the sum of their ih)
cudaError_t gather_pages_launch(const GatherPage* d_tab, int n, int total_rows, cudaStream_t s);
// `bytes` (a multiple of 16) of a host table into device memory dst (16-byte aligned), ordered on stream s: the bytes
// travel as kernel arguments, 3840 per launch, so the host table may be reused as soon as this returns and no pinned
// staging buffer or host wait orders the copy (ctd_preprocess_pages)
cudaError_t upload_table_launch(const void* host, size_t bytes, void* dst, cudaStream_t s);

// A caller's network outputs for one page (ctd_submit_outputs), all in device memory, float32 (half == 0) or float16
// (half == 1), element strides: blks (r, c) at blks + r * bsr + c * bsc for r < rows, c < no; mask (y, x) at mask +
// y * msh + x * msw; channel 0 of lines_map (y, x) at lines + y * lsh + x * lsw.
struct OutputGather {
  const void* blks;
  long long bsr, bsc;
  const void* mask;
  long long msh, msw;
  const void* lines;
  long long lsh, lsw;
  int rows, half;
};
// One launch over the n pages of d_tab (gather.cu), each h x w: per page the u8 mask `(uint8_t)(int32_t)truncf(p *
// 255.f)` (0 where the product is outside int32: numpy's float32 -> uint8 cast on x86-64) into mask_u8, channel 0 of
// lines_map into lines (page stride 2 * h * w floats, where segrep reads it), the DB bitmap `p > thresh` into bitmap,
// and the blks rows into blks at ws_rows rows per page, rows past `rows` padded with NaN objectness (never a
// candidate).  A float16 page does postprocess_mask and the binarize in half, as the reference does on half tensors:
// the mask byte from the product rounded to half, `p > half(thresh)`; its lines plane and blks rows are the half
// values widened exactly to float.  flags[i] (zeroed by the caller) gets bit 0 / 1 / 2 for a non-finite value in page
// i's blks / mask / lines; such a value is staged as 0.
cudaError_t gather_outputs_launch(const OutputGather* d_tab, int n, int h, int w, int no, int ws_rows, float thresh,
                                  uint8_t* mask_u8, float* lines, uint8_t* bitmap, float* blks, int32_t* flags,
                                  cudaStream_t s);

// refine_mask (refine_mk.cu): one kernel per phase over the window pixels of all pages of a batch, one CTA per chunk.
struct RefineWin {
  int x1, y1, x2, y2;     // window (python slice semantics: rows y1..y2-1, cols x1..x2-1)
  long long off;          // pixel offset of this window's planes inside each scratch plane (a multiple of 4)
  long long page_off;     // pixel offset of the window's page in the mask / mask_refined planes (x3 in the image)
  int pitch;              // width of that page = its row pitch in pixels
};
// Pixels [i0, i0 + rows * cols) of the window planes, i0 = y0 * rw + x0, cols = min(rw - x0, kRefineChunkPx).  A
// window of width rw <= kRefineChunkPx is cut into chunks of whole rows (x0 = 0, cols = rw); a wider window into row
// segments (rows = 1, x0 a multiple of kRefineChunkPx).  In the 1-bit planes (32 pixels per word) every chunk has its
// own run of ceil(rows * cols / 32) words from word `woff`: bit j of word w is chunk pixel 32 * w + j.  The chunks of
// a window are consecutive in the table, row by row.
struct RefineChunk { int win, y0, x0, rows, woff; };
constexpr int kRefineChunkPx = 8192;
// Rows per chunk of a window of width rw <= kRefineChunkPx: as many whole rows as fit, a multiple of 4 from 8 rows up
// (chunk starts 4-byte aligned in the window planes).  The host cuts the windows with it (RefineJob::add) and the
// labelling finds the chunk of a neighbouring pixel with it (refine_mk.cu).
__host__ __device__ constexpr int refine_rows_per_chunk(int rw) {
  return kRefineChunkPx / rw >= 8 ? (kRefineChunkPx / rw) & ~3 : (kRefineChunkPx / rw > 0 ? kRefineChunkPx / rw : 1);
}
// scratch planes for `total_px` window pixels (the sum of the window areas, each rounded up to 4) cut into n_chunks,
// whose bit-plane runs end at or below word total_px / 32 + n_chunks
size_t refine_scratch_bytes(size_t total_px, size_t n_chunks);
// d_state: refine_mk_state_bytes(n_wins) bytes of per-window state
size_t refine_mk_state_bytes(int n_wins);
// the first n_multi_chunks records of d_chunks are the chunks of windows that span more than one chunk.  The pages
// are located by each window's page_off / pitch; d_out must be 4-byte aligned.
cudaError_t refine_mk_launch(const uint8_t* d_img, const uint8_t* d_mask, const RefineWin* d_wins, int n_wins,
                             const RefineChunk* d_chunks, int n_chunks, int n_multi_chunks, void* d_state, size_t total_px,
                             void* scratch, int refine_mode, uint8_t* d_out, cudaStream_t s);

// ---- text-line crops (region.cu) ----
constexpr int kRegionTilePx = 256;   // output pixels per CTA of k_warp_regions = threads per CTA
// the u8 BGR page a crop reads, in device memory: byte (y, x, c) at data + y * sh + x * sw + c * sc, so a page is read
// where it is (a packed page: sh = iw * 3, sw = 3, sc = 1; a caller's tensor: any strides >= 0)
struct RegionPage {
  const uint8_t* data;
  long long sh, sw, sc;
  int ih, iw;
};
// one crop of a k_warp_regions launch: where its page and its output are, its shape and the inverse homography
struct RegionDev {
  long long offset;        // byte offset of the crop in the packed output
  const uint8_t* page;     // the crop's page (RegionPage::data) and its byte strides
  long long sh, sw, sc;
  int out_h, out_w;        // returned shape
  int warp_w, bw0;         // width of the warped (un-rotated) image, OpenCV's block width
  int rotate, ih, iw, pad;
  double m[9];             // inverse homography (destination -> page)
};
struct RegionTile { int region, first; };   // kRegionTilePx consecutive output pixels of one crop
// one CTA per tile; each crop reads its own page through RegionDev::page and its strides
cudaError_t warp_regions_launch(const RegionDev* d_regs, const RegionTile* d_tiles, int n_tiles, uint8_t* d_out,
                                cudaStream_t s);

}  // namespace ctd
