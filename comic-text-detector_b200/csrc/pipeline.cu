// Full-page pipeline of the engine: everything `TextDetector.__call__` does after the network (reference
// inference.py:148-178) behind the C ABI, with the page and its masks staying in HBM:
//
//   phase A (device)  forward + NMS + mask u8 + DB threshold + CCL + line boxes           (engine.cu)
//   phase B (host)    postprocess_yolo casts, box_thresh filter, `group_output` (group.cpp), expand_textwindow
//   phase C (device)  `refine_mask` on the resident page + mask (refine_mk.cu), optionally refine_undetected_mask
//
// ctd_submit_full / ctd_collect run batches of net-sized pages through A -> B -> C with two batches in flight per
// engine: the caller's thread enqueues phase A, a per-engine worker thread waits for A's small results, runs phase B
// for the pages of the batch on a few host threads and enqueues phase C on a second stream, so the host stage and
// the refine kernels of batch i overlap the forward of batch i+1.  ctd_detect_page is the blocking single-page form
// for pages of any size (letterbox + back-projection on the GPU), the call behind the drop-in TextDetector.
// ctd_submit_pages runs batches of pages of any size through the same two-in-flight schedule, with one letterbox and
// one back-projection launch per batch (TextDetector.detect_batch / detect_stream); with a textheight it also cuts
// every text line of every page of the batch out of the resident pages in one k_warp_regions launch (region.cu).  Its
// pages may already be in device memory (any strides; one gather_pages_kernel launch packs them, gather.cu) and the
// masks and crops may stay there (ctd_collect_device).  ctd_submit_refine runs phase C alone on caller pages, masks
// and block boxes (textmask.refine_mask / refine_undetected_mask, MaskRefiner) through the same two-slot schedule, and
// ctd_submit_regions the crop stage alone on caller pages and text lines (regions.RegionCropper).
// ctd_preprocess_pages letterboxes a batch of pages into a caller's network input tensor on the caller's stream, with
// no slot (preprocess.Preprocessor).
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "engine.h"

using namespace ctd;

#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return ctd_fail(h, CTD_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// ---- refine_mask plumbing ------------------------------------------------------------------------------------
namespace {
// python slice normalisation of one window bound pair on an axis of length n (negative indices wrap, then clamp)
inline void norm_slice(int& lo, int& hi, int n) {
  if (lo < 0) lo = std::max(lo + n, 0);
  if (hi < 0) hi = std::max(hi + n, 0);
  lo = std::min(lo, n);
  hi = std::min(hi, n);
  if (hi < lo) hi = lo;
}
}  // namespace

void RefineJob::add(int x1, int y1, int x2, int y2, size_t page_off, int iw, int ih) {
  norm_slice(x1, x2, iw);
  norm_slice(y1, y2, ih);
  const size_t a = (x2 > x1 && y2 > y1) ? size_t(x2 - x1) * (y2 - y1) : 0;
  if (a == 0) return;                                    // empty slice: the reference's loop body is a no-op
  const int wi = int(wins.size());
  const int rw = x2 - x1, rh = y2 - y1;
  // whole rows per chunk, or one row segment of <= kRefineChunkPx pixels per chunk when a row is longer
  const int rows_per = refine_rows_per_chunk(rw);
  for (int y0 = 0; y0 < rh; y0 += rows_per)
    for (int x0 = 0; x0 < rw; x0 += kRefineChunkPx) {
      const int rows = std::min(rows_per, rh - y0);
      chunks.push_back(RefineChunk{wi, y0, x0, rows, int(total_words)});
      total_words += (size_t(rows) * std::min(rw - x0, kRefineChunkPx) + 31) / 32;
    }
  wins.push_back(RefineWin{x1, y1, x2, y2, (long long)total_px, (long long)page_off, iw});
  total_px = (total_px + a + 3) / 4 * 4;
}
size_t RefineJob::table_bytes() const {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  return al(wins.size() * sizeof(RefineWin)) + al(chunks.size() * sizeof(RefineChunk));
}

// uploads the window tables of `job` into the refine scratch and launches the refine kernels: d_img / d_mask / d_out
// are device planes holding each window's page at its page_off.  Stream-ordered on `st`, the only stream that may use
// that scratch (it is grown here after synchronising `st`): the caller's calls use h->refine_scratch on h->stream, the
// pipeline worker h->post_refine on h->post.  `pinned` (optional) is a host staging buffer of >= job.table_bytes()
// bytes that stays valid until the copy has executed.
int launch_refine(ctd_handle* h, const RefineJob& job, const uint8_t* d_img, const uint8_t* d_mask, int refine_mode,
                  uint8_t* d_out, cudaStream_t st, DevBuf& scratch, char* pinned) {
  if (job.wins.empty()) return CTD_OK;
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t tb = job.table_bytes();   // a multiple of 256
  const size_t sb = refine_mk_state_bytes(int(job.wins.size()));
  if (int rc = scratch.grow(h, tb + sb + refine_scratch_bytes(job.total_px, job.chunks.size()), st, 2)) return rc;
  char* base = reinterpret_cast<char*>(scratch.p);
  const size_t wb = al(job.wins.size() * sizeof(RefineWin));
  std::vector<char> local;
  char* stage = pinned;
  if (!stage) { local.resize(tb); stage = local.data(); }
  memcpy(stage, job.wins.data(), job.wins.size() * sizeof(RefineWin));
  // chunk table: the chunks of windows that span SEVERAL chunks first -- only those have chunk borders to unite and
  // chunk-local roots to re-point (k_union_border / k_flat1 run on that prefix); the kernels are order-agnostic
  int n_multi = 0;
  {
    RefineChunk* hc = reinterpret_cast<RefineChunk*>(stage + wb);
    const size_t nc = job.chunks.size();
    size_t tail = nc;
    for (size_t i = 0; i < nc;) {
      size_t j = i;
      while (j < nc && job.chunks[j].win == job.chunks[i].win) ++j;
      if (j - i > 1) {
        for (size_t k = i; k < j; ++k) hc[n_multi++] = job.chunks[k];
      } else {
        hc[--tail] = job.chunks[i];
      }
      i = j;
    }
  }
  CK(cudaMemcpyAsync(base, stage, tb, cudaMemcpyHostToDevice, st));
  if (!pinned) CK(cudaStreamSynchronize(st));   // pageable staging dies with this frame
  CK(refine_mk_launch(d_img, d_mask, reinterpret_cast<const RefineWin*>(base), int(job.wins.size()),
                      reinterpret_cast<const RefineChunk*>(base + wb), int(job.chunks.size()), n_multi, base + tb,
                      job.total_px, base + tb + sb, refine_mode, d_out, st));
  return CTD_OK;
}

extern "C" int ctd_refine_mask(ctd_handle* h, const uint8_t* img, const uint8_t* mask, int32_t ih, int32_t iw,
                               const int32_t* windows, int32_t n_win, int32_t refine_mode, uint8_t* out) {
  if (!h || !img || !mask || !out || (n_win > 0 && !windows)) return CTD_E_INVALID;
  if (ih < 1 || iw < 1) return ctd_fail(h, CTD_E_SHAPE, "bad image size");
  CK(cudaSetDevice(h->cfg.device));
  RefineJob job;
  for (int i = 0; i < n_win; ++i) job.add(windows[4 * i], windows[4 * i + 1], windows[4 * i + 2], windows[4 * i + 3], 0, iw, ih);
  const size_t px = size_t(ih) * iw, pxa = (px + 255) / 256 * 256;
  if (int rc = h->io_scratch.grow(h, pxa * 5 + 1024, h->stream)) return rc;
  uint8_t* d_img = h->io_scratch.p;
  uint8_t* d_mask = d_img + pxa * 3;
  uint8_t* d_out = d_mask + pxa;
  CK(cudaMemcpyAsync(d_img, img, px * 3, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(d_mask, mask, px, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemsetAsync(d_out, 0, pxa, h->stream));
  if (int rc = launch_refine(h, job, d_img, d_mask, refine_mode, d_out, h->stream, h->refine_scratch, nullptr))
    return rc;
  CK(cudaMemcpyAsync(out, d_out, px, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

// ---- phase B for one page ------------------------------------------------------------------------------------------
namespace {
// Results of phase A for one page (host pointers into the result arena), scale of the page (1,1 for net-sized pages)
struct PageIn {
  const float* det; int n_det;                 // [n_det][6] x1,y1,x2,y2,conf,cls in net coordinates
  const int16_t* line_boxes; const float* line_scores; int n_lines;
  const uint8_t* mask; int im_w, im_h;          // page-sized mask
  float ratio_x, ratio_y;                      // resize_ratio (inference.py:148)
};

// page i of a batch whose phase-A rows are at `head` in `res` ([n][300][6] detections, [n] counts, [n][1000][8] line
// boxes, [n][1000] scores, [n] counts), with its page-sized host mask
PageIn page_in(const char* res, const PagesHead& head, int i, const JobPage& p, const uint8_t* mask) {
  PageIn in;
  in.det = reinterpret_cast<const float*>(res + head.det) + size_t(i) * 300 * 6;
  in.n_det = std::min(std::max(reinterpret_cast<const int32_t*>(res + head.cnt)[i], 0), 300);
  in.line_boxes = reinterpret_cast<const int16_t*>(res + head.lb) + size_t(i) * 1000 * 8;
  in.line_scores = reinterpret_cast<const float*>(res + head.ls) + size_t(i) * 1000;
  in.n_lines = std::min(std::max(reinterpret_cast<const int32_t*>(res + head.lc)[i], 0), 1000);
  in.mask = mask; in.im_w = p.iw; in.im_h = p.ih; in.ratio_x = p.ratio_x; in.ratio_y = p.ratio_y;
  return in;
}

// expand_textwindow(img.shape, xyxy, 16) (utils/imgproc_utils.py:151-161) on an im_w x im_h page: win = x1 y1 x2 y2,
// without the python slice normalisation (RefineJob::add applies it).  In int64: a caller's box of int32 corners can
// expand past int32 (ctd_refine_plan gives it status 2).
std::array<int64_t, 4> expand_textwindow(int64_t x1, int64_t y1, int64_t x2, int64_t y2, int im_w, int im_h) {
  const int64_t w = x2 - x1, h = y2 - y1;
  const int64_t pad = int64_t(nearbyint((double(std::max(h, w)) * 0.25 + double(std::min(h, w)) * 0.75) / 16.0));
  return {std::max<int64_t>(0, x1 - pad), std::max<int64_t>(0, y1 - pad), std::min<int64_t>(im_w - 1, x2 + pad),
          std::min<int64_t>(im_h - 1, y2 + pad)};
}

// inference.py:101-114 (postprocess_yolo casts), 158-172 (box_thresh, line rescale), textblock.group_output,
// expand_textwindow(.., 16): fills the page's block section and appends its refine windows
int host_group_page(const PageIn& in, char* section, const BlockSection& L, std::vector<int32_t>& win_out) {
  std::vector<int32_t> bxy(size_t(in.n_det) * 4), bcls(size_t(in.n_det));
  for (int i = 0; i < in.n_det; ++i) {
    const float* d = in.det + 6 * i;
    // det[..., [0, 2]] * ratio in float32 (numpy: float32 array * python float), then astype(int32)
    bxy[4 * i + 0] = int32_t(d[0] * in.ratio_x);
    bxy[4 * i + 1] = int32_t(d[1] * in.ratio_y);
    bxy[4 * i + 2] = int32_t(d[2] * in.ratio_x);
    bxy[4 * i + 3] = int32_t(d[3] * in.ratio_y);
    bcls[i] = int32_t(d[5]);
  }
  std::vector<int32_t> lines;
  lines.reserve(size_t(in.n_lines) * 8);
  for (int i = 0; i < in.n_lines; ++i) {
    if (!(in.line_scores[i] > 0.6f)) continue;           // box_thresh (inference.py:159-161), float32 compare
    const int16_t* b = in.line_boxes + 8 * i;
    for (int k = 0; k < 4; ++k) {                        // astype(float64) * ratio -> astype(int32)
      lines.push_back(int32_t(double(b[2 * k]) * double(in.ratio_x)));
      lines.push_back(int32_t(double(b[2 * k + 1]) * double(in.ratio_y)));
    }
  }
  ctd_page_blocks* hdr = reinterpret_cast<ctd_page_blocks*>(section);
  ctd_block* rec = reinterpret_cast<ctd_block*>(section + L.rec_off);
  int32_t* lout = reinterpret_cast<int32_t*>(section + L.lines_off);
  double* dout = reinterpret_cast<double*>(section + L.dist_off);
  int32_t nb = 0;
  int rc = ctd_group_output(bxy.data(), bcls.data(), in.n_det, lines.data(), int32_t(lines.size() / 8), in.im_w, in.im_h, in.mask,
                            1, rec, CTD_MAX_BLOCKS, lout, CTD_MAX_BLOCKS, dout, CTD_MAX_BLOCK_DIST, &nb);
  hdr->flags = 0;
  if (rc == CTD_E_CAPACITY) {
    // more distance values than the section holds (split blocks copy their parent's array): drop the distances,
    // keep blocks and lines (flag bit 0)
    std::vector<double> big(size_t(CTD_MAX_BLOCKS) * CTD_MAX_BLOCKS / 4);
    rc = ctd_group_output(bxy.data(), bcls.data(), in.n_det, lines.data(), int32_t(lines.size() / 8), in.im_w, in.im_h, in.mask, 1,
                          rec, CTD_MAX_BLOCKS, lout, CTD_MAX_BLOCKS, big.data(), int32_t(big.size()), &nb);
    if (rc == CTD_OK)
      for (int i = 0; i < nb; ++i) { rec[i].n_dist = 0; rec[i].dist_off = 0; }
    hdr->flags |= 1;
  }
  if (rc != CTD_OK) { hdr->n_blocks = 0; hdr->n_lines = 0; hdr->n_dist = 0; hdr->flags |= 2; return rc; }
  hdr->n_blocks = nb;
  int32_t tl = 0, td = 0;
  for (int i = 0; i < nb; ++i) { tl += rec[i].n_lines; td += rec[i].n_dist; }
  hdr->n_lines = tl;
  hdr->n_dist = td;
  win_out.resize(size_t(nb) * 4);
  for (int i = 0; i < nb; ++i) {
    const int32_t* xy = rec[i].xyxy;
    const auto win = expand_textwindow(xy[0], xy[1], xy[2], xy[3], in.im_w, in.im_h);   // inside the page
    for (int k = 0; k < 4; ++k) win_out[size_t(4 * i + k)] = int32_t(win[k]);
  }
  return CTD_OK;
}

// fn(i) for the n pages of a batch, on up to `threads` host threads
template <typename F>
void for_each_page(int n, int threads, F fn) {
  const int nthreads = std::max(1, std::min(n, threads));
  if (nthreads == 1) {
    for (int i = 0; i < n; ++i) fn(i);
    return;
  }
  std::vector<std::thread> th;
  for (int t = 0; t < nthreads; ++t)
    th.emplace_back([&, t] { for (int i = t; i < n; i += nthreads) fn(i); });
  for (auto& x : th) x.join();
}

__global__ void undetected_prep_kernel(uint8_t* __restrict__ mask, const uint8_t* __restrict__ refined,
                                       uint8_t* __restrict__ thr, size_t n) {
  // mask_pred[mask_refined > 30] = 0; cv2.threshold(mask_pred, 30, 255, THRESH_BINARY)  (textmask.py:136-137)
  const size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  uint8_t m = mask[i];
  if (refined[i] > 30) { m = 0; mask[i] = 0; }
  thr[i] = m > 30 ? 255 : 0;
}
__global__ void or_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, size_t n) {
  const size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i < n) dst[i] |= src[i];
}

// device planes of a set of pages, each page's at its pixel offset: the image (x3), the mask, mask_refined, and the
// second refine output and threshold planes of refine_undetected_mask; `total` pixels each
struct Planes {
  const uint8_t* img;
  uint8_t *mask, *ref, *ref2, *thr;
  size_t total;
};

// refine_undetected_mask (textmask.py:135-156) for a set of pages: one prep launch over all planes, connected
// components + stats of each page on `st` (the scratch `cc` grows here), the host loop over each page's stats rows
// against its blocks (boxes[i]: x1 y1 x2 y2 of each block of page i), then one refine launch for the extra windows of
// all pages and one OR launch.  The masks are modified in place, as in the reference.
// Synchronises `st` once for the label counts and once for the stats rows.
int refine_undetected(ctd_handle* h, const std::vector<JobPage>& pages, const std::vector<std::vector<int32_t>>& boxes,
                      const Planes& pl, int refine_mode, cudaStream_t st, DevBuf& cc, DevBuf& refine_scratch,
                      char* pinned, size_t pinned_cap) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const int n = int(pages.size());
  const size_t total_px = pl.total;
  undetected_prep_kernel<<<unsigned((total_px + 255) / 256), 256, 0, st>>>(pl.mask, pl.ref, pl.thr, total_px);
  CK(cudaGetLastError());
  // scratch: labels | 3 ints/px of CCL scratch for the largest page (reused page after page) | one stats table per
  // page (worst case of 8-connected components + background) | the label counts
  size_t max_px = 0;
  std::vector<int> cap(static_cast<size_t>(n));
  std::vector<size_t> stats_off(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) max_px = std::max(max_px, size_t(pages[i].ih) * pages[i].iw);
  const size_t o_scr = al(max_px * 4);
  size_t o = o_scr + al(max_px * 12);
  for (int i = 0; i < n; ++i) {
    cap[size_t(i)] = ((pages[i].ih + 1) / 2) * ((pages[i].iw + 1) / 2) + 2;
    stats_off[size_t(i)] = o;
    o += al(size_t(cap[size_t(i)]) * 5 * 4);
  }
  const size_t o_nl = o;
  if (int rc = cc.grow(h, o_nl + al(size_t(n) * 4), st)) return rc;
  uint8_t* base = cc.p;
  int32_t* d_labels = reinterpret_cast<int32_t*>(base);
  int32_t* d_scr = reinterpret_cast<int32_t*>(base + o_scr);
  int32_t* d_nl = reinterpret_cast<int32_t*>(base + o_nl);
  for (int i = 0; i < n; ++i) {
    const JobPage& p = pages[size_t(i)];
    int32_t* d_stats = reinterpret_cast<int32_t*>(base + stats_off[size_t(i)]);
    CK(ccl_launch(pl.thr + p.off, 1, p.ih, p.iw, d_labels, d_scr, d_nl + i, st));
    CK(ccl_stats_launch(d_labels, p.ih, p.iw, d_stats, cap[size_t(i)], st));
  }
  std::vector<int32_t> n_lab(static_cast<size_t>(n));
  CK(cudaMemcpyAsync(n_lab.data(), d_nl, size_t(n) * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  std::vector<std::vector<int32_t>> stats(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) {
    stats[size_t(i)].resize(size_t(std::max(n_lab[size_t(i)], 0)) * 5);
    if (n_lab[size_t(i)] > 0)
      CK(cudaMemcpyAsync(stats[size_t(i)].data(), base + stats_off[size_t(i)], stats[size_t(i)].size() * 4,
                         cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  RefineJob rj2;
  for (int i = 0; i < n; ++i) {
    const JobPage& p = pages[size_t(i)];
    const std::vector<int32_t>& xyxy = boxes[size_t(i)];
    const size_t nb = xyxy.size() / 4;
    bool first_valid = true;
    for (int li = 0; li < n_lab[size_t(i)]; ++li) {
      const int32_t* s5 = &stats[size_t(i)][size_t(li) * 5];
      if (!(s5[4] > 50)) continue;
      if (first_valid) { first_valid = false; continue; }        // valid_labels[1:]
      const int64_t bb[4] = {s5[0], s5[1], int64_t(s5[0]) + s5[2], int64_t(s5[1]) + s5[3]};
      int64_t score = -1;
      for (size_t b = 0; b < nb; ++b) {
        const int32_t* q = &xyxy[4 * b];
        const int64_t x1 = std::max<int64_t>(q[0], bb[0]), y1 = std::max<int64_t>(q[1], bb[1]);
        const int64_t x2 = std::min<int64_t>(q[2], bb[2]), y2 = std::min<int64_t>(q[3], bb[3]);
        const int64_t a = (y2 < y1 || x2 < x1) ? -1 : (y2 - y1) * (x2 - x1);
        if (a > score) score = a;
      }
      if (double(score) / double(s5[2]) / double(s5[3]) < 0.5) {
        const auto w4 = expand_textwindow(bb[0], bb[1], bb[2], bb[3], p.iw, p.ih);   // inside the page
        rj2.add(int(w4[0]), int(w4[1]), int(w4[2]), int(w4[3]), p.off, p.iw, p.ih);
      }
    }
  }
  if (!rj2.wins.empty()) {
    CK(cudaMemsetAsync(pl.ref2, 0, total_px, st));
    // the stream is idle here, so the pinned staging of an earlier launch is free again
    char* stage = rj2.table_bytes() <= pinned_cap ? pinned : nullptr;
    if (int rc = launch_refine(h, rj2, pl.img, pl.mask, refine_mode, pl.ref2, st, refine_scratch, stage)) return rc;
    or_kernel<<<unsigned((total_px + 255) / 256), 256, 0, st>>>(pl.ref, pl.ref2, total_px);
    CK(cudaGetLastError());
  }
  return CTD_OK;
}

// phase C of a set of pages, mask_refined already zeroed: one refine launch over the windows of every page
// (wins[i]: x1 y1 x2 y2 each), then with keep_undetected refine_undetected_mask against the pages' block boxes
// (boxes[i], read only then).  Stream-ordered on `st` with the scratch that belongs to it; `pinned` (optional,
// pinned_cap bytes) stages the window tables.
int phase_c(ctd_handle* h, const std::vector<JobPage>& pages, const std::vector<std::vector<int32_t>>& wins,
            const std::vector<std::vector<int32_t>>& boxes, const Planes& pl, int refine_mode, bool keep_undetected,
            cudaStream_t st, DevBuf& refine_scratch, DevBuf& cc, char* pinned, size_t pinned_cap) {
  RefineJob rj;
  for (size_t i = 0; i < pages.size(); ++i)
    for (size_t k = 0; k + 3 < wins[i].size(); k += 4)
      rj.add(wins[i][k], wins[i][k + 1], wins[i][k + 2], wins[i][k + 3], pages[i].off, pages[i].iw, pages[i].ih);
  char* stage = rj.table_bytes() <= pinned_cap ? pinned : nullptr;   // else: pageable + sync
  if (int rc = launch_refine(h, rj, pl.img, pl.mask, refine_mode, pl.ref, st, refine_scratch, stage)) return rc;
  if (!keep_undetected) return CTD_OK;
  return refine_undetected(h, pages, boxes, pl, refine_mode, st, cc, refine_scratch, pinned, pinned_cap);
}

// the block boxes of each page's block section (the detector's own blocks), for refine_undetected
std::vector<std::vector<int32_t>> section_boxes(const std::vector<JobPage>& pages) {
  const BlockSection bs = block_section_layout();
  std::vector<std::vector<int32_t>> boxes(pages.size());
  for (size_t i = 0; i < pages.size(); ++i) {
    const int nb = reinterpret_cast<const ctd_page_blocks*>(pages[i].section)->n_blocks;
    const ctd_block* rec = reinterpret_cast<const ctd_block*>(pages[i].section + bs.rec_off);
    for (int b = 0; b < nb; ++b) boxes[i].insert(boxes[i].end(), rec[b].xyxy, rec[b].xyxy + 4);
  }
  return boxes;
}
}  // namespace

extern "C" int ctd_results_layout(ctd_handle* h, ctd_results_layout_t* out) {
  if (!h || !out) return CTD_E_INVALID;
  const ArenaLayout& L = h->layout;
  out->max_batch = h->cfg.max_batch; out->max_h = h->cfg.max_h; out->max_w = h->cfg.max_w; out->reserved = 0;
  out->total_bytes = L.total;
  out->mask_u8 = 0; out->det = L.det; out->det_count = L.cnt; out->n_labels = L.nl;
  out->line_boxes = L.lb; out->line_scores = L.ls; out->line_count = L.lc;
  out->phase_a_bytes = L.a_bytes;
  out->mask_refined = L.refined; out->blocks = L.blocks; out->blocks_stride = L.blocks_stride;
  out->blk_records_off = L.rec_off; out->blk_lines_off = L.lines_off; out->blk_dist_off = L.dist_off;
  return CTD_OK;
}

// ---- pages of any size: batch layout ---------------------------------------------------------------------------------
PagesHead pages_head(int n) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t nb = size_t(n);
  PagesHead hd;
  hd.det = 0;
  hd.cnt = hd.det + al(nb * 300 * 6 * 4);
  hd.lb = hd.cnt + al(nb * 4);
  hd.ls = hd.lb + al(nb * 1000 * 8 * 2);
  hd.lc = hd.ls + al(nb * 1000 * 4);
  hd.masks = hd.lc + al(nb * 4);
  return hd;
}

// The pixel planes of a batch: page i's pixel offset P_i is the sum of the earlier pages' pixels, each rounded up to
// 256, and is the same in every plane: image bytes at 3 P_i, mask at P_i of the mask plane, mask_refined at P_i of the
// mask_refined plane, so refine_mask addresses the image and the mask planes of a page with one offset.  Fills page_off
// (3 P_i), mask_off (mask_plane + P_i) and refined_off (mask_off + T) of each entry and returns T, the pixels of a plane
// (the sum over the batch); the mask_refined plane follows the mask plane.
static size_t plan_planes(ctd_page_entry* pages, int n, size_t mask_plane) {
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    pages[i].page_off = int64_t(total * 3);
    pages[i].mask_off = int64_t(mask_plane + total);
    total += al(size_t(pages[i].ih) * size_t(pages[i].iw));
  }
  for (int i = 0; i < n; ++i) pages[i].refined_off = pages[i].mask_off + int64_t(total);
  return total;
}

// Results buffer: pages_head(n) | masks | mask_refined planes | block sections (plan_planes).
extern "C" int ctd_pages_plan(ctd_page_entry* pages, int32_t n, int32_t net_h, int32_t net_w, size_t* input_bytes,
                              size_t* results_bytes) {
  if (!input_bytes || !results_bytes || n < 0 || (n > 0 && !pages)) return CTD_E_INVALID;
  if (net_h < 64 || net_w < 64 || net_h % 64 || net_w % 64) return CTD_E_SHAPE;
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const PagesHead hd = pages_head(n);
  for (int i = 0; i < n; ++i) {
    Letterbox lb;
    if (!letterbox_of(pages[i].ih, pages[i].iw, net_h, net_w, lb)) return CTD_E_SHAPE;
    pages[i].unpad_h = lb.unpad_h;
    pages[i].unpad_w = lb.unpad_w;
  }
  const size_t total = plan_planes(pages, n, hd.masks);
  const size_t stride = al(block_section_layout().stride);
  const size_t blocks = hd.masks + 2 * total;
  for (int i = 0; i < n; ++i) pages[i].blocks_off = int64_t(blocks + size_t(i) * stride);
  *input_bytes = total * 3;
  *results_bytes = blocks + size_t(n) * stride;
  return CTD_OK;
}

// Input: the pages (3 T bytes), then a frame laid out as the results; results: masks | mask_refined (plan_planes).
extern "C" int ctd_refine_plan(ctd_page_entry* pages, int32_t n, const int32_t* xyxy, const int32_t* n_blocks,
                               int32_t* windows, int32_t* status, size_t* input_bytes, size_t* results_bytes) {
  if (!input_bytes || !results_bytes || n < 0 || (n > 0 && (!pages || !n_blocks))) return CTD_E_INVALID;
  int64_t nb = 0;
  for (int i = 0; i < n; ++i) {
    if (pages[i].ih < 1 || pages[i].iw < 1) return CTD_E_SHAPE;
    if (n_blocks[i] < 0) return CTD_E_INVALID;
    nb += n_blocks[i];
  }
  if (nb > INT32_MAX) return CTD_E_CAPACITY;
  if (nb > 0 && (!xyxy || !windows || !status)) return CTD_E_INVALID;
  for (int i = 0; i < n; ++i) {
    pages[i].unpad_h = pages[i].unpad_w = 0;
    pages[i].blocks_off = 0;
  }
  const size_t total = plan_planes(pages, n, 0);
  size_t b = 0;
  for (int i = 0; i < n; ++i) {
    const int ih = pages[i].ih, iw = pages[i].iw;
    for (int k = 0; k < n_blocks[i]; ++k, ++b) {
      const int32_t* q = xyxy + 4 * b;
      const auto w = expand_textwindow(q[0], q[1], q[2], q[3], iw, ih);
      bool fits = true;
      for (int j = 0; j < 4; ++j) {
        fits = fits && w[j] >= INT32_MIN && w[j] <= INT32_MAX;
        windows[4 * b + j] = int32_t(std::min<int64_t>(std::max<int64_t>(w[j], INT32_MIN), INT32_MAX));
      }
      // img[by1:by2, bx1:bx2] empty: cv2.cvtColor raises in get_topk_masklist
      int x1 = windows[4 * b], y1 = windows[4 * b + 1], x2 = windows[4 * b + 2], y2 = windows[4 * b + 3];
      norm_slice(x1, x2, iw);
      norm_slice(y1, y2, ih);
      status[b] = !fits ? 2 : (x2 > x1 && y2 > y1) ? 0 : 1;
    }
  }
  *input_bytes = total * 5;
  *results_bytes = total * 2;
  return CTD_OK;
}

// ctd_region_plan of every line of one page's block section, in block then line order (textblock.region_lines)
static int plan_page_regions(const char* section, const BlockSection& bs, int iw, int ih, int textheight,
                             std::vector<ctd_region>& plan, size_t* bytes) {
  const ctd_page_blocks* hdr = reinterpret_cast<const ctd_page_blocks*>(section);
  const ctd_block* rec = reinterpret_cast<const ctd_block*>(section + bs.rec_off);
  const int32_t* quads = reinterpret_cast<const int32_t*>(section + bs.lines_off);
  std::vector<ctd_region_line> lines;
  lines.reserve(size_t(std::max(hdr->n_lines, 0)));
  for (int b = 0; b < hdr->n_blocks; ++b)
    for (int k = 0; k < rec[b].n_lines; ++k) {
      ctd_region_line l{};
      const int32_t* q = quads + size_t(rec[b].line_off + k) * 8;
      for (int j = 0; j < 8; ++j) l.quad[j] = double(q[j]);
      l.language = rec[b].language;
      l.vertical = rec[b].vertical ? 1 : 0;
      l.font_size = rec[b].font_size;
      lines.push_back(l);
    }
  plan.resize(lines.size());
  *bytes = 0;
  if (lines.empty()) return CTD_OK;   // nothing to plan, whatever the page size
  return ctd_region_plan(lines.data(), int32_t(lines.size()), iw, ih, textheight, plan.data(), bytes);
}

// the device planes of a submitted batch
static Planes job_planes(const PipeJob& job) {
  return Planes{job.d_img, job.d_mask, job.d_ref, job.d_aux, job.d_aux ? job.d_aux + job.total : nullptr, job.total};
}

// the end of a batch on the worker's stream `st`: the masks refine_undetected_mask modified and mask_refined back to
// results_host (unless they stay on the device), then the batch's done event
static int finish_batch(ctd_handle* h, const PipeJob& job, cudaStream_t st) {
  if (!job.results_on_device) {
    char* res = job.results_host;
    if (job.keep_undetected) CK(cudaMemcpyAsync(res + job.head.masks, job.d_mask, job.total, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(res + job.refined, job.d_ref, job.total, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaEventRecord(h->slot[job.slot].ev_post_done, st));
  return CTD_OK;
}

// the pages of a batch as its crops read them: a page in device memory where it is (job.dev, ctd_submit_regions),
// every other page in the batch's packed page buffer
static std::vector<RegionPage> region_pages(const PipeJob& job) {
  std::vector<RegionPage> src;
  for (size_t i = 0; i < job.pages.size(); ++i) {
    const JobPage& p = job.pages[i];
    if (i < job.dev.size() && job.dev[i].data) {
      const ctd_device_page& d = job.dev[i];
      src.push_back(RegionPage{d.data, (long long)d.stride_h, (long long)d.stride_w, (long long)d.stride_c, p.ih, p.iw});
    } else {
      src.push_back(RegionPage{job.d_img + p.off * 3, (long long)p.iw * 3, 3, 1, p.ih, p.iw});
    }
  }
  return src;
}

// the crop stage of a batch, on the worker's stream `st`: the pages' plans (plans[i], plan_bytes[i] packed bytes each)
// concatenated with each page's crops after the previous page's into the slot's crop plan, the tables staged in the
// slot's pinned crop buffer, one k_warp_regions launch over every page where it is (src[i]), and the pixels back into
// the same pinned buffer after the tables (to_host), else left after the tables in d_crop.  A batch without a crop
// launches and allocates nothing.
static int crop_stage(ctd_handle* h, Slot& s, const std::vector<RegionPage>& src,
                      const std::vector<std::vector<ctd_region>>& plans, const std::vector<size_t>& plan_bytes,
                      bool to_host, cudaStream_t st) {
  const int n = int(src.size());
  RegionJob rg;
  s.crop_plan.clear();
  s.crop_first.assign(size_t(n) + 1, 0);
  s.crop_base.assign(size_t(n) + 1, 0);
  size_t base = 0;
  for (int i = 0; i < n; ++i) {
    const std::vector<ctd_region>& p = plans[size_t(i)];
    if (int bad = rg.add(p.data(), int(p.size()), src[size_t(i)], (long long)base); bad >= 0)
      return ctd_fail(h, CTD_E_INVALID, "malformed crop plan entry %d on page %d of the batch", bad, i);
    s.crop_first[size_t(i)] = int32_t(s.crop_plan.size());
    s.crop_base[size_t(i)] = base;
    for (ctd_region r : p) {
      r.offset += int64_t(base);
      s.crop_plan.push_back(r);
    }
    base += plan_bytes[size_t(i)];
  }
  s.crop_first[size_t(n)] = int32_t(s.crop_plan.size());
  s.crop_base[size_t(n)] = base;
  if (s.crop_plan.size() > size_t(INT32_MAX) || rg.tiles.size() > size_t(INT32_MAX))
    return ctd_fail(h, CTD_E_CAPACITY, "too many crops in one batch");
  s.crop_bytes = base;
  s.crop_px_off = 0;
  if (rg.tiles.empty()) return CTD_OK;
  // both buffers grow only after `st` is idle, since an earlier failed job of this slot may have left copies on it
  const size_t tb = rg.table_bytes(), px = s.crop_bytes;
  if (int rc = s.d_crop.grow(h, tb + px, st)) return rc;
  if (int rc = s.h_crop.grow(h, to_host ? tb + px : tb, st)) return rc;
  uint8_t* d_tab = s.d_crop.p;
  rg.write_tables(reinterpret_cast<char*>(s.h_crop.p));
  CK(cudaMemcpyAsync(d_tab, s.h_crop.p, tb, cudaMemcpyHostToDevice, st));
  const size_t rb = (rg.regs.size() * sizeof(RegionDev) + 255) / 256 * 256;
  CK(warp_regions_launch(reinterpret_cast<const RegionDev*>(d_tab), reinterpret_cast<const RegionTile*>(d_tab + rb),
                         int(rg.tiles.size()), d_tab + tb, st));
  if (to_host) CK(cudaMemcpyAsync(s.h_crop.p + tb, d_tab + tb, px, cudaMemcpyDeviceToHost, st));
  s.crop_px_off = tb;
  return CTD_OK;
}

// phases B and C of a submitted batch, on the worker thread
static int run_batch(ctd_handle* h, const PipeJob& job) {
  Slot& s = h->slot[job.slot];
  const int n = int(job.pages.size());
  CK(cudaEventSynchronize(s.ev_out_done));          // phase A results are in results_host
  for (int i = 0; job.nonfinite && i < n; ++i)
    if (const int32_t f = job.nonfinite[i])
      return ctd_fail(h, CTD_E_INVALID, "page %d of the batch: a non-finite value (NaN or inf) in its %s", i,
                      (f & 1) ? "blks" : (f & 2) ? "mask" : "lines_map");
  char* res = job.results_host;
  const BlockSection bs = block_section_layout();
  std::vector<std::vector<int32_t>> wins(static_cast<size_t>(n));
  std::vector<int> prc(size_t(n), CTD_OK);
  // text-line crops: each page's plan on the host threads, right after its group_output
  const bool crops = job.textheight > 0;
  std::vector<std::vector<ctd_region>> plans(crops ? size_t(n) : 0);
  std::vector<size_t> plan_bytes(size_t(n), 0);
  std::vector<int> crc(size_t(n), CTD_OK);
  for_each_page(n, h->host_threads, [&](int i) {
    const JobPage& p = job.pages[size_t(i)];
    const uint8_t* mask = reinterpret_cast<const uint8_t*>(res + job.head.masks + p.off);
    prc[size_t(i)] = host_group_page(page_in(res, job.head, i, p, mask), p.section, bs, wins[size_t(i)]);
    if (crops && prc[size_t(i)] == CTD_OK)
      crc[size_t(i)] = plan_page_regions(p.section, bs, p.iw, p.ih, job.textheight, plans[size_t(i)],
                                         &plan_bytes[size_t(i)]);
  });
  for (int i = 0; i < n; ++i)
    if (prc[size_t(i)] != CTD_OK) return ctd_fail(h, prc[size_t(i)], "group_output failed on page %d of the batch", i);
  for (int i = 0; i < n; ++i)
    if (crc[size_t(i)] != CTD_OK)
      return ctd_fail(h, crc[size_t(i)], "ctd_region_plan refused page %d of the batch (%dx%d, textheight %d)", i,
                      job.pages[size_t(i)].ih, job.pages[size_t(i)].iw, job.textheight);
  // phase C on the post stream over the slot's resident pages and masks
  cudaStream_t st = h->post;
  // enqueued here for ctd_submit_pages, not at submit: a wait enqueued at submit time would also hold this batch's
  // phase C behind the forward of every batch submitted before the worker reached it (ctd_submit_full enqueues it at
  // submit as well)
  CK(cudaStreamWaitEvent(st, s.ev_out_ready, 0));   // phase C never starts before its phase A copy
  // ctd_submit_full: block sections to the device arena copy (one gather then moves everything)
  if (job.d_blocks)
    CK(cudaMemcpyAsync(job.d_blocks, job.pages[0].section, job.blocks_bytes, cudaMemcpyHostToDevice, st));
  if (crops)
    if (int rc = crop_stage(h, s, region_pages(job), plans, plan_bytes, !job.results_on_device, st)) return rc;
  CK(cudaMemsetAsync(job.d_ref, 0, job.total, st));
  const auto boxes = job.keep_undetected ? section_boxes(job.pages) : std::vector<std::vector<int32_t>>();
  if (int rc = phase_c(h, job.pages, wins, boxes, job_planes(job), job.refine_mode, job.keep_undetected, st,
                       h->post_refine, h->pg_cc, s.pinned, h->pipe_pinned_cap))
    return rc;
  return finish_batch(h, job, st);
}

// ctd_submit_refine's batch on the worker: phase C on the caller's pages, masks and windows, or with a refined input
// refine_undetected_mask alone
static int run_refine_batch(ctd_handle* h, const PipeJob& job) {
  Slot& s = h->slot[job.slot];
  cudaStream_t st = h->post;
  CK(cudaStreamWaitEvent(st, s.ev_out_ready, 0));   // the packed pages and masks are in place
  const Planes pl = job_planes(job);
  if (job.refined_input) {
    if (int rc = refine_undetected(h, job.pages, job.boxes, pl, job.refine_mode, st, h->pg_cc, h->post_refine,
                                   s.pinned, h->pipe_pinned_cap))
      return rc;
  } else {
    CK(cudaMemsetAsync(job.d_ref, 0, job.total, st));
    if (int rc = phase_c(h, job.pages, job.wins, job.boxes, pl, job.refine_mode, job.keep_undetected, st,
                         h->post_refine, h->pg_cc, s.pinned, h->pipe_pinned_cap))
      return rc;
  }
  return finish_batch(h, job, st);
}

// ctd_submit_regions's batch on the worker: each page's lines planned on the host threads, then the crop stage
static int run_regions_batch(ctd_handle* h, const PipeJob& job) {
  Slot& s = h->slot[job.slot];
  const int n = int(job.pages.size());
  std::vector<size_t> first(size_t(n) + 1, 0);
  for (int i = 0; i < n; ++i) first[size_t(i) + 1] = first[size_t(i)] + size_t(job.n_lines[size_t(i)]);
  std::vector<std::vector<ctd_region>> plans(static_cast<size_t>(n));
  std::vector<size_t> plan_bytes(size_t(n), 0);
  std::vector<int> prc(size_t(n), CTD_OK);
  for_each_page(n, h->host_threads, [&](int i) {
    const JobPage& p = job.pages[size_t(i)];
    const int nl = job.n_lines[size_t(i)];
    plans[size_t(i)].resize(size_t(nl));
    if (nl > 0)
      prc[size_t(i)] = ctd_region_plan(job.lines.data() + first[size_t(i)], nl, p.iw, p.ih, job.textheight,
                                       plans[size_t(i)].data(), &plan_bytes[size_t(i)]);
  });
  for (int i = 0; i < n; ++i)
    if (prc[size_t(i)] != CTD_OK)
      return ctd_fail(h, prc[size_t(i)], "ctd_region_plan refused page %d of the batch (%dx%d, textheight %d)", i,
                      job.pages[size_t(i)].ih, job.pages[size_t(i)].iw, job.textheight);
  cudaStream_t st = h->post;
  CK(cudaStreamWaitEvent(st, s.ev_out_ready, 0));   // the host pages are in place, the device pages written
  if (int rc = crop_stage(h, s, region_pages(job), plans, plan_bytes, !job.results_on_device, st)) return rc;
  CK(cudaEventRecord(s.ev_post_done, st));
  return CTD_OK;
}

// ---- batch pipeline -------------------------------------------------------------------------------------------------
static void pipe_worker(ctd_handle* h) {
  cudaSetDevice(h->cfg.device);
  for (;;) {
    PipeJob job;
    {
      std::unique_lock<std::mutex> lk(h->pipe_mu);
      h->pipe_cv.wait(lk, [&] { return h->pipe_quit || !h->pipe_queue.empty(); });
      if (h->pipe_queue.empty()) return;    // quit requested and nothing left
      job = std::move(h->pipe_queue.front());
      h->pipe_queue.pop_front();
    }
    const int rc = job.refine ? run_refine_batch(h, job) : job.regions ? run_regions_batch(h, job) : run_batch(h, job);
    std::string err;
    if (rc != CTD_OK) err = h->err;
    {
      std::lock_guard<std::mutex> lk(h->pipe_mu);
      Slot& s = h->slot[job.slot];
      s.state = rc == CTD_OK ? 2 : 3;
      s.rc = rc;
      s.err = err;
    }
    h->pipe_done_cv.notify_all();
  }
}

// hands a submitted batch to the worker
static void queue_job(ctd_handle* h, PipeJob&& job) {
  Slot& s = h->slot[job.slot];
  {
    std::lock_guard<std::mutex> lk(h->pipe_mu);
    s.state = 1;
    h->pipe_queue.push_back(std::move(job));
  }
  h->pipe_cv.notify_one();
  s.busy = true;
}

// the handle's pipeline, set up by its first submission: copy streams, post stream, each slot's staging, events and
// pinned window tables, and the worker thread
static int ensure_full_pipeline(ctd_handle* h) {
  if (h->pipe_thread.joinable()) return CTD_OK;
  CK(cudaStreamCreateWithFlags(&h->copy_in, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&h->copy_out, cudaStreamNonBlocking));
  int lo = 0, hi = 0;
  CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CK(cudaStreamCreateWithPriority(&h->post, cudaStreamNonBlocking, hi));
  // window tables: <= CTD_MAX_BLOCKS windows per page (32 bytes each) and <= area / chunk + rows chunks per window
  // (16 bytes each)
  h->pipe_pinned_cap = size_t(h->cfg.max_batch) * (size_t(CTD_MAX_BLOCKS) * sizeof(RefineWin) +
                                                   size_t(CTD_MAX_BLOCKS) * sizeof(RefineChunk) * 8) + (size_t(8) << 20);
  const size_t in_bytes = size_t(h->cfg.max_batch) * h->cfg.max_h * h->cfg.max_w * 3;
  for (Slot& s : h->slot) {
    CK(cudaMalloc(&s.d_stage_in, in_bytes));
    CK(cudaMalloc(&s.d_stage_out, h->layout.total));
    for (cudaEvent_t* e : {&s.ev_in_done, &s.ev_in_free, &s.ev_out_ready, &s.ev_out_done, &s.ev_post_done})
      CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    CK(cudaHostAlloc(reinterpret_cast<void**>(&s.pinned), h->pipe_pinned_cap, cudaHostAllocDefault));
  }
  const char* ht = getenv("CTD_HOST_THREADS");
  const unsigned hc = std::thread::hardware_concurrency();
  h->host_threads = ht ? atoi(ht) : int(std::max(1u, std::min(8u, hc ? hc / 2 : 4u)));
  h->pipe_quit = false;
  h->pipe_thread = std::thread(pipe_worker, h);
  return CTD_OK;
}

// stops the worker and frees the handle-wide pipeline state (each slot's own: Slot::release)
void ctd_pipeline_shutdown(ctd_handle* h) {
  if (h->pipe_thread.joinable()) {
    {
      std::lock_guard<std::mutex> lk(h->pipe_mu);
      h->pipe_quit = true;
    }
    h->pipe_cv.notify_all();
    h->pipe_thread.join();
  }
  if (h->post) cudaStreamDestroy(h->post);
  h->post = nullptr;
  if (h->dev_out) cudaStreamDestroy(h->dev_out);
  h->dev_out = nullptr;
  h->pg_cc.release();
  h->post_refine.release();
}

// phase A of a batch of n net-sized pages on slot s:
//   copy_in:  [wait slot's staging free] H2D pages -> stage_in[slot]
//   compute:  [wait H2D] stage_in -> d_pages (D2D), forward, arena -> stage_out[slot] (D2D)
//   copy_out: [wait arena copy] D2H stage_out[slot] -> results_host
// so the H2D of batch i+1 and the D2H of batch i-1 run under the forward of batch i.  Device pages skip copy_in.
static int stage_phase_a(ctd_handle* h, Slot& s, const uint8_t* pages, bool pages_on_device, int n, int ph, int pw,
                         ShapePlan& sp, void* results_host) {
  const size_t bytes = size_t(n) * ph * pw * 3;
  if (!pages_on_device) {
    CK(cudaStreamWaitEvent(h->copy_in, s.ev_in_free, 0));   // no-op before the slot's first use
    CK(cudaMemcpyAsync(s.d_stage_in, pages, bytes, cudaMemcpyHostToDevice, h->copy_in));
    CK(cudaEventRecord(s.ev_in_done, h->copy_in));
    CK(cudaEventRecord(h->ev0, h->stream));
    CK(cudaStreamWaitEvent(h->stream, s.ev_in_done, 0));
    CK(cudaMemcpyAsync(h->d_pages, s.d_stage_in, bytes, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaEventRecord(s.ev_in_free, h->stream));
  } else {
    CK(cudaEventRecord(h->ev0, h->stream));
    CK(cudaMemcpyAsync(h->d_pages, pages, bytes, cudaMemcpyDeviceToDevice, h->stream));
  }
  if (int rc = enqueue_forward(h, n, ph, pw, sp)) return rc;
  CK(cudaStreamWaitEvent(h->stream, s.ev_out_done, 0));  // previous D2H of this slot has drained
  CK(cudaMemcpyAsync(s.d_stage_out, h->d_mask_u8, h->layout.a_bytes, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaEventRecord(s.ev_out_ready, h->stream));
  CK(cudaStreamWaitEvent(h->copy_out, s.ev_out_ready, 0));
  CK(cudaMemcpyAsync(results_host, s.d_stage_out, h->layout.a_bytes, cudaMemcpyDeviceToHost, h->copy_out));
  CK(cudaEventRecord(s.ev_out_done, h->copy_out));
  return CTD_OK;
}

extern "C" int ctd_submit_full(ctd_handle* h, int32_t slot, const uint8_t* pages, int32_t n, int32_t ph, int32_t pw,
                               int32_t pages_on_device, int32_t refine_mode, void* results_host) {
  if (!h || !pages || !results_host || slot < 0 || slot > 1) return CTD_E_INVALID;
  if (h->cfg.debug_skip_postproc) return ctd_fail(h, CTD_E_INVALID, "ctd_submit_full needs the full pipeline");
  Slot& s = h->slot[slot];
  if (s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has an uncollected submission", slot);
  ShapePlan* sp = nullptr;
  if (int rc = prepare_forward(h, n, ph, pw, &sp)) return rc;
  if (int rc = ensure_full_pipeline(h)) return rc;
  s.start(false, false);
  // the previous use of this slot's staging (refine reads stage_in / stage_out) ended with its collect
  if (int rc = stage_phase_a(h, s, pages, pages_on_device != 0, n, ph, pw, *sp, results_host)) return rc;
  CK(cudaStreamWaitEvent(h->post, s.ev_out_ready, 0));   // phase C never starts before its phase A copy
  // net-sized pages letterbox to themselves: resize_ratio 1
  const ArenaLayout& L = h->layout;
  const size_t px = size_t(ph) * pw;
  PipeJob job;
  job.slot = slot; job.refine_mode = refine_mode;
  job.results_host = static_cast<char*>(results_host);
  job.head = PagesHead{L.det, L.cnt, L.lb, L.ls, L.lc, 0};
  job.refined = L.refined;
  for (int i = 0; i < n; ++i)
    job.pages.push_back(JobPage{ph, pw, 1.f, 1.f, size_t(i) * px, job.results_host + L.blocks + size_t(i) * L.blocks_stride});
  job.total = size_t(n) * px;
  job.d_img = pages_on_device ? pages : s.d_stage_in;
  job.d_mask = s.d_stage_out;
  job.d_ref = s.d_stage_out + L.refined;
  job.d_blocks = s.d_stage_out + L.blocks;
  job.blocks_bytes = size_t(n) * L.blocks_stride;
  queue_job(h, std::move(job));
  return CTD_OK;
}

// true when [p, p + 1) is device memory of `device` (cudaPointerGetAttributes; clears the error it may leave)
static bool is_device_memory(const void* p, int device) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice && a.device == device;
}

// a page (ch = 3) or mask (ch = 1) of a batch in device memory: strides in range, and its first and last byte memory
// of the handle's GPU
static int check_device_image(ctd_handle* h, const char* what, int i, const ctd_device_page& d, int ih, int iw, int ch) {
  const int64_t kMaxStride = int64_t(1) << 31;   // keeps the image's last byte offset inside int64
  const int64_t sc = ch == 3 ? d.stride_c : 0;
  if (d.stride_h < 0 || d.stride_w < 0 || sc < 0 || d.stride_h > kMaxStride || d.stride_w > kMaxStride || sc > kMaxStride)
    return ctd_fail(h, CTD_E_INVALID, "%s %d: strides (%lld, %lld, %lld) out of range [0, 2^31]", what, i,
                    (long long)d.stride_h, (long long)d.stride_w, (long long)sc);
  const uint8_t* last = d.data + (ih - 1) * d.stride_h + (iw - 1) * d.stride_w + (ch - 1) * sc;
  if (!is_device_memory(d.data, h->cfg.device) || !is_device_memory(last, h->cfg.device))
    return ctd_fail(h, CTD_E_INVALID, "%s %d (%p) is not device memory of GPU %d", what, i, (const void*)d.data,
                    h->cfg.device);
  return CTD_OK;
}

// the slot's page tables, allocated at its first batch: max_batch PageGeom entries, then at pg_gather_off room for a
// GatherPage entry per page and per mask of a batch, at pg_out_off an OutputGather entry per page (ctd_submit_outputs),
// at pg_half_off its float16 flags (what NMS reads) and at pg_flag_off its non-finite flags (device: written by the
// ingest; host: their copy back)
static int ensure_page_tables(ctd_handle* h, Slot& s) {
  if (s.h_pg_tab) return CTD_OK;
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t nb = size_t(h->cfg.max_batch);
  h->pg_gather_off = al(nb * sizeof(PageGeom));
  h->pg_out_off = al(h->pg_gather_off + 2 * nb * sizeof(GatherPage));
  h->pg_half_off = al(h->pg_out_off + nb * sizeof(OutputGather));
  h->pg_flag_off = al(h->pg_half_off + nb * sizeof(int32_t));
  const size_t tab_bytes = h->pg_flag_off + nb * sizeof(int32_t);
  CK(cudaHostAlloc(reinterpret_cast<void**>(&s.h_pg_tab), tab_bytes, cudaHostAllocDefault));
  CK(cudaMalloc(reinterpret_cast<void**>(&s.d_pg_tab), tab_bytes));
  return CTD_OK;
}

// H2D on `st` of the byte ranges [off(i), off(i) + bytes(i)) from src to dst of the pages that are not on the device
// (dev[i].data == NULL, or dev NULL), one copy per run of consecutive such pages
template <typename Off, typename Len>
static int copy_host_runs(ctd_handle* h, const ctd_device_page* dev, int n, uint8_t* dst, const uint8_t* src, Off off,
                          Len bytes, cudaStream_t st) {
  for (int i = 0; i < n;) {
    if (dev && dev[i].data) { ++i; continue; }
    int j = i;
    while (j + 1 < n && !(dev && dev[j + 1].data)) ++j;
    const size_t lo = off(i), hi = off(j) + bytes(j);
    CK(cudaMemcpyAsync(dst + lo, src + lo, hi - lo, cudaMemcpyHostToDevice, st));
    i = j + 1;
  }
  return CTD_OK;
}

// a network output map of page i (ctd_submit_outputs), elements of esz bytes: device memory of the handle's GPU from
// its first to its last element (strides in [0, 2^31]), or a host pointer, whose byte span [p, p + *bytes) is returned
static int check_output_map(ctd_handle* h, const char* what, int i, const float* fp, size_t esz, int on_device,
                            int64_t s0, int64_t s1, int n0, int n1, size_t* bytes) {
  const char* p = reinterpret_cast<const char*>(fp);
  const int64_t kMaxStride = int64_t(1) << 31;
  *bytes = 0;
  if (n0 < 1 || n1 < 1) return CTD_OK;   // no element (blks with 0 rows)
  if (!p) return ctd_fail(h, CTD_E_INVALID, "page %d: %s is NULL", i, what);
  if (s0 < 0 || s1 < 0 || s0 > kMaxStride || s1 > kMaxStride)
    return ctd_fail(h, CTD_E_INVALID, "page %d: %s strides (%lld, %lld) out of range [0, 2^31]", i, what, (long long)s0,
                    (long long)s1);
  const char* last = p + ((n0 - 1) * s0 + (n1 - 1) * s1) * int64_t(esz);
  if (on_device) {
    if (!is_device_memory(p, h->cfg.device) || !is_device_memory(last, h->cfg.device))
      return ctd_fail(h, CTD_E_INVALID, "page %d: %s (%p) is not device memory of GPU %d", i, what, (const void*)p,
                      h->cfg.device);
  } else {
    *bytes = size_t(last - p) + esz;
  }
  return CTD_OK;
}

// ctd_submit_pages, and with `outs` ctd_submit_outputs_dtype: the caller's network outputs (page i in dtypes[i])
// staged in place of the letterbox and the forward
static int submit_pages_job(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, int32_t net_h,
                            int32_t net_w, const uint8_t* input_host, const ctd_device_page* dev,
                            const ctd_net_output* outs, const int32_t* dtypes, int32_t refine_mode,
                            int32_t keep_undetected, int32_t textheight, int32_t results_on_device, void* results_host) {
  const char* entry = outs ? "ctd_submit_outputs" : "ctd_submit_pages";
  if (!h || !pages || !results_host || slot < 0 || slot > 1 || n < 1) return CTD_E_INVALID;
  if (textheight != 0 && textheight < 2) return ctd_fail(h, CTD_E_INVALID, "textheight %d < 2", textheight);
  if (h->cfg.debug_skip_postproc) return ctd_fail(h, CTD_E_INVALID, "%s needs the full pipeline", entry);
  Slot& s = h->slot[slot];
  if (s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has an uncollected submission", slot);
  if (n > h->cfg.max_batch) return ctd_fail(h, CTD_E_CAPACITY, "batch %d exceeds max_batch %d", n, h->cfg.max_batch);
  // the offsets decide where the copies write: they must be the plan's
  std::vector<ctd_page_entry> pg(pages, pages + n);
  size_t in_bytes = 0, res_bytes = 0;
  if (int rc = ctd_pages_plan(pg.data(), n, net_h, net_w, &in_bytes, &res_bytes))
    return ctd_fail(h, rc, "the pages do not letterbox into a %dx%d net input", net_h, net_w);
  if (memcmp(pg.data(), pages, size_t(n) * sizeof(ctd_page_entry)) != 0)
    return ctd_fail(h, CTD_E_INVALID, "the page entries are not the ones ctd_pages_plan returns");
  size_t rows = 0;
  for (int i = 0; i < n; ++i) {
    rows += size_t(pg[size_t(i)].ih);
    if (keep_undetected && size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) > kCclMaxPixels)
      return ctd_fail(h, CTD_E_CAPACITY, "page %d (%dx%d): refine_undetected_mask labels pages of at most 2^28 pixels", i,
                      pg[size_t(i)].ih, pg[size_t(i)].iw);
  }
  if (rows > size_t(INT32_MAX)) return ctd_fail(h, CTD_E_CAPACITY, "the pages of a batch have more than 2^31 rows");
  // pages in device memory: strides, and the first and last byte each page reads must be memory of this GPU
  CK(cudaSetDevice(h->cfg.device));
  int n_dev = 0;
  for (int i = 0; i < n; ++i) {
    if (!dev || !dev[i].data) {
      if (!input_host) return ctd_fail(h, CTD_E_INVALID, "page %d is in neither input_host nor device memory", i);
      continue;
    }
    if (int rc = check_device_image(h, "page", i, dev[i], pg[size_t(i)].ih, pg[size_t(i)].iw, 3)) return rc;
    ++n_dev;
  }
  // the outputs: shapes, and each map device memory of this GPU or a host span copied into the slot's out_in
  const int no = 5 + h->cfg.nc, ws_rows = rows_per_image(net_h, net_w);
  std::vector<std::array<size_t, 3>> host_bytes(outs ? size_t(n) : 0), host_off(outs ? size_t(n) : 0);
  size_t out_in_bytes = 0;
  if (outs) {
    if (net_h > h->cfg.max_h || net_w > h->cfg.max_w)
      return ctd_fail(h, CTD_E_SHAPE, "net input %dx%d exceeds the engine's %dx%d", net_h, net_w, h->cfg.max_h,
                      h->cfg.max_w);
    for (int i = 0; i < n; ++i) {
      const ctd_net_output& o = outs[i];
      if (dtypes[i] != CTD_DTYPE_F32 && dtypes[i] != CTD_DTYPE_F16)
        return ctd_fail(h, CTD_E_INVALID, "page %d: dtype %d is not a CTD_DTYPE_* value", i, dtypes[i]);
      const size_t esz = dtypes[i] == CTD_DTYPE_F16 ? 2 : 4;
      if (o.rows < 0 || o.rows > ws_rows)
        return ctd_fail(h, CTD_E_CAPACITY, "page %d: %d blks rows, the %dx%d workspace holds 0 to %d", i, o.rows, net_h,
                        net_w, ws_rows);
      auto& hb = host_bytes[size_t(i)];
      if (int rc = check_output_map(h, "blks", i, o.blks, esz, o.blks_on_device, o.blks_stride_r, o.blks_stride_c,
                                    o.rows, no, &hb[0]))
        return rc;
      if (int rc = check_output_map(h, "mask", i, o.mask, esz, o.mask_on_device, o.mask_stride_h, o.mask_stride_w,
                                    net_h, net_w, &hb[1]))
        return rc;
      if (int rc = check_output_map(h, "lines", i, o.lines, esz, o.lines_on_device, o.lines_stride_h,
                                    o.lines_stride_w, net_h, net_w, &hb[2]))
        return rc;
      for (int k = 0; k < 3; ++k) {
        host_off[size_t(i)][size_t(k)] = out_in_bytes;
        out_in_bytes += (hb[size_t(k)] + 255) / 256 * 256;
      }
    }
  }
  ShapePlan* sp = nullptr;
  if (!outs)
    if (int rc = prepare_forward(h, n, net_h, net_w, &sp)) return rc;
  if (int rc = ensure_full_pipeline(h)) return rc;
  const ArenaLayout& L = h->layout;
  const PagesHead hd = pages_head(n);
  const size_t total = size_t(pg[0].refined_off - pg[0].mask_off);
  const size_t d2h = size_t(pg[0].refined_off);                       // phase-A rows + masks
  s.start(textheight > 0, results_on_device != 0);
  // grown while the slot is idle: its collect has synchronised the work of its last batch
  if (int rc = s.pg_in.grow(h, in_bytes, std::nullopt)) return rc;
  if (int rc = s.pg_res.grow(h, d2h + total, std::nullopt)) return rc;
  if (keep_undetected)
    if (int rc = s.pg_aux.grow(h, 2 * total, std::nullopt)) return rc;
  if (out_in_bytes)
    if (int rc = s.out_in.grow(h, out_in_bytes, std::nullopt)) return rc;
  if (int rc = ensure_page_tables(h, s)) return rc;
  PageGeom* tab = s.h_pg_tab;
  GatherPage* gtab = reinterpret_cast<GatherPage*>(reinterpret_cast<char*>(tab) + h->pg_gather_off);
  int row0 = 0, n_gather = 0, gather_rows = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    tab[i] = PageGeom{e.page_off, e.mask_off - int64_t(hd.masks), e.ih, e.iw, e.unpad_h, e.unpad_w, row0, 0};
    row0 += e.ih;
    if (dev && dev[i].data) {
      const ctd_device_page& d = dev[i];
      gtab[n_gather++] = GatherPage{d.data, (long long)d.stride_h, (long long)d.stride_w, (long long)d.stride_c,
                                    s.pg_in.p + e.page_off, e.ih, e.iw, gather_rows,
                                    d.stride_c == 1 && d.stride_w == 3 ? 1 : 0, 3, 0};
      gather_rows += e.ih;
    }
  }
  // phase A: tables and host pages in on copy_in (a batch with device pages copies only its host pages' byte ranges,
  // one copy per run of consecutive host pages); the device pages' events, the gather of the device pages, letterbox,
  // forward, back-projection and the phase-A rows on the engine stream; rows + masks out on copy_out
  OutputGather* otab = reinterpret_cast<OutputGather*>(reinterpret_cast<char*>(tab) + h->pg_out_off);
  int32_t* half_tab = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(tab) + h->pg_half_off);
  for (int i = 0; outs && i < n; ++i) {
    const ctd_net_output& o = outs[i];
    // a host map is read from its copy in out_in, at the same strides
    auto at = [&](const float* p, int k) -> const void* {
      if (host_bytes[size_t(i)][size_t(k)]) return s.out_in.p + host_off[size_t(i)][size_t(k)];
      return p;
    };
    half_tab[i] = dtypes[i] == CTD_DTYPE_F16 ? 1 : 0;
    otab[i] = OutputGather{o.blks_on_device ? o.blks : at(o.blks, 0), (long long)o.blks_stride_r,
                           (long long)o.blks_stride_c, o.mask_on_device ? o.mask : at(o.mask, 1),
                           (long long)o.mask_stride_h, (long long)o.mask_stride_w,
                           o.lines_on_device ? o.lines : at(o.lines, 2), (long long)o.lines_stride_h,
                           (long long)o.lines_stride_w, o.rows, half_tab[i]};
  }
  const size_t tab_bytes = outs       ? h->pg_half_off + size_t(n) * sizeof(int32_t)
                           : n_gather ? h->pg_gather_off + size_t(n_gather) * sizeof(GatherPage)
                                      : size_t(n) * sizeof(PageGeom);
  CK(cudaMemcpyAsync(s.d_pg_tab, tab, tab_bytes, cudaMemcpyHostToDevice, h->copy_in));
  for (int i = 0; outs && i < n; ++i) {
    const float* src[3] = {outs[i].blks, outs[i].mask, outs[i].lines};
    for (int k = 0; k < 3; ++k)
      if (const size_t b = host_bytes[size_t(i)][size_t(k)])
        CK(cudaMemcpyAsync(s.out_in.p + host_off[size_t(i)][size_t(k)], src[k], b, cudaMemcpyHostToDevice, h->copy_in));
  }
  if (n_dev == 0) {
    CK(cudaMemcpyAsync(s.pg_in.p, input_host, in_bytes, cudaMemcpyHostToDevice, h->copy_in));
  } else {
    if (int rc = copy_host_runs(h, dev, n, s.pg_in.p, input_host, [&](int i) { return size_t(pg[size_t(i)].page_off); },
                                [&](int i) { return size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) * 3; },
                                h->copy_in))
      return rc;
  }
  CK(cudaEventRecord(s.ev_in_done, h->copy_in));
  CK(cudaEventRecord(h->ev0, h->stream));
  CK(cudaStreamWaitEvent(h->stream, s.ev_in_done, 0));
  if (n_gather) {
    for (int i = 0; i < n; ++i)
      if (dev[i].data && dev[i].event) CK(cudaStreamWaitEvent(h->stream, static_cast<cudaEvent_t>(dev[i].event), 0));
    CK(gather_pages_launch(reinterpret_cast<const GatherPage*>(reinterpret_cast<const char*>(s.d_pg_tab) +
                                                               h->pg_gather_off),
                           n_gather, gather_rows, h->stream));
  }
  if (outs) {
    // the caller's outputs into the workspace the forward would have written, then the forward's NMS and DB tail
    for (int i = 0; i < n; ++i)
      if (outs[i].event) CK(cudaStreamWaitEvent(h->stream, static_cast<cudaEvent_t>(outs[i].event), 0));
    int32_t* d_flags = reinterpret_cast<int32_t*>(reinterpret_cast<char*>(s.d_pg_tab) + h->pg_flag_off);
    CK(cudaMemsetAsync(d_flags, 0, size_t(n) * sizeof(int32_t), h->stream));
    CK(gather_outputs_launch(reinterpret_cast<const OutputGather*>(reinterpret_cast<const char*>(s.d_pg_tab) +
                                                                   h->pg_out_off),
                             n, net_h, net_w, no, ws_rows, h->cfg.db_thresh, h->d_mask_u8, h->d_lines, h->d_bitmap,
                             h->d_blks, d_flags, h->stream));
    int cnt = 0;
    if (int rc = launch_nms(h, n, net_h, net_w, h->stream, &cnt,
                            reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(s.d_pg_tab) + h->pg_half_off)))
      return rc;
    if (int rc = launch_db_post(h, n, net_h, net_w, h->stream, &cnt)) return rc;
  } else {
    CK(letterbox_batch_launch(s.pg_in.p, s.d_pg_tab, n, h->d_pages, net_h, net_w, h->stream));
    if (int rc = enqueue_forward(h, n, net_h, net_w, *sp)) return rc;
  }
  uint8_t* d_res = s.pg_res.p;
  CK(backproject_batch_launch(h->d_mask_u8, net_h, net_w, s.d_pg_tab, n, row0, d_res + hd.masks, h->stream));
  const size_t nb = size_t(n);
  CK(cudaMemcpyAsync(d_res + hd.det, h->d_mask_u8 + L.det, nb * 300 * 6 * 4, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(d_res + hd.cnt, h->d_mask_u8 + L.cnt, nb * 4, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(d_res + hd.lb, h->d_mask_u8 + L.lb, nb * 1000 * 8 * 2, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(d_res + hd.ls, h->d_mask_u8 + L.ls, nb * 1000 * 4, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(d_res + hd.lc, h->d_mask_u8 + L.lc, nb * 4, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaEventRecord(s.ev_out_ready, h->stream));
  CK(cudaStreamWaitEvent(h->copy_out, s.ev_out_ready, 0));
  CK(cudaMemcpyAsync(results_host, d_res, d2h, cudaMemcpyDeviceToHost, h->copy_out));
  PipeJob job;
  if (outs) {
    char* h_flags = reinterpret_cast<char*>(s.h_pg_tab) + h->pg_flag_off;
    CK(cudaMemcpyAsync(h_flags, reinterpret_cast<char*>(s.d_pg_tab) + h->pg_flag_off, size_t(n) * sizeof(int32_t),
                       cudaMemcpyDeviceToHost, h->copy_out));
    job.nonfinite = reinterpret_cast<const int32_t*>(h_flags);
  }
  CK(cudaEventRecord(s.ev_out_done, h->copy_out));
  job.slot = slot; job.refine_mode = refine_mode;
  job.results_host = static_cast<char*>(results_host);
  job.head = hd;
  job.refined = size_t(pg[0].refined_off);
  for (const ctd_page_entry& e : pg) {
    Letterbox lb;
    letterbox_of(e.ih, e.iw, net_h, net_w, lb);   // planned: cannot fail
    job.pages.push_back(JobPage{e.ih, e.iw, lb.ratio_x, lb.ratio_y, size_t(e.mask_off) - hd.masks,
                                job.results_host + e.blocks_off});
  }
  job.total = total;
  job.d_img = s.pg_in.p;
  job.d_mask = d_res + hd.masks;
  job.d_ref = d_res + pg[0].refined_off;
  job.d_aux = keep_undetected ? s.pg_aux.p : nullptr;
  job.keep_undetected = keep_undetected ? 1 : 0;
  job.textheight = textheight;
  job.results_on_device = results_on_device ? 1 : 0;
  if (results_on_device) s.dev_pages = std::move(pg);
  queue_job(h, std::move(job));
  return CTD_OK;
}

extern "C" int ctd_submit_pages(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, int32_t net_h,
                                int32_t net_w, const uint8_t* input_host, const ctd_device_page* dev,
                                int32_t refine_mode, int32_t keep_undetected, int32_t textheight,
                                int32_t results_on_device, void* results_host) {
  return submit_pages_job(h, slot, pages, n, net_h, net_w, input_host, dev, nullptr, nullptr, refine_mode,
                          keep_undetected, textheight, results_on_device, results_host);
}

extern "C" int ctd_submit_outputs(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n, int32_t net_h,
                                  int32_t net_w, const uint8_t* input_host, const ctd_device_page* dev_pages,
                                  const ctd_net_output* outs, int32_t refine_mode, int32_t keep_undetected,
                                  int32_t textheight, int32_t results_on_device, void* results_host) {
  // every page float32 (the job reads dtypes only once it has checked n against max_batch)
  const std::vector<int32_t> f32(h && n > 0 && n <= h->cfg.max_batch ? size_t(n) : 1, CTD_DTYPE_F32);
  return ctd_submit_outputs_dtype(h, slot, pages, n, net_h, net_w, input_host, dev_pages, outs, f32.data(), refine_mode,
                                  keep_undetected, textheight, results_on_device, results_host);
}

extern "C" int ctd_submit_outputs_dtype(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n,
                                        int32_t net_h, int32_t net_w, const uint8_t* input_host,
                                        const ctd_device_page* dev_pages, const ctd_net_output* outs,
                                        const int32_t* dtypes, int32_t refine_mode, int32_t keep_undetected,
                                        int32_t textheight, int32_t results_on_device, void* results_host) {
  if (!outs || !dtypes) return CTD_E_INVALID;
  return submit_pages_job(h, slot, pages, n, net_h, net_w, input_host, dev_pages, outs, dtypes, refine_mode,
                          keep_undetected, textheight, results_on_device, results_host);
}

static_assert(int(CTD_PRE_F32_NCHW) == int(PRE_F32_NCHW) && int(CTD_PRE_F16_NCHW) == int(PRE_F16_NCHW) &&
                  int(CTD_PRE_U8_NHWC) == int(PRE_U8_NHWC),
              "ctd_preprocess_pages formats");

extern "C" int ctd_preprocess_pages(ctd_handle* h, const ctd_page_entry* pages, int32_t n, int32_t net_h, int32_t net_w,
                                    const uint8_t* input_host, const ctd_device_page* dev, int32_t format,
                                    int32_t reverse_channels, void* dst, void* stream) {
  if (!h || !pages || !dst || n < 1) return CTD_E_INVALID;
  if (format != CTD_PRE_F32_NCHW && format != CTD_PRE_F16_NCHW && format != CTD_PRE_U8_NHWC)
    return ctd_fail(h, CTD_E_INVALID, "format %d is not a CTD_PRE_* format", format);
  if (n > h->cfg.max_batch) return ctd_fail(h, CTD_E_CAPACITY, "batch %d exceeds max_batch %d", n, h->cfg.max_batch);
  std::vector<ctd_page_entry> pg(pages, pages + n);
  size_t in_bytes = 0, res_bytes = 0;
  if (int rc = ctd_pages_plan(pg.data(), n, net_h, net_w, &in_bytes, &res_bytes))
    return ctd_fail(h, rc, "the pages do not letterbox into a %dx%d net input", net_h, net_w);
  if (memcmp(pg.data(), pages, size_t(n) * sizeof(ctd_page_entry)) != 0)
    return ctd_fail(h, CTD_E_INVALID, "the page entries are not the ones ctd_pages_plan returns");
  size_t rows = 0;
  for (int i = 0; i < n; ++i) rows += size_t(pg[size_t(i)].ih);
  if (rows > size_t(INT32_MAX)) return ctd_fail(h, CTD_E_CAPACITY, "the pages of a batch have more than 2^31 rows");
  CK(cudaSetDevice(h->cfg.device));
  const size_t elem = format == CTD_PRE_F32_NCHW ? 4 : format == CTD_PRE_F16_NCHW ? 2 : 1;
  const size_t out_bytes = size_t(n) * 3 * size_t(net_h) * size_t(net_w) * elem;
  if (reinterpret_cast<uintptr_t>(dst) % 16) return ctd_fail(h, CTD_E_INVALID, "dst must be 16-byte aligned");
  if (!is_device_memory(dst, h->cfg.device) || !is_device_memory(static_cast<char*>(dst) + out_bytes - 1, h->cfg.device))
    return ctd_fail(h, CTD_E_INVALID, "dst (%p, %zu bytes) is not device memory of GPU %d", dst, out_bytes,
                    h->cfg.device);
  int n_dev = 0;
  for (int i = 0; i < n; ++i) {
    if (!dev || !dev[i].data) {
      if (!input_host) return ctd_fail(h, CTD_E_INVALID, "page %d is in neither input_host nor device memory", i);
      continue;
    }
    if (int rc = check_device_image(h, "page", i, dev[i], pg[size_t(i)].ih, pg[size_t(i)].iw, 3)) return rc;
    ++n_dev;
  }
  // everything from here on is ordered on the caller's stream, after the last call's reads of the page buffer and the
  // tables (ev_pre): a larger page buffer is a stream-ordered allocation, the old one a stream-ordered free
  cudaStream_t cs = static_cast<cudaStream_t>(stream);
  auto al = [](size_t v) { return (v + 255) / 256 * 256; };
  const size_t gather_off = al(size_t(h->cfg.max_batch) * sizeof(PageGeom));
  if (!h->d_pre_tab)
    CK(cudaMalloc(reinterpret_cast<void**>(&h->d_pre_tab), gather_off + size_t(h->cfg.max_batch) * sizeof(GatherPage)));
  if (!h->ev_pre) CK(cudaEventCreateWithFlags(&h->ev_pre, cudaEventDisableTiming));
  CK(cudaStreamWaitEvent(cs, h->ev_pre, 0));   // a no-op before the first record
  if (in_bytes > h->pre_in_cap) {
    if (h->pre_in) CK(cudaFreeAsync(h->pre_in, cs));
    h->pre_in = nullptr;
    h->pre_in_cap = 0;
    CK(cudaMallocAsync(reinterpret_cast<void**>(&h->pre_in), in_bytes + in_bytes / 4, cs));
    h->pre_in_cap = in_bytes + in_bytes / 4;
  }
  // the tables: PageGeom per page, then at gather_off a GatherPage per device page
  std::vector<char> tab(gather_off + size_t(n_dev) * sizeof(GatherPage));
  PageGeom* geo = reinterpret_cast<PageGeom*>(tab.data());
  GatherPage* gtab = reinterpret_cast<GatherPage*>(tab.data() + gather_off);
  int n_gather = 0, gather_rows = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    geo[i] = PageGeom{e.page_off, 0, e.ih, e.iw, e.unpad_h, e.unpad_w, 0, 0};
    if (dev && dev[i].data) {
      const ctd_device_page& d = dev[i];
      gtab[n_gather++] = GatherPage{d.data, (long long)d.stride_h, (long long)d.stride_w, (long long)d.stride_c,
                                    h->pre_in + e.page_off, e.ih, e.iw, gather_rows,
                                    d.stride_c == 1 && d.stride_w == 3 ? 1 : 0, 3, 0};
      gather_rows += e.ih;
    }
  }
  const size_t tab_bytes = n_gather ? tab.size() : size_t(n) * sizeof(PageGeom);
  tab.resize((tab_bytes + 15) / 16 * 16);
  CK(upload_table_launch(tab.data(), tab.size(), h->d_pre_tab, cs));
  if (n_dev < n) {
    if (int rc = copy_host_runs(h, dev, n, h->pre_in, input_host, [&](int i) { return size_t(pg[size_t(i)].page_off); },
                                [&](int i) { return size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) * 3; }, cs))
      return rc;
  }
  if (n_gather) {
    for (int i = 0; i < n; ++i)
      if (dev[i].data && dev[i].event) CK(cudaStreamWaitEvent(cs, static_cast<cudaEvent_t>(dev[i].event), 0));
    CK(gather_pages_launch(reinterpret_cast<const GatherPage*>(h->d_pre_tab + gather_off), n_gather, gather_rows, cs));
  }
  CK(letterbox_tensor_launch(h->pre_in, reinterpret_cast<const PageGeom*>(h->d_pre_tab), n, dst, net_h, net_w, format,
                             reverse_channels != 0, cs));
  CK(cudaEventRecord(h->ev_pre, cs));
  return CTD_OK;
}

extern "C" int ctd_submit_refine(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n,
                                 const int32_t* xyxy, const int32_t* n_blocks, const uint8_t* input_host,
                                 const ctd_device_page* dev_pages, const ctd_device_page* dev_masks,
                                 int32_t refine_mode, int32_t keep_undetected, int32_t refined_input,
                                 int32_t results_on_device, void* results_host) {
  if (!h || !pages || !n_blocks || !results_host || slot < 0 || slot > 1 || n < 1) return CTD_E_INVALID;
  Slot& s = h->slot[slot];
  if (s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has an uncollected submission", slot);
  if (n > h->cfg.max_batch) return ctd_fail(h, CTD_E_CAPACITY, "batch %d exceeds max_batch %d", n, h->cfg.max_batch);
  if (refined_input && (!keep_undetected || !input_host))
    return ctd_fail(h, CTD_E_INVALID, "a refined input needs keep_undetected and input_host");
  // the offsets and windows decide what the copies and the refine touch: they must be the plan's
  std::vector<ctd_page_entry> pg(pages, pages + n);
  int64_t nb = 0;
  for (int i = 0; i < n; ++i) nb += std::max(n_blocks[i], 0);
  std::vector<int32_t> win(static_cast<size_t>(nb) * 4), status(static_cast<size_t>(nb));
  size_t in_bytes = 0, res_bytes = 0;
  if (int rc = ctd_refine_plan(pg.data(), n, xyxy, n_blocks, win.data(), status.data(), &in_bytes, &res_bytes))
    return ctd_fail(h, rc, "ctd_refine_plan refuses the batch");
  if (memcmp(pg.data(), pages, size_t(n) * sizeof(ctd_page_entry)) != 0)
    return ctd_fail(h, CTD_E_INVALID, "the page entries are not the ones ctd_refine_plan returns");
  const size_t total = in_bytes / 5;
  PipeJob job;
  job.wins.resize(size_t(n));
  job.boxes.resize(size_t(n));
  size_t rows = 0;
  for (int i = 0, b = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    rows += size_t(e.ih);
    if (keep_undetected && size_t(e.ih) * size_t(e.iw) > kCclMaxPixels)
      return ctd_fail(h, CTD_E_CAPACITY, "page %d (%dx%d): refine_undetected_mask labels pages of at most 2^28 pixels", i,
                      e.ih, e.iw);
    for (int k = 0; k < n_blocks[i]; ++k, ++b) {
      // refine_mask raises on such a block; refine_undetected_mask alone only compares the boxes
      if (!refined_input && status[size_t(b)] != 0)
        return ctd_fail(h, CTD_E_INVALID, "page %d, block %d (%d, %d, %d, %d): %s", i, k, xyxy[4 * b], xyxy[4 * b + 1],
                        xyxy[4 * b + 2], xyxy[4 * b + 3],
                        status[size_t(b)] == 1 ? "its window is empty, refine_mask raises on it"
                                               : "its window does not fit int32");
      job.wins[size_t(i)].insert(job.wins[size_t(i)].end(), &win[4 * size_t(b)], &win[4 * size_t(b)] + 4);
      job.boxes[size_t(i)].insert(job.boxes[size_t(i)].end(), xyxy + 4 * size_t(b), xyxy + 4 * size_t(b) + 4);
    }
  }
  if (rows > size_t(INT32_MAX)) return ctd_fail(h, CTD_E_CAPACITY, "the pages of a batch have more than 2^31 rows");
  CK(cudaSetDevice(h->cfg.device));
  int n_dev_pages = 0, n_dev_masks = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    for (int m = 0; m < 2; ++m) {
      const ctd_device_page* d = m ? dev_masks : dev_pages;
      if (d && d[i].data) {
        if (int rc = check_device_image(h, m ? "mask" : "page", i, d[i], e.ih, e.iw, m ? 1 : 3)) return rc;
        ++(m ? n_dev_masks : n_dev_pages);
      } else if (!input_host) {
        return ctd_fail(h, CTD_E_INVALID, "%s %d is in neither input_host nor device memory", m ? "mask" : "page", i);
      }
    }
  }
  if (int rc = ensure_full_pipeline(h)) return rc;
  s.start(false, results_on_device != 0);
  // grown while the slot is idle: its collect has synchronised the work of its last batch.  pg_in: the packed pages;
  // pg_res: the frame of masks and mask_refined planes the refine reads and writes in place
  if (int rc = s.pg_in.grow(h, 3 * total, std::nullopt)) return rc;
  if (int rc = s.pg_res.grow(h, res_bytes, std::nullopt)) return rc;
  if (keep_undetected)
    if (int rc = s.pg_aux.grow(h, 2 * total, std::nullopt)) return rc;
  if (int rc = ensure_page_tables(h, s)) return rc;
  GatherPage* gtab = reinterpret_cast<GatherPage*>(reinterpret_cast<char*>(s.h_pg_tab) + h->pg_gather_off);
  int n_gather = 0, gather_rows = 0;
  for (int i = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    if (dev_pages && dev_pages[i].data) {
      const ctd_device_page& d = dev_pages[i];
      gtab[n_gather++] = GatherPage{d.data, (long long)d.stride_h, (long long)d.stride_w, (long long)d.stride_c,
                                    s.pg_in.p + e.page_off, e.ih, e.iw, gather_rows,
                                    d.stride_c == 1 && d.stride_w == 3 ? 1 : 0, 3, 0};
      gather_rows += e.ih;
    }
    if (dev_masks && dev_masks[i].data) {
      const ctd_device_page& d = dev_masks[i];
      gtab[n_gather++] = GatherPage{d.data, (long long)d.stride_h, (long long)d.stride_w, 0, s.pg_res.p + e.mask_off,
                                    e.ih, e.iw, gather_rows, d.stride_w == 1 ? 1 : 0, 1, 0};
      gather_rows += e.ih;
    }
  }
  // the tables and the host pages and masks in on copy_in (only the byte ranges of the images in input_host); the
  // waits on the device images' events and one gather of every device page and mask on the engine stream
  cudaStream_t cin = h->copy_in;
  const uint8_t* host_frame = input_host ? input_host + 3 * total : nullptr;
  if (n_gather)
    CK(cudaMemcpyAsync(reinterpret_cast<char*>(s.d_pg_tab) + h->pg_gather_off, gtab, size_t(n_gather) * sizeof(GatherPage),
                       cudaMemcpyHostToDevice, cin));
  if (n_dev_pages < n)
    if (int rc = copy_host_runs(h, dev_pages, n, s.pg_in.p, input_host,
                                [&](int i) { return size_t(pg[size_t(i)].page_off); },
                                [&](int i) { return size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) * 3; }, cin))
      return rc;
  if (n_dev_masks < n)
    if (int rc = copy_host_runs(h, dev_masks, n, s.pg_res.p, host_frame,
                                [&](int i) { return size_t(pg[size_t(i)].mask_off); },
                                [&](int i) { return size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw); }, cin))
      return rc;
  if (refined_input) CK(cudaMemcpyAsync(s.pg_res.p + total, host_frame + total, total, cudaMemcpyHostToDevice, cin));
  CK(cudaEventRecord(s.ev_in_done, cin));
  CK(cudaStreamWaitEvent(h->stream, s.ev_in_done, 0));
  if (n_gather) {
    for (int i = 0; i < n; ++i)
      for (const ctd_device_page* d : {dev_pages, dev_masks})
        if (d && d[i].data && d[i].event) CK(cudaStreamWaitEvent(h->stream, static_cast<cudaEvent_t>(d[i].event), 0));
    CK(gather_pages_launch(reinterpret_cast<const GatherPage*>(reinterpret_cast<const char*>(s.d_pg_tab) +
                                                               h->pg_gather_off),
                           n_gather, gather_rows, h->stream));
  }
  CK(cudaEventRecord(s.ev_out_ready, h->stream));
  job.refine = true;
  job.slot = slot; job.refine_mode = refine_mode;
  job.results_host = static_cast<char*>(results_host);
  job.head.masks = 0;
  job.refined = total;
  for (const ctd_page_entry& e : pg) job.pages.push_back(JobPage{e.ih, e.iw, 1.f, 1.f, size_t(e.mask_off), nullptr});
  job.total = total;
  job.d_img = s.pg_in.p;
  job.d_mask = s.pg_res.p;
  job.d_ref = s.pg_res.p + total;
  job.d_aux = keep_undetected ? s.pg_aux.p : nullptr;
  job.keep_undetected = keep_undetected ? 1 : 0;
  job.refined_input = refined_input ? 1 : 0;
  job.results_on_device = results_on_device ? 1 : 0;
  if (results_on_device) s.dev_pages = std::move(pg);
  queue_job(h, std::move(job));
  return CTD_OK;
}

extern "C" int ctd_submit_regions(ctd_handle* h, int32_t slot, const ctd_page_entry* pages, int32_t n,
                                  const ctd_region_line* lines, const int32_t* n_lines, int32_t textheight,
                                  const uint8_t* input_host, const ctd_device_page* dev_pages,
                                  int32_t results_on_device) {
  if (!h || !pages || !n_lines || slot < 0 || slot > 1 || n < 1) return CTD_E_INVALID;
  if (textheight < 2) return ctd_fail(h, CTD_E_INVALID, "textheight %d < 2", textheight);
  Slot& s = h->slot[slot];
  if (s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has an uncollected submission", slot);
  if (n > h->cfg.max_batch) return ctd_fail(h, CTD_E_CAPACITY, "batch %d exceeds max_batch %d", n, h->cfg.max_batch);
  int64_t total_lines = 0;
  for (int i = 0; i < n; ++i) {
    if (n_lines[i] < 0) return ctd_fail(h, CTD_E_INVALID, "page %d: n_lines %d < 0", i, n_lines[i]);
    total_lines += n_lines[i];
  }
  if (total_lines > INT32_MAX) return ctd_fail(h, CTD_E_CAPACITY, "more than 2^31 lines in one batch");
  if (total_lines > 0 && !lines) return CTD_E_INVALID;
  for (int i = 0; i < n; ++i) {
    const int ih = pages[i].ih, iw = pages[i].iw;
    if (ih < 1 || iw < 1 || ih >= 32767 || iw >= 32767)
      return ctd_fail(h, CTD_E_SHAPE, "page %d (%dx%d): the crop planner takes pages with sides in [1, 32767)", i, ih, iw);
  }
  // the offsets decide where the copies write: they must be the ones ctd_refine_plan lays out (no blocks)
  std::vector<ctd_page_entry> pg(pages, pages + n);
  const std::vector<int32_t> no_blocks(static_cast<size_t>(n), 0);
  size_t in_bytes = 0, res_bytes = 0;
  if (int rc = ctd_refine_plan(pg.data(), n, nullptr, no_blocks.data(), nullptr, nullptr, &in_bytes, &res_bytes))
    return ctd_fail(h, rc, "ctd_refine_plan refuses the pages");
  if (memcmp(pg.data(), pages, size_t(n) * sizeof(ctd_page_entry)) != 0)
    return ctd_fail(h, CTD_E_INVALID, "the page entries are not the ones ctd_refine_plan returns");
  const size_t total = in_bytes / 5;
  CK(cudaSetDevice(h->cfg.device));
  int n_dev = 0;
  for (int i = 0; i < n; ++i) {
    if (dev_pages && dev_pages[i].data) {
      if (int rc = check_device_image(h, "page", i, dev_pages[i], pg[size_t(i)].ih, pg[size_t(i)].iw, 3)) return rc;
      ++n_dev;
    } else if (!input_host) {
      return ctd_fail(h, CTD_E_INVALID, "page %d is in neither input_host nor device memory", i);
    }
  }
  if (int rc = ensure_full_pipeline(h)) return rc;
  s.start(true, results_on_device != 0, false);
  // grown while the slot is idle: its collect has synchronised the work of its last batch.  The host pages are
  // copied into pg_in at their offsets; the device pages are read where they are
  if (n_dev < n) {
    if (int rc = s.pg_in.grow(h, 3 * total, std::nullopt)) return rc;
    if (int rc = copy_host_runs(h, dev_pages, n, s.pg_in.p, input_host,
                                [&](int i) { return size_t(pg[size_t(i)].page_off); },
                                [&](int i) { return size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) * 3; },
                                h->copy_in))
      return rc;
  }
  CK(cudaEventRecord(s.ev_in_done, h->copy_in));
  CK(cudaStreamWaitEvent(h->stream, s.ev_in_done, 0));
  if (dev_pages)
    for (int i = 0; i < n; ++i)
      if (dev_pages[i].data && dev_pages[i].event)
        CK(cudaStreamWaitEvent(h->stream, static_cast<cudaEvent_t>(dev_pages[i].event), 0));
  CK(cudaEventRecord(s.ev_out_ready, h->stream));
  PipeJob job;
  job.regions = true;
  job.slot = slot;
  job.textheight = textheight;
  job.results_on_device = results_on_device ? 1 : 0;
  for (const ctd_page_entry& e : pg) job.pages.push_back(JobPage{e.ih, e.iw, 1.f, 1.f, size_t(e.page_off) / 3, nullptr});
  job.total = total;
  job.d_img = s.pg_in.p;
  job.lines.assign(lines, lines + total_lines);
  job.n_lines.assign(n_lines, n_lines + n);
  if (dev_pages) job.dev.assign(dev_pages, dev_pages + n);
  if (results_on_device) s.dev_pages = std::move(pg);
  queue_job(h, std::move(job));
  return CTD_OK;
}

extern "C" int ctd_collect(ctd_handle* h, int32_t slot) {
  if (!h || slot < 0 || slot > 1) return CTD_E_INVALID;
  Slot& s = h->slot[slot];
  if (!s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has nothing in flight", slot);
  CK(cudaSetDevice(h->cfg.device));
  int rc;
  {
    std::unique_lock<std::mutex> lk(h->pipe_mu);
    h->pipe_done_cv.wait(lk, [&] { return s.state >= 2; });
    rc = s.rc;
    if (rc != CTD_OK) h->err = s.err;
    s.state = 0;
  }
  s.busy = false;
  if (rc != CTD_OK) return rc;
  CK(cudaEventSynchronize(s.ev_post_done));
  s.collected = true;
  return CTD_OK;
}

extern "C" int ctd_collect_device(ctd_handle* h, int32_t slot, void* const* page_dst) {
  if (!h || slot < 0 || slot > 1 || !page_dst) return CTD_E_INVALID;
  const Slot& s = h->slot[slot];
  if (s.busy || !s.collected || !s.on_device)
    return ctd_fail(h, CTD_E_INVALID, "slot %d holds no collected batch with results on the device", slot);
  CK(cudaSetDevice(h->cfg.device));
  const std::vector<ctd_page_entry>& pg = s.dev_pages;
  const int n = int(pg.size());
  // bytes page i receives: its two masks (none in a ctd_submit_regions batch), then its crops
  auto page_bytes = [&](int i) {
    const size_t m = s.masks ? 2 * size_t(pg[size_t(i)].ih) * size_t(pg[size_t(i)].iw) : 0;
    return m + (s.crops ? s.crop_base[size_t(i) + 1] - s.crop_base[size_t(i)] : 0);
  };
  for (int i = 0; i < n; ++i)
    if (page_bytes(i) > 0 && (!page_dst[i] || !is_device_memory(page_dst[i], h->cfg.device)))
      return ctd_fail(h, CTD_E_INVALID, "page_dst[%d] (%p) is not device memory of GPU %d", i, page_dst[i],
                      h->cfg.device);
  if (!h->dev_out) CK(cudaStreamCreateWithFlags(&h->dev_out, cudaStreamNonBlocking));
  // the slot's planes: the collect has synchronised the batch's last writes (ev_post_done)
  const uint8_t* d_res = s.pg_res.p;
  const uint8_t* d_px = s.crops ? s.d_crop.p + s.crop_px_off : nullptr;
  for (int i = 0; i < n; ++i) {
    const ctd_page_entry& e = pg[size_t(i)];
    const size_t px = s.masks ? size_t(e.ih) * size_t(e.iw) : 0;
    uint8_t* dst = static_cast<uint8_t*>(page_dst[i]);
    if (s.masks) {
      CK(cudaMemcpyAsync(dst, d_res + e.mask_off, px, cudaMemcpyDeviceToDevice, h->dev_out));
      CK(cudaMemcpyAsync(dst + px, d_res + e.refined_off, px, cudaMemcpyDeviceToDevice, h->dev_out));
    }
    if (s.crops) {
      const size_t b0 = s.crop_base[size_t(i)], b1 = s.crop_base[size_t(i) + 1];
      if (b1 > b0) CK(cudaMemcpyAsync(dst + 2 * px, d_px + b0, b1 - b0, cudaMemcpyDeviceToDevice, h->dev_out));
    }
  }
  CK(cudaStreamSynchronize(h->dev_out));
  return CTD_OK;
}

extern "C" int ctd_debug_read_slot(ctd_handle* h, int32_t slot, int32_t plane, size_t offset, uint8_t* out,
                                   size_t bytes) {
  if (!h || slot < 0 || slot > 1 || plane < 0 || plane > 2 || !out) return CTD_E_INVALID;
  const Slot& s = h->slot[slot];
  if (s.busy) return ctd_fail(h, CTD_E_INVALID, "slot %d has an uncollected submission", slot);
  const uint8_t* base = plane == 0 ? s.pg_in.p : plane == 1 ? s.pg_res.p : h->d_pages;
  const size_t size = plane == 0   ? s.pg_in.cap
                      : plane == 1 ? s.pg_res.cap
                      : h->have_forward ? size_t(h->n) * h->ph * h->pw * 3 : 0;
  if (offset > size || bytes > size - offset)
    return ctd_fail(h, CTD_E_INVALID, "plane %d holds %zu bytes: [%zu, +%zu) is past its end", plane, size, offset,
                    bytes);
  if (bytes == 0) return CTD_OK;
  CK(cudaSetDevice(h->cfg.device));
  // after the engine stream's work: the gather, the letterbox and the forward that reads d_pages run there
  CK(cudaMemcpyAsync(out, base + offset, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return CTD_OK;
}

extern "C" int ctd_collect_regions(ctd_handle* h, int32_t slot, const ctd_region** plan, int32_t* n_regions,
                                   const int32_t** page_first, const uint8_t** pixels, size_t* bytes) {
  if (!h || slot < 0 || slot > 1 || !plan || !n_regions || !page_first || !pixels || !bytes) return CTD_E_INVALID;
  const Slot& s = h->slot[slot];
  if (s.busy || !s.collected || !s.crops)
    return ctd_fail(h, CTD_E_INVALID,
                    "slot %d holds no collected ctd_submit_pages batch with a textheight or ctd_submit_regions batch", slot);
  *plan = s.crop_plan.data();
  *n_regions = int32_t(s.crop_plan.size());
  *page_first = s.crop_first.data();
  *bytes = s.crop_bytes;
  *pixels = s.crop_bytes && !s.on_device ? s.h_crop.p + s.crop_px_off : nullptr;
  return CTD_OK;
}

extern "C" int ctd_device_arena(ctd_handle* h, int32_t slot, void** base, void** post_stream) {
  if (!h || slot < 0 || slot > 1 || !base) return CTD_E_INVALID;
  if (!h->slot[slot].d_stage_out)
    return ctd_fail(h, CTD_E_INVALID, "no pipelined submission has been made on this handle");
  *base = h->slot[slot].d_stage_out;
  if (post_stream) *post_stream = h->post;
  return CTD_OK;
}

// ---- single page, any size --------------------------------------------------------------------------------------------
extern "C" int ctd_detect_page(ctd_handle* h, const uint8_t* page, int32_t ih, int32_t iw, int32_t net_h, int32_t net_w,
                               int32_t refine_mode, int32_t keep_undetected, uint8_t* mask_out, uint8_t* mask_refined_out,
                               ctd_block* blocks, int32_t blocks_cap, int32_t* lines_out, int32_t lines_cap, double* dist_out,
                               int32_t dist_cap, int32_t* n_blocks) {
  if (!h || !page || !mask_out || !mask_refined_out || !n_blocks) return CTD_E_INVALID;
  if (ih < 1 || iw < 1) return ctd_fail(h, CTD_E_SHAPE, "bad page size %dx%d", ih, iw);
  *n_blocks = 0;
  if (keep_undetected && size_t(ih) * iw > kCclMaxPixels)
    return ctd_fail(h, CTD_E_CAPACITY, "page %dx%d: refine_undetected_mask labels pages of at most 2^28 pixels", ih, iw);
  Letterbox geo;
  if (!letterbox_of(ih, iw, net_h, net_w, geo)) return ctd_fail(h, CTD_E_SHAPE, "page does not letterbox into the net input");
  ShapePlan* sp = nullptr;
  if (int rc = prepare_forward(h, 1, net_h, net_w, &sp)) return rc;
  const size_t px = size_t(ih) * iw, pxa = (px + 255) / 256 * 256;
  // io scratch: page (3 px) | page-sized mask | mask_refined | second refine output | thresholded mask
  if (int rc = h->io_scratch.grow(h, pxa * 7 + 1024, h->stream)) return rc;
  uint8_t* d_page = h->io_scratch.p;
  uint8_t* d_mask = d_page + pxa * 3;
  uint8_t* d_ref = d_mask + pxa;
  uint8_t* d_ref2 = d_ref + pxa;
  uint8_t* d_thr = d_ref2 + pxa;
  cudaStream_t st = h->stream;
  CK(cudaEventRecord(h->ev0, st));
  CK(cudaMemcpyAsync(d_page, page, px * 3, cudaMemcpyHostToDevice, st));
  const bool same = ih == net_h && iw == net_w;
  if (same) CK(cudaMemcpyAsync(h->d_pages, d_page, px * 3, cudaMemcpyDeviceToDevice, st));
  else CK(resize_linear_u8_launch(d_page, ih, iw, size_t(iw) * 3, 3, h->d_pages, geo.unpad_h, geo.unpad_w, net_h, net_w, st));
  if (int rc = enqueue_forward(h, 1, net_h, net_w, *sp)) return rc;
  // mask back-projection (inference.py:164-168)
  if (same) CK(cudaMemcpyAsync(d_mask, h->d_mask_u8, px, cudaMemcpyDeviceToDevice, st));
  else CK(resize_linear_u8_launch(h->d_mask_u8, geo.unpad_h, geo.unpad_w, size_t(net_w), 1, d_mask, ih, iw, ih, iw, st));
  // the phase-A rows of the page, laid out as those of a one-page batch
  const PagesHead hd = pages_head(1);
  std::vector<char> rows(hd.masks);
  CK(cudaMemcpyAsync(mask_out, d_mask, px, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(rows.data() + hd.det, h->d_det, 300 * 6 * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(rows.data() + hd.cnt, h->d_det_count, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(rows.data() + hd.lb, h->d_line_boxes, 1000 * 8 * 2, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(rows.data() + hd.ls, h->d_line_scores, 1000 * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(rows.data() + hd.lc, h->d_line_count, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemsetAsync(d_ref, 0, pxa, st));
  CK(cudaStreamSynchronize(st));
  // phase B
  const BlockSection L = block_section_layout();
  std::vector<char> section(L.stride);
  const std::vector<JobPage> pages{JobPage{ih, iw, geo.ratio_x, geo.ratio_y, 0, section.data()}};
  std::vector<std::vector<int32_t>> wins(1);
  if (int rc = host_group_page(page_in(rows.data(), hd, 0, pages[0], mask_out), section.data(), L, wins[0]))
    return ctd_fail(h, rc, "group_output failed");
  const ctd_page_blocks* hdr = reinterpret_cast<const ctd_page_blocks*>(section.data());
  const ctd_block* rec = reinterpret_cast<const ctd_block*>(section.data() + L.rec_off);
  const int nb = hdr->n_blocks;
  *n_blocks = nb;
  if (nb > blocks_cap || hdr->n_lines > lines_cap || hdr->n_dist > dist_cap || (nb > 0 && (!blocks || !lines_out)) ||
      (hdr->n_dist > 0 && !dist_out))
    return ctd_fail(h, CTD_E_CAPACITY, "%d blocks / %d lines / %d distances do not fit the output arrays", nb, hdr->n_lines, hdr->n_dist);
  if (nb > 0) {
    memcpy(blocks, rec, size_t(nb) * sizeof(ctd_block));
    memcpy(lines_out, section.data() + L.lines_off, size_t(hdr->n_lines) * 32);
    if (hdr->n_dist > 0) memcpy(dist_out, section.data() + L.dist_off, size_t(hdr->n_dist) * 8);
  }
  // phase C; refine_undetected_mask modifies the page mask in place and it is returned, as in the reference
  const Planes pl{d_page, d_mask, d_ref, d_ref2, d_thr, px};
  const auto boxes = keep_undetected ? section_boxes(pages) : std::vector<std::vector<int32_t>>();
  if (int rc = phase_c(h, pages, wins, boxes, pl, refine_mode, keep_undetected, st, h->refine_scratch, h->cc_scratch,
                       nullptr, 0))
    return rc;
  if (keep_undetected) CK(cudaMemcpyAsync(mask_out, d_mask, px, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(mask_refined_out, d_ref, px, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return CTD_OK;
}
