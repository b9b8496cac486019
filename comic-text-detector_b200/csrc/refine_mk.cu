// refine_mask on the GPU, phase-synchronous form (reference utils/textmask.py:159-169 and callees 16-132).
//
// Why one kernel per phase: a single cooperative kernel with a CTA (or an 8-CTA cluster) per block window and barriers
// between the phases, measured on the synthetic 1024^2 pages, ran every phase as a latency-bound sweep with one pixel
// per thread iteration: a 1 Mpx window kept 8 SMs busy for 15 ms while the other 140 idled, and a batch of 16 pages
// (~50 Mpx of overlapping windows) cost 29 ms -- 4.5x the network.  Here every phase is its own kernel over ALL window
// pixels of the batch: the windows are cut into chunks (RefineChunk, kernels.h: whole rows of <= kChunkPx pixels, or
// row segments of <= kChunkPx pixels when a window row is longer; table built by the host, which knows the window
// sizes), one CTA per chunk, so a giant window is spread over the whole GPU and the kernel boundary is the barrier.
// Per-window reductions (histograms, xor sums, the two largest hole areas) go through a small per-window state record
// in global memory; per-window scalar decisions are one-CTA-per-window kernels.  Results are bit-identical to the
// oracle (tests/test_gpu_refine.py).
//
// The binary planes are BIT planes, 32 pixels per word, in global memory as in shared memory: the six positive
// candidates (k_xor thresholds every pixel once), the predicted mask, `merged` and the dilation's output.  One thread per
// (half) word does the work of 16 - 32 pixels with funnel shifts, ANDs and popcounts -- the erosions of phase 0, the
// dilation, the run contacts of the labelling, the per-label sums and the merges (one update per RUN, not per pixel).
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>

#include "kernels.h"

namespace ctd {

namespace {

constexpr int kThreads = 256;
constexpr int kChunkPx = kRefineChunkPx;

struct WinState {
  int hist[4][256];               // [0] grey of the eroded-mask pixels, [1..3] B, G, R of the whole window
  unsigned long long xs[12];      // xor sums: [k][pos/neg] for 3 colours, then 3 channels
  int lo[3], hi[3], otsu_t[3], ncol;
  int nproc, proc_kind[4], proc_neg[4];
  int area0, max1, cnt1, max2;
  int pad[2];
};

struct Ctx {
  const uint8_t* img_all;
  const uint8_t* mask_all;
  uint32_t* out_all;
  const RefineWin* wins;
  const RefineChunk* chunks;
  WinState* st;
  int mode;
  // planes (window-pixel indexed)
  uint16_t* lab;     // chunk-local root of every pixel, as an offset in its chunk; kNoLabel = background
  uint16_t* roots;   // chunk-local roots of each chunk (offsets), at the chunk's own pixel range; nroots[chunk] of them
  int* nroots;       // per chunk
  int* P;            // union-find parents of the chunk-local roots (only root entries are ever touched)
  int* acc;
  uint8_t* grey;
  // bit planes, each chunk's words at its RefineChunk::woff; the bits past a chunk's last pixel are zero
  unsigned* cand;    // 6 planes of plane_words: grey in [lo, hi] of colour 0..2, then channel B, G, R > its Otsu threshold
  unsigned *pred, *merged, *tmp;
  size_t plane_words;
};
constexpr uint16_t kNoLabel = 0xffffu;
constexpr unsigned kMergeBit = 0x8000u;   // of a root list entry: the root's component merges (k_decide_roots)
static_assert(kChunkPx <= int(kMergeBit), "a chunk-local offset fits the 15 bits below kMergeBit");

// A chunk's pixels are contiguous in the window planes: chunk pixel k is window pixel i0 + k, at window row
// y0 + k / cols and column x0 + k % cols.  A chunk is one row (rows == 1) or whole rows (x0 == 0, cols == rw).
struct View {
  RefineWin win;
  int w, rw, rh, y0, x0, rows, cols, i0, cnt, woff;   // woff: the chunk's first word in the bit planes
  const uint8_t* img;
  const uint8_t* mask;
};

__device__ __forceinline__ View view_of(const Ctx& c, int chunk) {
  View v;
  const RefineChunk ch = c.chunks[chunk];
  v.w = ch.win;
  v.win = c.wins[ch.win];
  v.rw = v.win.x2 - v.win.x1;
  v.rh = v.win.y2 - v.win.y1;
  v.y0 = ch.y0;
  v.x0 = ch.x0;
  v.rows = ch.rows;
  v.cols = min(v.rw - ch.x0, kChunkPx);
  v.i0 = ch.y0 * v.rw + ch.x0;
  v.cnt = ch.rows * v.cols;
  v.woff = ch.woff;
  v.img = c.img_all + size_t(v.win.page_off) * 3;
  v.mask = c.mask_all + size_t(v.win.page_off);
  return v;
}

// Window pixel index of the first pixel of the chunk that holds window pixel (y, x): the host's cut (RefineJob::add,
// pipeline.cu) into whole rows per chunk, or row segments of kChunkPx pixels when a row is longer.
__device__ __forceinline__ int chunk_start(int y, int x, int rw) {
  if (rw > kChunkPx) return y * rw + (x & ~(kChunkPx - 1));
  const int rows_per = refine_rows_per_chunk(rw);
  return (y / rows_per) * rows_per * rw;
}
static_assert((kChunkPx & (kChunkPx - 1)) == 0, "row segments start on multiples of kChunkPx");

// ---- union-find over a window's chunk-local roots (other CTAs update it: parent reads bypass L1) ---------------------
__device__ __forceinline__ int uf_find(const int* L, int a) {
  int p = __ldcg(L + a);
  while (p != a) {
    a = p;
    p = __ldcg(L + a);
  }
  return a;
}
__device__ __forceinline__ int uf_find_compress(int* L, int a) {
  const int r = uf_find(L, a);
  while (a != r) {
    const int p = __ldcg(L + a);
    if (p <= r) break;
    atomicMin(&L[a], r);
    a = p;
  }
  return r;
}
__device__ __forceinline__ void uf_union(int* L, int a, int b) {
  bool done;
  do {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a < b) {
      const int old = atomicMin(&L[b], a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(&L[a], b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

__device__ __forceinline__ void hist_add(int* hist, int bin) {
  // flat regions (page background, solid strokes): the whole warp hits one bin -> one atomic, no match.any
  const int b0 = __shfl_sync(0xffffffffu, bin, 0);
  if (__all_sync(0xffffffffu, bin == b0)) {
    if ((threadIdx.x & 31) == 0 && bin >= 0) atomicAdd(&hist[bin], 32);
    return;
  }
  // mixed warp: plain shared-memory atomics (the hardware serialises equal bins; measured faster than a match.any vote)
  if (bin >= 0) atomicAdd(&hist[bin], 1);
}

// i = q * d + r for 0 <= i < 2^24 (exact in float; |q error| <= 1 before the correction), else integer division.
// Every sweep below turns window-local pixel indices into (y, x): a runtime integer division per pixel was a
// quarter of the instructions of the lean kernels.
struct DivW { int d; float inv; bool fast; };
__device__ __forceinline__ DivW make_div(int d, int n) { return DivW{d, __frcp_rn(float(d)), n < (1 << 24)}; }
__device__ __forceinline__ void divmod(int i, const DivW& dv, int& q, int& r) {
  if (dv.fast) {
    q = __float2int_rz(__int2float_rn(i) * dv.inv);
    r = i - q * dv.d;
    if (r < 0) { --q; r += dv.d; } else if (r >= dv.d) { ++q; r -= dv.d; }
  } else {
    q = i / dv.d;
    r = i - q * dv.d;
  }
}

// ---- bit-plane words of a chunk -----------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned tail_mask(int w, int cnt) {   // the bits of word w that are pixels of the chunk
  const int rem = cnt - 32 * w;
  return rem >= 32 ? 0xffffffffu : (1u << rem) - 1u;
}
// of 32 consecutive pixels from column x0 of rows rw wide: the bits whose pixel is the first of its row
__device__ __forceinline__ unsigned row_start_bits(int x0, int rw) {
  unsigned rs = 0u;
  for (int j = x0 == 0 ? 0 : rw - x0; j < 32; j += rw) rs |= 1u << j;
  return rs;
}
// A run: consecutive foreground pixels of one row and one word.  M: foreground bits; S = run starts = M & (~(M << 1) | row
// starts).  Last bit of the run that starts at bit sbit, and the bits lo..hi:
__device__ __forceinline__ int run_end(unsigned M, unsigned S, int sbit) {
  const unsigned stop = (~M | S) & (0xfffffffeu << sbit);          // first position after the run
  return stop ? __ffs(stop) - 2 : 31;
}
__device__ __forceinline__ unsigned span_bits(int lo, int hi) {
  return (hi == 31 ? 0xffffffffu : ((2u << hi) - 1u)) & ~((1u << lo) - 1u);
}
// Word d of a bit array into which the `len` bits of `src` from bit sb on are copied at bit db (0 where the word holds
// none of them).  May read the word after the last one that holds a copied bit.
__device__ __forceinline__ unsigned copied_word(const unsigned* src, int sb, int len, int db, int d) {
  const int r = 32 * d - db;                      // index in the copied range of the word's bit 0
  if (r <= -32 || r >= len) return 0u;
  const int pos = sb + max(r, 0);
  unsigned o = __funnelshift_r(src[pos >> 5], src[(pos >> 5) + 1], pos & 31);
  if (len - max(r, 0) < 32) o &= (1u << (len - max(r, 0))) - 1u;
  return r < 0 ? o << -r : o;
}

// ---- phase 0: grey, pred bits (cross erosion > 60), merged = 0, histograms ------------------------------------------
constexpr int kU = 4;   // pixels per thread and outer iteration: the loads of all kU pixels are issued before the first use
// Halo rectangle of a chunk: its rows plus one row above and below, its columns plus one column left and right, clipped
// to the window.  Whole rows: <= 3 * kChunkPx pixels (the rows of a chunk, two halo rows of <= kChunkPx); a row
// segment: 3 rows of <= kChunkPx + 2 pixels.  3 * (kChunkPx + 2) = 24582 bits = 769 words, read up to one word past
// the last written one: kExtWords holds both.
constexpr int kExtWords = (3 * kChunkPx) / 32 + 4;
static_assert(3 * (kChunkPx + 2) / 32 + 2 < kExtWords, "a row segment's halo rectangle fits the shared bit masks");
struct Halo {
  int ystart, xs, ew, ext, off;   // first row / column, width (the row stride of the bit masks), pixels, chunk offset
};
__device__ __forceinline__ Halo halo_of(const View& v) {
  Halo h;
  h.ystart = v.y0 > 0 ? v.y0 - 1 : 0;
  h.xs = v.x0 > 0 ? v.x0 - 1 : 0;
  h.ew = min(v.x0 + v.cols + 1, v.rw) - h.xs;
  h.ext = (min(v.y0 + v.rows + 1, v.rh) - h.ystart) * h.ew;
  // chunk pixel k sits at rectangle position k + off: a chunk is one row, or its rows are as wide as the rectangle
  h.off = (v.y0 - h.ystart) * h.ew + v.x0 - h.xs;
  return h;
}
__device__ __forceinline__ unsigned bits_from(const unsigned* M, int pos) {   // 32 bits starting at pixel `pos` (< 0 reads 0)
  if (pos <= -32) return 0u;
  if (pos < 0) return M[0] << (-pos);
  const int w = pos >> 5, sft = pos & 31;
  return __funnelshift_r(M[w], M[w + 1], sft);
}
// 32 pixels of a chunk starting at window column x: the bits whose pixel is the first (rs) / last (re) of its window row
// (bits past the end of a row segment are not pixels of the chunk)
__device__ __forceinline__ void row_ends(int x, int rw, unsigned& rs, unsigned& re) {
  rs = row_start_bits(x, rw);
  int xe = x + 32;                                  // column of the pixel after the 32
  if (xe >= rw) xe %= rw;
  re = (rs >> 1) | (xe == 0 ? 0x80000000u : 0u);
}
// The two erosions of the mask crop are threshold tests of a minimum: min over the cross > 60 <=> NO pixel of the cross is
// <= 60.  So the chunk's halo rectangle is packed into two "bad pixel" bit masks (mask <= 60, mask <= 127) by warp
// ballots -- ONE mask load per pixel instead of nine bounds-checked ones -- and one thread per 32-pixel word ORs the
// 5 / 9 shifted views (window row ends masked; outside the window reads 0 = not bad = BORDER_CONSTANT +inf).
__global__ void __launch_bounds__(kThreads) k_phase0(Ctx c) {
  __shared__ int sh[4][256];
  __shared__ unsigned N60[kExtWords], N127[kExtWords];
  __shared__ unsigned F127[kChunkPx / 32 + 1];
  const View v = view_of(c, blockIdx.x);
  for (int i = threadIdx.x; i < 1024; i += kThreads) (&sh[0][0])[i] = 0;
  for (int i = threadIdx.x; i < kExtWords; i += kThreads) { N60[i] = 0u; N127[i] = 0u; }
  __syncthreads();
  uint8_t* grey = c.grey + v.win.off;
  const Halo hl = halo_of(v);
  const DivW dv = make_div(hl.ew, 3 * (kChunkPx + 2) + 1);
  for (int e0 = 0; e0 < hl.ext; e0 += kThreads) {
    const int e = e0 + threadIdx.x;
    int mv = 255;
    if (e < hl.ext) {
      int ye, xe;
      divmod(e, dv, ye, xe);
      mv = v.mask[size_t(v.win.y1 + hl.ystart + ye) * v.win.pitch + v.win.x1 + hl.xs + xe];
    }
    const unsigned b60 = __ballot_sync(0xffffffffu, mv <= 60), b127 = __ballot_sync(0xffffffffu, mv <= 127);
    if ((threadIdx.x & 31) == 0 && e < hl.ext) { N60[e >> 5] = b60; N127[e >> 5] = b127; }
  }
  __syncthreads();
  const int ew = hl.ew;
  for (int w = threadIdx.x; w * 32 < v.cnt; w += kThreads) {
    const int p = w * 32 + hl.off;
    int ye, xe;
    divmod(p, dv, ye, xe);
    unsigned rs, re;
    row_ends(hl.xs + xe, v.rw, rs, re);
    // cross (textmask.py:86-89, MORPH_CROSS 3x3) on the <= 60 mask: the predicted mask is the cross erosion > 60
    const unsigned f60 = bits_from(N60, p) | bits_from(N60, p - ew) | bits_from(N60, p + ew) | (bits_from(N60, p - 1) & ~rs) |
                         (bits_from(N60, p + 1) & ~re);
    c.pred[v.woff + w] = ~f60 & tail_mask(w, v.cnt);
    c.merged[v.woff + w] = 0u;
    // full 3x3 (textmask.py:60, the eroded mask of get_topk_color) on the <= 127 mask
    F127[w] = bits_from(N127, p) | bits_from(N127, p - ew) | bits_from(N127, p + ew) |
              ((bits_from(N127, p - 1) | bits_from(N127, p - ew - 1) | bits_from(N127, p + ew - 1)) & ~rs) |
              ((bits_from(N127, p + 1) | bits_from(N127, p - ew + 1) | bits_from(N127, p + ew + 1)) & ~re);
  }
  __syncthreads();
  const DivW dvw = make_div(v.rw, v.rw * v.rh);
  for (int k0 = 0; k0 < v.cnt; k0 += kThreads * kU) {
    int b[kU], g[kU], r[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int k = k0 + u * kThreads + threadIdx.x;
      b[u] = -1; g[u] = -1; r[u] = -1;
      if (k < v.cnt) {
        int y, x;
        divmod(v.i0 + k, dvw, y, x);
        const size_t gp = size_t(v.win.y1 + y) * v.win.pitch + v.win.x1 + x;
        b[u] = v.img[gp * 3]; g[u] = v.img[gp * 3 + 1]; r[u] = v.img[gp * 3 + 2];
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int k = k0 + u * kThreads + threadIdx.x;
      const bool in = k < v.cnt;
      int gr = 0;
      bool core = false;
      if (in) {
        const int i = v.i0 + k;
        // cv2.COLOR_BGR2GRAY on 8u (OpenCV 4.13): 15-bit fixed point, equal to cv2 on all 2^24 colours.  The 14-bit
        // coefficients (1868, 9617, 4899) differ by one grey level on 43 864 of them.
        gr = (b[u] * 3735 + g[u] * 19235 + r[u] * 9798 + 16384) >> 15;
        grey[i] = (uint8_t)gr;
        core = !((F127[k >> 5] >> (k & 31)) & 1u);                       // 3x3 erosion > 127 (textmask.py:60)
      }
      if (k0 + u * kThreads < v.cnt) {   // CTA-uniform: skip the histogram votes of iterations past the chunk
        hist_add(sh[1], b[u]);
        hist_add(sh[2], g[u]);
        hist_add(sh[3], r[u]);
        hist_add(sh[0], core ? gr : -1);
      }
    }
  }
  __syncthreads();
  int* gh = &c.st[v.w].hist[0][0];
  for (int i = threadIdx.x; i < 1024; i += kThreads) {
    const int val = (&sh[0][0])[i];
    if (val) atomicAdd(&gh[i], val);
  }
}

// ---- phase 1 (one CTA per window): np.histogram(bins=255), top-k colours, Otsu ---------------------------------------
constexpr int kDecideThreads = 64;   // mostly serial per-window work: small CTAs so that many windows are resident per SM
__global__ void __launch_bounds__(kDecideThreads) k_decide1(Ctx c) {
  __shared__ int cnt255[256];
  __shared__ int order[256];
  __shared__ double edges[256];
  __shared__ int s_first, s_last, s_total;
  __shared__ int hist_s[4][256];   // the serial loops below read every bin: from shared memory, not one global load per step
  WinState& st = c.st[blockIdx.x];
  const RefineWin win = c.wins[blockIdx.x];
  const int n = (win.x2 - win.x1) * (win.y2 - win.y1);
  for (int i = threadIdx.x; i < 1024; i += kDecideThreads) (&hist_s[0][0])[i] = (&st.hist[0][0])[i];
  const int* hist_g = hist_s[0];
  for (int i = threadIdx.x; i < 256; i += kDecideThreads) cnt255[i] = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    int first = -1, last = -1, total = 0;
    for (int v = 0; v < 256; ++v)
      if (hist_g[v]) { if (first < 0) first = v; last = v; total += hist_g[v]; }
    s_first = first; s_last = last; s_total = total;
  }
  __syncthreads();
  {
    // outer edges (numpy _get_outer_edges): empty -> (0,1); equal -> (v-0.5, v+0.5)
    double fe, le;
    if (s_total == 0) { fe = 0.0; le = 1.0; }
    else if (s_first == s_last) { fe = s_first - 0.5; le = s_last + 0.5; }
    else { fe = s_first; le = s_last; }
    const double step = (le - fe) / 255.0;  // np.linspace(fe, le, 256): arange * step + start, last = stop
    for (int i = threadIdx.x; i < 256; i += kDecideThreads) edges[i] = (i == 255) ? le : __dadd_rn(__dmul_rn((double)i, step), fe);
    __syncthreads();
    for (int v = threadIdx.x; v < 256; v += kDecideThreads) {
      if (!hist_g[v]) continue;
      const double a = (double)v;
      const double f = ((a - fe) / (le - fe)) * 255.0;  // numpy fast path: (tmp_a - first_edge) / norm_denom * n_bins
      int idx = (int)f;
      if (idx == 255) idx = 254;
      if (a < edges[idx]) --idx;
      if (a >= edges[idx + 1] && idx != 254) ++idx;
      atomicAdd(&cnt255[idx], hist_g[v]);
    }
  }
  __syncthreads();
  // stable descending order of the 255 bins (documented normalisation of np.argsort's tie order)
  for (int b = threadIdx.x; b < 255; b += kDecideThreads) {
    int rank = 0;
    const int cb = cnt255[b];
    for (int q = 0; q < 255; ++q) rank += (cnt255[q] > cb) || (cnt255[q] == cb && q < b);
    order[rank] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // get_topk_color (textmask.py:16-27): colour = LEFT EDGE of the bin (textmask.py:61-62 swaps the names)
    double top[3];
    int nt = 1;
    top[0] = edges[order[0]];
    const double tol = (double)s_total * 0.001;
    for (int j = 1; j < 255; ++j) {
      const double col = edges[order[j]];
      double dmin = 1e300;
      for (int t = 0; t < nt; ++t) dmin = fmin(dmin, fabs(top[t] - col));
      if (dmin > 10.0) top[nt++] = col;
      if (nt >= 3 || (double)cnt255[order[j]] < tol) break;
    }
    st.ncol = nt;
    for (int t = 0; t < nt; ++t) {
      const double c_top = fmin(top[t] + 30.0, 255.0);
      const double c_bot = c_top - 60.0;
      // cv2.inRange with float bounds on 8u data: cvRound (half to even) + saturate
      st.lo[t] = (int)fmin(fmax(rint(c_bot), 0.0), 255.0);
      st.hi[t] = (int)fmin(fmax(rint(c_top), 0.0), 255.0);
    }
  }
  if (threadIdx.x >= 32 && threadIdx.x < 35) {
    // cv2.threshold(..., THRESH_OTSU): getThreshVal_Otsu_8u
    const int* hh = hist_s[1 + threadIdx.x - 32];
    const double scale = 1.0 / (double)n;
    double mu = 0;
    for (int i = 0; i < 256; ++i) mu = __dadd_rn(mu, __dmul_rn((double)i, (double)hh[i]));
    mu = __dmul_rn(mu, scale);
    double mu1 = 0, q1 = 0, max_sigma = 0;
    int max_val = 0;
    for (int i = 0; i < 256; ++i) {
      const double p_i = __dmul_rn((double)hh[i], scale);
      mu1 = __dmul_rn(mu1, q1);
      q1 = __dadd_rn(q1, p_i);
      const double q2 = 1.0 - q1;
      if (fmin(q1, q2) < 1.1920929e-07 || fmax(q1, q2) > 1.0 - 1.1920929e-07) continue;
      // explicit roundings: the x86 build of OpenCV has no FMA contraction here
      mu1 = __ddiv_rn(__dadd_rn(mu1, __dmul_rn((double)i, p_i)), q1);
      const double mu2 = __ddiv_rn(__dsub_rn(mu, __dmul_rn(q1, mu1)), q2);
      const double dm = __dsub_rn(mu1, mu2);
      const double sigma = __dmul_rn(__dmul_rn(__dmul_rn(q1, q2), dm), dm);
      if (sigma > max_sigma) { max_sigma = sigma; max_val = i; }
    }
    st.otsu_t[threadIdx.x - 32] = max_val;
  }
}

// ---- phase 2: xor sums of every candidate and of its negative against the mask crop; the positive candidates' bit
// planes (a warp's 32 pixels are one word of the chunk).  No later kernel reads grey, the image or the mask.
__global__ void __launch_bounds__(kThreads) k_xor(Ctx c) {
  __shared__ unsigned long long sx[12];
  __shared__ unsigned Cw[6][kChunkPx / 32];   // the chunk's candidate words, written to the planes coalesced at the end
  const View v = view_of(c, blockIdx.x);
  const WinState& st = c.st[v.w];
  if (threadIdx.x < 12) sx[threadIdx.x] = 0ull;
  __syncthreads();
  const uint8_t* grey = c.grey + v.win.off;
  const int ncol = st.ncol;
  int lo[3], hi[3], ot[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { lo[k] = st.lo[k]; hi[k] = st.hi[k]; ot[k] = st.otsu_t[k]; }
  // per thread <= kChunkPx / kThreads pixels x 255: 32-bit partial sums.  Only the POSITIVE candidates are summed: for
  // t in {0, 255}, (255 - t) ^ m == 255 - (t ^ m), so the negative's sum is 255 * pixels - the positive's sum.
  unsigned pos[6], npx = 0;
#pragma unroll
  for (int k = 0; k < 6; ++k) pos[k] = 0u;
  const DivW dv = make_div(v.rw, v.rw * v.rh);
  for (int k0 = 0; k0 < v.cnt; k0 += kThreads * kU) {
    int mk[kU], gr[kU], ch[kU][3];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int k = k0 + u * kThreads + threadIdx.x;
      mk[u] = -1; gr[u] = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) ch[u][q] = 0;
      if (k < v.cnt) {
        int y, x;
        divmod(v.i0 + k, dv, y, x);
        const size_t gp = size_t(v.win.y1 + y) * v.win.pitch + v.win.x1 + x;
        mk[u] = v.mask[gp];
        gr[u] = grey[v.i0 + k];
#pragma unroll
        for (int q = 0; q < 3; ++q) ch[u][q] = v.img[gp * 3 + q];
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int kb = k0 + u * kThreads + (int(threadIdx.x) & ~31);   // the first pixel of the warp's word
      if (kb >= v.cnt) continue;                                      // warp-uniform
      const bool in = mk[u] >= 0;
      npx += in;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const bool t = in && gr[u] >= lo[k] && gr[u] <= hi[k];          // only read for k < ncol
        const bool t2 = in && ch[u][k] > ot[k];
        if (in) {
          pos[k] += (unsigned)((t ? 255 : 0) ^ mk[u]);
          pos[3 + k] += (unsigned)((t2 ? 255 : 0) ^ mk[u]);
        }
        const unsigned b = __ballot_sync(0xffffffffu, t), b2 = __ballot_sync(0xffffffffu, t2);
        if ((threadIdx.x & 31) == 0) { Cw[k][kb >> 5] = b; Cw[3 + k][kb >> 5] = b2; }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const bool used = k >= 3 || k < ncol;
    unsigned long long sp = used ? pos[k] : 0ull, sn = used ? 255ull * npx - pos[k] : 0ull;
    for (int o = 16; o > 0; o >>= 1) {
      sp += __shfl_down_sync(0xffffffffu, sp, o);
      sn += __shfl_down_sync(0xffffffffu, sn, o);
    }
    // xs layout: [2k] positive, [2k+1] negative for the 3 colours, then the 3 channels
    if ((threadIdx.x & 31) == 0) {
      if (sp) atomicAdd(&sx[2 * k], sp);
      if (sn) atomicAdd(&sx[2 * k + 1], sn);
    }
  }
  __syncthreads();
  if (threadIdx.x < 12 && sx[threadIdx.x]) atomicAdd(&c.st[v.w].xs[threadIdx.x], sx[threadIdx.x]);
  const int nw = (v.cnt + 31) >> 5;
  for (int k = 0; k < 6; ++k) {
    if (k < 3 && k >= ncol) continue;   // no round reads the plane of a colour the window does not have
    unsigned* cw = c.cand + k * c.plane_words + v.woff;
    for (int w = threadIdx.x; w < nw; w += kThreads) cw[w] = Cw[k][w];
  }
}

// candidate order (one thread per window): minxor_thresh + sort
__global__ void k_decide2(Ctx c, int n_wins) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_wins) return;
  WinState& st = c.st[w];
  const unsigned long long* xs = st.xs;
  // minxor_thresh (textmask.py:29-41): negative wins only if strictly smaller
  unsigned long long best[4];
  int kind[4], neg[4], np_ = 0;
  for (int k = 0; k < st.ncol; ++k) {
    const bool ng = xs[2 * k + 1] < xs[2 * k];
    best[np_] = ng ? xs[2 * k + 1] : xs[2 * k];
    kind[np_] = k; neg[np_] = ng; ++np_;
  }
  // Otsu: best channel (stable sort by xor sum -> first minimum in B,G,R order)  (textmask.py:43-54)
  int bc = 0, bneg = 0;
  unsigned long long bv = ~0ull;
  for (int ch = 0; ch < 3; ++ch) {
    const bool ng = xs[6 + 2 * ch + 1] < xs[6 + 2 * ch];
    const unsigned long long val = ng ? xs[6 + 2 * ch + 1] : xs[6 + 2 * ch];
    if (val < bv) { bv = val; bc = ch; bneg = ng; }
  }
  best[np_] = bv; kind[np_] = 3 + bc; neg[np_] = bneg; ++np_;
  // mask_list.sort(key=xor_sum) (textmask.py:74): stable insertion sort
  for (int i = 1; i < np_; ++i) {
    const unsigned long long val = best[i];
    const int kk = kind[i], nn = neg[i];
    int j = i - 1;
    while (j >= 0 && best[j] > val) { best[j + 1] = best[j]; kind[j + 1] = kind[j]; neg[j + 1] = neg[j]; --j; }
    best[j + 1] = val; kind[j + 1] = kk; neg[j + 1] = nn;
  }
  for (int i = 0; i < np_; ++i) { st.proc_kind[i] = kind[i]; st.proc_neg[i] = neg[i]; }
  st.nproc = np_;
  st.area0 = 0; st.max1 = -1; st.cnt1 = 0; st.max2 = -1;
}

// ---- labelling of a source plane: candidate `round` (0..3) or, round == 4, the inverse of `merged` (hole filling) -----
// Level 1, one CTA per chunk (<= kChunkPx pixels), everything in SHARED memory: the source words, the run starts inside
// each word, each word seam a run crosses linked to the run's first pixel, and the contacts between the rows of the
// chunk united in a shared union-find; every
// pixel's chunk-local root goes to the 16-bit `lab` plane as an offset in its chunk, and the chunk's roots (the nodes of
// the global forest P, which only ever touches root entries) to the chunk's root list.  Level 2: only the first row of
// every chunk issues global unions with the row above it, and the first pixel of a row segment with the last pixel of
// the segment to its left.  Level 3: compress from the roots of the list; a pixel's global root is then
// P[chunk start + lab].
// In the chunk-local passes a chunk pixel k is treated as at column k % rw of row k / rw: right for whole rows, and for
// a row segment (k < cnt <= kChunkPx < rw) one row whose first pixel starts a run and which has no row above.
// The labelling's passes are short and separated by CTA barriers, each bound by shared-memory and L2 latency: what
// hides that latency is the number of chunks resident per SM.  256 threads and 39 registers (ptxas, sm_90a) with
// 36.9 KB of shared memory fit six CTAs per SM; 512-thread CTAs fit three, and the kernel took 25 % longer (measured
// on an H100 SXM on the bench batch; 384 threads, four CTAs: 17 % longer).
constexpr int kLabelThreads = 256;
constexpr int kLabelCtasPerSm = 6;

// The source of a labelling round as words of the chunk: foreground word w = (words[w] ^ flip) & tail_mask(w, cnt)
struct Source { const unsigned* words; unsigned flip; };
__device__ __forceinline__ Source source_of(const Ctx& c, const WinState& st, const View& v, int round) {
  if (round == 4) return Source{c.merged + v.woff, 0xffffffffu};
  return Source{c.cand + size_t(st.proc_kind[round]) * c.plane_words + v.woff, st.proc_neg[round] ? 0xffffffffu : 0u};
}

// The merge of labelling round `round` (textmask.py:92-108 / 118-131), for one chunk, by all threads of its CTA: every run
// of the round's source whose root merges (kMergeBit in the chunk's root list, k_decide_roots) is ORed into the chunk's
// `merged` words.  The runs are the labelling's, recomputed from the same source words (in round 4 the source is `merged`
// itself, untouched since the labelling), and a run's root is the label at its first pixel.  `dec`: kChunkPx / 32 words
// of shared memory.
// Who applies which round: `merged` is current up to round r - 2 when k_label_local(r) starts, r = 1..3, and that
// kernel applies round r - 1 to its own chunk before it reads `merged` (also for a window whose last candidate round
// was r - 1, which then returns); k_merge applies round 3 before the dilation, which reads neighbouring chunks, and the
// hole filling; k_or applies round 4.
__device__ void apply_merges(const Ctx& c, const View& v, int chunk, int round, unsigned* dec) {
  for (int i = threadIdx.x; i < kChunkPx / 32; i += blockDim.x) dec[i] = 0u;
  __syncthreads();
  const uint16_t* roots = c.roots + v.win.off + v.i0;
  const int nr = c.nroots[chunk];
  bool any = false;
  for (int j = threadIdx.x; j < nr; j += blockDim.x) {
    const unsigned e = roots[j];
    if (e & kMergeBit) { atomicOr(&dec[(e ^ kMergeBit) >> 5], 1u << (e & 31)); any = true; }
  }
  if (!__syncthreads_or(any)) return;   // no root of the chunk merges
  const uint16_t* lab = c.lab + v.win.off + v.i0;
  const Source src = source_of(c, c.st[v.w], v, round);
  unsigned* merged = c.merged + v.woff;
  const DivW dv = make_div(v.rw, kChunkPx + 1);
  // two threads per word, each with the run starts of its half; the even lane writes the word.  The trip count is
  // the same for a whole warp: both lanes have read the source word (`merged` itself in round 4) before the shuffle.
  for (int hw0 = 0; hw0 * 16 < v.cnt; hw0 += blockDim.x) {
    const int hw = hw0 + threadIdx.x, w = hw >> 1;
    unsigned add = 0u;
    if (hw * 16 < v.cnt) {
      const unsigned M = (src.words[w] ^ src.flip) & tail_mask(w, v.cnt);
      if (M) {
        int yl, x0;
        divmod(w * 32, dv, yl, x0);
        const unsigned S = M & (~(M << 1) | row_start_bits(x0, v.rw));
        for (unsigned f = S & ((hw & 1) ? 0xffff0000u : 0x0000ffffu); f; f &= f - 1u) {
          const int sbit = __ffs(f) - 1;
          const unsigned l = lab[w * 32 + sbit];
          if ((dec[l >> 5] >> (l & 31)) & 1u) add |= span_bits(sbit, run_end(M, S, sbit));
        }
      }
    }
    add |= __shfl_xor_sync(0xffffffffu, add, 1);
    if (add && !(hw & 1)) merged[w] |= add;
  }
  __syncthreads();
}

__device__ __forceinline__ int suf_find(const int* L, int a) {
  int p = L[a];
  while (p != a) {
    a = p;
    p = L[a];
  }
  return a;
}
// find with path halving: every visited node is re-pointed at its grandparent (atomicMin: parents have smaller indices
// than their children, and concurrent unions only ever lower a root's entry).  The walks of the union phase were ~10 hops.
__device__ __forceinline__ int suf_find_halve(int* L, int a) {
  int p = L[a];
  while (p != a) {
    const int gp = L[p];
    if (gp != p) atomicMin(&L[a], gp);
    a = p;
    p = gp;
  }
  return a;
}
__device__ __forceinline__ void suf_union(int* L, int a, int b) {
  bool done;
  do {
    a = suf_find_halve(L, a);
    b = suf_find_halve(L, b);
    if (a < b) {
      const int old = atomicMin(&L[b], a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(&L[a], b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

// Pass timing of k_label_local (scripts/refine_table.py --passes builds a second library with -DCTD_REFINE_PASS_CLOCKS):
// thread 0 of every CTA adds the clock64() ticks between two pass boundaries, each behind a CTA barrier, to
// g_pass_clocks[round][pass], and every warp adds its threads' union counts to g_pass_counts[round]: [0] word seams a
// run crosses (linked in pass 1b), [1] shared unions of vertical and diagonal contacts (pass 2).  Without the macro
// nothing is compiled in.  PASS_COUNT is called by all threads of the CTA.
#ifdef CTD_REFINE_PASS_CLOCKS
__device__ unsigned long long g_pass_clocks[5][8];
__device__ unsigned long long g_pass_counts[5][2];
#define PASS_COUNT(i, n)                                                                        \
  do {                                                                                          \
    const unsigned pc_ = __reduce_add_sync(0xffffffffu, unsigned(n));                           \
    if ((threadIdx.x & 31) == 0 && pc_)                                                         \
      atomicAdd(&g_pass_counts[round][i], (unsigned long long)pc_);                             \
  } while (0)
#define PASS_CLOCK_BEGIN() long long pass_t0 = clock64()
#define PASS_CLOCK(pass)                                                                        \
  do {                                                                                          \
    __syncthreads();                                                                            \
    if (threadIdx.x == 0) {                                                                     \
      const long long t = clock64();                                                            \
      atomicAdd(&g_pass_clocks[round][pass], (unsigned long long)(t - pass_t0));                \
      pass_t0 = t;                                                                              \
    }                                                                                           \
  } while (0)
#else
#define PASS_COUNT(i, n) (void)(n)
#define PASS_CLOCK_BEGIN()
#define PASS_CLOCK(pass)
#endif

__global__ void __launch_bounds__(kLabelThreads, kLabelCtasPerSm) k_label_local(Ctx c, int round) {
  __shared__ int Ls[kChunkPx];
  __shared__ unsigned Mw[kChunkPx / 32 + 2];      // foreground bits, 32 pixels per word (+ zero padding)
  __shared__ unsigned Sw[kChunkPx / 32];          // run-start bits (the only nodes of the chunk-local forest)
  __shared__ unsigned Gw[kChunkPx / 32];          // foreground & not yet merged & predicted     ("gain" pixels)
  __shared__ unsigned Bw[kChunkPx / 32];          // foreground & not yet merged & not predicted ("loss" pixels)
  __shared__ unsigned Tw[kChunkPx / 32 / 32];     // words that a run passes through (pass 1b), one bit per word
  __shared__ int s_fg, s_nroot;
  const View v = view_of(c, blockIdx.x);
  WinState& st = c.st[v.w];
  PASS_CLOCK_BEGIN();
  if (round >= 1 && round <= 3 && round - 1 < st.nproc) apply_merges(c, v, blockIdx.x, round - 1, Sw);
  if (round < 4 && round >= st.nproc) return;
  PASS_CLOCK(0);
  for (int i = threadIdx.x; i < kChunkPx / 32 + 2; i += kLabelThreads) Mw[i] = 0u;
  if (threadIdx.x == 0) { s_fg = 0; s_nroot = 0; }
  __syncthreads();
  uint16_t* lab = c.lab + v.win.off + v.i0;
  uint16_t* roots = c.roots + v.win.off + v.i0;
  int* P = c.P + v.win.off;
  int* acc = c.acc + 4 * v.win.off;
  const int n = v.rw * v.rh;
  int* area = acc; int* gain = acc + n; int* loss = acc + 2 * n; int* maxi = acc + 3 * n;
  const DivW dv = make_div(v.rw, kChunkPx + 1);   // chunk-local indices: k = row * rw + x, k < kChunkPx
  // pass 1: the source, `merged` and `pred` words -> foreground / gain / loss masks and the run starts inside each word
  // (a foreground pixel whose left neighbour in the same row AND word is not foreground), two threads per word
  {
    const Source src = source_of(c, st, v, round);
    const unsigned* mgw = c.merged + v.woff;
    const unsigned* pdw = c.pred + v.woff;
    for (int hw = threadIdx.x; hw * 16 < v.cnt; hw += kLabelThreads) {
      const int w = hw >> 1;
      const unsigned M = (src.words[w] ^ src.flip) & tail_mask(w, v.cnt);
      int yl, x0;
      divmod(w * 32, dv, yl, x0);
      const unsigned S = M & (~(M << 1) | row_start_bits(x0, v.rw));
      if (!(hw & 1)) {
        const unsigned un = M & ~mgw[w], pd = pdw[w];
        Mw[w] = M; Sw[w] = S; Gw[w] = un & pd; Bw[w] = un & ~pd;
      }
      // forest nodes = run starts; any other foreground pixel maps to its run start via start_of()
      for (unsigned f = S & ((hw & 1) ? 0xffff0000u : 0x0000ffffu); f; f &= f - 1u) {
        const int k = w * 32 + __ffs(f) - 1;
        Ls[k] = k;
      }
    }
  }
  __syncthreads();
  // pass 1b: a run that crosses word seams is ONE forest node, its first pixel.  Bit 0 of a word that continues the run
  // of the word before it (the same row, both pixels foreground) is linked straight to that run's first pixel, with a
  // plain store: a parent has a smaller index than its child, and the pass-2 unions only ever lower a root's entry.
  // The run's first pixel is the highest run start of the last word before this one that the run does not pass through
  // (a word passes through when it is foreground throughout and its bit 0 continues the run: Sw == 1 and cont).
  static_assert(kChunkPx / 32 <= kLabelThreads, "pass 1b: one thread per word");
  {
    const int w = threadIdx.x;
    bool cont = false;
    if (w > 0 && w * 32 < v.cnt && (Mw[w] & 1u) && (Mw[w - 1] >> 31)) {
      int yl, x0;
      divmod(w * 32, dv, yl, x0);
      cont = x0 != 0;                               // bit 0 does not start a row
    }
    const unsigned tb = __ballot_sync(0xffffffffu, cont && Sw[w] == 1u);
    if ((threadIdx.x & 31) == 0 && threadIdx.x < kChunkPx / 32) Tw[threadIdx.x >> 5] = tb;
    __syncthreads();
    if (cont) {                                     // word 0 never passes through: the walk ends
      int u = w - 1;
      unsigned t = ~Tw[u >> 5] & (0xffffffffu >> (31 - (u & 31)));
      while (!t) {
        u = (u & ~31) - 1;
        t = ~Tw[u >> 5];
      }
      u = (u & ~31) + 31 - __clz(t);
      Ls[w * 32] = u * 32 + 31 - __clz(Sw[u]);
    }
    PASS_COUNT(0, cont);
  }
  __syncthreads();
  PASS_CLOCK(1);
  // pass 2: contacts with the row above inside the chunk -- on the foreground BIT masks, two
  // threads per 32-pixel word: the neighbour tests of 32 pixels are a handful of shifts and ANDs, and only the pixels
  // that really start a (run x upper run) contact walk the union-find (first version: every foreground pixel tested
  // its four neighbours with byte loads; half of the kernel's instructions, ncu).
  // run start of foreground pixel p: the highest run-start bit at or below p in its word (a node of the forest; one
  // that continues the run of the word before points at the run's first pixel since pass 1b)
  auto start_of = [&](int pos) -> int {
    return (pos & ~31) + 31 - __clz(Sw[pos >> 5] & (0xffffffffu >> (31 - (pos & 31))));
  };
  auto bits_at = [&](int pos) -> unsigned {        // 32 foreground bits starting at pixel `pos` (pixels < 0 read as 0)
    if (pos <= -32) return 0u;
    if (pos < 0) return Mw[0] << (-pos);
    const int w = pos >> 5, sft = pos & 31;
    return __funnelshift_r(Mw[w], Mw[w + 1], sft);
  };
  unsigned n_contacts = 0;   // shared unions of this thread (counted in the CTD_REFINE_PASS_CLOCKS build)
  for (int hw = threadIdx.x; hw * 16 < v.cnt; hw += kLabelThreads) {
    const int w = hw >> 1;
    const unsigned half = (hw & 1) ? 0xffff0000u : 0x0000ffffu;
    const unsigned cur = Mw[w];
    if (!(cur & half)) continue;
    const int k0 = w * 32;
    int yl, x0;
    divmod(k0, dv, yl, x0);
    const unsigned rs = row_start_bits(x0, v.rw);   // bits whose pixel is the FIRST of its row (x == 0)
    int xe = x0 + 32;                               // x of the pixel after this word
    if (xe >= v.rw) xe %= v.rw;
    const unsigned re = (rs >> 1) | (xe == 0 ? 0x80000000u : 0u);   // bits whose pixel is the LAST of its row
    const unsigned lft = bits_at(k0 - 1);           // fg(k - 1)
    if (k0 + 32 <= v.rw) continue;                  // the whole word lies in the first row of the chunk
    const unsigned vup = (k0 >= v.rw ? 0xffffffffu : (0xffffffffu << (v.rw - k0))) & half;   // pixels that have a row above
    const unsigned up = bits_at(k0 - v.rw), upl = bits_at(k0 - v.rw - 1), upr = bits_at(k0 - v.rw + 1);
    // pixel and the pixel above are foreground: only the first pixel of each (current run x upper run) overlap unions
    unsigned f = cur & up & vup & (rs | ~lft | ~upl);
    n_contacts += __popc(f) + __popc(cur & ~up & vup & upl & ~rs) + __popc(cur & ~up & vup & upr & ~re);
    while (f) {
      const int j = __ffs(f) - 1;
      f &= f - 1u;
      suf_union(Ls, start_of(k0 + j), start_of(k0 + j - v.rw));
    }
    const unsigned nb = cur & ~up & vup;
    f = nb & upl & ~rs;                             // diagonal contacts when the pixel above is background
    while (f) {
      const int j = __ffs(f) - 1;
      f &= f - 1u;
      suf_union(Ls, start_of(k0 + j), start_of(k0 + j - v.rw - 1));
    }
    f = nb & upr & ~re;
    while (f) {
      const int j = __ffs(f) - 1;
      f &= f - 1u;
      suf_union(Ls, start_of(k0 + j), start_of(k0 + j - v.rw + 1));
    }
  }
  PASS_COUNT(1, n_contacts);
  __syncthreads();
  PASS_CLOCK(3);
  // pass 3a: flatten the forest.  Its nodes are the run starts only (every other foreground pixel points at its run
  // start and is never re-parented): after this pass every run start points straight at its root, so the root of ANY
  // foreground pixel is Ls[Ls[k]] -- two loads instead of a walk (the walks were 10 hops on average, ncu).  The roots
  // zero their per-label sums here (area, gain, loss, max pixel index), start their tree of P and join the root list.
  int fgc = 0;
  for (int hw = threadIdx.x; hw * 16 < v.cnt; hw += kLabelThreads) {
    const unsigned half = (hw & 1) ? 0xffff0000u : 0x0000ffffu;
    unsigned f = Sw[hw >> 1] & half;
    fgc += __popc(Mw[hw >> 1] & half);
    const int k0 = (hw >> 1) * 32;
    while (f) {
      const int s0 = k0 + __ffs(f) - 1;
      f &= f - 1u;
      const int r = suf_find(Ls, s0);
      if (r != s0) {
        atomicMin(&Ls[s0], r);
      } else {
        const int gi = v.i0 + s0;
        area[gi] = 0; gain[gi] = 0; loss[gi] = 0; maxi[gi] = -1;
        P[gi] = gi;
        roots[atomicAdd(&s_nroot, 1)] = uint16_t(s0);
      }
    }
  }
  if (round == 4) {   // label 0 of the inverse = the pixels already in `merged`
    for (int o = 16; o > 0; o >>= 1) fgc += __shfl_down_sync(0xffffffffu, fgc, o);
    if ((threadIdx.x & 31) == 0 && fgc) atomicAdd(&s_fg, fgc);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    c.nroots[blockIdx.x] = s_nroot;
    const int a0 = v.cnt - s_fg;
    if (round == 4 && a0) atomicAdd(&st.area0, a0);
  }
  PASS_CLOCK(4);
  // pass 3b: chunk-local root of every pixel to global memory (an offset in the chunk; kNoLabel = background)
  for (int k = threadIdx.x; k < v.cnt; k += kLabelThreads)
    lab[k] = ((Mw[k >> 5] >> (k & 31)) & 1u) ? uint16_t(Ls[start_of(k)]) : kNoLabel;
  PASS_CLOCK(5);
  // pass 3c: per-label sums, one update per RUN (popcounts of the run's bits in the foreground / gain / loss masks) into
  // the sums of its chunk-local root.  k_flat1 adds the sums of the chunk roots of a multi-chunk window to their global
  // root; there is no per-pixel accumulation sweep any more.
  for (int hw = threadIdx.x; hw * 16 < v.cnt; hw += kLabelThreads) {
    const int w = hw >> 1;
    const unsigned M = Mw[w], S = Sw[w];
    unsigned f = S & ((hw & 1) ? 0xffff0000u : 0x0000ffffu);
    if (!f) continue;
    const unsigned G = Gw[w], B = Bw[w];
    const int k0 = w * 32;
    while (f) {
      const int sbit = __ffs(f) - 1;
      f &= f - 1u;
      const int e = run_end(M, S, sbit);                               // last pixel of the run
      const unsigned rm = span_bits(sbit, e);
      const int gi = v.i0 + Ls[k0 + sbit];
      atomicAdd(&area[gi], __popc(rm));
      atomicMax(&maxi[gi], v.i0 + k0 + e);
      const int g_ = __popc(rm & G), l_ = __popc(rm & B);
      if (g_) atomicAdd(&gain[gi], g_);
      if (l_) atomicAdd(&loss[gi], l_);
    }
  }
  PASS_CLOCK(6);
}
// level 2: the first row of every chunk against the row above it (x-1, x, x+1, possibly in the neighbouring row
// segments), and the first pixel of a row segment against the last pixel of the segment to its left
constexpr int kBorderThreads = 256;  // (64-thread CTAs measured 3x slower: a window row is up to thousands of pixels)
__global__ void __launch_bounds__(kBorderThreads) k_union_border(Ctx c, int round) {
  const View v = view_of(c, blockIdx.x);
  if (round < 4 && round >= c.st[v.w].nproc) return;
  if (v.i0 == 0) return;      // the window's first chunk
  const uint16_t* lab = c.lab + v.win.off;   // foreground <=> lab != kNoLabel (written for every pixel by k_label_local)
  int* P = c.P + v.win.off;
  // chunk-local root of the foreground pixel at window row y, column x, as a window pixel index
  auto root_at = [&](int y, int x) { const int i = y * v.rw + x; return chunk_start(y, x, v.rw) + lab[i]; };
  const int y = v.y0;
  if (v.x0 > 0 && threadIdx.x == 0 && lab[v.i0] != kNoLabel && lab[v.i0 - 1] != kNoLabel)
    uf_union(P, v.i0 + lab[v.i0], root_at(y, v.x0 - 1));
  if (y == 0) return;
  for (int k = threadIdx.x; k < v.cols; k += int(blockDim.x)) {
    const int i = v.i0 + k, x = v.x0 + k;
    if (lab[i] == kNoLabel) continue;
    const int up = i - v.rw;
    const int r = v.i0 + lab[i];
    if (lab[up] != kNoLabel) {
      // only the first pixel of each (run x run above) overlap: the pixels left of it are united with it (in the chunk
      // or across the segment seam) and so are the ones above
      const bool first = x == 0 || lab[i - 1] == kNoLabel || lab[up - 1] == kNoLabel;
      if (first) uf_union(P, r, root_at(y - 1, x));
    } else {
      if (x > 0 && lab[up - 1] != kNoLabel) uf_union(P, r, root_at(y - 1, x - 1));
      if (x + 1 < v.rw && lab[up + 1] != kNoLabel) uf_union(P, r, root_at(y - 1, x + 1));
    }
  }
}
// level 3: every chunk-local root of the chunk's list points straight at its global root
__global__ void __launch_bounds__(kThreads) k_flat1(Ctx c, int round) {
  const View v = view_of(c, blockIdx.x);
  if (round < 4 && round >= c.st[v.w].nproc) return;
  const uint16_t* roots = c.roots + v.win.off + v.i0;
  const int nr = c.nroots[blockIdx.x];
  int* P = c.P + v.win.off;
  int* acc = c.acc + 4 * v.win.off;
  const int n = v.rw * v.rh;
  int* area = acc; int* gain = acc + n; int* loss = acc + 2 * n; int* maxi = acc + 3 * n;
  for (int j = threadIdx.x; j < nr; j += kThreads) {
    // chunk-local root: point it straight at its global root and hand its sums (complete since k_label_local) over
    const int cr = v.i0 + roots[j];
    const int g = uf_find_compress(P, cr);
    if (g != cr) {
      atomicAdd(&area[g], area[cr]);
      atomicMax(&maxi[g], maxi[cr]);
      const int g_ = gain[cr], l_ = loss[cr];
      if (g_) atomicAdd(&gain[g], g_);
      if (l_) atomicAdd(&loss[g], l_);
    }
  }
}
// ---- merge step (textmask.py:92-108 / 118-131) -------------------------------------------------------------------------
// hole filling only: the two largest areas over all labels incl. label 0, as a multiset (max1 with its multiplicity, max2)
__global__ void __launch_bounds__(kThreads) k_top_a(Ctx c) {
  const View v = view_of(c, blockIdx.x);
  WinState& st = c.st[v.w];
  const int* P = c.P + v.win.off;
  const int* area = c.acc + 4 * v.win.off;
  const uint16_t* roots = c.roots + v.win.off + v.i0;   // chunk-local roots: the only candidates for a global root
  const int nr = c.nroots[blockIdx.x];
  int m = -1;
  for (int j = threadIdx.x; j < nr; j += kThreads) {
    const int i = v.i0 + roots[j];
    if (P[i] == i) m = max(m, area[i]);
  }
  if (v.i0 == 0 && threadIdx.x == 0) m = max(m, st.area0);   // once per window: its first chunk
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(&st.max1, m);
}
__global__ void __launch_bounds__(kThreads) k_top_b(Ctx c) {
  const View v = view_of(c, blockIdx.x);
  WinState& st = c.st[v.w];
  const int* P = c.P + v.win.off;
  const int* area = c.acc + 4 * v.win.off;
  const uint16_t* roots = c.roots + v.win.off + v.i0;
  const int nr = c.nroots[blockIdx.x];
  const int m1 = st.max1;
  int m2 = -1, c1 = 0;
  auto push = [&](int a) { if (a == m1) ++c1; else m2 = max(m2, a); };
  for (int j = threadIdx.x; j < nr; j += kThreads) {
    const int i = v.i0 + roots[j];
    if (P[i] == i) push(area[i]);
  }
  if (v.i0 == 0 && threadIdx.x == 0) push(st.area0);
  for (int o = 16; o > 0; o >>= 1) {
    m2 = max(m2, __shfl_down_sync(0xffffffffu, m2, o));
    c1 += __shfl_down_sync(0xffffffffu, c1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (c1) atomicAdd(&st.cnt1, c1);
    if (m2 >= 0) atomicMax(&st.max2, m2);
  }
}
// The merge decision of every chunk-local root, from the sums of its global root (P[cr]: k_flat1, or cr itself in a
// single-chunk window), as kMergeBit of its root list entry.  It has a kernel of its own because a global root's sums
// are complete only when k_flat1 has ended, and the next labelling of the root's chunk zeroes them.  apply_merges ORs
// the runs of the merging roots into `merged`.
__global__ void __launch_bounds__(kThreads) k_decide_roots(Ctx c, int round) {
  const View v = view_of(c, blockIdx.x);
  const WinState& st = c.st[v.w];
  if (round < 4 && round >= st.nproc) return;
  const int* P = c.P + v.win.off;
  const int* acc = c.acc + 4 * v.win.off;
  const int n = v.rw * v.rh;
  const int* area = acc; const int* gain = acc + n; const int* loss = acc + 2 * n; const int* maxi = acc + 3 * n;
  // sorted_area[-2] if more than one label else sorted_area[-1] (textmask.py:114-118); label 0 always exists
  const int second = st.cnt1 >= 2 ? st.max1 : st.max2;
  const int thresh = second >= 0 ? second : st.max1;
  uint16_t* roots = c.roots + v.win.off + v.i0;
  const int nr = c.nroots[blockIdx.x];
  for (int j = threadIdx.x; j < nr; j += kThreads) {
    const int cl = roots[j];
    const int g = P[v.i0 + cl];
    const int a = area[g];
    bool ok;
    if (round < 4) {
      // `if w * h < 3: continue` (textmask.py:97): bounding boxes 1x1, 1x2, 2x1.  g and mx are the first and last
      // pixel; a horizontal pair is mx == g + 1 in ONE row (in a window 2 px wide an anti-diagonal pair, a 2x2 box,
      // is mx == g + 1 too, across a row end)
      const int mx = maxi[g];
      ok = !(a == 1 || (a == 2 && ((mx == g + 1 && mx % v.rw != 0) || mx == g + v.rw)));
    } else {
      ok = a < thresh;  // textmask.py:120
    }
    if (ok && gain[g] > loss[g]) roots[j] = uint16_t(cl | kMergeBit);
  }
}
__global__ void __launch_bounds__(kThreads) k_merge(Ctx c, int round) {
  __shared__ unsigned dec[kChunkPx / 32];
  const View v = view_of(c, blockIdx.x);
  if (round >= c.st[v.w].nproc) return;
  apply_merges(c, v, blockIdx.x, round, dec);
}

// ---- dilate 3x3 (inpaint mode): merged -> tmp; the caller swaps the two planes afterwards -----------------------------
// The 3x3 maximum of a binary plane is an OR of nine shifted copies of its bits.  The chunk's halo rectangle (see
// k_phase0) is gathered into shared-memory words at the rectangle's row stride -- its rows above and below, and for a
// row segment the columns left and right, are bits of the neighbouring chunks' words -- and one thread per 32-pixel
// word ORs the nine views (window row ends masked) and writes the word of `tmp`.
__global__ void __launch_bounds__(kThreads) k_dilate(Ctx c) {
  __shared__ unsigned Mw[kExtWords];
  const View v = view_of(c, blockIdx.x);
  for (int i = threadIdx.x; i < kExtWords; i += kThreads) Mw[i] = 0u;
  __syncthreads();
  const Halo hl = halo_of(v);
  const int ew = hl.ew;
  const DivW dv = make_div(ew, 3 * (kChunkPx + 2) + 1);
  // The chunks of a window are consecutive in the table, row by row: whole-row chunks one after the other (all but the
  // window's last have refine_rows_per_chunk rows), row segments nseg per window row.
  const bool seg = v.rw > kChunkPx;
  const int nseg = (v.rw + kChunkPx - 1) / kChunkPx;
  const int rows_up = seg ? 1 : refine_rows_per_chunk(v.rw);
  if (!seg) {
    // whole rows: the rectangle is the last row of the chunk above, the chunk, and the first row of the chunk below,
    // one after the other -- three copies of consecutive bits
    const bool up = v.y0 > 0, down = v.y0 + v.rows < v.rh;
    const unsigned* mu = up ? c.merged + c.chunks[blockIdx.x - 1].woff : nullptr;
    const unsigned* md = down ? c.merged + c.chunks[blockIdx.x + 1].woff : nullptr;
    for (int d = threadIdx.x; d * 32 < hl.ext; d += kThreads) {
      unsigned m = copied_word(c.merged + v.woff, 0, v.cnt, hl.off, d);
      if (up) m |= copied_word(mu, (rows_up - 1) * v.rw, v.rw, 0, d);
      if (down) m |= copied_word(md, 0, v.rw, hl.off + v.cnt, d);
      Mw[d] = m;
    }
  }
  for (int e0 = 0; seg && e0 < hl.ext; e0 += kThreads) {
    const int e = e0 + threadIdx.x;
    bool bit = false;
    if (e < hl.ext) {
      int ye, xe;
      divmod(e, dv, ye, xe);
      const int y = hl.ystart + ye, x = hl.xs + xe;
      const int dy = y < v.y0 ? -1 : (y >= v.y0 + v.rows ? 1 : 0);
      // the chunk that holds window pixel (y, x), and the pixel's offset k in it
      int ch = int(blockIdx.x) + dy * (seg ? nseg : 1), k;
      if (seg) {
        ch += x / kChunkPx - v.x0 / kChunkPx;
        k = x % kChunkPx;
      } else {
        k = (dy < 0 ? rows_up - 1 : (dy > 0 ? 0 : y - v.y0)) * v.rw + x;
      }
      const int wo = ch == int(blockIdx.x) ? v.woff : c.chunks[ch].woff;
      bit = (c.merged[wo + (k >> 5)] >> (k & 31)) & 1u;
    }
    const unsigned m = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0 && e < hl.ext) Mw[e >> 5] = m;
  }
  __syncthreads();
  for (int w = threadIdx.x; w * 32 < v.cnt; w += kThreads) {
    const int p = w * 32 + hl.off;
    int ye, xe;
    divmod(p, dv, ye, xe);
    unsigned rs, re;
    row_ends(hl.xs + xe, v.rw, rs, re);
    unsigned o = bits_from(Mw, p) | bits_from(Mw, p - ew) | bits_from(Mw, p + ew);
    o |= (bits_from(Mw, p - 1) | bits_from(Mw, p - ew - 1) | bits_from(Mw, p + ew - 1)) & ~rs;
    o |= (bits_from(Mw, p + 1) | bits_from(Mw, p - ew + 1) | bits_from(Mw, p + ew + 1)) & ~re;
    c.tmp[v.woff + w] = o & tail_mask(w, v.cnt);
  }
}
// the hole filling's merge, then mask_refined[window] |= merged (textmask.py:168); windows may overlap -> atomic OR,
// issued for the set bits only
__global__ void __launch_bounds__(kThreads) k_or(Ctx c) {
  __shared__ unsigned dec[kChunkPx / 32];
  const View v = view_of(c, blockIdx.x);
  apply_merges(c, v, blockIdx.x, 4, dec);
  const unsigned* merged = c.merged + v.woff;
  const DivW dv = make_div(v.rw, v.rw * v.rh);
  for (int k = threadIdx.x; k < v.cnt; k += kThreads) {   // a warp reads one word and spreads its set bits over its lanes
    if (!((merged[k >> 5] >> (k & 31)) & 1u)) continue;
    int y, x;
    divmod(v.i0 + k, dv, y, x);
    const size_t gp = size_t(v.win.page_off) + size_t(v.win.y1 + y) * v.win.pitch + v.win.x1 + x;
    atomicOr(&c.out_all[gp >> 2], 0xffu << (8 * (gp & 3)));
  }
}

}  // namespace

#ifdef CTD_REFINE_PASS_CLOCKS
// copies g_pass_clocks to out[0, 5 * 8) and g_pass_counts to out[5 * 8, 5 * 8 + 5 * 2), and zeroes both
extern "C" __attribute__((visibility("default"))) int ctd_refine_pass_clocks(unsigned long long* out) {
  static const unsigned long long zero[5 * 8] = {};
  cudaError_t e = cudaMemcpyFromSymbol(out, g_pass_clocks, sizeof(g_pass_clocks));
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out + 5 * 8, g_pass_counts, sizeof(g_pass_counts));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_pass_clocks, zero, sizeof(g_pass_clocks));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_pass_counts, zero, sizeof(g_pass_counts));
  return int(e);
}
#endif

size_t refine_mk_state_bytes(int n_wins) { return (size_t(n_wins) * sizeof(WinState) + 255) / 256 * 256; }
// per window pixel: P (4 B) and the per-root sums (16 B), of which only root entries are touched; lab and the root
// lists (2 B each); grey (1 B).  Per chunk: its root count.  Nine bit planes (six candidates, pred, merged, tmp) of
// plane_words 4-byte words, 1.1 B per window pixel together.
static size_t plane_words(size_t total_px, size_t n_chunks) { return total_px / 32 + n_chunks + 1; }
size_t refine_scratch_bytes(size_t total_px, size_t n_chunks) {
  return total_px * (4 + 16 + 2 + 2 + 1) + n_chunks * 4 + 9 * 4 * plane_words(total_px, n_chunks) + 4096;
}

// d_wins: n_wins windows; d_chunks: n_chunks chunks (RefineChunk, kernels.h); d_state: refine_mk_state_bytes(n_wins)
// bytes (zeroed here); scratch: refine_scratch_bytes(total_px, n_chunks) bytes.  img / mask / out hold the pages' planes at the
// windows' page_off (3 bytes per pixel in img).
cudaError_t refine_mk_launch(const uint8_t* d_img, const uint8_t* d_mask, const RefineWin* d_wins, int n_wins,
                             const RefineChunk* d_chunks, int n_chunks, int n_multi_chunks, void* d_state, size_t total_px,
                             void* scratch, int refine_mode, uint8_t* d_out, cudaStream_t s) {
  if (n_wins <= 0 || n_chunks <= 0) return cudaSuccess;
  Ctx c;
  c.img_all = d_img; c.mask_all = d_mask; c.out_all = reinterpret_cast<uint32_t*>(d_out);
  c.wins = d_wins;
  c.chunks = d_chunks;
  c.st = static_cast<WinState*>(d_state);
  c.mode = refine_mode;
  char* p = static_cast<char*>(scratch);
  c.P = reinterpret_cast<int*>(p); p += total_px * 4;
  c.acc = reinterpret_cast<int*>(p); p += total_px * 16;
  c.lab = reinterpret_cast<uint16_t*>(p); p += total_px * 2;
  c.roots = reinterpret_cast<uint16_t*>(p); p += total_px * 2;
  c.nroots = reinterpret_cast<int*>(p); p += size_t(n_chunks) * 4;
  c.grey = reinterpret_cast<uint8_t*>(p); p += total_px;   // total_px is a multiple of 4: the words below are aligned
  c.plane_words = plane_words(total_px, size_t(n_chunks));
  c.cand = reinterpret_cast<unsigned*>(p); p += 6 * 4 * c.plane_words;
  c.pred = reinterpret_cast<unsigned*>(p); p += 4 * c.plane_words;
  c.merged = reinterpret_cast<unsigned*>(p); p += 4 * c.plane_words;
  c.tmp = reinterpret_cast<unsigned*>(p);
  cudaError_t e = cudaMemsetAsync(d_state, 0, refine_mk_state_bytes(n_wins), s);
  if (e != cudaSuccess) return e;
  const unsigned g = unsigned(n_chunks);
  k_phase0<<<g, kThreads, 0, s>>>(c);
  k_decide1<<<unsigned(n_wins), kDecideThreads, 0, s>>>(c);
  k_xor<<<g, kThreads, 0, s>>>(c);
  k_decide2<<<unsigned((n_wins + 127) / 128), 128, 0, s>>>(c, n_wins);
  for (int round = 0; round < 5; ++round) {
    if (round == 4) k_merge<<<g, kThreads, 0, s>>>(c, 3);
    if (round == 4 && refine_mode == 0) {
      k_dilate<<<g, kThreads, 0, s>>>(c);
      unsigned* t = c.merged; c.merged = c.tmp; c.tmp = t;   // the dilated plane IS `merged` from here on (no copy back)
    }
    k_label_local<<<g, kLabelThreads, 0, s>>>(c, round);
    if (n_multi_chunks > 0) {   // single-chunk windows: the chunk-local roots ARE the global roots
      k_union_border<<<unsigned(n_multi_chunks), kBorderThreads, 0, s>>>(c, round);
      k_flat1<<<unsigned(n_multi_chunks), kThreads, 0, s>>>(c, round);
    }
    if (round == 4) {
      k_top_a<<<g, kThreads, 0, s>>>(c);
      k_top_b<<<g, kThreads, 0, s>>>(c);
    }
    k_decide_roots<<<g, kThreads, 0, s>>>(c, round);
  }
  k_or<<<g, kThreads, 0, s>>>(c);
  return cudaGetLastError();
}

}  // namespace ctd
