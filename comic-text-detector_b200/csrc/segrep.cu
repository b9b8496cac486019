// SegDetectorRepresenter.boxes_from_bitmap on the GPU (reference utils/db_utils.py:123-166):
//   cv2.findContours(bitmap, RETR_LIST, CHAIN_APPROX_SIMPLE)  -> contour set + OpenCV order + 1000 cap
//   get_mini_boxes / box_score_fast / unclip / get_mini_boxes -> (4,2) int16 box + f32 score per contour
//
// No border following: everything downstream of findContours only needs, per contour, (a) its position
// in OpenCV's list, (b) the convex hull of its points, (c) the set of pixels inside it (for the score).
//  * outer border of an 8-connected foreground component C: discovered at C's first raster pixel;
//    hull = hull(C); inside = C + everything C encloses.
//  * hole border of a 4-connected background component Q that does not touch the image frame:
//    discovered at Q's first raster pixel (the scan meets the fg->bg transition there); its points
//    are the foreground pixels 4-adjacent to Q (the "ring"); inside = ring + Q + everything Q encloses.
//  * OpenCV returns the list in REVERSE discovery order; the reference keeps the first 1000.
// "Everything enclosed" is the subtree in the component adjacency tree (parent of a fg component = the
// bg component left of its first pixel; parent of a hole = the fg component left of its first pixel).
#include <cuda_runtime.h>
#include <limits.h>

#include "geom.h"
#include "kernels.h"

namespace ctd {

using ctdgeom::IPt;

__device__ __forceinline__ int uf_find_g(const int* L, int a) {
  int p = L[a];
  while (p != a) {
    a = p;
    p = L[a];
  }
  return a;
}
__device__ __forceinline__ void uf_union_g(int* L, int a, int b) {
  bool done;
  do {
    a = uf_find_g(L, a);
    b = uf_find_g(L, b);
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

// ---- 4-connectivity labelling of the BACKGROUND (bitmap == 0), same tile-local + border scheme as ccl_*
__global__ void __launch_bounds__(1024) bg_local_kernel(const uint8_t* __restrict__ img, int h, int w, int* __restrict__ Lall) {
  __shared__ int s[32 * 32];
  const int page = blockIdx.z;
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int x = blockIdx.x * 32 + lx, y = blockIdx.y * 32 + ly;
  const bool inb = x < w && y < h;
  const size_t o = size_t(page) * h * w;
  const int l = threadIdx.x;
  const bool bg = inb && img[o + size_t(y) * w + x] == 0;
  const unsigned m = __ballot_sync(0xffffffffu, bg);
  const unsigned zeros_below = ~m & ((1u << lx) - 1u);
  const int start = zeros_below ? 32 - __clz(zeros_below) : 0;
  s[l] = bg ? (ly << 5) + start : -1;
  __syncthreads();
  if (bg && ly > 0 && s[l - 32] >= 0) {
    const bool first = (lx == start) || s[l - 33] < 0;
    if (first) uf_union_g(s, l, l - 32);
  }
  __syncthreads();
  if (inb) {
    int g = -1;
    if (bg) {
      const int r = uf_find_g(s, l);
      g = (blockIdx.y * 32 + (r >> 5)) * w + blockIdx.x * 32 + (r & 31);
    }
    Lall[o + size_t(y) * w + x] = g;
  }
}
__global__ void bg_border_kernel(int h, int w, int* __restrict__ Lall) {
  const int page = blockIdx.y;
  int* L = Lall + size_t(page) * h * w;
  const int nvl = (w - 1) / 32, nhl = (h - 1) / 32;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nvl * h) {
    const int x = (i / h + 1) * 32, y = i % h;
    const int p = y * w + x;
    if (L[p] >= 0 && L[p - 1] >= 0) uf_union_g(L, p, p - 1);
  } else if (i < nvl * h + nhl * w) {
    const int j = i - nvl * h;
    const int y = (j / w + 1) * 32, x = j % w;
    const int p = y * w + x;
    if (L[p] >= 0 && L[p - w] >= 0) uf_union_g(L, p, p - w);
  }
}
// flatten; every root marks its parent "not decided" (-1)
__global__ void bg_flatten_kernel(int h, int w, int* __restrict__ Lall, int* __restrict__ parent_all) {
  const int page = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  int* L = Lall + size_t(page) * h * w;
  if (L[p] < 0) return;
  const int r = uf_find_g(L, p);
  L[p] = r;
  if (r == p) parent_all[size_t(page) * h * w + p] = -1;
}

// ---- component tree ---------------------------------------------------------------------------
// parent[root]: >= 0 parent root pixel, kFrame = the image frame / an outside background component
constexpr int kFrame = -2;

// bg components touching the frame are "outside": mark their roots
// (and reset the contours' y ranges)
__global__ void mark_outside_kernel(int h, int w, const int* __restrict__ Lb_all, int* __restrict__ parent_all,
                                    int* __restrict__ c_yrange, int max_cand) {
  const int page = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < max_cand) {
    c_yrange[(page * max_cand + i) * 2] = INT_MAX;
    c_yrange[(page * max_cand + i) * 2 + 1] = -1;
  }
  const int per = 2 * w + 2 * h;
  if (i >= per) return;
  int x, y;
  if (i < w) { x = i; y = 0; }
  else if (i < 2 * w) { x = i - w; y = h - 1; }
  else if (i < 2 * w + h) { x = 0; y = i - 2 * w; }
  else { x = w - 1; y = i - 2 * w - h; }
  const size_t o = size_t(page) * h * w;
  const int r = Lb_all[o + size_t(y) * w + x];
  if (r >= 0) parent_all[o + r] = kFrame;
}

// ---- discovery order -> contour ids (OpenCV returns the reverse discovery order) ----------------
// The roots of a page are numbered in raster order.  A 256-thread CTA owns a segment of kSeg pixels and sweeps it in
// kSeg / 256 coalesced steps; roots_kernel counts the segment's roots, flag_scan_top scans the counts, and
// assign_cid_kernel ranks each root inside its segment.
constexpr int kSeg = 2048;

// a CTA-wide exclusive prefix of one flag per thread (raster order = thread order); returns the CTA's total
__device__ __forceinline__ int cta_flag_prefix(bool flag, int* excl, int* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, flag);
  __syncthreads();   // wsum of the previous call has been read
  if (lane == 0) wsum[warp] = __popc(b);
  __syncthreads();
  int off = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    off += k < warp ? wsum[k] : 0;
    tot += wsum[k];
  }
  *excl = off + __popc(b & ((1u << lane) - 1u));
  return tot;
}

// per pixel: roots get their parent and zeroed accumulators; per segment: the count of discovery points (the first
// pixels of foreground components and of holes)
__global__ void __launch_bounds__(256) roots_kernel(int h, int w, const int* __restrict__ Lf_all, const int* __restrict__ Lb_all,
                                                    int* __restrict__ parent_all, double* __restrict__ own_sum,
                                                    int* __restrict__ own_cnt, double* __restrict__ tot_sum,
                                                    int* __restrict__ tot_cnt, double* __restrict__ ring_sum,
                                                    int* __restrict__ ring_cnt, int* __restrict__ segsum, int nseg) {
  __shared__ int wsum[8];
  const int page = blockIdx.y, seg = blockIdx.x;
  const int hw = h * w;
  const size_t o = size_t(page) * hw;
  int cnt = 0;
  for (int e = 0; e < kSeg / 256; ++e) {
    const int p = seg * kSeg + e * 256 + threadIdx.x;
    if (p >= hw) break;
    const int lf = Lf_all[o + p], lb = Lb_all[o + p];
    if (lf == p) {
      const int x = p % w;
      int par = kFrame;
      if (x > 0) {
        const int q = Lb_all[o + p - 1];  // bg (p is the component's first raster pixel)
        par = (q >= 0 && parent_all[o + q] != kFrame) ? q : kFrame;
      }
      parent_all[o + p] = par;
      ++cnt;
    } else if (lb == p) {
      if (parent_all[o + p] != kFrame) {  // a hole: its left neighbour is foreground
        parent_all[o + p] = Lf_all[o + p - 1];
        ++cnt;
      }
    }
    if (lf == p || lb == p) {
      own_sum[o + p] = 0.0; own_cnt[o + p] = 0;
      tot_sum[o + p] = 0.0; tot_cnt[o + p] = 0;
      ring_sum[o + p] = 0.0; ring_cnt[o + p] = 0;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int k = 0; k < 8; ++k) t += wsum[k];
    segsum[page * nseg + seg] = t;
  }
}

__global__ void __launch_bounds__(1024) flag_scan_top_kernel(int* __restrict__ segsum, int nseg, int* __restrict__ total) {
  // exclusive scan of up to 4096 segment sums: 4 consecutive entries per thread, block scan of the per-thread sums
  __shared__ int part[1024];
  const int page = blockIdx.x;
  int* sgs = segsum + page * nseg;
  int v[4], loc = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = threadIdx.x * 4 + k;
    v[k] = i < nseg ? sgs[i] : 0;
    loc += v[k];
  }
  part[threadIdx.x] = loc;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    int u = 0;
    if (threadIdx.x >= off) u = part[threadIdx.x - off];
    __syncthreads();
    part[threadIdx.x] += u;
    __syncthreads();
  }
  int run = part[threadIdx.x] - loc;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = threadIdx.x * 4 + k;
    if (i < nseg) sgs[i] = run;
    run += v[k];
  }
  if (threadIdx.x == 1023) total[page] = part[1023];
}
// each discovery point (a root whose parent roots_kernel decided: every foreground root, and the background roots that
// are not outside) gets its discovery rank; cid[root] = its position in OpenCV's list if < max_candidates else -1,
// written at roots only; the contour table; the list of roots in discovery order, for tree_kernel
__global__ void __launch_bounds__(256) assign_cid_kernel(int h, int w, const int* __restrict__ Lf_all,
                                                         const int* __restrict__ Lb_all, const int* __restrict__ parent_all,
                                                         const int* __restrict__ segoff, int nseg, const int* __restrict__ total,
                                                         int max_cand, int* __restrict__ cid_all, int* __restrict__ c_root,
                                                         int* __restrict__ root_list) {
  __shared__ int wsum[8];
  const int page = blockIdx.y, seg = blockIdx.x;
  const int hw = h * w;
  const size_t o = size_t(page) * hw;
  int base = segoff[page * nseg + seg];
  for (int e = 0; e < kSeg / 256; ++e) {
    const int p = seg * kSeg + e * 256 + threadIdx.x;
    if (seg * kSeg + e * 256 >= hw) break;   // CTA-uniform
    bool fg_root = false, flag = false;
    if (p < hw) {
      fg_root = Lf_all[o + p] == p;
      flag = fg_root || (Lb_all[o + p] == p && parent_all[o + p] != kFrame);
    }
    int excl;
    const int tot = cta_flag_prefix(flag, &excl, wsum);
    if (flag) {
      const int rank = base + excl;
      root_list[o + rank] = p;
      const int c = total[page] - 1 - rank;
      int cid = -1;
      if (c < max_cand) {
        cid = c;
        // bit 31 of the table entry: 1 = hole contour
        c_root[page * max_cand + c] = fg_root ? p : (p | int(0x80000000u));
      }
      cid_all[o + p] = cid;
    }
    base += tot;
  }
}
// Every row a contour's pixels reach lies in its y range: reset those rows to all ones (min 0xffffffff as unsigned,
// max -1), so that the next launch finds the whole rows area reset without clearing n x max_cand x h entries.
__global__ void rows_clear_kernel(int h, int max_cand, const int* __restrict__ total, const int* __restrict__ c_yrange,
                                  int2* __restrict__ rows) {
  const int page = blockIdx.y, c = blockIdx.x;
  if (c >= total[page]) return;
  const int y0 = c_yrange[(page * max_cand + c) * 2], y1 = c_yrange[(page * max_cand + c) * 2 + 1];
  int2* r = rows + (size_t(page) * max_cand + c) * h;
  for (int y = y0 + int(threadIdx.x); y <= y1; y += blockDim.x) r[y] = make_int2(-1, -1);
}

// ---- per-pixel accumulation ----------------------------------------------------------------------
// Warp-aggregated: the 32 lanes of a warp are 32 consecutive pixels of one row, which mostly share their
// component, so lanes with the same (component, row) key elect a leader that issues ONE set of atomics.
__global__ void accumulate_kernel(int h, int w, const float* __restrict__ pred_all, size_t pred_page_stride,
                                  const int* __restrict__ Lf_all, const int* __restrict__ Lb_all,
                                  const int* __restrict__ parent_all, const int* __restrict__ cid_all,
                                  double* __restrict__ own_sum, int* __restrict__ own_cnt, double* __restrict__ ring_sum,
                                  int* __restrict__ ring_cnt, int2* __restrict__ rows, int* __restrict__ c_yrange,
                                  int max_cand) {
  const int page = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  const bool live = p < hw;
  const size_t o = size_t(page) * hw;
  const int lane = threadIdx.x & 31;
  float v = 0.f;
  int y = 0, x = 0, lf = -1, key = -1;
  if (live) {
    v = pred_all[size_t(page) * pred_page_stride + p];
    y = p / w;
    x = p - y * w;
    lf = Lf_all[o + p];
    if (lf >= 0) key = lf;
    else {
      const int lb = Lb_all[o + p];
      if (parent_all[o + lb] != kFrame) key = lb;
    }
  }
  const unsigned long long k64 = (unsigned long long)(unsigned)key | ((unsigned long long)(unsigned)y << 32);
  const unsigned peers = __match_any_sync(0xffffffffu, k64);
  const int leader = __ffs(peers) - 1;
  double s = 0.0;
  int c = 0;
  if (__all_sync(0xffffffffu, peers == 0xffffffffu)) {
    // the common case, one (component, row) run covers the whole warp: 5-step tree instead of 32 shuffles
    s = (double)v;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
    c = 32;   // only lane 0 (the leader) holds the full sum, and only the leader uses it
  } else {
#pragma unroll 4
    for (int l = 0; l < 32; ++l) {
      const float ov = __shfl_sync(0xffffffffu, v, l);
      if ((peers >> l) & 1u) {
        s += (double)ov;
        ++c;
      }
    }
  }
  if (live && key >= 0 && lane == leader) {
    atomicAdd(&own_sum[o + key], s);
    atomicAdd(&own_cnt[o + key], c);
    if (lf >= 0) {
      const int cid = cid_all[o + lf];
      if (cid >= 0) {
        const int last = 31 - __clz(peers);
        const size_t ro = (size_t(page) * max_cand + cid) * h + y;
        atomicMin(reinterpret_cast<unsigned*>(&rows[ro].x), unsigned(x));   // the leader is the left-most peer
        atomicMax(&rows[ro].y, x + (last - lane));
        atomicMin(&c_yrange[(page * max_cand + cid) * 2], y);
        atomicMax(&c_yrange[(page * max_cand + cid) * 2 + 1], y);
      }
    }
  }
  if (live && lf >= 0) {
    // ring membership: distinct holes among the 4-neighbours (boundary pixels only -> plain atomics)
    int hs[4];
    int nh = 0;
    const int nb[4] = {x > 0 ? p - 1 : -1, x + 1 < w ? p + 1 : -1, y > 0 ? p - w : -1, y + 1 < h ? p + w : -1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (nb[k] < 0) continue;
      const int q = Lb_all[o + nb[k]];
      // the hole border runs over pixels of the component that SURROUNDS the hole (its tree parent); islands
      // inside the hole touch it too but belong to its interior
      if (q < 0 || parent_all[o + q] != lf) continue;
      bool dup = false;
      for (int e = 0; e < nh; ++e) dup |= hs[e] == q;
      if (!dup) hs[nh++] = q;
    }
    for (int e = 0; e < nh; ++e) {
      const int q = hs[e];
      atomicAdd(&ring_sum[o + q], (double)v);
      atomicAdd(&ring_cnt[o + q], 1);
      const int c2 = cid_all[o + q];
      if (c2 >= 0) {
        const size_t ro = (size_t(page) * max_cand + c2) * h + y;
        atomicMin(reinterpret_cast<unsigned*>(&rows[ro].x), unsigned(x));
        atomicMax(&rows[ro].y, x);
        atomicMin(&c_yrange[(page * max_cand + c2) * 2], y);
        atomicMax(&c_yrange[(page * max_cand + c2) * 2 + 1], y);
      }
    }
  }
}

// every node (a root of root_list) adds its own sums to itself and to all its ancestors
__global__ void tree_kernel(int h, int w, const int* __restrict__ root_list, const int* __restrict__ total,
                            const int* __restrict__ parent_all, const double* __restrict__ own_sum,
                            const int* __restrict__ own_cnt, double* __restrict__ tot_sum, int* __restrict__ tot_cnt) {
  const int page = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total[page]) return;
  const size_t o = size_t(page) * h * w;
  const int p = root_list[o + i];
  const double s = own_sum[o + p];
  const int c = own_cnt[o + p];
  int a = p;
  int guard = 0;
  while (a >= 0 && guard++ < 4096) {
    atomicAdd(&tot_sum[o + a], s);
    atomicAdd(&tot_cnt[o + a], c);
    a = parent_all[o + a];
  }
}

// ---- per-contour geometry: one thread per candidate -------------------------------------------------
// CAP = vertex capacity of the hull / offset buffers.  The kernel runs twice: CAP = 128 for every contour (4.5 KB of
// shared memory per warp -> 48 contours in flight per SM instead of 12; the per-contour work is serial, latency-bound
// lane-0 code, so contours in flight is what sets the pace), then CAP = ctdgeom::kMaxHull for the few contours whose
// hull or offset polygon did not fit (collected in an overflow list by the first pass).
template <int CAP>
struct ContourScratchT {
  IPt hull[CAP];
  IPt tmp[CAP];
  IPt off[CAP];
  float f0[CAP], f1[CAP], f2[CAP];
};
struct ContourScratch;   // (unused global-memory variant of the first design)

// ---- warp-cooperative pieces of the per-contour geometry (bit-identical to the serial forms in geom.h) ------------
// rotate so that hull[0] is the max-x (ties: max-y) vertex; all 32 lanes, hull/tmp in shared memory
__device__ __forceinline__ void hull_start_maxx_warp(IPt* hull, int n, IPt* tmp, int lane) {
  if (n < 3) return;
  int bx = INT_MIN, by = INT_MIN, bi = 0;
  for (int i = lane; i < n; i += 32) {
    const IPt q = hull[i];
    if (q.x > bx || (q.x == bx && q.y > by)) { bx = q.x; by = q.y; bi = i; }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const int ox = __shfl_xor_sync(0xffffffffu, bx, off), oy = __shfl_xor_sync(0xffffffffu, by, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (ox > bx || (ox == bx && oy > by)) { bx = ox; by = oy; bi = oi; }   // hull vertices are distinct: no index ties
  }
  if (bi == 0) return;   // warp-uniform
  for (int i = lane; i < n; i += 32) { int j = i + bi; if (j >= n) j -= n; tmp[i] = hull[j]; }
  __syncwarp();
  for (int i = lane; i < n; i += 32) hull[i] = tmp[i];
  __syncwarp();
}

// first pass of min_area_rect across the warp: per-edge vectors / inverse lengths (element-wise, same expressions as
// ctdgeom::mar_edge) and the FIRST index of each extreme
__device__ __forceinline__ ctdgeom::MarExt mar_prepass_warp(const IPt* hull, int n, float* vx, float* vy, float* inv, int lane) {
  float lx = 3.402823466e+38f, rx = -3.402823466e+38f, ty = -3.402823466e+38f, by = 3.402823466e+38f;
  int li = 0x7fffffff, ri = 0x7fffffff, ti = 0x7fffffff, bi = 0x7fffffff;
  for (int i = lane; i < n; i += 32) {
    const float px = (float)hull[i].x, py = (float)hull[i].y;
    if (px < lx) { lx = px; li = i; }
    if (px > rx) { rx = px; ri = i; }
    if (py > ty) { ty = py; ti = i; }
    if (py < by) { by = py; bi = i; }
    ctdgeom::mar_edge(hull, n, i, vx, vy, inv);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    float o; int oi;
    o = __shfl_xor_sync(0xffffffffu, lx, off); oi = __shfl_xor_sync(0xffffffffu, li, off);
    if (o < lx || (o == lx && oi < li)) { lx = o; li = oi; }
    o = __shfl_xor_sync(0xffffffffu, rx, off); oi = __shfl_xor_sync(0xffffffffu, ri, off);
    if (o > rx || (o == rx && oi < ri)) { rx = o; ri = oi; }
    o = __shfl_xor_sync(0xffffffffu, ty, off); oi = __shfl_xor_sync(0xffffffffu, ti, off);
    if (o > ty || (o == ty && oi < ti)) { ty = o; ti = oi; }
    o = __shfl_xor_sync(0xffffffffu, by, off); oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (o < by || (o == by && oi < bi)) { by = o; bi = oi; }
  }
  __syncwarp();
  return ctdgeom::MarExt{li, bi, ri, ti};
}

// Longest-job-first order: the serial per-contour geometry costs roughly in proportion to the rows a contour spans,
// and the kernel is bound by its longest contour.  One CTA per page sorts (rows desc, id asc) with a bitonic network
// so that contour_kernel starts the tall contours first and fills the tail with the small ones.
__global__ void __launch_bounds__(1024) contour_order_kernel(int max_cand, const int* __restrict__ total,
                                                             const int* __restrict__ c_yrange, int* __restrict__ perm) {
  __shared__ unsigned int key[1024];
  const int page = blockIdx.x, i = threadIdx.x;
  int ncont = total[page];
  if (ncont > max_cand) ncont = max_cand;
  unsigned int k = 0xffffffffu;   // ascending sort of (~rows, id): padding last
  if (i < max_cand) {
    int rows = 0;
    if (i < ncont) {
      const int y0 = c_yrange[(page * max_cand + i) * 2], y1 = c_yrange[(page * max_cand + i) * 2 + 1];
      rows = y1 >= y0 ? y1 - y0 + 1 : 0;
      if (rows > 0xfffff) rows = 0xfffff;
    }
    k = ((0xfffffu - (unsigned int)rows) << 12) | (unsigned int)i;   // max_cand <= 1024 < 4096
  }
  key[i] = k;
  __syncthreads();
  for (int size = 2; size <= 1024; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int j = i ^ stride;
      if (j > i) {
        const unsigned int a = key[i], b = key[j];
        const bool up = (i & size) == 0;
        if ((a > b) == up) { key[i] = b; key[j] = a; }
      }
      __syncthreads();
    }
  if (i < max_cand) perm[page * max_cand + i] = int(key[i] & 0xfffu);
}

// One WARP per candidate (lane 0 runs the serial geometry; the working set lives in shared memory instead
// of per-thread local memory), 4 candidates per CTA.
constexpr int kContourWarps = 4;
template <int CAP>
__global__ void __launch_bounds__(32 * kContourWarps) contour_kernel(int h, int w, int max_cand, const int* __restrict__ total,
                                                     const int* __restrict__ c_root, const int2* __restrict__ rows,
                                                     const int* __restrict__ c_yrange,
                                                     const double* __restrict__ tot_sum,
                                                     const int* __restrict__ tot_cnt, const double* __restrict__ ring_sum,
                                                     const int* __restrict__ ring_cnt, ContourScratch* __restrict__ scratch,
                                                     int16_t* __restrict__ boxes, float* __restrict__ scores,
                                                     int* __restrict__ n_out, int dst_w, int dst_h, float unclip_ratio,
                                                     const int* __restrict__ perm, int n_pages,
                                                     int* __restrict__ ovf_count, int* __restrict__ ovf_list, int second) {
  extern __shared__ __align__(16) unsigned char csm[];
  ContourScratchT<CAP>& S = reinterpret_cast<ContourScratchT<CAP>*>(csm)[threadIdx.x >> 5];
  (void)scratch;
  // 1-D grid, page fastest: every page's tallest contours are scheduled before anybody's small ones
  const int page = int(blockIdx.x) % n_pages;
  const int slot = (int(blockIdx.x) / n_pages) * kContourWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  int ncont = total[page];
  if (ncont > max_cand) ncont = max_cand;
  if (!second && slot == 0 && lane == 0) n_out[page] = ncont;
  if (slot >= max_cand) return;
  int c;
  if (second) {
    if (slot >= ovf_count[page]) return;   // warp-uniform: only the contours the first pass could not hold
    c = ovf_list[page * max_cand + slot];
  } else {
    c = perm[page * max_cand + slot];
  }
  // a contour that overflows this pass's buffers is handed to the next pass (its row stays zero if there is none)
  auto defer = [&]() {
    if (!second && lane == 0) ovf_list[page * max_cand + atomicAdd(&ovf_count[page], 1)] = c;
  };
  int16_t* bo = boxes + (size_t(page) * max_cand + c) * 8;
  float* so = scores + size_t(page) * max_cand + c;
  if (lane < 8) bo[lane] = 0;
  if (lane == 0) *so = 0.f;
  if (c >= ncont) return;   // warp-uniform
  const int entry = c_root[page * max_cand + c];
  const bool is_hole = entry < 0;
  const int root = entry & 0x7fffffff;
  const size_t o = size_t(page) * h * w;
  const int2* rr = rows + (size_t(page) * max_cand + c) * h;
  // monotone chain over the row extremes; rows are sorted by y, so the chain runs in the transposed
  // plane (x' = y, y' = x) and the result is transposed back (which mirrors the orientation -> reversed).
  // The rows are prefetched 64 at a time by the whole warp (coalesced) and consumed by lane 0.
  const int y_lo = max(0, c_yrange[(page * max_cand + c) * 2]), y_hi = min(h - 1, c_yrange[(page * max_cand + c) * 2 + 1]);
  int* rbuf = reinterpret_cast<int*>(S.f0);  // 128 ints; f0 is free until the calipers run
  int k = 0;
  bool overflow = false;
  for (int y0 = y_lo; y0 <= y_hi; y0 += 64) {
    for (int e = lane; e < 64; e += 32) {
      const int y = y0 + e;
      rbuf[e] = y <= y_hi ? rr[y].x : INT_MAX;
      rbuf[64 + e] = y <= y_hi ? rr[y].y : -1;
    }
    __syncwarp();
    if (lane == 0 && !overflow) {
      for (int e = 0; e < 64 && y0 + e <= y_hi && !overflow; ++e) {
        const int a = rbuf[e], b = rbuf[64 + e];
        if (b < 0) continue;
        for (int q = 0; q < (a == b ? 1 : 2); ++q) {
          const IPt pt{y0 + e, q == 0 ? a : b};
          while (k >= 2 && ctdgeom::cross3(S.hull[k - 2], S.hull[k - 1], pt) <= 0) --k;
          if (k >= CAP) { overflow = true; break; }
          S.hull[k++] = pt;
        }
      }
    }
    __syncwarp();
  }
  const int lower = k + 1;
  bool first = true;
  for (int y1 = y_hi; y1 >= y_lo; y1 -= 64) {
    for (int e = lane; e < 64; e += 32) {
      const int y = y1 - e;
      rbuf[e] = y >= y_lo ? rr[y].x : INT_MAX;
      rbuf[64 + e] = y >= y_lo ? rr[y].y : -1;
    }
    __syncwarp();
    if (lane == 0 && !overflow) {
      for (int e = 0; e < 64 && y1 - e >= y_lo && !overflow; ++e) {
        const int a = rbuf[e], b = rbuf[64 + e];
        if (b < 0) continue;
        for (int q = 0; q < (a == b ? 1 : 2); ++q) {
          const IPt pt{y1 - e, q == 0 ? b : a};
          if (first) { first = false; continue; }  // the very last point of the forward pass
          while (k >= lower && ctdgeom::cross3(S.hull[k - 2], S.hull[k - 1], pt) <= 0) --k;
          if (k >= CAP) { overflow = true; break; }
          S.hull[k++] = pt;
        }
      }
    }
    __syncwarp();
  }
  // ---- geometry: the element-wise parts run across the warp, the calipers / offset / hull stay on lane 0 ----------
  overflow = __shfl_sync(0xffffffffu, int(overflow), 0) != 0;
  k = __shfl_sync(0xffffffffu, k, 0);
  if (overflow) { defer(); return; }
  if (k > 1) --k;
  // transpose back + reverse (the chain ran in the transposed plane)
  for (int i = lane; i < k; i += 32) S.tmp[i] = IPt{S.hull[k - 1 - i].y, S.hull[k - 1 - i].x};
  __syncwarp();
  for (int i = lane; i < k; i += 32) S.hull[i] = S.tmp[i];
  __syncwarp();
  if (k < 3) return;                                  // contour_stage1: 1-2 points / collinear -> skipped
  hull_start_maxx_warp(S.hull, k, S.tmp, lane);
  const ctdgeom::MarExt e1 = mar_prepass_warp(S.hull, k, S.f0, S.f1, S.f2, lane);
  int m = 0;
  __syncwarp();   // S.off / S.tmp of the previous use are dead for every lane before lane 0 rewrites S.off
  if (lane == 0) {
    const ctdgeom::RRect r1 = ctdgeom::mar_core(S.hull, k, S.f0, S.f1, S.f2, e1);
    const float sside = r1.w < r1.h ? r1.w : r1.h;
    if (sside >= 2.f) {
      float px[4], py[4], ox[4], oy[4];
      ctdgeom::box_points(r1, px, py);
      ctdgeom::order_mini_box(px, py, ox, oy);
      m = ctdgeom::unclip_offset(ox, oy, (double)unclip_ratio, S.off, CAP);
      if (m >= 0 && m < 3) m = 0;
    }
  }
  m = __shfl_sync(0xffffffffu, m, 0);
  __syncwarp();   // lane 0's S.off writes are visible to the lanes that rank-sort them (racecheck: shfl is no fence)
  if (m < 0) { defer(); return; }   // more offset vertices than this pass holds
  if (m == 0) return;
  // cooperative rank sort of the offset points by (x, y) into S.tmp, then back
  for (int i = lane; i < m; i += 32) {
    const IPt p = S.off[i];
    int rank = 0;
    for (int j = 0; j < m; ++j) {
      const IPt q = S.off[j];
      rank += (q.x < p.x) || (q.x == p.x && (q.y < p.y || (q.y == p.y && j < i)));
    }
    S.tmp[rank] = p;
  }
  __syncwarp();
  for (int i = lane; i < m; i += 32) S.off[i] = S.tmp[i];
  __syncwarp();
  int nh2 = 0;
  if (lane == 0) nh2 = ctdgeom::hull_sorted(S.off, m, S.hull, CAP);
  nh2 = __shfl_sync(0xffffffffu, nh2, 0);
  __syncwarp();
  if (nh2 < 0) { defer(); return; }
  if (nh2 < 3) return;
  hull_start_maxx_warp(S.hull, nh2, S.tmp, lane);
  const ctdgeom::MarExt e2 = mar_prepass_warp(S.hull, nh2, S.f0, S.f1, S.f2, lane);
  if (lane != 0) return;
  const ctdgeom::RRect r2 = ctdgeom::mar_core(S.hull, nh2, S.f0, S.f1, S.f2, e2);
  float px[4], py[4], ox[4], oy[4];
  ctdgeom::box_points(r2, px, py);
  ctdgeom::order_mini_box(px, py, ox, oy);
  int16_t box[8];
  for (int q = 0; q < 4; ++q) {
    box[2 * q] = ctdgeom::quantise(ox[q], w, dst_w);
    box[2 * q + 1] = ctdgeom::quantise(oy[q], h, dst_h);
  }
  // box_score_fast (db_utils.py:197-211): mean of pred over the filled contour polygon.  cv2.mean scales the double
  // sum by the reciprocal of the pixel count rather than dividing by it; the two differ in the last bit of the float
  // score on about 3 contours in 100 000 (tests/golden/seg_score_reciprocal.npz)
  double sum = tot_sum[o + root];
  long long cnt = tot_cnt[o + root];
  if (is_hole) {
    sum += ring_sum[o + root];
    cnt += ring_cnt[o + root];
  }
  *so = cnt > 0 ? (float)D_MUL(sum, D_DIV(1.0, (double)cnt)) : 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) bo[e] = box[e];
}

__global__ void binarize_kernel(const float* __restrict__ pred, size_t count, float thresh, uint8_t* __restrict__ bitmap) {
  const size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x;
  if (i < count) bitmap[i] = pred[i] > thresh ? 1 : 0;  // db_utils.py:71-72
}
cudaError_t binarize_launch(const float* pred, size_t count, float thresh, uint8_t* bitmap, cudaStream_t s) {
  binarize_kernel<<<unsigned((count + 255) / 256), 256, 0, s>>>(pred, count, thresh, bitmap);
  return cudaGetLastError();
}

size_t segrep_scratch_bytes(int n, int h, int w, int max_cand) {
  const size_t hw = size_t(n) * h * w;
  return hw * 4 * 5            // Lb, parent, cid, root_list, own_cnt
         + hw * 4 * 2          // tot_cnt, ring_cnt
         + hw * 8 * 3          // own_sum, tot_sum, ring_sum
         + size_t(n) * max_cand * 20          // c_root, c_yrange, perm, overflow list
         + size_t(n) * 8192 * 4               // segsum (<= 4096 per page) + totals
         + 65536;                             // 256-byte alignment slack of the 17 sub-arrays
}

cudaError_t segrep_launch(const uint8_t* bitmap, const float* pred, size_t pred_page_stride, const int* Lf, int n, int h,
                          int w, int max_cand, float unclip_ratio, void* scratch, int2* rows, int16_t* boxes,
                          float* scores, int* n_contours, cudaStream_t s) {
  const size_t hw = size_t(h) * w, nhw = size_t(n) * hw;
  char* p = static_cast<char*>(scratch);
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) / 256 * 256; return r; };
  int* Lb = reinterpret_cast<int*>(take(nhw * 4));
  int* parent = reinterpret_cast<int*>(take(nhw * 4));
  int* cid = reinterpret_cast<int*>(take(nhw * 4));
  int* root_list = reinterpret_cast<int*>(take(nhw * 4));
  int* own_cnt = reinterpret_cast<int*>(take(nhw * 4));
  int* tot_cnt = reinterpret_cast<int*>(take(nhw * 4));
  int* ring_cnt = reinterpret_cast<int*>(take(nhw * 4));
  double* own_sum = reinterpret_cast<double*>(take(nhw * 8));
  double* tot_sum = reinterpret_cast<double*>(take(nhw * 8));
  double* ring_sum = reinterpret_cast<double*>(take(nhw * 8));
  int* c_root = reinterpret_cast<int*>(take(size_t(n) * max_cand * 4));
  int* c_yrange = reinterpret_cast<int*>(take(size_t(n) * max_cand * 8));
  int* perm = reinterpret_cast<int*>(take(size_t(n) * max_cand * 4));
  int* segsum = reinterpret_cast<int*>(take(size_t(n) * 4096 * 4));
  int* total = reinterpret_cast<int*>(take(size_t(n) * 4));
  int* ovf_count = reinterpret_cast<int*>(take(size_t(n) * 4));
  int* ovf_list = reinterpret_cast<int*>(take(size_t(n) * max_cand * 4));
  ContourScratch* cs = nullptr;
  const int nseg = int((hw + kSeg - 1) / kSeg);
  if (nseg > 4096) return cudaErrorInvalidValue;
  if (max_cand > 1024) return cudaErrorInvalidValue;

  dim3 tgrid((w + 31) / 32, (h + 31) / 32, n);
  dim3 grid(unsigned((hw + 255) / 256), n);
  dim3 sgrid(unsigned(nseg), n);
  bg_local_kernel<<<tgrid, 1024, 0, s>>>(bitmap, h, w, Lb);
  const int nborder = ((w - 1) / 32) * h + ((h - 1) / 32) * w;
  if (nborder > 0) bg_border_kernel<<<dim3((nborder + 255) / 256, n), 256, 0, s>>>(h, w, Lb);
  bg_flatten_kernel<<<grid, 256, 0, s>>>(h, w, Lb, parent);
  mark_outside_kernel<<<dim3((max(2 * w + 2 * h, max_cand) + 255) / 256, n), 256, 0, s>>>(h, w, Lb, parent, c_yrange,
                                                                                          max_cand);
  roots_kernel<<<sgrid, 256, 0, s>>>(h, w, Lf, Lb, parent, own_sum, own_cnt, tot_sum, tot_cnt, ring_sum, ring_cnt, segsum,
                                     nseg);
  flag_scan_top_kernel<<<n, 1024, 0, s>>>(segsum, nseg, total);
  assign_cid_kernel<<<sgrid, 256, 0, s>>>(h, w, Lf, Lb, parent, segsum, nseg, total, max_cand, cid, c_root, root_list);
  accumulate_kernel<<<grid, 256, 0, s>>>(h, w, pred, pred_page_stride, Lf, Lb, parent, cid, own_sum, own_cnt, ring_sum,
                                         ring_cnt, rows, c_yrange, max_cand);
  tree_kernel<<<grid, 256, 0, s>>>(h, w, root_list, total, parent, own_sum, own_cnt, tot_sum, tot_cnt);
  constexpr int kCapSmall = 128, kCapLarge = ctdgeom::kMaxHull;
  const size_t sm_small = sizeof(ContourScratchT<kCapSmall>) * kContourWarps, sm_large = sizeof(ContourScratchT<kCapLarge>) * kContourWarps;
  // per device, so set on every launch (cheap; a process may own engines on several GPUs)
  cudaFuncSetAttribute(contour_kernel<kCapLarge>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sm_large));
  contour_order_kernel<<<n, 1024, 0, s>>>(max_cand, total, c_yrange, perm);
  cudaError_t e = cudaMemsetAsync(ovf_count, 0, size_t(n) * 4, s);
  if (e != cudaSuccess) return e;
  const unsigned cgrid = unsigned((max_cand + kContourWarps - 1) / kContourWarps) * unsigned(n);
  contour_kernel<kCapSmall><<<cgrid, 32 * kContourWarps, sm_small, s>>>(
      h, w, max_cand, total, c_root, rows, c_yrange, tot_sum, tot_cnt, ring_sum, ring_cnt, cs, boxes, scores,
      n_contours, w, h, unclip_ratio, perm, n, ovf_count, ovf_list, 0);
  contour_kernel<kCapLarge><<<cgrid, 32 * kContourWarps, sm_large, s>>>(
      h, w, max_cand, total, c_root, rows, c_yrange, tot_sum, tot_cnt, ring_sum, ring_cnt, cs, boxes, scores,
      n_contours, w, h, unclip_ratio, perm, n, ovf_count, ovf_list, 1);
  rows_clear_kernel<<<dim3(max_cand, n), 128, 0, s>>>(h, max_cand, total, c_yrange, rows);
  return cudaGetLastError();
}

}  // namespace ctd
