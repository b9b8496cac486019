// Post-processing kernels: YOLO candidate filter + NMS (utils/yolov5_utils.py:124-218 with
// torchvision.ops.nms semantics) and 8-connectivity connected-components labelling with OpenCV's
// label numbering (cv2.connectedComponentsWithStats as called from utils/textmask.py:93,113,138).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <limits.h>

#include "kernels.h"

namespace ctd {

// =========================================================================================
// NMS
constexpr int kCandStride = 8;  // x1,y1,x2,y2,conf,cls,row(int bits),pad
constexpr int kMaxDet = 300;    // max_det (yolov5_utils.py:125)
constexpr float kMaxWh = 4096.f;  // class offset (yolov5_utils.py:143,198)

size_t nms_workspace_bytes(int n, int cap) {
  return size_t(n) * cap * kCandStride * 4 * 2 + size_t(n) * 4 * 8 + size_t(n) * cap * (cap / 64) * 8;
}
void nms_workspace_bind(NmsWorkspace& ws, void* base, int n, int cap) {
  char* p = static_cast<char*>(base);
  ws.cap = cap;
  ws.mask = reinterpret_cast<unsigned long long*>(p);
  p += size_t(n) * cap * (cap / 64) * 8;
  ws.cand = reinterpret_cast<float*>(p);
  p += size_t(n) * cap * kCandStride * 4;
  ws.sorted = reinterpret_cast<float*>(p);
  p += size_t(n) * cap * kCandStride * 4;
  ws.cand_count = reinterpret_cast<int*>(p);
  p += size_t(n) * 4 * 4;
  ws.cand_total = reinterpret_cast<int*>(p);
}

__device__ __forceinline__ float round_half(float v) { return __half2float(__float2half_rn(v)); }

// the best class score of row x and its class, or 0 (no candidate): obj > conf -> cls *= obj -> best class -> conf >
// thres (yolov5_utils.py:136,169,179-180).  hf: the row holds float16 values and the reference's arithmetic is half's:
// conf_thres is half(conf_thres) there, and each product is rounded to half (the float product of two halves is
// exact, so this is RN_half of the exact product).  Positive floats: the bit pattern is monotone in the value.
__device__ __forceinline__ unsigned nms_score_key(const float* __restrict__ x, int no, float conf_thres, bool hf,
                                                  int* cls) {
  const float obj = x[4];
  if (!(obj > conf_thres)) return 0u;
  float best = -INFINITY;
  int bj = 0;
  for (int j = 5; j < no; ++j) {
    float c = __fmul_rn(x[j], obj);
    if (hf) c = round_half(c);
    if (c > best) {
      best = c;
      bj = j - 5;
    }
  }
  if (!(best > conf_thres)) return 0u;
  *cls = bj;
  return __float_as_uint(best);
}

// the candidate row torch.cat((box, conf, j.float()), 1) (yolov5_utils.py:172,180): xywh2xyxy, in half for a float16
// row, widened exactly to float32 by the cat
__device__ __forceinline__ void write_cand(float* __restrict__ o, const float* __restrict__ x, bool hf, unsigned key,
                                           int cls, int r) {
  float hw = x[2] / 2.f, hh = x[3] / 2.f;
  if (hf) {
    hw = round_half(hw);
    hh = round_half(hh);
    o[0] = round_half(x[0] - hw); o[1] = round_half(x[1] - hh); o[2] = round_half(x[0] + hw); o[3] = round_half(x[1] + hh);
  } else {
    o[0] = x[0] - hw; o[1] = x[1] - hh; o[2] = x[0] + hw; o[3] = x[1] + hh;
  }
  o[4] = __uint_as_float(key); o[5] = float(cls); o[6] = __int_as_float(r); o[7] = 0.f;
}

// conf_thres as page img compares it: half(conf_thres) for a float16 page
__device__ __forceinline__ float page_conf(const int32_t* __restrict__ half, int img, float conf_thres, bool* hf) {
  *hf = half && half[img];
  return *hf ? round_half(conf_thres) : conf_thres;
}

// yolov5_utils.py:136,152,169-182: one thread per row, candidates appended at atomic slots
__global__ void nms_filter_kernel(const float* __restrict__ blks, int rows, int no, float conf_thres,
                                  const int32_t* __restrict__ half, float* __restrict__ cand,
                                  int* __restrict__ cand_count, int cap) {
  const int img = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  bool hf;
  const float conf = page_conf(half, img, conf_thres, &hf);
  const float* x = blks + (size_t(img) * rows + r) * no;
  int cls = 0;
  const unsigned key = nms_score_key(x, no, conf, hf, &cls);
  if (key == 0u) return;
  const int slot = atomicAdd(&cand_count[img], 1);
  if (slot >= cap) return;
  write_cand(cand + (size_t(img) * cap + slot) * kCandStride, x, hf, key, cls, r);
}

// Overflow path (more candidates than the workspace holds, `cap`): the atomicAdd slots above are claimed in
// scheduling order, so WHICH rows survived would be nondeterministic.  The reference keeps every candidate up to
// max_nms = 30000 and beyond that the highest scores (yolov5_utils.py:143,191-194); here the cap is lower, so on
// overflow this kernel rebuilds the page's candidate list as exactly the `cap` best rows by (score descending, row
// ascending) -- a 3-level radix select over the score bits, then an ordered compaction -- and records the true
// candidate count so the host can see that the cap was hit (ctd_get_nms_status).  One CTA per page; returns at once
// when the page did not overflow.
__global__ void __launch_bounds__(1024) nms_overflow_kernel(const float* __restrict__ blks, int rows, int no,
                                                            float conf_thres, const int32_t* __restrict__ half,
                                                            float* __restrict__ cand,
                                                            int* __restrict__ cand_count, int* __restrict__ cand_total,
                                                            int cap) {
  __shared__ int hist[2048];
  __shared__ unsigned s_prefix, s_maskbits;
  __shared__ int s_need, s_base_take, s_base_tie;
  __shared__ int wsum_take[32], wsum_tie[32];
  const int img = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int total = cand_count[img];
  if (t == 0) cand_total[img] = total;
  if (total <= cap) return;
  bool hf;
  const float conf = page_conf(half, img, conf_thres, &hf);
  const float* pb = blks + size_t(img) * rows * no;
  if (t == 0) { s_prefix = 0u; s_maskbits = 0u; s_need = cap; }
  const int shifts[3] = {21, 10, 0}, nbins[3] = {2048, 2048, 1024};
#pragma unroll
  for (int lvl = 0; lvl < 3; ++lvl) {
    for (int i = t; i < 2048; i += 1024) hist[i] = 0;
    __syncthreads();
    const unsigned prefix = s_prefix, maskbits = s_maskbits;
    for (int r = t; r < rows; r += 1024) {
      int cls;
      const unsigned key = nms_score_key(pb + size_t(r) * no, no, conf, hf, &cls);
      if (key != 0u && (key & maskbits) == prefix) atomicAdd(&hist[(key >> shifts[lvl]) & unsigned(nbins[lvl] - 1)], 1);
    }
    __syncthreads();
    if (t == 0) {
      int need = s_need, cum = 0, digit = 0;
      for (int b = nbins[lvl] - 1; b >= 0; --b) {
        if (cum + hist[b] >= need) { digit = b; break; }
        cum += hist[b];
      }
      s_need = need - cum;                       // still to take among keys sharing the extended prefix
      s_prefix = prefix | (unsigned(digit) << shifts[lvl]);
      s_maskbits = maskbits | (unsigned(nbins[lvl] - 1) << shifts[lvl]);
    }
    __syncthreads();
  }
  const unsigned T = s_prefix;                   // key of the cap-th best score
  const int need_ties = s_need;                  // rows with key == T to take, lowest row index first
  if (t == 0) { s_base_take = 0; s_base_tie = 0; }
  __syncthreads();
  float* out = cand + size_t(img) * cap * kCandStride;
  for (int r0 = 0; r0 < rows; r0 += 1024) {
    const int r = r0 + t;
    int cls = 0;
    unsigned key = 0u;
    if (r < rows) key = nms_score_key(pb + size_t(r) * no, no, conf, hf, &cls);
    const bool tie = key == T && key != 0u;
    const unsigned tb = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) wsum_tie[wid] = __popc(tb);
    __syncthreads();
    int tie_rank = s_base_tie + __popc(tb & ((1u << lane) - 1u));
    for (int w2 = 0; w2 < wid; ++w2) tie_rank += wsum_tie[w2];
    const bool take = key > T || (tie && tie_rank < need_ties);
    const unsigned kb = __ballot_sync(0xffffffffu, take);
    if (lane == 0) wsum_take[wid] = __popc(kb);
    __syncthreads();
    if (take) {
      int slot = s_base_take + __popc(kb & ((1u << lane) - 1u));
      for (int w2 = 0; w2 < wid; ++w2) slot += wsum_take[w2];
      if (slot < cap) write_cand(out + size_t(slot) * kCandStride, pb + size_t(r) * no, hf, key, cls, r);
    }
    __syncthreads();
    if (t == 0) {
      int a = 0, b = 0;
      for (int w2 = 0; w2 < 32; ++w2) { a += wsum_take[w2]; b += wsum_tie[w2]; }
      s_base_take += a;
      s_base_tie += b;
    }
    __syncthreads();
  }
  if (t == 0) cand_count[img] = cap;
}

// stable descending sort by score (ties: original row order) -- torchvision nms_kernel sorts with
// stable=true.  One CTA per page, bitonic network in shared memory.
template <int P>
__global__ void __launch_bounds__(1024) nms_sort_kernel(const float* __restrict__ cand, int* __restrict__ cand_count,
                                                        float* __restrict__ sorted, int cap) {
  __shared__ float skey[P];
  __shared__ int srow[P];
  __shared__ int sslot[P];
  const int img = blockIdx.x;
  int m = cand_count[img];
  if (m > cap) m = cap;
  const float* c = cand + size_t(img) * cap * kCandStride;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    if (i < m) {
      skey[i] = c[i * kCandStride + 4];
      srow[i] = __float_as_int(c[i * kCandStride + 6]);
      sslot[i] = i;
    } else {
      skey[i] = -INFINITY;
      srow[i] = INT_MAX;
      sslot[i] = -1;
    }
  }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool up = (i & k) == 0;  // ascending position order == "better first"
          const float ka = skey[i], kb = skey[ixj];
          const int ra = srow[i], rb = srow[ixj];
          const bool a_first = (ka > kb) || (ka == kb && ra < rb);
          if (a_first != up) {
            skey[i] = kb; skey[ixj] = ka;
            srow[i] = rb; srow[ixj] = ra;
            const int t = sslot[i]; sslot[i] = sslot[ixj]; sslot[ixj] = t;
          }
        }
      }
      __syncthreads();
    }
  }
  float* o = sorted + size_t(img) * cap * kCandStride;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const int sl = sslot[i];
#pragma unroll
    for (int e = 0; e < kCandStride; ++e) o[i * kCandStride + e] = c[sl * kCandStride + e];
  }
}

// IoU bit matrix over class-offset boxes (yolov5_utils.py:198-200; torchvision nms_kernel arithmetic)
__global__ void __launch_bounds__(64) nms_mask_kernel(const float* __restrict__ sorted, const int* __restrict__ cand_count,
                                                      unsigned long long* __restrict__ mask, int cap, float iou_thres) {
  const int img = blockIdx.z;
  int m = cand_count[img];
  if (m > cap) m = cap;
  const int rb = blockIdx.y, cb = blockIdx.x;
  if (rb * 64 >= m || cb * 64 >= m || cb < rb) return;
  __shared__ float cbox[64][5];
  const float* s = sorted + size_t(img) * cap * kCandStride;
  const int cj = cb * 64 + threadIdx.x;
  if (cj < m) {
    const float off = s[cj * kCandStride + 5] * kMaxWh;
    cbox[threadIdx.x][0] = s[cj * kCandStride + 0] + off;
    cbox[threadIdx.x][1] = s[cj * kCandStride + 1] + off;
    cbox[threadIdx.x][2] = s[cj * kCandStride + 2] + off;
    cbox[threadIdx.x][3] = s[cj * kCandStride + 3] + off;
    cbox[threadIdx.x][4] = __fmul_rn(cbox[threadIdx.x][2] - cbox[threadIdx.x][0], cbox[threadIdx.x][3] - cbox[threadIdx.x][1]);
  }
  __syncthreads();
  const int i = rb * 64 + threadIdx.x;
  if (i >= m) return;
  const float off = s[i * kCandStride + 5] * kMaxWh;
  const float x1 = s[i * kCandStride + 0] + off, y1 = s[i * kCandStride + 1] + off;
  const float x2 = s[i * kCandStride + 2] + off, y2 = s[i * kCandStride + 3] + off;
  const float area = __fmul_rn(x2 - x1, y2 - y1);
  unsigned long long bits = 0;
  const int jmax = min(64, m - cb * 64);
  for (int j = 0; j < jmax; ++j) {
    if (cb * 64 + j <= i) continue;
    const float xx1 = fmaxf(x1, cbox[j][0]), yy1 = fmaxf(y1, cbox[j][1]);
    const float xx2 = fminf(x2, cbox[j][2]), yy2 = fminf(y2, cbox[j][3]);
    const float w = fmaxf(0.f, xx2 - xx1), h = fmaxf(0.f, yy2 - yy1);
    const float inter = __fmul_rn(w, h);
    const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area, cbox[j][4]), inter));
    if (ovr > iou_thres) bits |= 1ull << j;
  }
  mask[(size_t(img) * cap + i) * (cap / 64) + cb] = bits;
}

// greedy scan, one CTA per page, candidates in chunks of 64: the 64x64 diagonal block of a chunk is
// resolved serially by one thread from registers/shared memory, then every thread ORs the rows of the
// chunk's kept candidates into its own word of the suppression vector (coalesced row reads).  Stops at
// max_det kept rows like yolov5_utils.py:201-202.
__global__ void __launch_bounds__(64) nms_scan_kernel(const float* __restrict__ sorted, const int* __restrict__ cand_count,
                                                      const unsigned long long* __restrict__ mask, int cap,
                                                      float* __restrict__ det, int* __restrict__ det_count) {
  __shared__ unsigned long long remv[64];      // cap <= 4096 -> <= 64 words
  __shared__ unsigned long long diag[64];
  __shared__ unsigned long long s_keepbits;
  __shared__ int s_kept;
  const int img = blockIdx.x, t = threadIdx.x;
  int m = cand_count[img];
  if (m > cap) m = cap;
  const int words = cap / 64;
  const int wlast = (m + 63) >> 6;
  remv[t] = 0ull;
  if (t == 0) s_kept = 0;
  __syncthreads();
  const unsigned long long* mbase = mask + size_t(img) * cap * words;
  const float* s = sorted + size_t(img) * cap * kCandStride;
  float* o = det + size_t(img) * kMaxDet * 6;
  for (int c = 0; c < wlast; ++c) {
    const int i = c * 64 + t;
    diag[t] = (i < m) ? mbase[size_t(i) * words + c] : 0ull;
    __syncthreads();
    if (t == 0) {
      unsigned long long rw = remv[c], keep = 0ull;
      int kept = s_kept;
      const int lim = min(64, m - c * 64);
      for (int j = 0; j < lim && kept < kMaxDet; ++j) {
        if ((rw >> j) & 1ull) continue;
        keep |= 1ull << j;
        rw |= diag[j];
        ++kept;
      }
      s_keepbits = keep;
    }
    __syncthreads();
    const unsigned long long keep = s_keepbits;
    const int base_kept = s_kept;
    // write the kept rows (thread j writes its own row if kept)
    if ((keep >> t) & 1ull) {
      const int pos = base_kept + __popcll(keep & ((1ull << t) - 1ull));
      const float* r = s + size_t(c * 64 + t) * kCandStride;
#pragma unroll
      for (int e = 0; e < 6; ++e) o[pos * 6 + e] = r[e];
    }
    // OR the kept rows into the later words: thread t owns word t
    if (t > c && t < wlast) {
      unsigned long long acc = remv[t], kb = keep;
      while (kb) {
        const int j = __ffsll((long long)kb) - 1;
        kb &= kb - 1;
        acc |= mbase[size_t(c * 64 + j) * words + t];
      }
      remv[t] = acc;
    }
    __syncthreads();
    if (t == 0) s_kept = base_kept + __popcll(keep);
    __syncthreads();
    if (s_kept >= kMaxDet) break;
  }
  if (t == 0) det_count[img] = s_kept;
}

cudaError_t nms_launch(const float* blks, int n, int rows, int nc, float conf, float iou, NmsWorkspace& ws, float* det,
                       int* det_count, cudaStream_t s, const int32_t* half) {
  cudaError_t e = cudaMemsetAsync(ws.cand_count, 0, sizeof(int) * n, s);
  if (e != cudaSuccess) return e;
  // rows of `mask` below the diagonal block are never read; words at/after are always written
  nms_filter_kernel<<<dim3((rows + 255) / 256, n), 256, 0, s>>>(blks, rows, 5 + nc, conf, half, ws.cand, ws.cand_count,
                                                                 ws.cap);
  nms_overflow_kernel<<<n, 1024, 0, s>>>(blks, rows, 5 + nc, conf, half, ws.cand, ws.cand_count, ws.cand_total, ws.cap);
  if (ws.cap == 4096) nms_sort_kernel<4096><<<n, 1024, 0, s>>>(ws.cand, ws.cand_count, ws.sorted, ws.cap);
  else if (ws.cap == 1024) nms_sort_kernel<1024><<<n, 1024, 0, s>>>(ws.cand, ws.cand_count, ws.sorted, ws.cap);
  else return cudaErrorInvalidValue;
  const int blocks = ws.cap / 64;
  nms_mask_kernel<<<dim3(blocks, blocks, n), 64, 0, s>>>(ws.sorted, ws.cand_count, ws.mask, ws.cap, iou);
  if (ws.cap > 4096) return cudaErrorInvalidValue;
  nms_scan_kernel<<<n, 64, 0, s>>>(ws.sorted, ws.cand_count, ws.mask, ws.cap, det, det_count);
  return cudaGetLastError();
}

// =========================================================================================
// Connected components, 8-connectivity, OpenCV numbering.
//
// OpenCV's 8-connectivity labeller scans 2x2 blocks in raster order and, after flattening its
// union-find, numbers components by their smallest provisional label, i.e. by the first 2x2
// block (raster order over blocks) that holds one of the component's pixels (SURVEY section 7,
// App. D #16).  All pixels of one 2x2 block are mutually 8-adjacent, so that block identifies the
// component uniquely.  Here: union-find over pixels (Playne-Hawick atomicMin unions), per-root
// minimum block index, a prefix sum over "is a first block" flags gives the final label.

__device__ __forceinline__ int uf_find(const int* L, int a) {
  int p = L[a];
  while (p != a) {
    a = p;
    p = L[a];
  }
  return a;
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

constexpr int kCclTile = 32;  // 32x32-pixel tiles, one thread per pixel
constexpr int kScanSeg = 2048;

// Pass 1: union-find inside a 32x32 tile in shared memory (one warp per tile row).  Every pixel
// starts as the first pixel of its horizontal run (ballot + clz, no chains inside a row); vertical /
// diagonal contacts with the row above are then united.  Afterwards every pixel points at the
// GLOBAL raster index of its tile-local root (the smallest index of its local component).
__global__ void __launch_bounds__(1024) ccl_local_kernel(const uint8_t* __restrict__ img, int h, int w,
                                                         int* __restrict__ Lall, int* __restrict__ keymin_all) {
  __shared__ int s[kCclTile * kCclTile];
  const int page = blockIdx.z;
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int x = blockIdx.x * kCclTile + lx, y = blockIdx.y * kCclTile + ly;
  const bool inb = x < w && y < h;
  const size_t o = size_t(page) * h * w;
  const int l = threadIdx.x;
  const bool fg = inb && img[o + size_t(y) * w + x] != 0;
  const unsigned m = __ballot_sync(0xffffffffu, fg);
  const unsigned zeros_below = ~m & ((1u << lx) - 1u);
  const int start = zeros_below ? 32 - __clz(zeros_below) : 0;
  s[l] = fg ? (ly << 5) + start : -1;
  __syncthreads();
  if (fg && ly > 0) {
    const bool un = s[l - 32] >= 0;
    if (un) {
      // N contact: only the first pixel of each (current run x upper run) overlap issues the union
      const bool first = (lx == start) || s[l - 33] < 0;
      if (first) uf_union(s, l, l - 32);
    } else {
      if (lx > 0 && s[l - 33] >= 0) uf_union(s, l, l - 33);
      if (lx < 31 && s[l - 31] >= 0) uf_union(s, l, l - 31);
    }
  }
  __syncthreads();
  if (inb) {
    int g = -1;
    if (fg) {
      const int r = uf_find(s, l);
      g = (blockIdx.y * kCclTile + (r >> 5)) * w + blockIdx.x * kCclTile + (r & 31);
    }
    Lall[o + size_t(y) * w + x] = g;
    keymin_all[o + size_t(y) * w + x] = INT_MAX;
  }
}

// Pass 2: unions across tile borders only (global memory).
__global__ void ccl_border_kernel(int h, int w, int* __restrict__ Lall) {
  const int page = blockIdx.y;
  int* L = Lall + size_t(page) * h * w;
  const int nvl = (w - 1) / kCclTile;  // vertical border lines at x = 32, 64, ...
  const int nhl = (h - 1) / kCclTile;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nvl * h) {
    const int x = (i / h + 1) * kCclTile, y = i % h;
    const int p = y * w + x;
    if (L[p] < 0) return;
    if (L[p - 1] >= 0) uf_union(L, p, p - 1);
    if (y > 0 && L[p - w - 1] >= 0) uf_union(L, p, p - w - 1);
    if (y + 1 < h && L[p + w - 1] >= 0) uf_union(L, p, p + w - 1);
  } else if (i < nvl * h + nhl * w) {
    const int j = i - nvl * h;
    const int y = (j / w + 1) * kCclTile, x = j % w;
    const int p = y * w + x;
    if (L[p] < 0) return;
    if (L[p - w] >= 0) uf_union(L, p, p - w);
    if (x > 0 && L[p - w - 1] >= 0) uf_union(L, p, p - w - 1);
    if (x + 1 < w && L[p - w + 1] >= 0) uf_union(L, p, p - w + 1);
  }
}

// Pass 3: flatten + key.  The component's first 2x2 block (block-raster order) lies in the block row
// of its first pixel (= its root); its block column is the minimum over the component's pixels in
// that block row.  Only those pixels issue an atomic.
__global__ void ccl_flatten_key_kernel(int h, int w, int* __restrict__ Lall, int* __restrict__ keymin_all) {
  const int page = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (p >= hw) return;
  int* L = Lall + size_t(page) * hw;
  if (L[p] < 0) return;
  const int r = uf_find(L, p);
  L[p] = r;  // racing writers all store a valid ancestor; roots are fixed points
  const int y = p / w, x = p - y * w;
  if ((y >> 1) == ((r / w) >> 1)) atomicMin(&keymin_all[size_t(page) * hw + r], x >> 1);
}

// Pass 4: flag[first block] = 1 per component (bflag zeroed by a memset).
__global__ void ccl_markfirst_kernel(int h, int w, const int* __restrict__ Lall, const int* __restrict__ keymin_all,
                                     int* __restrict__ bflag_all) {
  const int page = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (p >= hw) return;
  const size_t o = size_t(page) * hw;
  if (Lall[o + p] == p) {
    const int bw = (w + 1) / 2;
    bflag_all[o + ((p / w) >> 1) * bw + keymin_all[o + p]] = 1;
  }
}

// Pass 5a: per 2048-flag segment: exclusive prefix in place + segment total.
__global__ void __launch_bounds__(256) ccl_scan_seg_kernel(int h, int w, int* __restrict__ bflag_all, int* __restrict__ segsum,
                                                           int nseg) {
  __shared__ int wsum[8];
  const int page = blockIdx.y, seg = blockIdx.x;
  const int nb = ((h + 1) / 2) * ((w + 1) / 2);
  int* f = bflag_all + size_t(page) * h * w + size_t(seg) * kScanSeg;
  const int base = seg * kScanSeg;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // each thread owns 8 consecutive flags
  int v[8], t = 0;
  const int i0 = threadIdx.x * 8;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    v[e] = (base + i0 + e < nb) ? f[i0 + e] : 0;
    t += v[e];
  }
  int incl = t;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += u;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int woff = 0;
  for (int k = 0; k < warp; ++k) woff += wsum[k];
  int run = woff + incl - t;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    if (base + i0 + e < nb) f[i0 + e] = run;
    run += v[e];
  }
  if (threadIdx.x == 255) segsum[page * nseg + seg] = woff + incl;
}
// Pass 5b: exclusive scan of the segment totals, n_labels.  Chunks of 4096 segments (4 consecutive entries per thread,
// block scan of the per-thread sums) with a running carry, so any segment count works: a 2^28-pixel image has 32768.
__global__ void __launch_bounds__(1024) ccl_scan_top_kernel(int* __restrict__ segsum, int nseg, int* __restrict__ n_labels) {
  __shared__ int part[1024];
  const int page = blockIdx.x;
  int* sgs = segsum + size_t(page) * nseg;
  int carry = 0;
  for (int c0 = 0; c0 < nseg; c0 += 4096) {
    int v[4], loc = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = c0 + threadIdx.x * 4 + k;
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
    int run = carry + part[threadIdx.x] - loc;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = c0 + threadIdx.x * 4 + k;
      if (i < nseg) sgs[i] = run;
      run += v[k];
    }
    carry += part[1023];
    __syncthreads();   // every thread has read part[1023] before the next chunk overwrites it
  }
  if (threadIdx.x == 0) n_labels[page] = carry + 1;
}

__global__ void ccl_relabel_kernel(int h, int w, const int* __restrict__ Lall, const int* __restrict__ keymin_all,
                                   const int* __restrict__ rank_all, const int* __restrict__ segoff, int nseg,
                                   int32_t* __restrict__ labels) {
  const int page = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (p >= hw) return;
  const size_t o = size_t(page) * hw;
  const int r = Lall[o + p];
  int lab = 0;
  if (r >= 0) {
    const int bw = (w + 1) / 2;
    const int key = ((r / w) >> 1) * bw + keymin_all[o + r];
    lab = segoff[page * nseg + key / kScanSeg] + rank_all[o + key] + 1;
  }
  labels[o + p] = lab;
}

// scratch: 3 * n*h*w ints (L, keymin, bflag/rank); segment sums live at the tail of the bflag area
cudaError_t ccl_launch(const uint8_t* img, int n, int h, int w, int32_t* labels, int32_t* scratch, int32_t* n_labels,
                       cudaStream_t s) {
  const int hw = h * w;
  int* L = scratch;
  int* keymin = scratch + size_t(n) * hw;
  int* bflag = scratch + size_t(2) * n * hw;
  const int nb = ((h + 1) / 2) * ((w + 1) / 2);
  const int nseg = (nb + kScanSeg - 1) / kScanSeg;
  // per page the bflag area has hw ints but only nb (<= hw/4 + ..) are used: keep segsum after them
  int* segsum = bflag + size_t(n - 1) * hw + nb;  // n*nseg ints, fits: nseg*n <= hw - nb for sane shapes
  if (size_t(n) * nseg > size_t(hw - nb)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemset2DAsync(bflag, size_t(hw) * sizeof(int), 0, size_t(nb) * sizeof(int), n, s);
  if (e != cudaSuccess) return e;
  dim3 tgrid((w + kCclTile - 1) / kCclTile, (h + kCclTile - 1) / kCclTile, n);
  ccl_local_kernel<<<tgrid, 1024, 0, s>>>(img, h, w, L, keymin);
  const int nborder = ((w - 1) / kCclTile) * h + ((h - 1) / kCclTile) * w;
  if (nborder > 0) ccl_border_kernel<<<dim3((nborder + 255) / 256, n), 256, 0, s>>>(h, w, L);
  dim3 grid((hw + 255) / 256, n);
  ccl_flatten_key_kernel<<<grid, 256, 0, s>>>(h, w, L, keymin);
  ccl_markfirst_kernel<<<grid, 256, 0, s>>>(h, w, L, keymin, bflag);
  ccl_scan_seg_kernel<<<dim3(nseg, n), 256, 0, s>>>(h, w, bflag, segsum, nseg);
  ccl_scan_top_kernel<<<n, 1024, 0, s>>>(segsum, nseg, n_labels);
  ccl_relabel_kernel<<<grid, 256, 0, s>>>(h, w, L, keymin, bflag, segsum, nseg, labels);
  return cudaGetLastError();
}

// stats rows: x, y, w, h, area (cv2.CC_STAT_*); single page
__global__ void ccl_stats_init_kernel(int32_t* stats, int cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  stats[i * 5 + 0] = INT_MAX;
  stats[i * 5 + 1] = INT_MAX;
  stats[i * 5 + 2] = -1;
  stats[i * 5 + 3] = -1;
  stats[i * 5 + 4] = 0;
}
__global__ void ccl_stats_acc_kernel(const int32_t* __restrict__ labels, int h, int w, int32_t* stats, int cap) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= h * w) return;
  const int l = labels[p];
  if (l >= cap) return;
  const int y = p / w, x = p - y * w;
  atomicMin(&stats[l * 5 + 0], x);
  atomicMin(&stats[l * 5 + 1], y);
  atomicMax(&stats[l * 5 + 2], x);
  atomicMax(&stats[l * 5 + 3], y);
  atomicAdd(&stats[l * 5 + 4], 1);
}
__global__ void ccl_stats_fin_kernel(int32_t* stats, int cap) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  if (stats[i * 5 + 4] == 0) {
    // OpenCV reports an empty label (only possible for background) as x=y=INT_MAX-ish; mirror cv2: zeros w/h
    stats[i * 5 + 2] = 0;
    stats[i * 5 + 3] = 0;
  } else {
    stats[i * 5 + 2] = stats[i * 5 + 2] - stats[i * 5 + 0] + 1;
    stats[i * 5 + 3] = stats[i * 5 + 3] - stats[i * 5 + 1] + 1;
  }
}
cudaError_t ccl_stats_launch(const int32_t* labels, int h, int w, int32_t* stats, int cap, cudaStream_t s) {
  ccl_stats_init_kernel<<<(cap + 255) / 256, 256, 0, s>>>(stats, cap);
  ccl_stats_acc_kernel<<<(h * w + 255) / 256, 256, 0, s>>>(labels, h, w, stats, cap);
  ccl_stats_fin_kernel<<<(cap + 255) / 256, 256, 0, s>>>(stats, cap);
  return cudaGetLastError();
}

}  // namespace ctd
